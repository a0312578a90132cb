"""Every host call walks its batch in chunks of the program's reservation.  With the chunk capped
(SOROBN_B200_CHUNK_ROWS) the same seeded batch runs in many chunks, the last one partial, so every chunk's row
offset into the caller's codes, likelihoods, weights and outputs is exercised: no per-row output may change by a
bit.  Count tables are summed chunk by chunk and differ only in summation order."""
import numpy as np
import pytest
import torch

from sorobn_b200 import engine, examples, planner, workloads

pytestmark = pytest.mark.gpu

NET = examples.asia()._compiled
OBSERVED = (0, 3, 7)
SOFT = (2, 6)      # two binary variables: four likelihood columns
MAP_VARS = (1, 4)


def on_device(a):
    return torch.as_tensor(a, device=torch.device("cuda", engine.default_device()))


def table_first(out):
    """(per-row outputs, count table) of a call that returns the count table first"""
    return out[1:], out[0]


# kind: (plan, call(program, codes, n_rows, lik, weights) -> (per-row outputs, count table or None), float64 twin)
CASES = {
    "run": (lambda: planner.build_plan(NET, [1], OBSERVED),
            lambda p, c, n, lik, w: ((p.run(c, n), p.evidence(c, n)), None), True),
    "run_marginals": (lambda: planner.build_marginals_plan(NET, OBSERVED),
                      lambda p, c, n, lik, w: ((p.run(c, n),), None), True),
    "run_soft": (lambda: planner.build_plan(NET, [1], OBSERVED, soft=SOFT),
                 lambda p, c, n, lik, w: (p.run_soft(c, lik, n, log_evidence=True), None), True),
    "counts": (lambda: planner.build_counts_plan(NET, OBSERVED),
               lambda p, c, n, lik, w: table_first(p.counts(c, n)), True),
    "counts_soft": (lambda: planner.build_pattern_plan(NET, "counts", OBSERVED, soft=SOFT),
                    lambda p, c, n, lik, w: table_first(p.counts(c, n, lik=lik, log_evidence=True)), True),
    "sample": (lambda: planner.build_sample_plan(NET, OBSERVED),
               lambda p, c, n, lik, w: (p.sample(c, n, 3, seed=5, row_base=17), None), True),
    "sample_soft": (lambda: planner.build_pattern_plan(NET, "sample", OBSERVED, soft=SOFT),
                    lambda p, c, n, lik, w: (p.sample(c, n, 3, seed=5, row_base=17, lik=lik, log_evidence=True), None),
                    True),
    "mpe": (lambda: planner.build_mpe_plan(NET, OBSERVED), lambda p, c, n, lik, w: (p.mpe(c, n), None), False),
    "mpe_soft": (lambda: planner.build_pattern_plan(NET, "mpe", OBSERVED, soft=SOFT),
                 lambda p, c, n, lik, w: (p.mpe(c, n, lik=lik), None), False),
    "map": (lambda: planner.build_map_plan(NET, OBSERVED, MAP_VARS), lambda p, c, n, lik, w: (p.map(c, n), None), False),
    "map_soft": (lambda: planner.build_pattern_plan(NET, "map", OBSERVED, soft=SOFT, map_vars=MAP_VARS),
                 lambda p, c, n, lik, w: (p.map(c, n, lik=lik), None), False),
    "grad_forward": (lambda: planner.build_pattern_plan(NET, "grad", OBSERVED, soft=SOFT),
                     lambda p, c, n, lik, w: (p.grad_forward(c, n, lik=lik), None), True),
    "grad_backward": (lambda: planner.build_pattern_plan(NET, "grad", OBSERVED, soft=SOFT),
                      lambda p, c, n, lik, w: table_first(p.grad_backward(c, n, w, lik=lik)), True),
    "grad_backward_device": (lambda: planner.build_pattern_plan(NET, "grad", OBSERVED, soft=SOFT),
                             lambda p, c, n, lik, w: table_first(
                                 p.grad_backward(c, n, on_device(w), lik=on_device(lik))), True),
    "joint": (lambda: planner.build_joint_plan(NET, OBSERVED), lambda p, c, n, lik, w: (p.joint(c, n), None), True),
    "joint_soft": (lambda: planner.build_joint_plan(NET, OBSERVED, soft=SOFT),
                   lambda p, c, n, lik, w: (p.joint(c, n, lik=lik), None), True),
}
DECODING = ("sample", "sample_soft", "mpe", "mpe_soft", "map", "map_soft")

PARAMS = [pytest.param(kind, f64, n_rows, cap, id=f"{kind}-{'f64' if f64 else 'f32'}-{n_rows}-cap{cap}")
          for kind, (_, _, twin) in CASES.items() for f64 in ((False, True) if twin else (False,))
          # 1,000 rows in chunks of 96: ten full chunks and a partial one.  Sample and MPE chunks replay a graph from
          # 4,096 rows only, so their 10,000 rows in chunks of 4,096 take two replays and a plain partial chunk.
          for n_rows, cap in ((1000, 96),) + (((10_000, 4096),) if kind in DECODING else ())]


@pytest.mark.parametrize("kind,f64,n_rows,cap", PARAMS)
def test_chunked_call_matches_one_chunk(monkeypatch, kind, f64, n_rows, cap):
    plan_of, call, _ = CASES[kind]
    program = engine.Program(plan_of(), f64=f64)
    codes = np.ascontiguousarray(workloads.forward_sample_codes(NET, n_rows, 3)[list(OBSERVED)])
    rng = np.random.default_rng(4)
    lik = rng.random((n_rows, 4)) * 10.0 ** rng.integers(-3, 3, size=(n_rows, 1)) + 1e-3
    weights = rng.random(n_rows) + 0.5

    def run():
        before = program.info()["launches"]
        out = call(program, codes, n_rows, lik, weights)
        return out, program.info()["launches"] - before

    try:
        monkeypatch.delenv("SOROBN_B200_CHUNK_ROWS", raising=False)
        (whole, whole_counts), n_whole = run()
        monkeypatch.setenv("SOROBN_B200_CHUNK_ROWS", str(cap))
        (chunked, chunked_counts), n_chunked = run()
    finally:
        program.close()
    assert n_chunked > n_whole  # the cap took effect
    assert len(chunked) == len(whole) > 0
    for a, b in zip(chunked, whole):
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), kind
    if whole_counts is not None:
        np.testing.assert_allclose(chunked_counts, whole_counts, rtol=1e-12)
