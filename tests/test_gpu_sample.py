"""Exact posterior draws on the device (BayesNet.sample_many, the sample kernel sbn_sample_step), against
the CPU replay of the same random stream (oracle/program_interp.py), marginals_many and the programs'
float64 twins."""
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

import kernel_corpus
from conftest import ROOT
from oracle import program_interp
from sorobn_b200 import engine, examples, planner, workloads

pytestmark = pytest.mark.gpu

ROWS = [1, 2, 127, 128, 129, 513]
CORPUS = ["dag9p2s4x1x4x4_seed54_q1-8_e2", "dag14p4s5x8_seed1_zeros_q10-13_e1", "dag8p2s37x3x2_seed3_q0-3_e2",
          "dag16p4s8_seed0_q15_e2", "grid7x7s5_seed39_q48_e18", "dag19p7s3_seed93_q12_e3"]
SKIPPED = {"draws": 0, "skipped": 0}


def networks():
    """(name, CompiledNet, observed var ids, codes of 513 rows [n_ev, 513])."""
    out = []
    for name in ["alarm", "asia", "sprinkler", "grades"]:
        net = getattr(examples, name)()._compiled
        observed = (0, len(net.names) - 1)
        out.append((name, net, observed, workloads.forward_sample_codes(net, 513, 1)[list(observed)]))
    for name in CORPUS:
        case = next(c for c in kernel_corpus.CASES if c["name"] == name)
        spec = kernel_corpus.make_spec(case)
        net = kernel_corpus.compiled_net(spec)
        evidence = [spec.nodes[k] for k in case["evidence"]]
        observed = tuple(sorted(net.index[e] for e in evidence))
        codes = kernel_corpus.evidence_rows(spec, [net.names[v] for v in observed], 513, seed=3)
        out.append((name, net, observed, codes))
    wl = workloads.grid10x10()
    bn = wl.build()
    net = bn._compiled
    observed = tuple(sorted(net.index[e] for e in wl.evidence))
    out.append(("grid10x10", net, observed, workloads.forward_sample_codes(net, 513, 2)[list(observed)]))
    return out


def replay(plan, program, codes, n_rows, n_draws, seed, f64, rtol):
    """Device draws, then the interpreter with each step conditioned on the device's own earlier draws:
    every draw whose margin exceeds `rtol` must be equal.  P(observed) must equal the float64
    interpreter's: to 1e-9 with the same NaN rows for a float64 program, to 1e-4 where a float32 program
    gives a value (its NaN rows are the range rule's, settled by the float64 program)."""
    codes = np.ascontiguousarray(codes[:, :n_rows])
    drawn, prob = program.sample(codes, n_rows, n_draws, seed)
    dtype = np.float64 if f64 else np.float32
    blob = plan.table_blob64 if f64 else plan.table_blob
    mine, p_mine, info = program_interp.run_sample(plan.words, blob, codes, n_rows=n_rows, n_draws=n_draws, seed=seed,
                                                   dtype=dtype, given=drawn)
    ok = ~np.isnan(prob)
    p_ref = program_interp.run_sample(plan.words, plan.table_blob64, codes, n_rows=n_rows, seed=seed)[1]
    if f64:
        assert np.array_equal(np.isnan(prob), np.isnan(p_ref))
    assert np.all(np.abs(prob[ok] - p_ref[ok]) <= (1e-9 if f64 else 1e-4) * p_ref[ok]), (n_rows, n_draws)
    for st in info:
        rows = slice(st["d_first"], st["d_first"] + len(st["cards"]))
        sure = (st["margin"] > rtol) & ok[None, :]
        SKIPPED["draws"] += int(ok.sum()) * n_draws * len(st["cards"])
        SKIPPED["skipped"] += int((~sure & ok[None, :]).sum()) * len(st["cards"])
        assert np.array_equal(drawn[rows][:, sure], mine[rows][:, sure]), (st["d_first"], n_rows, n_draws)
    return drawn, prob


@pytest.mark.parametrize("f64", [False, True])
def test_every_draw_follows_the_replay(f64):
    SKIPPED.update(draws=0, skipped=0)
    for name, net, observed, codes in networks():
        plan = planner.build_sample_plan(net, observed)
        program = engine.Program(plan, device=0, f64=f64)
        for n_rows in ROWS:
            for n_draws in (1, 3):
                _, prob = replay(plan, program, codes, n_rows, n_draws, seed=1000 + n_rows, f64=f64,
                                 rtol=1e-9 if f64 else 1e-5)
                assert np.isfinite(prob).mean() > 0.9, name
        program.close()
    print(f"\n{'float64' if f64 else 'float32'}: {SKIPPED['skipped']} of {SKIPPED['draws']} draws skipped for a small margin")
    assert SKIPPED["skipped"] < 1e-3 * SKIPPED["draws"]


def test_grid_marginals_of_200000_draws():
    wl = workloads.grid10x10()
    bn = wl.build(device=0)
    event = wl.events(1, seed=4, bn=bn)
    n = 200_000
    draws = bn.sample_many(event, n=n, seed=99)
    marg = bn.marginals_many(event)
    worst = 0.0
    for node in marg.columns.get_level_values(0).unique():
        p = marg[node].iloc[0]
        freq = draws[node].value_counts(normalize=True).reindex(p.index, fill_value=0.0).to_numpy()
        se = np.sqrt(np.maximum(p.to_numpy() * (1 - p.to_numpy()), 1e-12) / n)
        worst = max(worst, float(np.max(np.abs(freq - p.to_numpy()) / se)))
    assert worst < 6.0, worst


def test_determinism_chunking_and_seeds():
    wl = workloads.grid10x10()
    bn = wl.build(device=0)
    net = bn._compiled
    observed = tuple(sorted(net.index[e] for e in wl.evidence))
    plan = planner.build_sample_plan(net, observed)
    n = 100_007
    codes = np.ascontiguousarray(workloads.forward_sample_codes(net, n, 5)[list(observed)])
    program = engine.Program(plan, device=0)
    a, pa = program.sample(codes, n, 2, seed=2024)
    b, pb = program.sample(codes, n, 2, seed=2024)
    assert np.array_equal(a, b) and np.array_equal(pa, pb, equal_nan=True)
    program.set_graph(False)
    c, _ = program.sample(codes, n, 2, seed=2024)
    assert np.array_equal(a, c)
    program.set_graph(True)
    pieces = []
    for r0 in range(0, n, 4096):
        r1 = min(n, r0 + 4096)
        pieces.append(program.sample(np.ascontiguousarray(codes[:, r0:r1]), r1 - r0, 2, seed=2024, row_base=r0)[0])
    assert np.array_equal(np.concatenate(pieces, axis=2), a)
    d, _ = program.sample(codes, n, 2, seed=2025)
    assert (d != a).mean() > 0.1


def chain(n, card, rng):
    from sorobn_b200 import BayesNet

    names = [f"h{k:03d}" for k in range(n)]
    bn = BayesNet(*[(names[k - 1], names[k]) for k in range(1, n)], device=0)
    bn.P[names[0]] = pd.Series({0: 0.3, 1: 0.3, 2: 0.4})
    for k in range(1, n):
        t = rng.dirichlet(np.ones(card) * 0.3, size=card)
        bn.P[names[k]] = pd.DataFrame([(a, b, t[a, b]) for a in range(card) for b in range(card)],
                                      columns=[names[k - 1], names[k], "p"])
    bn.prepare()
    return bn, names


def test_rows_below_the_float32_range_are_drawn_in_float64():
    """A batch of 60-node chain rows whose P(observed) is below the float32 range (1e-30): every row is
    flagged by the float32 program, and `sample_many` draws all of them with the float64 program, at their
    own positions."""
    bn, names = chain(60, 3, np.random.default_rng(5))
    rows = pd.DataFrame(np.random.default_rng(6).integers(0, 3, size=(200, 57)), columns=names[1:58])
    net = bn._compiled
    observed = tuple(net.index[c] for c in rows.columns)
    codes = np.ascontiguousarray(rows.to_numpy().T.astype(np.uint8))
    plan = planner.build_sample_plan(net, observed)
    _, p64, _ = program_interp.run_sample(plan.words, plan.table_blob64, codes)
    # random codes on 57 of 60 nodes: with these seeds every row has a positive probability below 1e-30; the
    # filter keeps the test's premise should the generator change
    keep = np.flatnonzero((p64 > 0) & (p64 < 1e-30))
    assert len(keep) > 20
    rows, codes = rows.iloc[keep].reset_index(drop=True), np.ascontiguousarray(codes[:, keep])
    n = len(keep)
    _, p32 = engine.Program(plan, device=0).sample(codes, n, 4, seed=77)
    assert np.isnan(p32).all()
    got = bn.sample_many(rows, n=4, seed=77)
    f64 = engine.Program(plan, device=0, f64=True)
    replay(plan, f64, codes, n, 4, seed=77, f64=True, rtol=1e-9)
    drawn, prob = f64.sample(codes, n, 4, seed=77)
    assert np.isfinite(prob).all()
    for j, v in enumerate(plan.sampled):
        assert list(got[net.names[v]]) == list(np.asarray(net.domains[v])[drawn[j].T.reshape(-1)])


def test_kernel_census_in_a_fresh_interpreter():
    script = f"""
import sys
sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]
from kernel_census import census
from sorobn_b200 import engine, examples, planner, workloads
net = examples.alarm()._compiled
plan = planner.build_sample_plan(net, [0])
codes = workloads.forward_sample_codes(net, 1000, 1)[[0]]
for f64 in (False, True):
    p = engine.Program(plan, device=0, f64=f64)
    class Run:
        def run(self, c, n):
            p.sample(c, n, 2, 5)
        def set_graph(self, g):
            p.set_graph(g)
    print(sorted({{name for name, _ in census(Run(), codes, 1000)}}))
"""
    out = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, check=True).stdout
    assert "sbn_sample_step<float>" in out and "sbn_sample_step<double>" in out, out


def test_the_abi_refuses_other_programs_by_return_code():
    net = examples.asia()._compiled
    lib = engine.load()
    sample = engine.Program(planner.build_sample_plan(net, [0]), device=0)
    other = engine.Program(planner.build_plan(net, [1], [0]), device=0)
    counts = engine.Program(planner.build_counts_plan(net, [0]), device=0)
    codes = np.zeros((1, 4), dtype=np.uint8)
    out = np.zeros((7, 1, 4), dtype=np.uint8)
    prob = np.zeros(4, dtype=np.float32)
    for prog in (other, counts):
        assert lib.sbn_program_sample_host(prog._h, codes.ctypes.data, 4, 4, 1, 1, 0, out.ctypes.data, prob.ctypes.data) != 0
    post = np.zeros((2, 4), dtype=np.float32)
    assert lib.sbn_program_run_host(sample._h, codes.ctypes.data, 4, 4, post.ctypes.data, 4) != 0
    assert lib.sbn_program_evidence_host(sample._h, codes.ctypes.data, 4, 4, prob.ctypes.data) != 0
    cnt = np.zeros(counts.plan.n_counts, dtype=np.float64)
    assert lib.sbn_program_counts_host(sample._h, codes.ctypes.data, 4, 4, cnt.ctypes.data, cnt.size, prob.ctypes.data) != 0
    # the float64 entry point refuses a float32 program
    p64 = np.zeros(4, dtype=np.float64)
    assert lib.sbn_program_sample_host_f64(sample._h, codes.ctypes.data, 4, 4, 1, 1, 0, out.ctypes.data, p64.ctypes.data) != 0
    # and the program still works
    drawn, p = sample.sample(codes, 4, 1, 1)
    assert drawn.shape == (7, 1, 4) and np.isfinite(p).all()
