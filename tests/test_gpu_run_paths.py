"""Every program kind runs through one issue loop and one graph cache: with the CUDA graph on, a run must give
the bits of plain launches and advance `info()["launches"]` by the same amount, on the first (captured) and a
later (replayed) call alike."""
import numpy as np
import pytest

from sorobn_b200 import engine, examples, planner, workloads

pytestmark = pytest.mark.gpu

NET = examples.asia()._compiled
OBSERVED = (0, 3, len(NET.names) - 1)
QUERY = 1  # not observed


def plan_and_call(kind):
    """(plan, call(program, codes, n_rows) -> tuple of output arrays) of one program kind."""
    if kind == "posterior":
        return planner.build_plan(NET, [QUERY], list(OBSERVED)), lambda p, c, n: (p.run(c, n),)
    if kind == "marginals":
        return planner.build_marginals_plan(NET, list(OBSERVED)), lambda p, c, n: (p.run(c, n),)
    if kind == "counts":
        return planner.build_counts_plan(NET, list(OBSERVED)), lambda p, c, n: p.counts(c, n)
    if kind == "sample":
        return planner.build_sample_plan(NET, OBSERVED), lambda p, c, n: p.sample(c, n, 2, seed=11)
    return planner.build_mpe_plan(NET, OBSERVED), lambda p, c, n: p.mpe(c, n)


def counted(program, call):
    before = program.info()["launches"]
    out = call()
    return out, program.info()["launches"] - before


@pytest.mark.parametrize("n_rows", [1000, 10_000])  # sample / MPE: below and above the 4,096-row graph threshold
@pytest.mark.parametrize("kind", ["posterior", "marginals", "counts", "sample", "mpe"])
def test_graph_and_plain_launches_agree(kind, n_rows):
    plan, call = plan_and_call(kind)
    program = engine.Program(plan, device=0)
    codes = np.ascontiguousarray(workloads.forward_sample_codes(NET, n_rows, 7)[list(OBSERVED)])
    program.set_graph(False)
    plain, n_plain = counted(program, lambda: call(program, codes, n_rows))
    assert n_plain > 0
    program.set_graph(True)
    for _ in range(2):  # capture, then replay
        got, n_got = counted(program, lambda: call(program, codes, n_rows))
        assert n_got == n_plain, kind
        for a, b in zip(got, plain):
            assert a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8)), kind
    program.close()


def test_pipelined_graph_and_plain_launches_agree():
    """A transfer-bound posterior batch from pinned host buffers runs as ONE replay of the pipelined graph."""
    plan, _ = plan_and_call("posterior")
    program = engine.Program(plan, device=0)
    n_rows = 200_003  # >= 4 x 32768 rows and >= 2 MB of copies
    codes = engine.PinnedArray((len(OBSERVED), n_rows), np.uint8)
    codes.array[:] = workloads.forward_sample_codes(NET, n_rows, 8)[list(OBSERVED)]
    plain, graph = (engine.PinnedArray((program.Q, n_rows), np.float32) for _ in range(2))
    program.set_graph(False)
    _, n_plain = counted(program, lambda: program.run(codes.array, n_rows, out=plain.array))
    assert n_plain > 0
    program.set_graph(True)
    for _ in range(2):  # capture, then replay
        graph.array[:] = -1.0
        _, n_got = counted(program, lambda: program.run(codes.array, n_rows, out=graph.array))
        assert n_got == n_plain
        assert np.array_equal(graph.array.view(np.uint32), plain.array.view(np.uint32))
    for a in (codes, plain, graph):
        a.free()
    program.close()
