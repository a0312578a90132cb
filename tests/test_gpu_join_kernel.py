"""The row-block join kernel (csrc/sbn_join.cu) on batches large enough to take it.

It replaces the tiled kernel's several-variable (MX) launches on two batched operands only when the
batch has at least 2 x SMs x R rows (R = 16 or 32 rows per block), so every other test, which runs
small batches, reaches the tiled kernel instead.  Here: the kernel must run where it is claimed, its
output must be bitwise equal to the same batch run in pieces below that threshold (the tiled kernel),
and a sample of rows must match the float64 oracle.  Every row count is ragged (not a multiple of R).
"""
import numpy as np
import pytest

import kernel_census
import kernel_corpus
from oracle import ve_oracle

pytestmark = pytest.mark.gpu

RTOL = 1e-6
PIECE = 2048  # below the threshold at any R, on any GPU with at least 64 SMs


def join_launches(program, codes, n):
    return [name for name, _ in kernel_census.census(program, codes, n) if name.startswith("sbn_join_kernel")]


def check_pieces_and_oracle(plan, codes, n, dn, query, evidence, value_of, order):
    from sorobn_b200 import engine

    big = engine.Program(plan)
    ran = join_launches(big, codes, n)
    out = big.run(codes, n)
    small = engine.Program(plan)
    assert not join_launches(small, np.ascontiguousarray(codes[:, :PIECE]), PIECE)
    pieces = [small.run(np.ascontiguousarray(codes[:, lo:lo + PIECE]), min(PIECE, n - lo)) for lo in range(0, n, PIECE)]
    assert np.array_equal(np.concatenate(pieces, axis=1), out, equal_nan=True)
    worst = 0.0
    for b in list(range(0, n, max(1, n // 12))) + [n - 1]:
        ev = {v: value_of(v, codes[i, b]) for i, v in enumerate(evidence)}
        want = ve_oracle.query(dn, *query, event=ev, order=order)[1].reshape(-1)
        if np.isnan(want).all():
            assert np.isnan(out[:, b]).all()
            continue
        pos = want > 0
        assert (out[~pos, b] == 0).all()
        worst = max(worst, float(np.max(np.abs(out[pos, b] - want[pos]) / want[pos])))
    assert worst < RTOL, worst
    return ran


def test_join_kernel_full_size_grid():
    """The benchmark grid (10x10, 5 states) at 100,007 rows: the join kernel runs the two several-variable
    steps on two batched operands (`625 <- sum_25 t5e2 x B625 x B625 x t25e1` and `125 <- sum_25 B125 x B625 x
    t125`)."""
    from sorobn_b200 import planner, workloads

    wl = workloads.grid10x10()
    bn = wl.build()
    net = bn._compiled
    n = 100_007
    codes = wl.codes(bn, n, seed=11)
    plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    order = [net.names[v] for v in plan.order]
    ran = check_pieces_and_oracle(plan, codes, n, dn, wl.query, wl.evidence,
                                  lambda v, c: int(net.domains[net.index[v]][c]), order)
    assert sorted(ran) == ["sbn_join_kernel<0, 1, 2>", "sbn_join_kernel<2, 1, 1>"], ran


@pytest.mark.parametrize("name", ["grid10x10s5_seed60_q99_e26", "grid8x8s5_seed74_q63_e11"])
def test_join_kernel_corpus_grid(name):
    """Corpus grids whose programs have several-variable steps on two batched operands, at 20,011 rows."""
    case = next(c for c in kernel_corpus.CASES if c["name"] == name)
    spec, net, dn, plan, query, evidence = kernel_corpus.build(case)
    n = 20_011
    codes = kernel_corpus.evidence_rows(spec, evidence, n, seed=case["seed"])
    order = [net.names[v] for v in plan.order]
    ran = check_pieces_and_oracle(plan, codes, n, dn, query, evidence, lambda v, c: int(c), order)
    assert ran, "the join kernel did not run"
