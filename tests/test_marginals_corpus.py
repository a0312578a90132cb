"""Marginals plans of every network of the variant corpus (tests/kernel_corpus.py), on the CPU.

oracle/program_interp.py runs each plan: in float64 against the float64 oracle at 1e-12, and in
float32 with the readout kernel's arithmetic (float32 products summed in runs of 32, the runs' sums
added in float64) against the float64 run at the project's 1e-6.  A readout sums every joint state
of its bucket but the target per entry -- 625 on the benchmark grid, 2,187 and 2,560 on two corpus
networks -- and a single float32 running sum of that many terms does not hold 1e-6:
test_float32_readout_accumulator_breaks_1e6 shows it, so the float32 check is known to see the
difference.  Also: which networks reach which readout path, and the planner's refusal of a readout
the engine cannot take.
"""
import numpy as np
import pytest

import kernel_corpus
from oracle import program_interp, ve_oracle
from sorobn_b200 import planner

N_ROWS = 64


def runs(name):
    """The corpus network's marginals plan, 64 evidence rows, the float64 run of the plan, and P(e)."""
    spec, net, dn, plan, evidence = kernel_corpus.build_marginals(name)
    codes = kernel_corpus.evidence_rows(spec, evidence, N_ROWS, seed=1)
    want = program_interp.run_marginals(plan.words, plan.table_blob64, codes, n_rows=N_ROWS)
    p_e = np.array([ve_oracle.evidence_probability(dn, dict(zip(evidence, map(int, codes[:, b])))) if evidence else 1.0
                    for b in range(N_ROWS)])
    return spec, net, dn, plan, evidence, codes, want, p_e


@pytest.mark.parametrize("name", kernel_corpus.MARGINALS_CASES)
def test_corpus_marginals_plan(name):
    spec, net, dn, plan, evidence, codes, want, p_e = runs(name)
    starts = program_interp.segment_starts(plan)
    assert plan.Q == sum(int(net.card[t]) for t in plan.targets)
    assert sorted(plan.targets) == sorted(set(range(len(net.names))) - {net.index[e] for e in evidence})
    # float64 against the oracle, every target, on rows 0, n - 1 and others between
    rows = sorted({0, N_ROWS - 1, *range(0, N_ROWS, 4 if len(plan.targets) < 100 else 32)})
    for b in rows:
        ev = dict(zip(evidence, map(int, codes[:, b])))
        if p_e[b] == 0:
            assert np.isnan(want[:, b]).all(), b
            continue
        for t, q0 in zip(plan.targets, starts):
            ref = ve_oracle.query(dn, net.names[t], event=ev)[1].reshape(-1)
            got = want[q0:q0 + len(ref), b]
            assert np.allclose(got, ref, rtol=1e-12, atol=1e-300), (b, net.names[t], got, ref)
            assert (got[ref == 0] == 0).all(), (b, net.names[t], got, ref)
    # float32 tables and steps, the readout kernel's double partial sums, at 1e-6 on every entry
    got32 = program_interp.run_marginals(plan.words, plan.table_blob, codes, n_rows=N_ROWS, dtype=np.float32)
    worst, flagged = program_interp.check_posterior(got32, want, starts, p_event=p_e)
    assert worst < 1e-6, worst


# corpus networks whose float32-accumulated readouts exceed 1e-6 on the 64 rows: (name, largest cz)
FLOAT32_ACC_FAILS = [
    ("grid10x10s5_seed0_q99_e30", 625),
    ("grid8x8s5_seed74_q63_e11", 625),
    ("grid8x8s4x5_seed10_q63_e9", 500),
    ("dag14p4s5x8_seed1_zeros_q10-13_e1", 2560),
    ("dag19p7s3_seed93_q12_e3", 2187),
]


@pytest.mark.parametrize("name,cz", FLOAT32_ACC_FAILS)
def test_float32_readout_accumulator_breaks_1e6(name, cz):
    """The readout as it was first written, a float32 accumulator, on the networks where it misses 1e-6."""
    spec, net, dn, plan, evidence, codes, want, p_e = runs(name)
    assert max(st.cx for st in plan.steps if st.kind == planner.KIND_MARGINAL) == cz
    starts = program_interp.segment_starts(plan)
    old = program_interp.run_marginals(plan.words, plan.table_blob, codes, n_rows=N_ROWS, dtype=np.float32,
                                       readout_acc=np.float32)
    worst, _ = program_interp.check_posterior(old, want, starts, p_event=p_e)
    assert worst > 1e-6, worst


READOUT_ITEM_CASES = {
    "readout multi-pass": {"dag8p2s37x3x2_seed3_q0-3_e2", "dag7p2s13x9x4_seed5_q6_e2", "dag6p2s37x2_seed1_q2_e2",
                           "dag300p1s17_seed2_q0_e5", "dag300p1s17_seed5_q0_e6", "dag300p1s17_seed16_q0_e7",
                           "dag300p1s17_seed34_q0_e8", kernel_corpus.NAIVE_BAYES_12},
    "readout unstaged tables": {"dag14p4s5x8_seed1_zeros_q10-13_e1"},
    "readout tables only": {"dag15p4s6_seed79_q7_e2"},
    "readout card 1": {"dag9p2s4x1x4x4_seed54_q1-8_e2", "dag16p4s5x8_seed63_single8-0_q14_e3"},
}


def test_readout_items_of_the_corpus():
    """Which corpus networks' marginals plans reach each readout path the plan shows (the GPU coverage
    test relies on them)."""
    hits = {item: set() for item in kernel_corpus.READOUT_ITEMS}
    for name in kernel_corpus.MARGINALS_CASES:
        for item in kernel_corpus.readout_items(kernel_corpus.build_marginals(name)[3]):
            hits[item].add(name)
    assert hits == READOUT_ITEM_CASES


def star(n_parents, parent_card):
    """A child `t` (2 states) of `n_parents` roots with `parent_card` states each.  Eliminated first, `t`
    is in one bucket, whose readout sums out parent_card ** n_parents joint states."""
    yes = np.random.default_rng(0).uniform(0.1, 0.9, (parent_card,) * n_parents)
    return planner.CompiledNet(
        names=[*(f"p{k}" for k in range(n_parents)), "t"],
        domains=[list(range(parent_card))] * n_parents + [[0, 1]],
        parents=[[]] * n_parents + [list(range(n_parents))],
        cpt=[np.full(parent_card, 1.0 / parent_card)] * n_parents + [np.stack([1 - yes, yes], axis=-1)],
    )


def test_readout_size_limit_is_the_engines():
    """A readout may sum out at most planner.MARGINAL_MAX_Z = 2^21 joint states (the engine's bound on
    its offset table).  128^3 = 2^21 plans; 130^3 is refused with ValueError at planning time, not
    when the engine parses the program."""
    plan = planner.build_marginals_plan(star(3, 128), [], order=[3, 0, 1, 2])  # `t` first: its only bucket
    assert max(st.cx for st in plan.steps if st.kind == planner.KIND_MARGINAL) == planner.MARGINAL_MAX_Z
    with pytest.raises(ValueError, match="too large for a readout"):
        planner.build_marginals_plan(star(3, 130), [], order=[3, 0, 1, 2])
