"""The two references of the log-domain GPU test (tests/test_gpu_log_domain_variants.py) against each other, on the
CPU: over every log-domain case of the variant corpus (kernel_corpus.LOG_DOMAIN_CASES) and its MAP sets, the float64
replay of the MPE and marginal MAP words (oracle/program_interp.run_mpe on `table_blob64`) against the float64
oracles (tests/mpe_oracle.py, tests/map_oracle.py).  log P agrees to 1e-9 x max(1, |L*|), with -inf on the same
rows, and a decoded state that differs from the oracle's is an exact tie: its own log P is L* within that
tolerance."""
import numpy as np
import pytest

import kernel_corpus
import map_oracle
import mpe_oracle
from oracle import program_interp
from sorobn_b200 import planner

TOL64 = 1e-9  # x max(1, |L*|): float64 sums of the same logs in another order
LOG_FLT_MIN = float(np.log(np.finfo(np.float32).tiny))  # -87.34: below it P underflows float32's normal range


class Oracle:
    """The float64 oracle's answer of one program (MPE, or marginal MAP of `plan.sampled`) per evidence row, cached
    per distinct evidence code."""

    def __init__(self, net, dn, observed, plan, codes):
        self.net, self.dn, self.plan, self.codes = net, dn, plan, codes
        self.ev_names = [net.names[v] for v in observed]
        self.map_names = [net.names[v] for v in plan.sampled]
        self.cache = {}

    def event(self, b):
        return dict(zip(self.ev_names, (int(c) for c in self.codes[:, b])))

    def __call__(self, b):
        """(x* {name: state}, L*, gap to the runner-up: inf for MPE, which the tests do not read)."""
        key = tuple(int(c) for c in self.codes[:, b])
        if key not in self.cache:
            ev = self.event(b)
            if self.plan.version == planner.VERSION_MAP:
                self.cache[key] = map_oracle.solve(self.dn, ev, self.map_names)
            else:
                self.cache[key] = (*mpe_oracle.max_sum(self.dn, ev), np.inf)
        return self.cache[key]

    def log_p(self, b, decoded):
        """log P of the row's event and the decoded states `decoded` [n_decoded] (codes in `plan.sampled` order)."""
        mine = {n: int(c) for n, c in zip(self.map_names, decoded)}
        if self.plan.version == planner.VERSION_MAP:
            return map_oracle.log_prob(self.dn, self.event(b), mine)
        return mpe_oracle.log_joint(self.dn, {**self.event(b), **mine})

    def check(self, b, decoded, lp, rtol):
        """Row b: log P `lp` within rtol x max(1, |L*|) of the oracle's (-inf where L* is), and `decoded`, where it
        is not the oracle's state, a tie within the same tolerance.  Returns whether it differs."""
        x, L, _ = self(b)
        assert not np.isnan(lp), b
        if L == -np.inf:
            assert lp == -np.inf, (b, lp)
            return False
        tol = rtol * max(1.0, abs(L))
        assert abs(float(lp) - L) <= tol, (b, float(lp), L)
        if {n: int(c) for n, c in zip(self.map_names, decoded)} == x:
            return False
        assert abs(self.log_p(b, decoded) - L) <= tol, (b, decoded, L)
        return True


def programs(name, n_rows=kernel_corpus.LOG_DOMAIN_ORACLE_ROWS):
    """(CompiledNet, DenseNet, observed ids, codes [n_observed, n_rows], [(label, plan)]) of a case: its MPE plan,
    then one marginal MAP plan per MAP set."""
    _, net, dn, observed, codes = kernel_corpus.build_log_domain(name, n_rows)
    plans = [("mpe", planner.build_mpe_plan(net, observed))]
    plans += [(f"map{m}", planner.build_map_plan(net, observed, m)) for m in kernel_corpus.MAP_SETS[name]]
    return net, dn, observed, codes, plans


@pytest.mark.parametrize("name", kernel_corpus.LOG_DOMAIN_CASES)
def test_float64_replay_agrees_with_the_oracles(name):
    net, dn, observed, codes, plans = programs(name)
    n = codes.shape[1]
    for label, plan in plans:
        decoded, lp = program_interp.run_mpe(plan.words, plan.table_blob64, codes, dtype=np.float64)
        oracle = Oracle(net, dn, observed, plan, codes)
        for b in range(n):
            oracle.check(b, decoded[:, b], lp[b], TOL64)
        if name == kernel_corpus.NAIVE_BAYES_60 and label != "mpe":
            lo, hi = kernel_corpus.NAIVE_BAYES_60_LOG_P
            assert lo <= lp.min() and lp.max() <= hi < LOG_FLT_MIN, (lp.min(), lp.max())


@pytest.mark.parametrize("name", kernel_corpus.LOG_DOMAIN_CASES)
def test_claimed_plan_items_are_the_plans(name):
    """The plan-derived items a case claims are exactly those its plans show."""
    _, _, _, _, plans = programs(name)
    got = set().union(*[kernel_corpus.log_domain_items(p) for _, p in plans])
    assert got == set(kernel_corpus.LOG_DOMAIN_CLAIMS[name]) & set(kernel_corpus.LOG_DOMAIN_PLAN_ITEMS)


def test_the_structural_zero_case_sums_buckets_of_impossible_states():
    """The MAP programs of the structural-zero case sum out buckets whose terms are all -inf, in a batched and in
    a flat log-sum-exp step: the output entry is -inf, never NaN, and the row's log P stays finite."""
    name = "dag14p4s5x8_seed1_zeros_q10-13_e1"
    _, _, _, codes, plans = programs(name)
    kinds = set()
    for label, plan in plans[1:]:
        prog = program_interp._Program(plan.words, plan.table_blob64, codes, codes.shape[1], np.float64, (9,))
        for st in prog.steps:
            if st["kind"] == planner.KIND_ARGMAX:
                continue
            prog.contract(st)
            out = prog.bufs[st["out_slot"]]
            assert not np.isnan(out).any(), label
            if st["reduce"] == program_interp.REDUCE_LOGSUMEXP and np.isneginf(out).any():
                kinds.add(st["kind"])
        assert np.isfinite(prog.post_rows()).all(), label
    assert kinds == {planner.KIND_FLAT, planner.KIND_BATCHED}, kinds
