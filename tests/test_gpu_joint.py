"""Joint programs and `BayesNet.joint_marginals_many` on the H100, against the CPU replay of their words
(tests/joint_interp.py) and the float64 oracle (test_joint_plan.oracle_group)."""
import numpy as np
import pandas as pd
import pytest
import torch

import joint_interp
import soft_oracle
from kernel_census import census_many
from sorobn_b200 import BayesNet, engine, examples, planner, synthetic, workloads
from test_joint_host import ASIA_COLS, frame, joint_golden_check
from test_joint_plan import missing_patterns, network, oracle_group

pytestmark = pytest.mark.gpu

ROWS = [1, 127, 129, 4099]


def rows_of(net, ev, soft, n, seed):
    """(codes [n_ev, n], likelihoods [n, n_lik] or None) of n rows drawn from the network, the likelihoods over 6
    orders of magnitude."""
    rng = np.random.default_rng(seed)
    full = workloads.forward_sample_codes(net, n, seed)
    codes = np.ascontiguousarray(full[list(ev)]) if ev else np.zeros((0, n), dtype=np.uint8)
    n_lik = sum(int(net.card[v]) for v in soft)
    lik = rng.random((n, n_lik)) * 10.0 ** rng.integers(-3, 3, size=(n, 1)) if soft else None
    return codes, lik


def run(plan, codes, lik, f64=False):
    prog = engine.Program(plan, f64=f64)
    try:
        return prog.joint(codes, codes.shape[1] if codes.size else len(lik), lik=lik)
    finally:
        prog.close()


def cases(net, seed):
    """(observed var ids, soft var ids) per case: missing cells, latent nodes and soft evidence."""
    rng = np.random.default_rng(seed)
    perm = [int(v) for v in rng.permutation(len(net.names))]
    pats = missing_patterns(net, seed, 2)
    soft = tuple(sorted(perm[:2], key=lambda v: net.names[v]))
    return [(pats[0], ()), (pats[1], ()), (tuple(v for v in pats[0] if v not in soft), soft)]


@pytest.mark.parametrize("name", ["alarm", "asia", "grades", "sprinkler", "dag12", "dag20"])
@pytest.mark.parametrize("n_rows", ROWS)
def test_device_matches_the_replay_and_the_oracle(name, n_rows):
    net = network(name)
    dn = soft_oracle.dense(net)
    for k, (ev, soft) in enumerate(cases(net, n_rows)):
        plan = planner.build_pattern_plan(net, "joint", ev, soft=soft)
        codes, lik = rows_of(net, ev, plan.soft, n_rows, k)
        n = n_rows
        out, prob = run(plan, codes, lik)
        r32, p32, _ = joint_interp.run_joint(plan.words, plan.table_blob, codes, lik=lik, n_rows=n, dtype=np.float32)
        r64, p64, _ = joint_interp.run_joint(plan.words, plan.table_blob64, codes, lik=lik, n_rows=n)
        ok = ~np.isnan(prob)
        assert ok.all(), "no row of these networks is below the float32 range"
        np.testing.assert_allclose(prob, p32, rtol=2e-6)
        for ref in (r32, r64):
            np.testing.assert_allclose(out, ref, rtol=2e-6, atol=1e-7)
        # the oracle on a few rows
        rows = soft_oracle.rows(net, ev, codes, plan.soft, lik if lik is not None else np.zeros((n, 0)))
        for b in range(0, n, max(1, n // 5)):
            hard, s = rows[b]
            for g, q0 in zip(plan.groups, plan.group_rows):
                M = [u for u in g if u not in ev]
                if M:
                    want = oracle_group(net, dn, M, hard, s)
                    np.testing.assert_allclose(out[q0:q0 + len(want), b], want, rtol=2e-6, atol=1e-7)


def test_frames_sum_to_the_expected_counts():
    bn = examples.alarm()
    X = frame(bn, 5000, 3, ("John calls", "Mary calls", "Earthquake"), frac=0.3)
    got = bn.joint_marginals_many(X)
    counts = bn.expected_counts(X)
    for node, df in got.items():
        np.testing.assert_allclose(df.sum(axis=1).to_numpy(), 1.0, atol=1e-6)
        np.testing.assert_allclose(df.sum(axis=0).to_numpy(), counts[node].to_numpy(), rtol=1e-6, atol=1e-6 * len(X))


def test_groups_with_a_table_of_ones_on_the_device():
    bn = examples.asia()
    X = frame(bn, 300, 5, ASIA_COLS, frac=0.5)
    groups = [("Visit to Asia", "Dispnea"), ("Smoker", "Tuberculosis", "Positive X-ray"), "TB or cancer"]
    got = bn.joint_marginals_many(X, groups=groups)
    net = bn._compiled
    dn = soft_oracle.dense(net)
    for b in range(0, len(X), 29):
        row = X.iloc[b]
        hard = {c: v for c, v in row.items() if v is not None and v == v}
        for g in groups[:2]:
            M = [n for n in g if n not in hard]
            if not M:
                continue
            want = oracle_group(net, dn, [net.index[n] for n in M], hard, {})
            vals = got[g].iloc[b].to_numpy().reshape([2] * len(g))
            index = tuple(int(hard[n]) if n in hard else slice(None) for n in g)
            sub = vals[index]
            np.testing.assert_allclose(sub.transpose().reshape(-1), want, rtol=2e-6, atol=1e-7)


def test_float64_rescue_of_a_long_chain():
    """P(row) ~ 1e-40 is below the float32 range: the float32 program flags every row and the float64 twin answers."""
    spec = synthetic.chain(120, 4, seed=3)
    bn = synthetic.load(spec, BayesNet)
    net = bn._compiled
    n = 64
    full = workloads.forward_sample_codes(net, n, 1)
    cols = [spec.nodes[k] for k in range(0, 120) if k % 5 != 2]
    X = pd.DataFrame({c: np.asarray(net.domains[net.index[c]], dtype=object)[full[net.index[c]]] for c in cols})
    plan = planner.build_joint_plan(net, tuple(sorted(net.index[c] for c in cols)),
                                    [(net.index[spec.nodes[k]],) for k in (2, 57, 117)])
    codes = np.ascontiguousarray(full[list(plan.evidence)])
    _, p32 = run(plan, codes, None)
    assert np.isnan(p32).all()
    out64, p64 = run(plan, codes, None, f64=True)
    assert (p64 < 1e-35).all() and (p64 > 0).all()
    got = bn.joint_marginals_many(X, groups=[spec.nodes[k] for k in (2, 57, 117)])
    r64, _, _ = joint_interp.run_joint(plan.words, plan.table_blob64, codes, n_rows=n)
    dn = soft_oracle.dense(net)
    for k, node in zip(range(3), (2, 57, 117)):
        df = got[spec.nodes[node]]
        assert np.isfinite(df.to_numpy()).all()
        np.testing.assert_allclose(df.sum(axis=1).to_numpy(), 1.0, atol=1e-9)
    np.testing.assert_allclose(out64, r64, rtol=1e-12, atol=1e-15)
    hard = {c: X[c].iloc[0] for c in cols}
    want = oracle_group(net, dn, [net.index[spec.nodes[57]]], hard, {})
    np.testing.assert_allclose(out64[plan.group_rows[1]:plan.group_rows[1] + 4, 0], want, rtol=1e-9)


def test_soft_evidence_from_a_cuda_tensor_is_read_in_place():
    net = network("alarm")
    soft = (net.index["Alarm"], net.index["Burglary"])
    plan = planner.build_pattern_plan(net, "joint", (net.index["John calls"],), soft=soft)
    codes, lik = rows_of(net, plan.evidence, plan.soft, 3000, 2)
    prog = engine.Program(plan)
    try:
        want = prog.joint(codes, 3000, lik=lik)
        got = prog.joint(codes, 3000, lik=torch.tensor(lik, dtype=torch.float32, device="cuda"))
    finally:
        prog.close()
    assert want[0].tobytes() == got[0].tobytes() and want[1].tobytes() == got[1].tobytes()
    bn = examples.alarm()
    X = pd.DataFrame({"John calls": np.asarray(net.domains[net.index["John calls"]], dtype=object)[codes[0]]})
    liks = {net.names[v]: lik[:, sum(int(net.card[u]) for u in plan.soft[:k]):][:, :int(net.card[v])]
            for k, v in enumerate(plan.soft)}
    a = bn.joint_marginals_many(X, likelihoods=liks)
    b = bn.joint_marginals_many(X, likelihoods={k: torch.tensor(v, device="cuda") for k, v in liks.items()})
    for k in a:
        np.testing.assert_allclose(a[k].to_numpy(), b[k].to_numpy(), rtol=1e-6, atol=1e-7)


def grid_case(n_rows):
    wl = workloads.grid10x10()
    bn = wl.build()
    net = bn._compiled
    ev = tuple(sorted(net.index[v] for v in wl.evidence))
    codes = np.ascontiguousarray(workloads.forward_sample_codes(net, n_rows, 9)[list(ev)])
    return net, planner.build_joint_plan(net, ev), codes


def test_grid_is_bitwise_deterministic_and_chunking_invariant():
    net, plan, codes = grid_case(100_003)
    prog = engine.Program(plan)
    try:
        out, prob = prog.joint(codes, codes.shape[1])
        out2, prob2 = prog.joint(codes, codes.shape[1])
        assert out.tobytes() == out2.tobytes() and prob.tobytes() == prob2.tobytes()
        parts = [(0, 40_000), (40_000, 40_129), (40_129, 100_003)]
        for a, b in parts:
            o, p = prog.joint(np.ascontiguousarray(codes[:, a:b]), b - a)
            assert o.tobytes() == np.ascontiguousarray(out[:, a:b]).tobytes() and p.tobytes() == prob[a:b].tobytes()
        prog.set_graph(False)
        o, p = prog.joint(codes, codes.shape[1])
        assert o.tobytes() == out.tobytes() and p.tobytes() == prob.tobytes()
    finally:
        prog.close()
    ok = ~np.isnan(prob)
    assert ok.mean() > 0.99
    r32, p32, _ = joint_interp.run_joint(plan.words, plan.table_blob, codes[:, :6], n_rows=6, dtype=np.float32)
    np.testing.assert_allclose(out[:, :6], r32, rtol=2e-6, atol=1e-7)


def test_other_run_calls_refuse_a_joint_program():
    net = network("asia")
    plan = planner.build_joint_plan(net, (0,))
    prog = engine.Program(plan)
    try:
        codes = np.zeros((1, 4), dtype=np.uint8)
        with pytest.raises(engine.EngineError, match="sbn_program_joint_host"):
            prog.run(codes, 4)
        with pytest.raises(engine.EngineError, match="sbn_program_joint_host"):
            prog.counts(codes, 4)
    finally:
        prog.close()
    counts = engine.Program(planner.build_counts_plan(net, (0,)))
    try:
        with pytest.raises(engine.EngineError, match="sbn_program_counts_host"):
            engine._check(engine.load().sbn_program_joint_host(counts._h, codes.ctypes.data, 4, 4, None, 0, 0,
                                                               np.zeros(64, np.float32).ctypes.data, 4,
                                                               np.zeros(4, np.float32).ctypes.data))
    finally:
        counts.close()


class _JointRun:
    """A joint program behind the `run` / `set_graph` calls the census drives."""

    def __init__(self, prog):
        self.prog = prog

    def run(self, codes, n_rows):
        return self.prog.joint(codes, n_rows)

    def set_graph(self, on):
        self.prog.set_graph(on)


def test_census_every_joint_instantiation_ran():
    net, plan, codes = grid_case(2000)  # families of 5, 25 and 125 unobserved states: C = 8, passes beyond
    asia = network("asia")
    small = planner.build_joint_plan(asia, (0, 1), [(2,), (0, 2, 5)])  # 2 and 4 unobserved states
    progs = [engine.Program(p, f64=f64) for p in (plan, small) for f64 in (False, True)]
    try:
        runs = [(_JointRun(p), codes if p.plan is plan else np.zeros((2, 500), np.uint8), 2000 if p.plan is plan else 500)
                for p in progs]
        seen = census_many(runs)
    finally:
        for p in progs:
            p.close()
    names = {n for s in seen for n, _ in s}
    for t in ("float", "double"):
        for c in (2, 4, 8):
            assert f"sbn_joint_step<{t}, {c}>" in names, (t, c, sorted(names))
    assert max(int(np.prod(st.cards)) for st in plan.steps if st.kind == planner.KIND_JOINT) == 125


@pytest.mark.parametrize("name", ["alarm", "asia", "grades", "sprinkler"])
def test_reference_joint_goldens(name):
    assert joint_golden_check(getattr(examples, name)(), name, rtol=2e-6) > 50
