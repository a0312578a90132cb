"""Soft evidence on the GPU (engine.Program.run_soft, the likelihoods= keyword): the device against the float64
virtual-evidence oracle (tests/soft_oracle.py) and the CPU replay of the words (tests/soft_interp.py)."""
import numpy as np
import pandas as pd
import pytest

import soft_interp
import soft_oracle
from sorobn_b200 import engine, examples, planner, workloads

pytestmark = pytest.mark.gpu


def lik_for(rng, net, soft, n_rows, zeros=True):
    n_lik = sum(int(net.card[v]) for v in soft)
    lik = rng.random((n_rows, n_lik)) * 10.0 ** rng.integers(-4, 4, size=(n_rows, 1))
    if zeros:
        lik[rng.random(lik.shape) < 0.1] = 0.0
        lik[0] = 0.0
    return lik


def codes_for(net, evidence, n_rows, seed):
    allc = workloads.forward_sample_codes(net, n_rows, seed)
    return np.ascontiguousarray(allc[list(evidence)])


@pytest.mark.parametrize("name", ["asia", "alarm", "sprinkler", "grades"])
def test_posterior_and_log_evidence_against_oracle(name):
    net = getattr(examples, name)()._compiled
    rng = np.random.default_rng(0)
    n = len(net.names)
    dn = soft_oracle.dense(net)
    for trial in range(3):
        perm = [int(v) for v in rng.permutation(n)]
        soft, ev = tuple(perm[:2]), tuple(perm[3:3 + trial])
        query = (perm[2],) if trial != 1 else (perm[0],)  # trial 1: a soft variable is queried
        plan = planner.build_plan(net, query, ev, soft=soft)
        B = 64
        codes, lik = codes_for(net, ev, B, trial), lik_for(rng, net, plan.soft, B)
        prog = engine.Program(plan)
        post, log_ev = prog.run_soft(codes, lik, B, log_evidence=True)
        for b, (hard, s) in enumerate(soft_oracle.rows(net, ev, codes, plan.soft, lik)):
            want = soft_oracle.posterior(dn, [net.names[v] for v in plan.query], hard, s)
            if np.isnan(want).all():
                assert np.isnan(post[:, b]).all() and np.isnan(log_ev[b])
                continue
            np.testing.assert_allclose(post[:, b], want, rtol=1e-6, atol=1e-7)
            le = soft_oracle.log_evidence(dn, hard, s)
            assert abs(log_ev[b] - le) <= 1e-6 * max(1.0, abs(le))
        mplan = planner.build_marginals_plan(net, ev, soft=soft)
        mpost = engine.Program(mplan).run_soft(codes, lik, B)
        ref = soft_interp.run_marginals(mplan.words, mplan.table_blob64, codes, lik, n_rows=B)
        np.testing.assert_allclose(mpost, ref, rtol=1e-5, atol=1e-6)


def test_one_hot_is_hard_evidence_and_ones_drop_the_column():
    bn = examples.alarm()
    net = bn._compiled
    n = 1000
    X = workloads.Workload("alarm", "", ("Burglary",), ("Alarm", "John calls"), n, example="alarm").events(n, 3, bn)
    hard = bn.query_many("Burglary", events=X)
    dom = net.domains[net.index["Alarm"]]
    onehot = (np.asarray(X["Alarm"].to_numpy())[:, None] == np.asarray(dom, dtype=object)[None, :]).astype(float) * 0.25
    soft = bn.query_many("Burglary", events=X[["John calls"]], likelihoods={"Alarm": onehot})
    np.testing.assert_allclose(soft.to_numpy(), hard.to_numpy(), rtol=1e-6)
    dropped = bn.query_many("Burglary", events=X[["John calls"]])
    ones = bn.query_many("Burglary", events=X[["John calls"]], likelihoods={"Alarm": np.ones((n, len(dom)))})
    np.testing.assert_allclose(ones.to_numpy(), dropped.to_numpy(), rtol=1e-6)


def test_scale_invariance_and_log_evidence_shift():
    net = examples.alarm()._compiled
    rng = np.random.default_rng(4)
    soft = (net.index["Alarm"], net.index["Mary calls"])
    plan = planner.build_plan(net, (net.index["Burglary"],), (net.index["John calls"],), soft=soft)
    B = 4096
    codes, lik = codes_for(net, plan.evidence, B, 5), lik_for(rng, net, plan.soft, B, zeros=False)
    prog = engine.Program(plan)
    p0, l0 = prog.run_soft(codes, lik, B, log_evidence=True)
    # any scale: the float32 likelihoods round differently, so the answers agree to float32 rounding
    c = 10.0 ** rng.uniform(-5, 5, size=(B, len(soft)))
    cols = np.repeat(c, [int(net.card[v]) for v in plan.soft], axis=1)
    p1, l1 = prog.run_soft(codes, lik * cols, B, log_evidence=True)
    np.testing.assert_allclose(p1, p0, rtol=1e-6)
    np.testing.assert_allclose(l1, l0 + np.log(c).sum(axis=1), rtol=0, atol=1e-6)  # 1e-6 relative on P(e, lik)
    # powers of two scale exactly: the packed slots are bitwise the same, and only the double log(max) moves
    c = 2.0 ** rng.integers(-20, 20, size=(B, len(soft)))
    cols = np.repeat(c, [int(net.card[v]) for v in plan.soft], axis=1)
    p2, l2 = prog.run_soft(codes, lik * cols, B, log_evidence=True)
    np.testing.assert_array_equal(p2, p0)
    np.testing.assert_allclose(l2, l0 + np.log(c).sum(axis=1), rtol=0, atol=1e-9)


def test_host_and_device_likelihoods_graphs_and_replays_agree_bitwise():
    torch = pytest.importorskip("torch")
    w = workloads.grid10x10()
    bn = w.build()
    net = bn._compiled
    rng = np.random.default_rng(6)
    hidden = [v for v in range(len(net.names)) if net.names[v] not in w.evidence and net.names[v] not in w.query]
    soft = tuple(int(v) for v in rng.choice(hidden, size=5, replace=False))
    plan = planner.build_plan(net, [net.index[q] for q in w.query], [net.index[e] for e in w.evidence], soft=soft)
    B = 20000
    codes, lik = w.codes(bn, B, 7), lik_for(rng, net, plan.soft, B, zeros=False)
    prog = engine.Program(plan)
    a = prog.run_soft(codes, lik, B)
    b = prog.run_soft(codes, torch.as_tensor(lik, device="cuda"), B)
    np.testing.assert_array_equal(a, b)
    # a second call on the same buffers with other likelihoods: the graph replay reads the new values
    lik2 = lik_for(rng, net, plan.soft, B, zeros=False)
    c = prog.run_soft(codes, lik2, B)
    prog.set_graph(0)
    np.testing.assert_array_equal(prog.run_soft(codes, lik2, B), c)
    np.testing.assert_array_equal(prog.run_soft(codes, lik, B), a)
    assert not np.array_equal(a, c)
    # the replay of the words on the CPU, for a few rows
    rows = np.array([1, 2, 3, 4999, B - 1])
    ref = soft_interp.run(plan.words, plan.table_blob64, np.ascontiguousarray(codes[:, rows]), lik2[rows])[0]
    np.testing.assert_allclose(c[:, rows], ref, rtol=2e-5)


@pytest.mark.parametrize("n_soft", [1, 5, 10])
def test_benchmark_grid_with_soft_evidence(n_soft):
    w = workloads.grid10x10()
    bn = w.build()
    net = bn._compiled
    rng = np.random.default_rng(100 + n_soft)
    hidden = [v for v in range(len(net.names)) if net.names[v] not in w.evidence and net.names[v] not in w.query]
    soft = tuple(int(v) for v in rng.choice(hidden, size=n_soft, replace=False))
    plan = planner.build_plan(net, [net.index[q] for q in w.query], [net.index[e] for e in w.evidence], soft=soft)
    B = 100_000
    codes, lik = w.codes(bn, B, 8), lik_for(rng, net, plan.soft, B, zeros=False)
    prog = engine.Program(plan)
    on = prog.run_soft(codes, lik, B)
    prog.set_tiled(10)  # no paired steps
    off = prog.run_soft(codes, lik, B)
    prog.set_tiled(11)
    ok = ~np.isnan(on).any(axis=0)
    assert ok.mean() > 0.99
    np.testing.assert_allclose(on[:, ok], off[:, ok], rtol=2e-5, atol=1e-7)
    rows = np.array([0, 1, 777, 31337, B - 1])
    rows = rows[ok[rows]]
    ref = soft_interp.run(plan.words, plan.table_blob64, np.ascontiguousarray(codes[:, rows]), lik[rows])[0]
    np.testing.assert_allclose(on[:, rows], ref, rtol=2e-5, atol=1e-7)


def test_tiny_likelihoods_are_flagged_and_settled_in_float64():
    w = workloads.grid10x10()
    bn = w.build()
    net = bn._compiled
    rng = np.random.default_rng(9)
    n = 64
    X = w.events(n, 10, bn)
    hidden = [net.names[v] for v in range(len(net.names)) if net.names[v] not in w.evidence and net.names[v] not in w.query]
    soft = sorted(rng.choice(hidden, size=10, replace=False).tolist())
    # each likelihood favours one state by 1e8: rows where the favoured states are improbable fall below 1e-30
    lik = {}
    for s in soft:
        card = len(net.domains[net.index[s]])
        m = np.full((n, card), 1e-8)
        m[np.arange(n), rng.integers(0, card, n)] = 1.0
        lik[s] = m
    got = bn.query_many(*w.query, events=X, likelihoods=lik)
    plan = planner.build_plan(net, [net.index[q] for q in w.query], [net.index[e] for e in w.evidence],
                              soft=[net.index[s] for s in soft])
    L = np.concatenate([lik[s] for s in soft], axis=1)
    codes = w.codes(bn, n, 10)
    ref, total, _ = soft_interp.run(plan.words, plan.table_blob64, codes, L)
    low = total < 1e-30
    assert low.any(), "no row below the float32 range: the case does not test the rescue"
    np.testing.assert_allclose(got.to_numpy().T, ref, rtol=2e-5, atol=1e-7)
    np.testing.assert_allclose(got.to_numpy().T[:, low], ref[:, low], rtol=1e-9)  # settled in float64


def test_other_entry_points_refuse_soft_programs():
    net = examples.asia()._compiled
    plan = planner.build_plan(net, (net.index["Lung cancer"],), (), soft=(net.index["Dispnea"],))
    prog = engine.Program(plan)
    with pytest.raises(engine.EngineError, match="run_soft_host"):
        prog.run(np.zeros((0, 4), np.uint8), 4)
    plain = engine.Program(planner.build_plan(net, (net.index["Lung cancer"],), ()))
    lik, out = np.ones(2, np.float32), np.empty(2, np.float32)
    with pytest.raises(engine.EngineError, match="run_host"):
        engine._check(engine.load().sbn_program_run_soft_host(plain._h, None, 1, 1, lik.ctypes.data, 2, 0,
                                                              out.ctypes.data, 1, None))


@pytest.mark.parametrize("name", ["alarm", "asia", "grades", "sprinkler"])
def test_reference_goldens(name):
    from test_soft_host import golden_check

    assert golden_check(getattr(examples, name)(), name, 1e-6) > 0
