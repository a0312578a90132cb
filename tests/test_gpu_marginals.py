"""Marginals of every variable on the device (BayesNet.marginals / marginals_many, the readout
kernel sbn_marginal_step), against the reference's goldens, the float64 oracle and per-variable
query_many."""
import numpy as np
import pandas as pd
import pytest

from conftest import build_network, case_event, dense_answer, golden_names, load_golden
from oracle import ve_oracle

pytestmark = pytest.mark.gpu

# Both the marginals program and a per-variable program are float32, each within 1e-6 relative of the
# float64 answer (checked against the oracle below); their difference is bounded by the sum of the two.
RTOL_VS_QUERY_MANY = 2e-6


def rel_err(got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return float(np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-30)))


def grid():
    from sorobn_b200 import workloads

    wl = workloads.grid10x10()
    return wl, wl.build(device=0)


@pytest.mark.parametrize("name", golden_names())
def test_marginals_match_goldens_on_device(name):
    golden = load_golden(name)
    bn = build_network(golden)
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    single = [c for c in golden["cases"] if len(c["query"]) == 1][:40]
    assert single
    for case in single:
        ev = case_event(case)
        got = bn.marginals(ev)
        q = case["query"][0]
        want = dense_answer(case, dn.domains)
        if want.sum() == 0:
            assert got[q].empty
            continue
        full = pd.Series(want, index=pd.Index(dn.domains[q], name=q))
        assert rel_err(got[q].to_numpy(), full[full > 0].to_numpy()) < 1e-12, case
        assert list(got[q].index) == list(full.index[full > 0])
    # the batched float32 program against the oracle and against per-variable query_many
    patterns = {}
    for case in golden["cases"]:
        patterns.setdefault(tuple(v for v, _ in case["event"]), []).append(case)
    for ev_vars, cases in list(patterns.items())[:3]:
        if not ev_vars:
            continue
        rows = pd.DataFrame([[dict(c["event"])[v] for v in ev_vars] for c in cases[:20]], columns=list(ev_vars))
        got = bn.marginals_many(rows)
        targets = sorted(set(got.columns.get_level_values(0)))
        assert targets == sorted(n for n in bn.nodes if n not in ev_vars)
        for t in targets[:12]:
            per_var = bn.query_many(t, events=rows).to_numpy()
            mine = got[t].to_numpy()
            ok = ~np.isnan(per_var).any(axis=1)
            assert np.array_equal(np.isnan(mine).any(axis=1), ~ok)
            assert rel_err(mine[ok], per_var[ok]) < RTOL_VS_QUERY_MANY
            for b in range(0, len(rows), 7):
                if ok[b]:
                    want = ve_oracle.query(dn, t, event=rows.iloc[b].to_dict())[1].reshape(-1)
                    assert rel_err(mine[b], want) < 1e-6


def test_single_event_equals_query():
    from sorobn_b200 import examples

    bn = examples.build(examples.NETWORKS["asia"])
    event = {"Smoker": True, "Dispnea": True}
    got = bn.marginals(event)
    assert sorted(got) == sorted(n for n in bn.nodes if n not in event)
    for v, s in got.items():
        want = bn.query(v, event=event)
        pd.testing.assert_series_equal(s, want, rtol=1e-12)
    sub = bn.marginals(event, variables=["Lung cancer"])
    assert list(sub) == ["Lung cancer"]
    with pytest.raises(ValueError):
        bn.marginals(event, variables=["Smoker"])
    with pytest.raises(ValueError):
        bn.marginals_many(pd.DataFrame({"Smoker": [True]}), variables=["Smoker"])
    # impossible evidence: every Series empty, as query
    impossible = bn.marginals({"Tuberculosis": False, "Lung cancer": False, "TB or cancer": True})
    assert all(s.empty for s in impossible.values())


@pytest.mark.parametrize("n", [1, 31, 33, 127, 129, 511, 513, 4095, 4097, 33791, 33793, 67583, 67585])
def test_batch_sizes_around_block_edges(n):
    wl, bn = grid()
    events = wl.events(n, seed=n, bn=bn)
    got = bn.marginals_many(events)
    assert got.shape == (n, 70 * 5)
    assert np.allclose(got.T.groupby(level=0).sum().to_numpy(), 1.0, atol=1e-5)
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    for t in ("g0000", "g0909", sorted(set(got.columns.get_level_values(0)))[33]):
        per_var = bn.query_many(t, events=events).to_numpy()
        assert rel_err(got[t].to_numpy(), per_var) < RTOL_VS_QUERY_MANY
        for b in sorted({0, n // 2, n - 1}):
            want = ve_oracle.query(dn, t, event=events.iloc[b].to_dict())[1].reshape(-1)
            assert rel_err(got[t].iloc[b].to_numpy(), want) < 1e-6


def test_full_benchmark_grid():
    wl, bn = grid()
    n = 100_000
    events = wl.events(n, seed=11, bn=bn)
    a = bn.marginals_many(events).to_numpy()
    b = bn.marginals_many(events).to_numpy()
    assert np.isfinite(a).all()
    assert np.allclose(a.reshape(n, 70, 5).sum(axis=2), 1.0, atol=1e-5)
    assert np.array_equal(a, b), "two runs differ"
    half = n // 2 + 17
    c = np.concatenate([bn.marginals_many(events.iloc[:half]).to_numpy(), bn.marginals_many(events.iloc[half:]).to_numpy()])
    assert np.array_equal(a, c), "results depend on the batch the row is in"
    perm = np.random.default_rng(0).permutation(n)
    d = bn.marginals_many(events.iloc[perm].reset_index(drop=True)).to_numpy()
    assert np.array_equal(a[perm], d), "results depend on the row order"
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    cols = bn.marginals_many(events.iloc[:1]).columns
    targets = list(dict.fromkeys(cols.get_level_values(0)))
    for r in (0, 4242, 99_999):
        ev = events.iloc[r].to_dict()
        for k in (0, 17, 69):
            want = ve_oracle.query(dn, targets[k], event=ev)[1].reshape(-1)
            assert rel_err(a[r, 5 * k:5 * k + 5], want) < 1e-6


def test_bad_rows_are_nan():
    from sorobn_b200 import examples

    bn = examples.build(examples.NETWORKS["asia"])
    rows = pd.DataFrame({"Tuberculosis": [False, True, False], "Lung cancer": [False, False, False],
                         "TB or cancer": [True, True, "maybe"]})
    got = bn.marginals_many(rows)
    assert np.isnan(got.iloc[0]).all()
    assert np.isfinite(got.iloc[1]).all()
    assert np.isnan(got.iloc[2]).all()


def chain(n, prefix, card, rng=None):
    from sorobn_b200 import BayesNet

    names = [f"{prefix}{k:03d}" for k in range(n)]
    bn = BayesNet(*[(names[k - 1], names[k]) for k in range(1, n)])
    if card == 2:
        bn.P[names[0]] = pd.Series({0: 0.5, 1: 0.5})
        for k in range(1, n):
            bn.P[names[k]] = pd.DataFrame({names[k - 1]: [0, 0, 1, 1], names[k]: [0, 1, 0, 1], "p": [0.99, 0.01, 0.02, 0.98]})
    else:
        bn.P[names[0]] = pd.Series({0: 0.3, 1: 0.3, 2: 0.4})
        for k in range(1, n):
            t = rng.dirichlet(np.ones(3) * 0.3, size=3)
            bn.P[names[k]] = pd.DataFrame([(a, b, t[a, b]) for a in range(3) for b in range(3)], columns=[names[k - 1], names[k], "p"])
    bn.prepare()
    return bn, names


def test_extremely_unlikely_row_is_rescued_in_float64():
    bn, names = chain(120, "c", 2)
    ev_vars = names[1:]
    rows = pd.DataFrame([[k % 2 for k in range(1, 120)], [0] * 119], columns=ev_vars)
    got = bn.marginals_many(rows)
    assert list(got.columns.get_level_values(0).unique()) == [names[0]]
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    for b in range(2):
        ev = {v: int(rows[v].iloc[b]) for v in ev_vars}
        want = ve_oracle.query(dn, names[0], event=ev)[1].reshape(-1)
        assert rel_err(got.iloc[b].to_numpy(), want) < (1e-9 if b == 0 else 1e-6)
    single = bn.marginals({v: int(rows[v].iloc[0]) for v in ev_vars})[names[0]]
    assert rel_err(got.iloc[0].to_numpy(), single.to_numpy()) < 1e-12


def test_batch_of_unlikely_rows_goes_through_the_batched_float64_program():
    bn, names = chain(60, "h", 3, np.random.default_rng(5))
    ev_vars = names[1:58]  # two hidden leaves at the end, and the root: three targets
    rows = pd.DataFrame(np.random.default_rng(6).integers(0, 3, size=(40, len(ev_vars))), columns=ev_vars)
    got = bn.marginals_many(rows)
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    targets = list(got.columns.get_level_values(0).unique())
    assert targets == [names[0], names[58], names[59]]
    for b in range(0, 40, 3):
        ev = {v: int(rows[v].iloc[b]) for v in ev_vars}
        for t in targets:
            want = ve_oracle.query(dn, t, event=ev)[1].reshape(-1)
            assert rel_err(got[t].iloc[b].to_numpy(), want) < 1e-9


def test_kernel_census_shows_both_readout_instantiations():
    from kernel_census import census
    from sorobn_b200 import engine, planner

    wl, bn = grid()
    net = bn._compiled
    plan = planner.build_marginals_plan(net, [net.index[e] for e in wl.evidence])
    codes = wl.codes(bn, 1000, seed=2)
    names32 = {name for name, _ in census(engine.Program(plan, device=0), codes, 1000)}
    names64 = {name for name, _ in census(engine.Program(plan, device=0, f64=True), codes, 1000)}
    assert any(n.startswith("sbn_marginal_step<float") for n in names32), names32
    assert any(n.startswith("sbn_marginal_step<double") for n in names64), names64
    assert not any("normalise" in n for n in names32 | names64)


def test_other_engine_paths_agree(monkeypatch):
    from sorobn_b200 import engine, planner

    wl, bn = grid()
    net = bn._compiled
    plan = planner.build_marginals_plan(net, [net.index[e] for e in wl.evidence])
    codes = wl.codes(bn, 3000, seed=4)
    ref = engine.Program(plan, device=0).run(codes, 3000).astype(np.float64)
    assert np.isfinite(ref).all()

    def check(prog):
        got = prog.run(codes, 3000).astype(np.float64)
        assert np.max(np.abs(got - ref)) < 3e-6
        prog.close()

    monkeypatch.setenv("SOROBN_B200_PAIR", "0")
    check(engine.Program(plan, device=0))
    monkeypatch.delenv("SOROBN_B200_PAIR")
    for mode in (0, 4, 7, 9):
        p = engine.Program(plan, device=0)
        p.set_tiled(mode)
        check(p)
    for g in (0, 3):
        p = engine.Program(plan, device=0)
        p.set_graph(g)
        check(p)
    for var in ("SOROBN_B200_CHAIN", "SOROBN_B200_TMA"):
        monkeypatch.setenv(var, "1")
        check(engine.Program(plan, device=0))
        monkeypatch.delenv(var)
    # the P(event) entry point refuses a marginals program
    with pytest.raises(engine.EngineError):
        engine.Program(plan, device=0).evidence(codes, 3000)
