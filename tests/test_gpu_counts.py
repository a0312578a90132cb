"""Expected counts and EM on the device (BayesNet.expected_counts / fit_em, the count kernel
sbn_count_step), against the float64 oracle (tests/em_oracle.py), marginals_many, fit and the
programs' own float64 twins."""
import numpy as np
import pandas as pd
import pytest

import em_oracle
from oracle import ve_oracle
from sorobn_b200 import examples, planner, workloads

pytestmark = pytest.mark.gpu

RTOL = 2e-6


def oracle_net(bn):
    return ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)


def frame(bn, n, seed, missing=(), frac=1.0, latent=()):
    """n forward-sampled rows; the columns in `missing` are NaN in a fraction `frac` of the rows, the
    nodes in `latent` have no column."""
    net = bn._compiled
    codes = workloads.forward_sample_codes(net, n, seed)
    rng = np.random.default_rng(seed + 1)
    cols = {}
    for v, name in enumerate(net.names):
        if name in latent:
            continue
        values = np.asarray(net.domains[v], dtype=object)[codes[v]]
        if name in missing:
            values = values.copy()
            values[rng.random(n) < frac] = None
        cols[name] = values
    return pd.DataFrame(cols)


def oracle_counts(bn, X):
    rows = [{k: v for k, v in r.items() if v is not None and v == v} for r in X.to_dict("records")]
    return em_oracle.expected_counts(oracle_net(bn), rows)


def assert_close(got, want, rtol=RTOL):
    for node, series in got.items():
        w = want[node].reshape(-1)
        g = series.to_numpy()
        assert g.shape == w.shape, node
        assert np.all(np.abs(g - w) <= rtol * np.abs(w) + 1e-12 * max(1.0, w.sum())), (node, np.max(np.abs(g - w)))


@pytest.mark.parametrize("name", ["alarm", "asia", "sprinkler", "grades"])
def test_examples_against_the_oracle(name):
    bn = getattr(examples, name)(device=0)
    nodes = bn.nodes
    for miss in ([nodes[0]], nodes[1:3], nodes[-3:]):
        X = frame(bn, 700, 3, missing=miss, frac=0.4)
        got = bn.expected_counts(X)
        assert list(got) == list(nodes)
        for node, s in got.items():
            assert list(s.index.names) == [*bn.parents.get(node, []), node]
            assert abs(s.sum() - len(X)) < 1e-6 * len(X)  # float32 posteriors sum to one within 1e-7
        assert_close(got, oracle_counts(bn, X))
    # a latent variable
    X = frame(bn, 500, 4, latent=[nodes[len(nodes) // 2]])
    assert_close(bn.expected_counts(X), oracle_counts(bn, X))


@pytest.mark.parametrize("n", [1, 127, 128, 129, 4 * 132 * 128 - 1, 4 * 132 * 128 + 1, 3 * 4 * 132 * 128 + 77])
def test_row_counts_around_block_and_grid_edges(n):
    bn = examples.asia(device=0)
    X = frame(bn, n, 11, missing=["Smoker", "Tuberculosis"], frac=0.5)
    assert_close(bn.expected_counts(X), oracle_counts(bn, X))


def test_benchmark_grid_on_a_row_sample():
    wl = workloads.grid10x10()
    bn = wl.build(device=0)
    latent = [n for n in bn.nodes if n not in wl.evidence][:20]
    X = frame(bn, 8, 5, missing=list(wl.evidence[:2]), frac=0.5, latent=latent)
    assert_close(bn.expected_counts(X), oracle_counts(bn, X))


def test_dag50_with_three_missing_columns():
    wl = workloads.dag50()
    bn = wl.build(device=0)
    X = frame(bn, 12, 6, missing=list(wl.evidence[:3]), frac=1.0)
    X = X[list(wl.evidence)]
    assert_close(bn.expected_counts(X), oracle_counts(bn, X))


def test_single_unobserved_member_equals_marginals_many():
    bn = examples.asia(device=0)
    X = frame(bn, 5000, 8, missing=["Lung cancer"], frac=1.0)
    got = bn.expected_counts(X)
    obs = X.drop(columns=["Lung cancer"])
    marg = bn.marginals_many(obs, variables=["Lung cancer"])["Lung cancer"]
    # family of "Lung cancer" = (Smoker, Lung cancer): sum the marginal per Smoker value
    want = marg.groupby(obs["Smoker"].to_numpy()).sum()
    s = got["Lung cancer"]
    for smoker in want.index:
        for state in want.columns:
            w = want.loc[smoker, state]
            assert abs(s.loc[(smoker, state)] - w) <= RTOL * w


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


def test_rows_below_the_float32_range_are_settled_in_float64():
    bn, names = chain(60, 3, np.random.default_rng(5))
    rows = pd.DataFrame(np.random.default_rng(6).integers(0, 3, size=(40, 57)), columns=names[1:58])
    dn = oracle_net(bn)
    p = [ve_oracle.evidence_probability(dn, {k: int(v) for k, v in r.items()}) for r in rows.to_dict("records")]
    keep = [b for b in range(40) if p[b] > 0]
    rows = rows.iloc[keep].reset_index(drop=True)
    assert sum(p[b] < 1e-30 for b in keep) > 8  # more than a handful: the batched float64 program runs
    got = bn.expected_counts(rows)
    want = oracle_counts(bn, rows.astype(object))
    assert_close(got, want, rtol=1e-9)


def test_impossible_rows_raise():
    bn = examples.sprinkler(device=0)
    X = pd.DataFrame({"Rain": [False, True], "Sprinkler": [False, True], "Wet grass": [True, True]})
    with pytest.raises(ValueError, match="probability zero"):
        bn.expected_counts(X)
    with pytest.raises(ValueError, match="not a state"):
        bn.expected_counts(pd.DataFrame({"Rain": ["maybe"]}))


def test_two_runs_are_bitwise_equal():
    wl = workloads.grid10x10()
    bn = wl.build(device=0)
    X = frame(bn, 20000, 9, missing=list(wl.evidence[:2]), frac=0.3,
              latent=[n for n in bn.nodes if n not in wl.evidence])
    a = bn.expected_counts(X)
    b = bn.expected_counts(X)
    for node in a:
        assert a[node].to_numpy().tobytes() == b[node].to_numpy().tobytes()


def test_set_tables_equals_a_fresh_program_bitwise():
    from sorobn_b200 import engine

    wl = workloads.dag50()
    bn = wl.build(device=0)
    net = bn._compiled
    observed = [net.index[e] for e in wl.evidence[3:]]
    plan = planner.build_counts_plan(net, observed)
    codes = np.ascontiguousarray(workloads.forward_sample_codes(net, 3000, 1)[observed])
    rng = np.random.default_rng(2)
    cpts = []
    for c in net.cpt:
        x = rng.random(c.shape) + 0.05
        cpts.append(x / x.sum(axis=-1, keepdims=True))
    fresh_plan = planner.build_counts_plan(planner.CompiledNet(net.names, net.domains, net.parents, cpts), observed)
    for f64 in (False, True):
        prog = engine.Program(plan, device=0, f64=f64)
        prog.counts(codes, 3000)  # captures the graph
        blob32, blob64 = planner.refresh_tables(plan, cpts)
        prog.set_tables(blob64 if f64 else blob32)
        got, p_got = prog.counts(codes, 3000)  # replays it
        fresh = engine.Program(fresh_plan, device=0, f64=f64)
        want, p_want = fresh.counts(codes, 3000)
        assert got.tobytes() == want.tobytes() and p_got.tobytes() == p_want.tobytes()
        with pytest.raises(engine.EngineError):
            prog.run(codes, 3000)
        prog.close()
        fresh.close()
    p4 = planner.build_plan(net, [0], observed)
    with pytest.raises(engine.EngineError):
        engine.Program(p4, device=0).set_tables(p4.table_blob)


def test_fit_em_on_complete_data_is_fit():
    bn = examples.sprinkler(device=0)
    X = frame(bn, 20000, 12)
    ref = examples.sprinkler(device=0)
    ref.P = {}
    ref.fit(X)
    em = examples.sprinkler(device=0)
    em.P = {}
    em.fit_em(X)
    assert len(em.em_log_likelihood_) == 2
    for node in ref.P:
        assert list(em.P[node].index) == list(ref.P[node].index), node
        assert np.allclose(em.P[node].to_numpy(), ref.P[node].to_numpy(), rtol=1e-12, atol=0)


def test_fit_em_recovers_cpts_where_available_case_fit_does_not():
    truth = examples.sprinkler(device=0)
    X = frame(truth, 200_000, 13)
    rng = np.random.default_rng(14)
    # Rain is missing at random given Wet grass: mostly when the grass is wet
    p_miss = np.where(X["Wet grass"].to_numpy(dtype=bool), 0.7, 0.1)
    X.loc[rng.random(len(X)) < p_miss, "Rain"] = None
    avail = examples.sprinkler(device=0)
    avail.P = {}
    avail.fit(X)
    em = examples.sprinkler(device=0)
    em.P = {}
    em.fit_em(X)
    lls = em.em_log_likelihood_
    assert all(b >= a - 1e-9 * abs(a) for a, b in zip(lls, lls[1:])), lls
    ta, tb = oracle_net(truth), oracle_net(em)
    for node in truth.nodes:
        assert np.max(np.abs(tb.cpt[node] - ta.cpt[node])) < 0.02, node
    assert np.max(np.abs(oracle_net(avail).cpt["Rain"] - ta.cpt["Rain"])) > 0.02
    # a later partial_fit continues from the expected counts: every row is behind each family's totals
    assert abs(em._P_sizes["Rain"].sum() - len(X)) < 1e-6 * len(X)
    assert abs(em._P_sizes["Cloudy"] - len(X)) < 1e-6 * len(X)


def test_fit_em_with_a_latent_variable_needs_a_start():
    bn = examples.sprinkler(device=0)
    X = frame(bn, 1000, 15, latent=["Cloudy"])
    fresh = examples.sprinkler(device=0)
    fresh.P = {}
    with pytest.raises(ValueError, match="initial CPTs"):
        fresh.fit_em(X)
    bn.fit_em(X, max_iter=20)
    lls = bn.em_log_likelihood_
    assert all(b >= a - 1e-9 * abs(a) for a, b in zip(lls, lls[1:])), lls


def test_kernel_census_shows_the_count_kernel():
    import kernel_census

    bn = examples.asia(device=0)
    net = bn._compiled
    plan = planner.build_counts_plan(net, [0, 1, 2, 3])
    from sorobn_b200 import engine

    prog = engine.Program(plan, device=0)
    codes = np.ascontiguousarray(workloads.forward_sample_codes(net, 1000, 3)[[0, 1, 2, 3]])

    class Run:  # the census calls run(); a counts program runs through counts()
        def set_graph(self, mode):
            prog.set_graph(mode)

        def run(self, codes, n):
            return prog.counts(codes, n)

    names = {name for name, _ in kernel_census.census(Run(), codes, 1000)}
    assert any(n.startswith("sbn_count_step<float") for n in names), names
    assert "sbn_count_reduce" in names, names


def test_more_missingness_patterns_than_cached_programs():
    bn = examples.asia(device=0)
    bn.max_cached_programs = 8
    net = bn._compiled
    codes = workloads.forward_sample_codes(net, 400, 21)
    rng = np.random.default_rng(22)
    cols = {}
    for v, name in enumerate(net.names):
        values = np.asarray(net.domains[v], dtype=object)[codes[v]]
        values[rng.random(400) < 0.3] = None
        cols[name] = values
    X = pd.DataFrame(cols)
    assert len(bn._count_patterns(X)) > 3 * bn.max_cached_programs
    assert_close(bn.expected_counts(X), oracle_counts(bn, X))
    assert len(bn._engine_cache) <= bn.max_cached_programs
