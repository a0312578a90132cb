"""Counts plans (planner.build_counts_plan, version-6 programs) and the EM oracle, checked on the CPU.

oracle/program_interp.py executes the serialised words with numpy, so a pass here means the bucket
choice, the keys, the strides, the count-table offsets and the slot reuse the device will see are
right: the counts must equal tests/em_oracle.py (per row, `ve_oracle.query` of the unobserved family
members given the observed cells)."""

import numpy as np
import pytest

import em_oracle
from oracle import program_interp, ve_oracle
from sorobn_b200 import examples, planner, workloads

EXAMPLES = ["alarm", "asia", "sprinkler", "grades"]


def oracle_net(bn):
    return ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)


def rows_of(net, codes, observed):
    return [{net.names[v]: net.domains[v][int(codes[i, b])] for i, v in enumerate(observed)} for b in range(codes.shape[1])]


def oracle_vector(net, dn, rows):
    want = em_oracle.expected_counts(dn, rows)
    return np.concatenate([want[n].reshape(-1) for n in net.names])


def sample(net, n, seed, observed):
    allc = workloads.forward_sample_codes(net, n, seed)
    return np.ascontiguousarray(allc[list(observed)])


def check(bn, missing, n=40, seed=0, rtol=1e-12):
    net = bn._compiled
    dn = oracle_net(bn)
    observed = [v for v in range(len(net.names)) if v not in set(missing)]
    plan = planner.build_counts_plan(net, observed)
    assert plan.version == 6 and plan.words[1] == 6 and plan.n_counts == planner.count_layout(net)[1]
    codes = sample(net, n, seed, observed)
    got, prob = program_interp.run_counts(plan.words, plan.table_blob64, codes, n_rows=n)
    rows = rows_of(net, codes, observed)
    want = oracle_vector(net, dn, rows)
    assert np.allclose(got, want, rtol=rtol, atol=1e-12 * n), (missing, np.max(np.abs(got - want)))
    p_want = np.array([em_oracle._p(dn, r) for r in rows])
    assert np.allclose(prob, p_want, rtol=1e-12)
    # every family's counts sum to the number of rows
    offsets, _ = planner.count_layout(net)
    for v in range(len(net.names)):
        assert abs(got[offsets[v]:offsets[v] + net.cpt[v].size].sum() - n) < 1e-9 * n
    return plan, got


@pytest.mark.parametrize("name", EXAMPLES)
def test_every_single_missing_column_matches_the_oracle(name):
    bn = getattr(examples, name)()
    for v in range(len(bn.nodes)):
        check(bn, (v,))


@pytest.mark.parametrize("name", EXAMPLES)
def test_several_missing_columns_match_the_oracle(name):
    bn = getattr(examples, name)()
    n_vars = len(bn.nodes)
    rng = np.random.default_rng(1)
    for k in (2, 3):
        for _ in range(4):
            check(bn, tuple(sorted(rng.choice(n_vars, size=k, replace=False).tolist())), seed=k)


@pytest.mark.parametrize("name", EXAMPLES)
def test_a_fully_observed_pattern_is_the_histogram(name):
    bn = getattr(examples, name)()
    net = bn._compiled
    n = 200
    codes = sample(net, n, 5, range(len(net.names)))
    plan = planner.build_counts_plan(net, range(len(net.names)))
    assert all(st.kind == planner.KIND_COUNT and not st.inputs for st in plan.steps if st.kind == planner.KIND_COUNT)
    got, _ = program_interp.run_counts(plan.words, plan.table_blob64, codes)
    offsets, _ = planner.count_layout(net)
    for v in range(len(net.names)):
        scope = net.scope(v)
        want = np.zeros(net.cpt[v].shape)
        np.add.at(want, tuple(codes[u] for u in scope), 1.0)
        assert np.array_equal(got[offsets[v]:offsets[v] + want.size], want.reshape(-1))


def test_a_latent_variable():
    bn = examples.sprinkler()
    check(bn, (bn._compiled.index["Cloudy"],))
    bn = examples.asia()
    net = bn._compiled
    check(bn, (net.index["TB or cancer"], net.index["Tuberculosis"]))


def test_rows_without_any_observed_cell_give_the_prior():
    bn = examples.grades()
    net = bn._compiled
    plan = planner.build_counts_plan(net, ())
    got, prob = program_interp.run_counts(plan.words, plan.table_blob64, np.zeros((0, 3), np.uint8), n_rows=3)
    want = oracle_vector(net, oracle_net(bn), [{}] * 3)
    assert np.allclose(got, want, rtol=1e-12) and np.allclose(prob, 1.0)


@pytest.mark.parametrize("wl", ["grid10x10", "dag50"])
def test_large_networks_with_several_latent_variables(wl):
    w = workloads.WORKLOADS[wl]()
    bn = w.build()
    net = bn._compiled
    hidden = [v for v in range(len(net.names)) if net.names[v] not in w.evidence]
    # the workload's unobserved variables are latent, plus three of its columns
    missing = tuple(sorted(hidden + [net.index[e] for e in w.evidence[:3]]))
    plan, _ = check(bn, missing, n=3, seed=2, rtol=1e-10)
    # the readouts go through the downward pass: some count step reads a bucket whose message comes from above
    assert sum(st.kind == planner.KIND_COUNT and any(f.is_slot for f, _, _ in st.inputs) for st in plan.steps) > 5


def test_float32_interpretation_stays_within_2e_6():
    w = workloads.grid10x10()
    bn = w.build()
    net = bn._compiled
    observed = [net.index[e] for e in w.evidence[3:]]
    plan = planner.build_counts_plan(net, observed)
    codes = sample(net, 64, 4, observed)
    got64, _ = program_interp.run_counts(plan.words, plan.table_blob64, codes)
    got32, prob = program_interp.run_counts(plan.words, plan.table_blob, codes, dtype=np.float32)
    assert np.isfinite(prob).all()
    big = got64 > 1e-3
    assert np.max(np.abs(got32 - got64)[big] / got64[big]) < 2e-6


def test_rows_out_of_range_and_impossible_rows_add_nothing():
    bn = examples.sprinkler()
    net = bn._compiled
    ev = [net.index["Rain"], net.index["Sprinkler"], net.index["Wet grass"]]
    plan = planner.build_counts_plan(net, ev)
    # Rain = F, Sprinkler = F, Wet grass = T has probability zero
    codes = np.array([[0, 1], [0, 1], [1, 1]], dtype=np.uint8)  # domains sorted: False = 0
    got, prob = program_interp.run_counts(plan.words, plan.table_blob64, codes)
    assert np.isnan(prob[0]) and prob[1] > 0
    want = oracle_vector(net, oracle_net(bn), rows_of(net, codes[:, 1:], ev))
    assert np.allclose(got, want, rtol=1e-12)


def test_a_count_step_beyond_the_readout_bound_is_refused(monkeypatch):
    w = workloads.dag50()
    bn = w.build()
    net = bn._compiled
    planner.build_counts_plan(net, [net.index[e] for e in w.evidence])
    monkeypatch.setattr(planner, "MARGINAL_MAX_Z", 8)
    with pytest.raises(ValueError, match="too large for a count step"):
        planner.build_counts_plan(net, [net.index[e] for e in w.evidence])


@pytest.mark.parametrize("wl", ["grid10x10", "dag50"])
def test_refreshed_tables_equal_a_fresh_plan_bitwise(wl):
    w = workloads.WORKLOADS[wl]()
    bn = w.build()
    net = bn._compiled
    observed = [net.index[e] for e in w.evidence[2:]]
    plan = planner.build_counts_plan(net, observed)
    rng = np.random.default_rng(0)
    cpts = []
    for c in net.cpt:
        x = rng.random(c.shape)
        cpts.append(x / x.sum(axis=-1, keepdims=True))
    blob32, blob64 = planner.refresh_tables(plan, cpts)
    fresh = planner.build_counts_plan(planner.CompiledNet(net.names, net.domains, net.parents, cpts), observed)
    assert np.array_equal(fresh.words, plan.words)
    assert blob64.tobytes() == fresh.table_blob64.tobytes()
    assert blob32.tobytes() == fresh.table_blob.tobytes()


@pytest.mark.parametrize("wl", ["grid10x10", "dag50"])
def test_refreshed_tables_of_a_marginals_plan_are_its_own_blobs(wl):
    w = workloads.WORKLOADS[wl]()
    net = w.build()._compiled
    plan = planner.build_marginals_plan(net, [net.index[e] for e in w.evidence[2:]])
    blob32, blob64 = planner.refresh_tables(plan, net.cpt)
    assert blob64.tobytes() == plan.table_blob64.tobytes()
    assert blob32.tobytes() == plan.table_blob.tobytes()


def test_version_4_and_5_words_are_unchanged_by_the_counts_planner():
    bn = examples.asia()
    net = bn._compiled
    p5 = planner.build_marginals_plan(net, [0, 2])
    assert p5.version == 5 and all(st.kind != planner.KIND_COUNT for st in p5.steps)
    assert p5.words[8] == -1 and p5.words[10] == 0


def test_oracle_em_never_decreases_the_log_likelihood_with_a_latent_cloudy():
    bn = examples.sprinkler()
    dn = oracle_net(bn)
    net = bn._compiled
    codes = sample(net, 300, 3, range(len(net.names)))
    rows = [r for r in rows_of(net, codes, range(len(net.names)))]
    for r in rows:
        del r["Cloudy"]
    # a start that breaks the symmetry of the latent variable
    start = ve_oracle.DenseNet(nodes=list(dn.nodes), parents=dict(dn.parents), domains=dict(dn.domains))
    rng = np.random.default_rng(7)
    for v in dn.nodes:
        x = rng.random(dn.cpt[v].shape) + 0.1
        start.cpt[v] = x / x.sum(axis=-1, keepdims=True)
    lls, cur = [], start
    for _ in range(12):
        cur, ll = em_oracle.em_step(cur, rows)
        lls.append(ll)
    assert all(b >= a - 1e-9 * abs(a) for a, b in zip(lls, lls[1:])), lls
    assert lls[-1] > lls[0]
