"""Joint plans (planner.build_joint_plan, version-11 programs), checked on the CPU.

tests/joint_interp.py replays the words as the device runs them.  The float64 ground truth is `ve_oracle.query`
of each group's unobserved members given the row's observed cells, asked on Pearl's virtual-child network of the
row when it has likelihoods (soft_oracle), the way tests/em_oracle.py asks it per family."""
import numpy as np
import pytest

import joint_interp
import soft_oracle
from oracle import program_interp, ve_oracle
from sorobn_b200 import examples, planner, synthetic, workloads
from sorobn_b200.bayes_net import BayesNet

EXAMPLES = ["alarm", "asia", "sprinkler", "grades"]


def network(name):
    if name in EXAMPLES:
        return getattr(examples, name)()._compiled
    n, p, s = {"dag12": (12, 3, 3), "dag20": (20, 2, (2, 3, 4)), "dag30": (30, 3, 2)}[name]
    return synthetic.load(synthetic.random_dag(n, p, s, seed=len(name)), BayesNet)._compiled


def oracle_group(net, dn, M, hard, soft):
    """P(M | hard, soft) as a compact float64 vector over the members M (var ids), the first one fastest; NaN
    throughout for an impossible row."""
    names = [net.names[u] for u in M]
    vnet, event, _ = soft_oracle.virtual(dn, soft)
    size = int(np.prod([int(net.card[u]) for u in M]))
    if event is None or ({**hard, **event} and ve_oracle.evidence_probability(vnet, {**hard, **event}) <= 0):
        return np.full(size, np.nan)
    got, values, _ = ve_oracle.query(vnet, *names, event={**hard, **event})
    arr = np.transpose(values, [list(got).index(n) for n in names])  # member order, the first slowest
    return np.transpose(arr, list(reversed(range(len(M))))).reshape(-1)


def check(net, evidence, groups=None, soft=(), n=24, seed=0, lik_zero_row=False):
    """Replay the plan in float64 against the oracle (1e-9) and return (plan, output, P(observed))."""
    rng = np.random.default_rng(seed)
    plan = planner.build_pattern_plan(net, "joint", evidence, soft=soft, groups=groups)
    assert plan.version == 11 and int(plan.words[1]) == 11 and int(plan.words[10]) == 0
    full = workloads.forward_sample_codes(net, n, seed)
    codes = np.ascontiguousarray(full[list(evidence)]) if evidence else np.zeros((0, n), dtype=np.uint8)
    n_lik = sum(int(net.card[v]) for v in plan.soft)
    lik = rng.random((n, n_lik)) * 10.0 ** rng.integers(-3, 3, size=(n, 1)) if plan.soft else None
    if lik is not None and lik_zero_row:
        lik[0] = 0.0
    out, prob, _ = joint_interp.run_joint(plan.words, plan.table_blob64, codes, lik=lik, n_rows=n)
    dn = soft_oracle.dense(net)
    rows = soft_oracle.rows(net, evidence, codes, plan.soft, lik if lik is not None else np.zeros((n, 0)))
    for g, q0 in zip(plan.groups, plan.group_rows):
        M = [u for u in g if u not in evidence]
        assert (q0 < 0) == (not M)
        if not M:
            continue
        cs = int(np.prod([int(net.card[u]) for u in M]))
        for b, (hard, s) in enumerate(rows):
            want = oracle_group(net, dn, M, hard, s)
            got = out[q0:q0 + cs, b]
            if np.isnan(want).all():
                assert np.isnan(got).all() and np.isnan(prob[b])
                continue
            assert np.allclose(got, want, rtol=1e-9, atol=1e-12), ([net.names[u] for u in g], b, got, want)
    return plan, out, prob, codes, lik


def missing_patterns(net, seed, k=3):
    rng = np.random.default_rng(seed)
    n = len(net.names)
    out = []
    for j in range(k):
        hidden = set(int(v) for v in rng.choice(n, size=min(n - 1, 1 + j * max(1, n // 4)), replace=False))
        out.append(tuple(v for v in range(n) if v not in hidden))
    return out


@pytest.mark.parametrize("name", EXAMPLES + ["dag12", "dag20", "dag30"])
def test_family_posteriors_match_the_oracle(name):
    net = network(name)
    for j, ev in enumerate(missing_patterns(net, 7)):
        check(net, ev, seed=j)


@pytest.mark.parametrize("name", ["alarm", "asia", "dag12"])
def test_latent_nodes_and_no_evidence(name):
    net = network(name)
    check(net, ())
    check(net, tuple(range(0, len(net.names), 2)), seed=3)


@pytest.mark.parametrize("name", ["alarm", "asia", "grades", "dag20"])
def test_soft_evidence_matches_the_virtual_evidence_oracle(name):
    net = network(name)
    rng = np.random.default_rng(11)
    perm = [int(v) for v in rng.permutation(len(net.names))]
    soft, ev = tuple(perm[:2]), tuple(perm[2:2 + len(perm) // 3])
    plan, out, prob, _, _ = check(net, ev, soft=soft, seed=5, lik_zero_row=True)
    assert np.isnan(prob[0]) and np.isnan(out[:, 0]).all() and not np.isnan(out[:, 1:]).any()


def test_pairs_outside_any_family_get_a_table_of_ones_and_keep_their_values():
    net = network("alarm")
    idx = net.index
    fam = ("Alarm", "Burglary")  # within the family of Alarm
    far = ("John calls", "Burglary")  # in no CPT's scope
    groups = [tuple(idx[n] for n in fam), tuple(idx[n] for n in far), (idx["Burglary"],)]
    plan, *_ = check(net, (), groups=groups)
    assert plan.ones == ((idx["John calls"], idx["Burglary"]),)
    assert int(plan.words[4]) == len(plan.tables) + 1
    # observing one member leaves a single unobserved member: no table needed
    plan, *_ = check(net, (idx["Burglary"],), groups=groups)
    assert plan.ones == () and plan.group_rows[2] == -1
    # the default groups (families) never need one
    assert planner.build_joint_plan(net, ()).ones == ()
    # the families plan the counts plan's upward pass
    fams = planner.build_joint_plan(net, (idx["Mary calls"],))
    counts = planner.build_counts_plan(net, (idx["Mary calls"],))
    assert fams.order == counts.order and fams.tables == counts.tables


@pytest.mark.parametrize("name", ["asia", "sprinkler", "dag12"])
def test_explicit_groups_with_and_without_ones(name):
    net = network(name)
    n = len(net.names)
    groups = [(0, n - 1), (n - 1, 0), (1,), (2, 0, 1), tuple(range(min(4, n)))[::-1]]
    for j, ev in enumerate([(), (n - 1,), (0, 2)]):
        check(net, ev, groups=groups, seed=j)


@pytest.mark.parametrize("name", ["alarm", "dag20"])
def test_rows_sum_to_the_expected_counts(name):
    net = network(name)
    ev = missing_patterns(net, 2)[1]
    plan, out, prob, codes, _ = check(net, ev, n=30)
    counts_plan = planner.build_counts_plan(net, ev)
    want, p_counts = program_interp.run_counts(counts_plan.words, counts_plan.table_blob64, codes)
    assert np.allclose(prob, p_counts, rtol=1e-12)
    offsets, _ = planner.count_layout(net)
    got = np.zeros_like(want)
    for v, q0 in zip(range(len(net.names)), plan.group_rows):
        scope = net.scope(v)
        shape = [int(net.card[u]) for u in scope]
        dense = np.zeros([out.shape[1], *shape])
        M = [u for u in scope if u not in ev]
        for b in range(out.shape[1]):
            index = [int(codes[ev.index(u), b]) if u in ev else slice(None) for u in scope]
            if not M:
                dense[(b, *index)] = 1.0
                continue
            cs = int(np.prod([int(net.card[u]) for u in M]))
            block = out[q0:q0 + cs, b].reshape([int(net.card[u]) for u in reversed(M)]).transpose()
            dense[(b, *index)] = block
        got[offsets[v]:offsets[v] + dense[0].size] = dense.sum(axis=0).reshape(-1)
    assert np.allclose(got, want, rtol=1e-10, atol=1e-12)


def test_kind_7_words():
    net = network("asia")
    ev = (net.index["Smoker"],)
    groups = [(net.index["Dispnea"], net.index["Smoker"], net.index["Tuberculosis"])]
    plan = planner.build_joint_plan(net, ev, groups)
    hdr = [int(x) for x in plan.words[:12]]
    assert hdr[:4] == [planner.MAGIC, 11, 1, 1] and hdr[7] == plan.Q == 4 and hdr[10] == 0 and hdr[11] == 0
    _, _, _, _, steps = joint_interp.parse(plan.words)
    (st,) = [s for s in steps if s["kind"] == 7]
    assert st["out_slot"] == -1 and st["q_offset"] == 0 and st["cards"] == [2, 2]
    assert plan.steps[-1].out_vars == (net.index["Dispnea"], net.index["Tuberculosis"])


def test_bad_groups_raise():
    net = network("asia")
    with pytest.raises(ValueError, match="duplicate"):
        planner.build_joint_plan(net, (), [(0, 0)])
    with pytest.raises(ValueError, match="observed completely"):
        planner.build_joint_plan(net, (0, 1), [(0, 1)])
    with pytest.raises(ValueError, match="groups go with kind 'joint'"):
        planner.build_pattern_plan(net, "counts", (), groups=[(0,)])


def test_a_group_too_large_for_a_readout_names_the_group():
    spec = synthetic.random_dag(12, 0, 8, seed=1)  # independent nodes: a group of 8 spans no CPT
    net = synthetic.load(spec, BayesNet)._compiled
    with pytest.raises(ValueError, match=r"group \['v00'"):
        planner.build_joint_plan(net, (), [tuple(range(8))])


def test_other_kinds_keep_their_words():
    """A joint group argument changes nothing for the other kinds: the counts plan is the same with or without the
    joint machinery (the committed digests of tests/golden/plan_words_parent.json pin every other kind)."""
    net = network("alarm")
    a = planner.build_counts_plan(net, (0, 3))
    b = planner.build_pattern_plan(net, "counts", (0, 3))
    assert np.array_equal(a.words, b.words)
