"""Gibbs sampling on the device (BASELINE.json configs[4]; reference: bayes_net.py:665-737).

The reference's chain cannot be reproduced draw for draw (its RNG is Python's `random` plus a
Cython alias sampler), so parity is distributional: the chain's frequencies must converge to
the exact posterior -- which is itself pinned to the reference -- and the run must be
reproducible from the seed."""
import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu


def test_gibbs_converges_to_exact_posterior_on_reference_examples():
    from sorobn_b200 import examples

    cases = [
        (examples.sprinkler, ("Rain",), {"Sprinkler": True}),            # bayes_net.py:683-688
        (examples.alarm, ("Burglary",), {"John calls": True, "Mary calls": True}),
        (examples.grades, ("Letter", "SAT"), {"Intelligence": "Smart"}),
        (examples.sprinkler, ("Cloudy", "Rain"), {}),
    ]
    for make, query, event in cases:
        bn = make(seed=42)
        exact = bn.query(*query, event=event)
        got = bn.query(*query, event=event, algorithm="gibbs", n_iterations=400_000)
        assert got.name == exact.name and list(got.index.names) == list(exact.index.names)
        assert np.isclose(got.sum(), 1.0, atol=1e-5)
        both = pd.concat([exact, got], axis=1).fillna(0.0)
        assert np.abs(both.iloc[:, 0] - both.iloc[:, 1]).max() < 0.01, both


def test_gibbs_is_reproducible_from_the_seed():
    from sorobn_b200 import examples

    a = examples.alarm(seed=7).query("Alarm", event={"John calls": True}, algorithm="gibbs", n_iterations=5000)
    b = examples.alarm(seed=7).query("Alarm", event={"John calls": True}, algorithm="gibbs", n_iterations=5000)
    c = examples.alarm(seed=8).query("Alarm", event={"John calls": True}, algorithm="gibbs", n_iterations=5000)
    pd.testing.assert_series_equal(a, b)
    assert not a.equals(c)


def test_one_chain_per_evidence_row_matches_exact_batch():
    """query_many(algorithm="gibbs"): chains are independent per row; their frequencies track
    the exact batched posteriors on a 4x4 grid with 3 states."""
    from sorobn_b200 import BayesNet, synthetic

    spec = synthetic.grid(4, 4, 3, seed=11)
    bn = synthetic.load(spec, BayesNet, seed=3)
    query = ("g0303",)
    evidence = ["g0001", "g0102", "g0210", "g0301"]
    evidence = [e for e in evidence if e in spec.nodes] or spec.nodes[1:5]
    B = 512
    events = synthetic.random_events(spec, evidence, B, seed=5)
    exact = bn.query_many(*query, events=events).to_numpy()
    gibbs = bn.query_many(*query, events=events, algorithm="gibbs", n_iterations=120_000).to_numpy()
    assert gibbs.shape == exact.shape
    assert np.allclose(gibbs.sum(axis=1), 1.0, atol=1e-5)
    err = np.abs(gibbs - exact)
    assert err.mean() < 0.01 and err.max() < 0.06, (err.mean(), err.max())


def test_gibbs_on_the_benchmark_grid_runs_and_tracks_exact():
    """configs[4] shape: the 100-node 5-state grid.  4096 independent chains for ONE event, pooled:
    the pooled frequencies are an average over chains, so their error shrinks with the number of
    chains and a wrong Markov-blanket term on any child shows as a bias far above it."""
    from sorobn_b200 import workloads

    wl = workloads.grid10x10()
    bn = wl.build(seed=1)
    one = wl.events(1, seed=2, bn=bn)
    events = pd.concat([one] * 4096, ignore_index=True)
    exact = bn.query_many(*wl.query, events=one).to_numpy()[0]
    # 70 non-event variables share the iterations: 400 draws of the query variable per chain
    gibbs = bn.query_many(*wl.query, events=events, algorithm="gibbs", n_iterations=70 * 400).to_numpy()
    assert np.allclose(gibbs.sum(axis=1), 1.0, atol=1e-5)
    pooled = gibbs.mean(axis=0)
    # standard error of the pooled estimate from the spread BETWEEN chains (they are independent)
    sem = gibbs.std(axis=0, ddof=1) / np.sqrt(len(gibbs))
    assert np.all(np.abs(pooled - exact) < 6 * sem + 2e-3), (pooled, exact, sem)
    assert np.abs(pooled - exact).max() < 0.01


def test_gibbs_conditionals_match_the_reference_tables():
    """The deterministic half of the sampler: P(var | Markov blanket) as the chain evaluates it
    (sbn_gibbs_conditional, the same device function the chains run) against the tables the
    reference precomputes in `_gibbs_sampling` (bayes_net.py:699-712; tests/golden/gibbs_conditionals_*),
    entry by entry on the four example networks."""
    from conftest import golden_names, load_golden
    from sorobn_b200 import engine, examples

    checked = 0
    for name in golden_names(("gibbs_conditionals",)):
        golden = load_golden(name)
        bn = examples.build(examples.NETWORKS[golden["network"]])
        net = bn._compiled
        ids = list(range(len(net.names)))
        sampler = engine.GibbsSampler(net, [0], [], sorted(ids, key=lambda v: net.names[v]))
        for node, g in golden["nodes"].items():
            v = net.index[node]
            scope = [net.index[u] for u in g["boundary"]] + [v]
            for key, want in zip(g["index"], g["values"]):
                joint = np.zeros(len(ids), dtype=np.uint8)
                for u, val in zip(scope, key):
                    joint[u] = net.domains[u].index(val)
                got = sampler.conditional(v, joint)
                assert abs(got[joint[v]] - want) <= 2e-6 * max(want, 1e-30), (name, node, key, got, want)
                assert abs(got.sum() - 1.0) < 1e-5
                checked += 1
        sampler.close()
    assert checked > 200


def test_rejection_sampling_converges_to_exact_posterior():
    from sorobn_b200 import examples

    for make, query, event in ((examples.sprinkler, ("Rain",), {"Sprinkler": True}),
                               (examples.grades, ("Grade",), {"Letter": "Strong", "SAT": "Success"}),
                               (examples.asia, ("Bronchitis",), {"Smoker": True, "Dispnea": True})):
        bn = make(seed=11)
        exact = bn.query(*query, event=event)
        got = bn.query(*query, event=event, algorithm="rejection", n_iterations=2_000_000)
        both = pd.concat([exact, got], axis=1).fillna(0.0)
        assert np.isclose(got.sum(), 1.0, atol=1e-5)
        assert np.abs(both.iloc[:, 0] - both.iloc[:, 1]).max() < 0.01, both
    # an event that never shows up: the reference's answer is empty
    bn = examples.asia(seed=1)
    assert len(bn.query("Smoker", event={"TB or cancer": False, "Lung cancer": True}, algorithm="rejection",
                        n_iterations=10_000)) == 0


def test_likelihood_weighting_matches_the_reference_estimator():
    from oracle.sampler_replay import lw_expectation
    from sorobn_b200 import examples

    for make, query, event in ((examples.sprinkler, ("Rain",), {"Sprinkler": True}),
                               (examples.alarm, ("Burglary",), {"John calls": True, "Mary calls": True}),
                               (examples.grades, ("Letter", "SAT"), {"Intelligence": "Smart"})):
        bn = make(seed=5)
        want = lw_expectation(bn._compiled, query, event)
        got = bn.query(*query, event=event, algorithm="likelihood", n_iterations=2_000_000)
        net = bn._compiled
        assert np.isclose(got.sum(), 1.0, atol=1e-5)
        for key, p in want.items():
            names = sorted(query)
            label = tuple(net.domains[net.index[n]][k] for n, k in zip(names, key))
            value = got[label if len(label) > 1 else label[0]]
            assert abs(value - p) < 0.01, (query, label, value, p)


def test_every_algorithm_answers_like_the_reference_check_query():
    # reference check_query (test_bayes_net.py:66-76): every algorithm returns an answer
    from sorobn_b200 import examples

    for make in (examples.alarm, examples.asia, examples.sprinkler, examples.grades):
        bn = make(seed=3)
        fjd = bn.full_joint_dist()
        event = dict(zip(fjd.index.names, fjd.index[0]))
        query = sorted(event)[0]
        del event[query]
        for algorithm in ("exact", "gibbs", "likelihood", "rejection"):
            ans = bn.query(query, event=event, algorithm=algorithm, n_iterations=2000)
            assert ans.name == f"P({query})"
            if len(ans):
                assert np.isclose(ans.sum(), 1.0, atol=1e-5)
    many = examples.alarm(seed=2).query_many("Alarm", events=pd.DataFrame({"John calls": [True, False, True]}),
                                             algorithm="likelihood", n_iterations=20_000)
    assert many.shape == (3, 2) and np.allclose(many.sum(axis=1), 1.0, atol=1e-5)


def test_straight_line_gibbs_kernel_equals_the_generic_one_bit_for_bit():
    """Small networks run the chain through fixed-size records (sbn_gibbs_flat_kernel); same random
    stream, same arithmetic as the generic kernel, so the frequencies must be identical."""
    from sorobn_b200 import engine, workloads

    wl = workloads.grid10x10()
    bn = wl.build()
    net = bn._compiled
    cycle = [net.index[v] for v in sorted(set(bn.nodes) - set(wl.evidence))]
    sampler = engine.GibbsSampler(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence], cycle)
    codes = wl.codes(bn, 777, seed=3)
    flat = sampler.run(codes, 777, 3001, seed=99, algorithm="gibbs")
    generic = sampler.run(codes, 777, 3001, seed=99, algorithm="gibbs_generic")
    assert np.array_equal(flat, generic)
    assert np.allclose(flat.sum(axis=0), 1.0, atol=1e-5)
