"""Constraint-based structure learning on the device (engine.Tally.tests, structure.ci_tests / pc_cpdag / pc;
csrc/sbn_tally.cu) against the numpy oracle (tests/ci_oracle.py): exact degrees of freedom, statistics and p-values
on both count paths and both stratum layouts, bitwise reproducible calls, and searches equal to the host search
driven by the oracle."""
import math

import numpy as np
import pytest
from scipy import stats

import ci_oracle
import pc_oracle
from sorobn_b200 import BayesNet, engine, examples, structure, synthetic

pytestmark = pytest.mark.gpu

# column: states; columns 4 and 9 use only some of their states (empty rows and columns of every table)
CARDS = [2, 3, 1, 5, 7, 255, 4, 2, 16, 255, 3]


def make_codes(n, seed):
    rng = np.random.default_rng(seed)
    codes = np.empty((len(CARDS), n), dtype=np.uint8)
    for v, r in enumerate(CARDS):
        codes[v] = rng.integers(0, r, n)
    codes[4] = rng.choice([0, 3, 6], n)             # 7 states, 3 seen
    codes[9] = rng.integers(0, 40, n)               # 255 states, 40 seen
    codes[1] = np.where(rng.random(n) < 0.7, codes[0], codes[1])  # a dependence: column 1 follows column 0
    codes[6] = np.where(rng.random(n) < 0.5, (codes[3] + codes[1]) % 4, codes[6])
    codes[10] = np.where(codes[7] == 1, 0, codes[10])  # stratum 7 = 1 leaves one state of 10: dof 0 there
    return codes


TESTS = [
    [0, 1], [1, 0], [0, 2], [2, 0], [0, 1, 2], [3, 6], [3, 6, 1], [6, 3, 1, 0], [6, 3, 1, 0, 7],  # S of 0 to 4
    [4, 6, 3], [4, 9], [9, 4, 0, 7], [5, 1], [1, 5, 7], [5, 9],              # empty rows and columns; 255 x 255
    [5, 8, 1], [8, 5, 3, 1], [9, 5, 2], [5, 9, 0],                         # tables over 32,768 entries
    [10, 0, 7], [10, 3, 7, 2], [2, 10], [0, 3, 8, 4, 10], [7, 8, 3, 6, 10],  # dof 0 strata, many strata
    [0, 3, 8, 4, 10, 7], [6, 0, 1, 3, 7, 2],
]


def oracle_rows(codes, tests, kind):
    data = {v: codes[v].astype(np.int64) for v in range(len(CARDS))}
    cards = dict(enumerate(CARDS))
    return [ci_oracle.statistic(ci_oracle.table(data, cards, t[0], t[1], tuple(t[2:])), kind) for t in tests]


@pytest.mark.parametrize("kind", ["g2", "chi2"])
@pytest.mark.parametrize("n", [1, 31, 1000, (1 << 20) + 7])
def test_tests_match_the_oracle(n, kind):
    codes = make_codes(n, n)
    assert any(math.prod(CARDS[v] for v in t) > engine.TALLY_SMEM_BINS for t in TESTS)
    tally = engine.Tally(codes, CARDS)
    try:
        got = tally.tests(TESTS, kind)
        again = tally.tests(TESTS, kind)
    finally:
        tally.close()
    assert got.shape == (len(TESTS), 3) and got.dtype == np.float64
    assert np.array_equal(got.view(np.uint64), again.view(np.uint64))
    for t, (stat, dof, _), (g_stat, g_dof, g_p) in zip(TESTS, oracle_rows(codes, TESTS, kind), got):
        assert g_dof == dof, (t, g_dof, dof)
        assert abs(g_stat - stat) <= 1e-12 * n + 1e-9 * abs(stat), (t, g_stat, stat)
        if g_dof == 0:
            assert g_p == 1.0, t
            continue
        want = stats.chi2.sf(g_stat, g_dof)
        if want >= 1e-300:
            assert abs(g_p - want) <= 1e-9 * want, (t, g_p, want)
        else:
            assert 0.0 <= g_p <= 1e-290, (t, g_p, want)
    assert any(d == 0 for _, d, _ in got) or n == 1


def test_p_values_across_the_range_of_dof():
    """Strongly and weakly dependent tables with up to ~2^20 degrees of freedom: p from 1 down past underflow."""
    n = (1 << 20) + 7
    rng = np.random.default_rng(5)
    cards = [255, 255, 16, 4]
    codes = np.empty((4, n), dtype=np.uint8)
    codes[0] = rng.integers(0, 255, n)
    codes[1] = np.where(rng.random(n) < 0.002, codes[0], rng.integers(0, 255, n))
    codes[2] = rng.integers(0, 16, n)
    codes[3] = np.where(rng.random(n) < 0.5, codes[2] % 4, rng.integers(0, 4, n))
    tests = [[0, 1], [1, 0, 2], [0, 1, 2, 3], [2, 3], [3, 2, 0], [0, 2], [2, 0, 1]]
    tally = engine.Tally(codes, cards)
    try:
        got = tally.tests(tests, "g2")
    finally:
        tally.close()
    data = {v: codes[v].astype(np.int64) for v in range(4)}
    for t, (stat, dof, _), (g_stat, g_dof, g_p) in zip(tests, [ci_oracle.statistic(
            ci_oracle.table(data, dict(enumerate(cards)), t[0], t[1], tuple(t[2:])), "g2") for t in tests], got):
        assert g_dof == dof and abs(g_stat - stat) <= 1e-12 * n + 1e-9 * abs(stat)
        want = stats.chi2.sf(g_stat, g_dof)
        assert abs(g_p - want) <= 1e-9 * want if want >= 1e-300 else g_p <= 1e-290
    assert got[:, 1].max() > 500_000


def test_ci_tests_matches_tally_tests():
    X = examples.asia(seed=3).sample(20_000)
    tests = [("Smoker", "Dispnea", ()), ("Dispnea", "Smoker", ("Bronchitis",)),
             ("Tuberculosis", "Lung cancer", ("TB or cancer", "Smoker"))]
    got = structure.ci_tests(X, tests, test="chi2")
    codes, cards = ci_oracle.codes_of(X)
    want = [ci_oracle.statistic(ci_oracle.table(codes, cards, x, y, g), "chi2") for x, y, g in tests]
    assert np.allclose(got, np.array(want), rtol=1e-9, atol=1e-12)


def test_tally_tests_refuses_bad_words():
    tally = engine.Tally(make_codes(100, 1), CARDS)
    try:
        with pytest.raises(engine.EngineError):
            tally.tests([[0]])
        with pytest.raises(engine.EngineError):
            tally.tests([[0, 0]])
        with pytest.raises(KeyError):
            tally.tests([[0, 1]], "x2")
    finally:
        tally.close()


# ------------------------------------------------------------------------------------ searches
def sample(name, n, seed):
    if name == "dag12":
        return synthetic.load(synthetic.random_dag(12, 3, 3, seed=seed), BayesNet, seed=seed).sample(n)
    return getattr(examples, name)(seed=seed).sample(n)


@pytest.mark.parametrize("test", ["g2", "chi2"])
@pytest.mark.parametrize("name,n,alpha", [("asia", 50_000, 0.05), ("alarm", 100_000, 0.01), ("dag12", 50_000, 0.05)])
def test_device_search_equals_host_search(name, n, alpha, test):
    X = sample(name, n, 0)
    inner = ci_oracle.tester(X, test)
    seen = []

    def tester(tests):
        ps = inner(tests)
        seen.extend(ps)
        return ps

    _, card = ci_oracle.codes_of(X)
    want = structure.pc_search(list(X.columns), [card[c] for c in X.columns], tester, alpha)
    # a p-value this close to alpha could fall on either side with the device's rounding
    assert not any(abs(p - alpha) <= 1e-6 * alpha for p in seen)
    got = structure.pc_cpdag(X, alpha=alpha, test=test)
    assert got == want
    items = structure.pc(X, alpha=alpha, test=test)
    edges = [i for i in items if isinstance(i, tuple)]
    assert edges == structure._dag_edges(list(X.columns), want)


def test_pc_recovers_the_true_cpdag_at_a_million_rows():
    spec = synthetic.random_dag(7, 2, 3, seed=1)  # the host tester recovers it at 1M rows
    X = synthetic.load(spec, BayesNet, seed=1).sample(1_000_000)
    nodes, edges = list(spec.nodes), list(spec.edges)
    directed, undirected, kept = pc_oracle.cpdag(nodes, edges)
    assert directed and undirected
    got = structure.pc_cpdag(X, alpha=0.01)
    assert set(got.directed) == directed and {frozenset(e) for e in got.undirected} == undirected
    dag = [i for i in structure.pc(X, alpha=0.01) if isinstance(i, tuple)]
    assert set(dag) in kept


def test_learned_network_fits_and_answers_queries():
    X = sample("asia", 20_000, 3)
    bn = BayesNet(*structure.pc(X)).fit(X)
    assert sorted(bn.nodes) == sorted(X.columns)
    post = bn.query_many("Lung cancer", events=X[["Smoker", "Dispnea"]].head(100))
    assert post.shape[0] == 100 and np.allclose(post.sum(axis=1), 1.0, atol=1e-5)
