"""Structure learning on the device (engine.Tally, structure.family_scores / hill_climb; csrc/sbn_tally.cu)
against the float64 oracle (tests/structure_oracle.py): exact counts on both count paths, scores within
1e-10, and the search's graphs."""
import itertools
import math

import numpy as np
import pandas as pd
import pytest

import structure_oracle as oracle
from sorobn_b200 import BayesNet, engine, examples, structure, synthetic

pytestmark = pytest.mark.gpu


def random_codes(cards, n, seed):
    """Codes with skew (most rows in state 0 for every third column) and a column copied from another, so
    that tables have hot bins."""
    rng = np.random.default_rng(seed)
    codes = np.empty((len(cards), n), dtype=np.uint8)
    for v, r in enumerate(cards):
        if v % 3 == 2 and r > 1:
            codes[v] = np.where(rng.random(n) < 0.9, 0, rng.integers(0, r, n))
        else:
            codes[v] = rng.integers(0, r, n)
    if len(cards) > 1 and cards[1] == cards[0]:
        codes[1] = codes[0]
    return codes


def oracle_counts(codes, cards, fam):
    data = {v: (codes[v].astype(np.int64), int(cards[v])) for v in fam}
    return oracle.counts(data, fam[0], tuple(fam[1:]))


def check_counts(codes, cards, families):
    tally = engine.Tally(codes, cards)
    try:
        got = tally.counts(families)
    finally:
        tally.close()
    assert len(got) == len(families)
    for fam, g in zip(families, got):
        want = oracle_counts(codes, cards, fam)
        assert g.dtype == np.uint64 and np.array_equal(g.astype(np.int64), want), fam
        assert int(g.sum()) == codes.shape[1]


CARDS = [3, 3, 2, 4, 1, 5, 2, 7]  # column 4 has one state


@pytest.mark.parametrize("n", [1, 31, 1000, (1 << 20) + 7])
def test_counts_of_families_of_one_to_five_members(n):
    codes = random_codes(CARDS, n, seed=n)
    rng = np.random.default_rng(3)
    families = []
    for k in range(1, 6):
        for _ in range(6):
            families.append([int(x) for x in rng.choice(len(CARDS), size=k, replace=False)])
    families += [[4], [4, 0], [0, 4], [1, 0], [2, 5, 3, 7, 4]]
    check_counts(codes, CARDS, families)


@pytest.mark.parametrize("n", [1000, (1 << 20) + 7])
def test_counts_of_a_group_of_over_a_thousand_small_families(n):
    cards = [2 + (v % 3) for v in range(40)]
    codes = random_codes(cards, n, seed=7)
    families = [[v, u] for v in range(40) for u in range(40) if u != v]
    assert len(families) > 1000 and sum(cards[a] * cards[b] for a, b in families) <= engine.TALLY_SMEM_BINS
    check_counts(codes, cards, families + [[v] for v in range(40)])


@pytest.mark.parametrize("n", [31, (1 << 20) + 7])
def test_counts_of_a_family_over_the_shared_memory_budget(n):
    cards = [9, 9, 9, 9, 9, 2, 3]
    codes = random_codes(cards, n, seed=11)
    big = [0, 1, 2, 3, 4]
    assert math.prod(cards[v] for v in big) > engine.TALLY_SMEM_BINS
    # small families on either side of the big one: the groups around a global family stay in place
    check_counts(codes, cards, [[5, 6], big, [6, 5, 0], [2, 1, 0, 3, 4], [5]])


@pytest.mark.parametrize("n", [1000, 100_003])
def test_counts_of_consecutive_shared_groups(n):
    """More than 64 columns with more than one state, and small tables that together pass the shared-memory
    budget: the batch splits into consecutive shared groups, on the staged-column limit and on the bin budget,
    each with its own staged columns."""
    cards = [2 + (v % 2) for v in range(70)]
    codes = random_codes(cards, n, seed=13)
    # every child's pair families span all 70 columns: groups close on the staged-column limit
    families = [[v, u] for v in range(70) for u in range(70) if u != v]
    # 81-entry tables over 20 three-state columns: groups close on the bin budget
    rng = np.random.default_rng(1)
    odd = np.arange(1, 70, 2)[:20]
    quads = [[int(x) for x in rng.choice(odd, size=4, replace=False)] for _ in range(450)]
    assert sum(math.prod(cards[c] for c in fam) for fam in quads) > engine.TALLY_SMEM_BINS
    check_counts(codes, cards, families + quads + [[v, (v + 1) % 70, (v + 2) % 70] for v in range(70)])


def asia_frame(n, seed):
    return examples.asia(seed=seed).sample(n)


@pytest.mark.parametrize("score,ess", [("bic", 1.0), ("bdeu", 0.5), ("bdeu", 1.0), ("bdeu", 10.0)])
def test_family_scores_match_the_oracle(score, ess):
    X = asia_frame(100_000, 1)
    X["Tri"] = np.random.default_rng(2).integers(0, 3, len(X))
    cols = list(X.columns)
    families = [(c, ()) for c in cols]
    families += [(v, (u,)) for u, v in itertools.permutations(cols, 2)]
    families += [(cols[0], (cols[1], cols[8])), (cols[8], (cols[2], cols[3], cols[4])), ("Dispnea", ("Bronchitis", "TB or cancer"))]
    got = structure.family_scores(X, families, score=score, ess=ess)
    data = oracle.encode(X)
    want = np.array([oracle.family_score(data, c, ps, score, ess) for c, ps in families])
    assert got.shape == want.shape
    assert np.all(np.abs(got - want) <= 1e-10 * np.abs(want)), np.max(np.abs(got - want) / np.abs(want))


def sample(name, n, seed):
    if name == "dag12":
        return synthetic.load(synthetic.random_dag(12, 3, 3), BayesNet, seed=seed).sample(n)
    return getattr(examples, name)(seed=seed).sample(n)


@pytest.mark.parametrize("score", ["bic", "bdeu"])
@pytest.mark.parametrize("name,n", [("sprinkler", 50_000), ("asia", 100_000), ("alarm", 200_000), ("dag12", 50_000)])
def test_hill_climb_matches_the_oracle_search(name, n, score):
    X = sample(name, n, 0)
    items = structure.hill_climb(X, score=score, max_parents=3)
    edges = [i for i in items if isinstance(i, tuple)]
    data = oracle.encode(X)
    cards = {c: r for c, (_, r) in data.items()}
    cols = list(X.columns)

    def score_fn(c, ps):
        return oracle.family_score(data, c, ps, score)

    history = oracle.hill_climb(cols, cards, n, score_fn, 3, margin=1e-6)
    assert edges == history[-1]
    assert items[len(edges):] == [c for c in cols if not any(c in e for e in edges)]
    # a local optimum under the oracle's scores, and no worse than the empty graph
    assert len(oracle.hill_climb(cols, cards, n, score_fn, 3, start=edges)) == 1
    assert oracle.total_score(data, edges, score) >= oracle.total_score(data, [], score)


def test_learned_network_fits_and_answers_queries():
    X = sample("asia", 20_000, 3)
    bn = BayesNet(*structure.hill_climb(X)).fit(X)
    assert sorted(bn.nodes) == sorted(X.columns)
    post = bn.query_many("Lung cancer", events=X[["Smoker", "Dispnea"]].head(100))
    assert post.shape[0] == 100 and np.allclose(post.sum(axis=1), 1.0, atol=1e-5)


def test_hill_climb_respects_the_start_and_max_parents():
    X = sample("asia", 20_000, 4)
    start = [("Smoker", "Visit to Asia")]
    items = structure.hill_climb(X, score="bdeu", max_parents=1, start=start)
    edges = [i for i in items if isinstance(i, tuple)]
    children = [v for _, v in edges]
    assert len(children) == len(set(children))
    data = oracle.encode(X)
    cards = {c: r for c, (_, r) in data.items()}
    want = oracle.hill_climb(list(X.columns), cards, len(X), lambda c, ps: oracle.family_score(data, c, ps, "bdeu"),
                             1, start=start)[-1]
    assert edges == want


def test_constant_column_and_single_row():
    X = pd.DataFrame({"a": [1], "b": ["x"]})
    assert structure.hill_climb(X) == ["a", "b"]
    got = structure.family_scores(X, [("a", ()), ("a", ("b",))], score="bdeu")
    assert np.allclose(got, [0.0, 0.0])
