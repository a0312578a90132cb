"""Constraint-based structure learning on the CPU: structure.pc_search against the brute-force CPDAG under a
perfect d-separation tester and against a plain sequential PC-stable (tests/pc_oracle.py) under the numpy G^2
tester (tests/ci_oracle.py); the orientation and extension rules on hand-built graphs; the statistics oracle
against scipy; the wiring of ci_tests / pc_cpdag / pc with the device tally replaced by the oracle; every
ValueError."""
import itertools
import math

import numpy as np
import pandas as pd
import pytest
from scipy import stats

import ci_oracle
import pc_oracle
from sorobn_b200 import BayesNet, engine, examples, structure, synthetic


def check_recovery(nodes, parents):
    edges = [(p, c) for c, ps in parents.items() for p in ps]
    res = structure.pc_search(nodes, [2] * len(nodes), pc_oracle.d_sep_tester(parents))
    directed, undirected, kept = pc_oracle.cpdag(nodes, edges)
    assert set(res.directed) == directed
    assert {frozenset(e) for e in res.undirected} == undirected
    assert len(res.directed) == len(set(res.directed)) and len(res.undirected) == len(set(res.undirected))
    for (u, v), s in res.sepsets.items():
        assert nodes.index(u) < nodes.index(v)
        assert pc_oracle.d_separated(parents, u, v, s)
    skeleton = {frozenset(e) for e in edges}
    assert set(res.sepsets) == {(u, v) for u, v in itertools.combinations(nodes, 2)
                                if frozenset((u, v)) not in skeleton}
    assert set(structure._dag_edges(nodes, res)) in kept


@pytest.mark.parametrize("name", ["asia", "sprinkler", "grades", "alarm"])
def test_perfect_oracle_recovers_the_cpdag_of_the_examples(name):
    bn = getattr(examples, name)()
    check_recovery(list(bn.nodes), bn.parents)


def test_perfect_oracle_recovers_the_cpdag_of_random_dags():
    done = 0
    for seed in range(200):
        spec = synthetic.random_dag(5 + seed % 4, 3, 3, seed=seed)
        if len(list(spec.edges)) > 14:
            continue
        check_recovery(list(spec.nodes), spec.parents)
        done += 1
        if done == 24:
            break
    assert done == 24


# ------------------------------------------------------------------------------- batching = sequential
def sample(name, n, seed):
    if name == "dag12":
        return synthetic.load(synthetic.random_dag(12, 3, 3, seed=seed), BayesNet, seed=seed).sample(n)
    return getattr(examples, name)(seed=seed).sample(n)


def compare_with_sequential(X, alpha, max_cond, tester):
    cols = list(X.columns)
    _, card = ci_oracle.codes_of(X)
    cards = [card[c] for c in cols]
    calls = []

    def batched(tests):
        calls.append(list(tests))
        return tester(tests)

    res = structure.pc_search(cols, cards, batched, alpha, max_cond)
    directed, undirected, seps = pc_oracle.sequential_pc(cols, cards, lambda x, y, g: tester([(x, y, g)])[0],
                                                         alpha, max_cond)
    assert set(res.directed) == directed
    assert {frozenset(e) for e in res.undirected} == undirected
    assert res.sepsets == seps
    for tests in calls:  # one call per level, every test distinct, x before y, given in column order
        assert len(tests) == len(set(tests))
        for x, y, given in tests:
            assert cols.index(x) < cols.index(y)
            assert [cols.index(g) for g in given] == sorted(cols.index(g) for g in given)
        assert len({len(g) for _, _, g in tests}) == 1
    return res, calls


@pytest.mark.parametrize("max_cond", [None, 0, 1])
@pytest.mark.parametrize("name,n,alpha", [("asia", 3000, 0.05), ("alarm", 2000, 0.01), ("sprinkler", 500, 0.05),
                                          ("grades", 800, 0.05), ("dag12", 1500, 0.05)])
def test_batched_levels_equal_sequential_pc_stable(name, n, alpha, max_cond):
    X = sample(name, n, 1)
    res, calls = compare_with_sequential(X, alpha, max_cond, ci_oracle.tester(X))
    if max_cond is not None:
        assert len(calls) <= max_cond + 1


def test_nan_p_values_count_as_dependent():
    X = sample("dag12", 1500, 2)
    inner = ci_oracle.tester(X)
    dropped = []

    def tester(tests):
        ps = inner(tests)
        out = []
        for (x, y, given), p in zip(tests, ps):
            if (sum(map(ord, x + y)) + len(given)) % 3 == 0:
                dropped.append((x, y, given))
                p = math.nan
            out.append(p)
        return out

    res, _ = compare_with_sequential(X, 0.05, None, tester)
    assert dropped
    plain = structure.pc_search(list(X.columns), [3] * 12, inner)
    assert len(res.directed) + len(res.undirected) >= len(plain.directed) + len(plain.undirected)


def test_tests_over_the_table_limit_are_not_sent():
    cols = ["a", "b", "c", "d"]
    cards = [256, 256, 64, 2]  # a b c: 2^22 entries, a b c d: over
    seen = []

    def tester(tests):
        seen.extend(tests)
        return [1.0 if set(g) == {"c", "d"} else 0.0 for _, _, g in tests]

    res = structure.pc_search(cols, cards, tester)
    assert all(math.prod(cards[cols.index(m)] for m in (x, y, *g)) <= 1 << 22 for x, y, g in seen)
    assert ("a", "b", ("c",)) in seen and ("a", "b", ("c", "d")) not in seen
    assert ("a", "b") not in res.sepsets  # its separating test was never sent


# ------------------------------------------------------------------------------- hand-built cases
def pdag(n, undirected, directed):
    adj = [set() for _ in range(n)]
    for a, b in [*undirected, *directed]:
        adj[a].add(b)
        adj[b].add(a)
    return adj, set(directed)


def test_meek_rule_1():
    adj, d = pdag(3, [(1, 2)], [(0, 1)])  # 0 -> 1 - 2, 0 and 2 non-adjacent
    structure._meek(adj, d)
    assert d == {(0, 1), (1, 2)}


def test_meek_rule_2():
    adj, d = pdag(3, [(0, 2)], [(0, 1), (1, 2)])  # 0 -> 1 -> 2, 0 - 2
    structure._meek(adj, d)
    assert d == {(0, 1), (1, 2), (0, 2)}


def test_meek_rule_3():
    # 0 - 1 -> 3, 0 - 2 -> 3, 1 and 2 non-adjacent, 0 - 3: R3 gives 0 -> 3; R1 and R2 cannot fire
    adj, d = pdag(4, [(0, 1), (0, 2), (0, 3)], [(1, 3), (2, 3)])
    structure._meek(adj, d)
    assert d == {(1, 3), (2, 3), (0, 3)}


def test_meek_rules_chain_to_a_fixpoint():
    # 0 -> 1 - 2 - 3: R1 orients 1 -> 2, and then 2 -> 3
    adj, d = pdag(4, [(1, 2), (2, 3)], [(0, 1)])
    structure._meek(adj, d)
    assert d == {(0, 1), (1, 2), (2, 3)}


def independence_model(cols, edges, seps):
    """A tester that separates every non-edge by its set in `seps` (default: the empty set)."""
    def tester(tests):
        out = []
        for x, y, given in tests:
            if (x, y) in edges or (y, x) in edges:
                out.append(0.0)
            else:
                out.append(1.0 if tuple(given) == seps.get((x, y), ()) else 0.0)
        return out
    return tester


def test_collider_conflict_keeps_the_first_orientation():
    cols = ["a", "b", "c", "d"]
    edges = {("a", "b"), ("b", "c"), ("c", "d")}
    tester = independence_model(cols, edges, {})
    res = structure.pc_search(cols, [2] * 4, tester)
    # (a, c) orients a -> b <- c first; (b, d) then wants b -> c, already c -> b, and orients d -> c
    assert set(res.directed) == {("a", "b"), ("c", "b"), ("d", "c")} and res.undirected == []
    d, u, s = pc_oracle.sequential_pc(cols, [2] * 4, lambda x, y, g: tester([(x, y, g)])[0], 0.05)
    assert d == set(res.directed) and not u


def test_a_collider_that_would_close_a_cycle_is_skipped():
    cols = [f"n{i}" for i in range(6)]
    pairs = [(0, 1), (0, 3), (0, 4), (0, 5), (1, 5), (2, 3), (3, 4), (3, 5)]
    edges = {(cols[a], cols[b]) for a, b in pairs}
    tester = independence_model(cols, edges, {})
    res = structure.pc_search(cols, [2] * 6, tester)
    # (n1, n3) orients n0 -> n3 <- ... and n3 -> n5 before (n3, n?) asks for n5 -> n0, which would close
    # n0 -> n3 -> n5 -> n0; the edge stays undirected through the colliders and R2 then orients n0 -> n5
    assert ("n0", "n5") in res.directed and ("n5", "n0") not in res.directed
    assert pc_oracle._acyclic(cols, res.directed)
    d, u, s = pc_oracle.sequential_pc(cols, [2] * 6, lambda x, y, g: tester([(x, y, g)])[0], 0.05)
    assert d == set(res.directed) and u == {frozenset(e) for e in res.undirected}


def test_dor_tarsi_extension_and_its_fallback():
    cols = ["a", "b", "c", "d"]
    # an undirected 4-cycle without a chord: no node qualifies, so the lowest-position sink "a" takes its edges
    cyc = structure.CPDAG([], [("a", "b"), ("b", "c"), ("c", "d"), ("a", "d")], {})
    assert structure._dag_edges(cols, cyc) == [("b", "a"), ("d", "a"), ("c", "b"), ("d", "c")]
    # a chordal class: a - b - c, a - c, c -> d; "d" has an outgoing-free position but no undirected edge
    ch = structure.CPDAG([("c", "d")], [("a", "b"), ("a", "c"), ("b", "c")], {})
    got = structure._dag_edges(cols, ch)
    assert pc_oracle.extends(got, {("c", "d")}, {frozenset(e) for e in ch.undirected}, cols)
    assert pc_oracle.v_structures(got) == set()


# ------------------------------------------------------------------------------- statistics oracle
def scipy_sum(tab, kind):
    stat, dof = 0.0, 0
    for z in tab:
        obs = z[z.sum(axis=1) > 0][:, z.sum(axis=0) > 0]
        if obs.size == 0:
            continue
        if min(obs.shape) == 1:
            continue  # dof 0, statistic 0: scipy computes the same, but warns
        res = stats.chi2_contingency(obs, correction=False, lambda_="log-likelihood" if kind == "g2" else None)
        stat += res.statistic
        dof += res.dof
    return stat, dof


@pytest.mark.parametrize("kind", ["g2", "chi2"])
def test_statistics_oracle_matches_scipy(kind):
    rng = np.random.default_rng(0)
    for trial in range(60):
        nz, ry, rx = rng.integers(1, 5), rng.integers(1, 6), rng.integers(1, 6)
        tab = rng.integers(0, 20, size=(nz, ry, rx)) * (rng.random((nz, ry, rx)) < 0.8)
        if trial % 5 == 0:
            tab[:, rng.integers(0, ry)] = 0  # an empty y row in every stratum
        if trial % 7 == 0:
            tab[..., rng.integers(0, rx)] = 0  # an empty x column
        if trial % 3 == 0:
            tab[rng.integers(0, nz)] = 0  # an empty stratum
        stat, dof, p = ci_oracle.statistic(tab, kind)
        want_stat, want_dof = scipy_sum(tab, kind)
        assert dof == want_dof
        assert math.isclose(stat, want_stat, rel_tol=1e-10, abs_tol=1e-10)
        if dof > 0:
            assert math.isclose(p, stats.chi2.sf(stat, dof), rel_tol=1e-9)
        else:
            assert p == 1.0


def test_statistics_oracle_counts_the_frame():
    X = sample("asia", 2000, 3)
    codes, cards = ci_oracle.codes_of(X)
    tab = ci_oracle.table(codes, cards, "Dispnea", "Smoker", ("Bronchitis",))
    want = pd.crosstab([X["Bronchitis"], X["Smoker"]], X["Dispnea"]).to_numpy().reshape(tab.shape)
    assert np.array_equal(tab, want)


# ------------------------------------------------------------------------------- wiring, device tally faked
class FakeTally:
    """engine.Tally's tests() answered by the oracle."""
    calls = []

    def __init__(self, codes, cards, device=None):
        self.codes, self.cards = codes.astype(np.int64), np.asarray(cards, dtype=np.int32)

    def tests(self, tests, kind="g2"):
        FakeTally.calls.append(len(tests))
        codes = {i: self.codes[i] for i in range(len(self.cards))}
        cards = {i: int(r) for i, r in enumerate(self.cards)}
        return np.array([ci_oracle.statistic(ci_oracle.table(codes, cards, t[0], t[1], tuple(t[2:])), kind)
                         for t in tests], dtype=np.float64)

    def close(self):
        pass


def test_pc_and_ci_tests_wiring(monkeypatch):
    monkeypatch.setattr(engine, "Tally", FakeTally)
    monkeypatch.setattr(structure, "_BATCH_ENTRIES", 12)  # 4 + 8 entries, then 16
    X = sample("asia", 3000, 4)
    tests = [("Smoker", "Dispnea", ()), ("Smoker", "Dispnea", ("Bronchitis",)), ("Dispnea", "Smoker", ("TB or cancer", "Bronchitis"))]
    FakeTally.calls.clear()
    got = structure.ci_tests(X, tests, test="chi2")
    codes, cards = ci_oracle.codes_of(X)
    want = [ci_oracle.statistic(ci_oracle.table(codes, cards, x, y, g), "chi2") for x, y, g in tests]
    assert np.array_equal(got, np.array(want)) and len(FakeTally.calls) == 2
    cp = structure.pc_cpdag(X, alpha=0.01)
    res = structure.pc_search(list(X.columns), [2] * 8, ci_oracle.tester(X), alpha=0.01)
    assert cp == res
    items = structure.pc(X, alpha=0.01)
    edges = [i for i in items if isinstance(i, tuple)]
    assert edges == structure._dag_edges(list(X.columns), res)
    assert items[len(edges):] == [c for c in X.columns if not any(c in e for e in edges)]
    assert edges == sorted(edges, key=lambda e: (list(X.columns).index(e[1]), list(X.columns).index(e[0])))
    bn = BayesNet(*items).fit(X)
    assert sorted(bn.nodes) == sorted(X.columns)


# ------------------------------------------------------------------------------- refusals
def test_refusals():
    X = pd.DataFrame({"a": [0, 1, 0, 1], "b": [1, 1, 0, 0], "c": [0, 0, 1, 1]})
    for tests in ([("a", "zz", ())], [("a", "a", ())], [("a", "b", ("a",))], [("a", "b", ("b",))],
                  [("a", "b", ("c", "c"))], [("zz", "b", ())], [("a", "b", ("zz",))]):
        with pytest.raises(ValueError):
            structure.ci_tests(X, tests)
    with pytest.raises(ValueError):
        structure.ci_tests(X, [("a", "b", ())], test="g3")
    big = pd.DataFrame({f"c{i}": np.arange(255) for i in range(3)})  # 255^3 > 2^22 table entries
    with pytest.raises(ValueError, match="entries"):
        structure.ci_tests(big, [("c0", "c1", ("c2",))])
    holes = X.astype(object)
    holes.loc[1, "b"] = None
    for fn in (structure.pc, structure.pc_cpdag):
        with pytest.raises(ValueError, match="missing"):
            fn(holes)
        with pytest.raises(ValueError, match="missing"):
            structure.ci_tests(holes, [("a", "b", ())])
        for alpha in (0.0, 1.0, -0.1, 2.0, math.nan):
            with pytest.raises(ValueError, match="alpha"):
                fn(X, alpha=alpha)
        with pytest.raises(ValueError, match="max_cond"):
            fn(X, max_cond=-1)
        with pytest.raises(ValueError, match="test"):
            fn(X, test="x2")
        with pytest.raises(ValueError):
            fn(pd.DataFrame())
    with pytest.raises(ValueError, match="alpha"):
        structure.pc_search(["a", "b"], [2, 2], lambda t: [0.0] * len(t), alpha=1.5)
    with pytest.raises(ValueError, match="max_cond"):
        structure.pc_search(["a", "b"], [2, 2], lambda t: [0.0] * len(t), max_cond=-2)


def test_tally_tests_refuses_bad_words_before_the_device():
    """The C entry point's argument checks (k < 2, unknown kind) come before any device work, and the exported
    symbol is declared in the header."""
    lib = engine.load()
    words = np.array([1, 0], dtype=np.int32)
    out = np.empty(3)
    assert lib.sbn_tally_tests(None, words.ctypes.data, 2, 0, out.ctypes.data, 1) != 0
    assert engine.Tally.TESTS == {"g2": 0, "chi2": 1}
