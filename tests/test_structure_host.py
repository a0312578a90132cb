"""Score-based structure learning on the CPU: the float64 oracle (tests/structure_oracle.py) against its own
cross-checks, structure.climb driven by the oracle's scores against the oracle's search step by step, the
wiring of hill_climb with the device tally replaced by the oracle, and every ValueError."""
import math
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

import structure_oracle as oracle
from sorobn_b200 import BayesNet, engine, examples, structure, synthetic


def sample(name, n, seed):
    if name == "dag12":
        return synthetic.load(synthetic.random_dag(12, 3, 3), BayesNet, seed=seed).sample(n)
    return getattr(examples, name)(seed=seed).sample(n)


def oracle_search(X, score, max_parents, start=(), ess=1.0):
    data = oracle.encode(X)
    cards = {c: r for c, (_, r) in data.items()}
    return oracle.hill_climb(list(X.columns), cards, len(X),
                             lambda c, ps: oracle.family_score(data, c, ps, score, ess), max_parents, start)


def climb_steps(X, score, max_parents, start=(), ess=1.0):
    cards = [oracle.encode(X[[c]])[c][1] for c in X.columns]
    calls = []
    inner = oracle.scorer(X, score, ess)

    def scorer(families):
        calls.append(list(families))
        return inner(families)

    steps = list(structure.climb(list(X.columns), cards, len(X), scorer, max_parents, start))
    return steps, calls


# ------------------------------------------------------------------------------------------- oracle
def test_oracle_counts_and_scores_cross_check():
    X = sample("asia", 3000, 1)
    data = oracle.encode(X)
    child, parents = "Dispnea", ("Bronchitis", "TB or cancer")
    table = oracle.counts(data, child, parents)
    # the flat index puts the child fastest: compare with a groupby on the frame
    want = X.groupby([parents[1], parents[0], child]).size()
    dense = np.zeros((2, 2, 2), dtype=np.int64)
    for key, n in want.items():
        dense[tuple(sorted(set(X[c])).index(k) for c, k in zip((parents[1], parents[0], child), key))] = n
    assert np.array_equal(table, dense.reshape(-1))
    for ess in (0.5, 1.0, 10.0):
        assert math.isclose(oracle.bdeu(table, 2, ess), oracle.bdeu_gammaln(table, 2, ess), rel_tol=1e-12)


def test_oracle_bdeu_matches_brute_force_on_a_two_variable_table():
    rng = np.random.default_rng(5)
    parent = rng.integers(0, 3, 400)
    child = (parent + rng.integers(0, 2, 400)) % 4
    X = pd.DataFrame({"c": child, "p": parent})
    data = oracle.encode(X)
    table = oracle.counts(data, "c", ("p",))
    for ess in (0.5, 1.0, 10.0):
        want = oracle.bdeu_sequential(data["c"][0], data["p"][0], 4, 3, ess)
        assert math.isclose(oracle.bdeu(table, 4, ess), want, rel_tol=1e-10)


@pytest.mark.parametrize("score", ["bic", "bdeu"])
def test_oracle_scores_are_score_equivalent(score):
    X = sample("sprinkler", 2000, 2)
    data = oracle.encode(X)
    for u in X.columns:
        for v in X.columns:
            if u < v:
                uv = oracle.family_score(data, v, (u,), score) + oracle.family_score(data, u, (), score)
                vu = oracle.family_score(data, u, (v,), score) + oracle.family_score(data, v, (), score)
                assert math.isclose(uv, vu, rel_tol=1e-12), (u, v)


# ------------------------------------------------------------------------------------------- search
CASES = [("sprinkler", 3000, 0, 1), ("sprinkler", 3000, 0, 2), ("asia", 5000, 1, 2), ("asia", 5000, 1, 3),
         ("dag12", 4000, 2, 1), ("dag12", 4000, 2, 3)]


@pytest.mark.parametrize("score", ["bic", "bdeu"])
@pytest.mark.parametrize("name,n,seed,max_parents", CASES)
def test_climb_follows_the_oracle_search_step_by_step(name, n, seed, max_parents, score):
    X = sample(name, n, seed)
    steps, calls = climb_steps(X, score, max_parents)
    assert steps == oracle_search(X, score, max_parents)
    # one scorer call per step that needs new families, and no family is scored twice
    flat = [(c, tuple(ps)) for call in calls for c, ps in call]
    assert len(flat) == len(set(flat))
    assert len(calls) <= len(steps)


@pytest.mark.parametrize("score", ["bic", "bdeu"])
def test_climb_from_a_start_graph(score):
    X = sample("asia", 5000, 4)
    start = [("Smoker", "Visit to Asia"), ("Dispnea", "Positive X-ray")]
    steps, _ = climb_steps(X, score, 2, start=start)
    assert steps[0] == sorted(start, key=lambda e: (list(X.columns).index(e[1]), list(X.columns).index(e[0])))
    assert steps == oracle_search(X, score, 2, start=start)


def test_climb_without_parents_only_stops():
    X = sample("sprinkler", 500, 1)
    steps, calls = climb_steps(X, "bic", 0)
    assert steps == [[]] and calls == []


class OracleTally:
    """Stands in for engine.Tally: the same calls, answered by the oracle."""

    def __init__(self, codes, cards, device=None):
        self.cards = np.asarray(cards, dtype=np.int32)
        self.data = {i: (codes[i].astype(np.int64), int(r)) for i, r in enumerate(cards)}
        self.calls = 0

    def scores(self, families, kind="bic", ess=1.0):
        self.calls += 1
        return np.array([oracle.family_score(self.data, f[0], tuple(f[1:]), kind, ess) for f in families])

    def close(self):
        pass


def test_hill_climb_returns_constructor_items(monkeypatch):
    monkeypatch.setattr(engine, "Tally", OracleTally)
    X = sample("asia", 5000, 1)
    X["Constant"] = "x"
    items = structure.hill_climb(X, score="bdeu", max_parents=2)
    edges = [i for i in items if isinstance(i, tuple)]
    assert edges == oracle_search(X, "bdeu", 2)[-1]
    assert items[len(edges):] == [c for c in X.columns if not any(c in e for e in edges)]
    assert "Constant" in items
    bn = BayesNet(*items).fit(X)
    assert sorted(bn.nodes) == sorted(X.columns)
    want = [oracle.family_score(oracle.encode(X), c, (), "bic") for c in X.columns[:2]]
    got = structure.family_scores(X, [(c, ()) for c in X.columns[:2]])
    assert np.allclose(got, want, rtol=1e-12)


# ------------------------------------------------------------------------------------------- errors
def frame():
    return pd.DataFrame({"a": [0, 1, 1, 0], "b": ["x", "y", "y", "x"], "c": [True, False, True, True]})


@pytest.mark.parametrize("X,match", [
    (pd.DataFrame({"a": [0, None, 1]}, dtype=object), "missing"),
    (pd.DataFrame({"a": [0.0, np.nan, 1.0]}), "missing"),
    (pd.DataFrame({"a": np.arange(256)}), "256 states"),
    (pd.DataFrame({"a": []}), "at least one row"),
    (pd.DataFrame(), "at least one row"),
])
def test_bad_data_is_refused(X, match):
    with pytest.raises(ValueError, match=match):
        structure.family_scores(X, [("a", ())])
    with pytest.raises(ValueError, match=match):
        structure.hill_climb(X)


@pytest.mark.parametrize("families,match", [
    ([("z", ())], "unknown column 'z'"),
    ([("a", ("z",))], "unknown column 'z'"),
    ([("a", ("b", "b"))], "duplicate parent"),
    ([("a", ("a",))], "among its own parents"),
])
def test_bad_families_are_refused(families, match):
    with pytest.raises(ValueError, match=match):
        structure.family_scores(frame(), families)


def test_family_over_the_table_limit_is_refused():
    rng = np.random.default_rng(0)
    X = pd.DataFrame({c: rng.permutation(200) for c in "abc"})
    with pytest.raises(ValueError, match="more than 4194304 entries"):
        structure.family_scores(X, [("a", ("b", "c"))])


@pytest.mark.parametrize("kwargs,match", [
    (dict(score="aic"), "score must be one of"),
    (dict(score="bdeu", ess=0.0), "ess must be positive"),
    (dict(score="bdeu", ess=-1.0), "ess must be positive"),
])
def test_bad_scores_are_refused(kwargs, match):
    with pytest.raises(ValueError, match=match):
        structure.family_scores(frame(), [("a", ())], **kwargs)
    with pytest.raises(ValueError, match=match):
        structure.hill_climb(frame(), **kwargs)


@pytest.mark.parametrize("kwargs,match", [
    (dict(max_parents=-1), "max_parents must be >= 0"),
    (dict(start=[("a", "b"), ("b", "c"), ("c", "a")]), "cyclic"),
    (dict(start=[("a", "z")]), "unknown column 'z'"),
    (dict(start=[("a", "c"), ("b", "c")], max_parents=1), "max_parents is 1"),
])
def test_bad_searches_are_refused(kwargs, match):
    with pytest.raises(ValueError, match=match):
        structure.hill_climb(frame(), **kwargs)


def test_tally_refuses_codes_outside_their_states():
    with pytest.raises(engine.EngineError, match="column 1 holds code 3 of 3 states"):
        engine.Tally(np.array([[0, 1], [2, 3]], dtype=np.uint8), [2, 3])


def test_package_imports_with_docstrings_stripped():
    """Nothing at import time may depend on a docstring: `python -OO` drops them."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-OO", "-c", "import sorobn_b200.structure"], cwd=root,
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
