"""Host-side logic of the BayesNet mirror (no GPU needed) and the C-ABI library's
loadability.  Mirrors the reference's own tests (/root/reference/sorobn/test_bayes_net.py)
where they concern the exact-inference path."""
import ctypes
import os
import re

import numpy as np
import pandas as pd
import pytest

from sorobn_b200 import BayesNet, engine, examples

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def naive():
    bn = BayesNet("A", "B", "C")
    bn.P["A"] = pd.Series({True: 0.1, False: 0.9})
    bn.P["B"] = pd.Series({True: 0.3, False: 0.7})
    bn.P["C"] = pd.Series({True: 0.5, False: 0.5})
    bn.prepare()
    return bn


ALL = [examples.alarm, examples.asia, examples.sprinkler, examples.grades, naive]


@pytest.mark.parametrize("make", ALL, ids=lambda f: f.__name__)
def test_check_Ps(make):
    # reference check_Ps (test_bayes_net.py:52-63)
    bn = make()
    for child, parents in bn.parents.items():
        P = bn.P[child]
        assert P.index.names[-1] == child
        assert P.index.names[:-1] == parents
        assert np.allclose(P.groupby(parents).sum(), 1)
    for orphan in set(bn.nodes) - set(bn.parents):
        P = bn.P[orphan]
        assert P.index.name == orphan
        assert np.isclose(P.sum(), 1)


def test_structure_matches_reference_doctests():
    bn = examples.grades()
    # examples.py:257-264
    assert bn.nodes == ["Difficulty", "Intelligence", "Grade", "SAT", "Letter"]
    assert bn.children == {"Difficulty": ["Grade"], "Intelligence": ["Grade", "SAT"], "Grade": ["Letter"]}
    assert bn.parents == {"Grade": ["Difficulty", "Intelligence"], "SAT": ["Intelligence"], "Letter": ["Grade"]}
    # bayes_net.py:987-998
    assert BayesNet(("a", "b"), ("a", "c")).is_tree
    assert not BayesNet(("a", "c"), ("b", "c")).is_tree
    # bayes_net.py:1015-1031
    bn = BayesNet((0, 3), (1, 4), (2, 5), (3, 6), (4, 6), (5, 8), (6, 8), (6, 9), (7, 9), (7, 10), (8, 11), (8, 12))
    assert bn.markov_boundary(6) == [3, 4, 5, 7, 8, 9]
    # bayes_net.py:1049-1060
    assert list(examples.asia().iter_dfs()) == [
        "Smoker", "Bronchitis", "Dispnea", "Lung cancer", "TB or cancer", "Positive X-ray", "Visit to Asia",
        "Tuberculosis"]
    bn = examples.asia()
    assert bn.roots == ["Smoker", "Visit to Asia"]
    assert set(bn.leaves) == {"Dispnea", "Positive X-ray"}
    assert bn.ancestors("Dispnea") == {"Bronchitis", "Smoker", "TB or cancer", "Lung cancer", "Tuberculosis",
                                       "Visit to Asia"}


def test_structure_grammar_with_lists_and_cycles():
    import graphlib

    bn = BayesNet(("Smoker", ["Lung cancer", "Bronchitis"]), (["Tuberculosis", "Lung cancer"], "TB or cancer"))
    assert bn.parents["TB or cancer"] == ["Lung cancer", "Tuberculosis"]
    assert bn.children["Smoker"] == ["Bronchitis", "Lung cancer"]
    with pytest.raises(graphlib.CycleError):
        BayesNet(("a", "b"), ("b", "c"), ("c", "a"))


def test_cpt_dataframe_forms():
    # test_bayes_net.py:204-262
    def make(cols):
        bn = BayesNet(("A", "C"), ("B", "C"))
        bn.P["A"] = pd.Series({True: 0.7, False: 0.3})
        bn.P["B"] = pd.Series({True: 0.4, False: 0.6})
        data = {
            "A": [True, True, False, False],
            "B": [True, False, True, False],
            "C": [True, True, True, True],
            "p": [0.9, 0.8, 0.7, 0.1],
        }
        bn.P["C"] = pd.DataFrame({c: data[c] for c in cols})
        bn.prepare()
        return bn

    b1, b2 = make(["A", "B", "C", "p"]), make(["B", "C", "A", "p"])
    pd.testing.assert_series_equal(b1.P["C"], b2.P["C"])
    assert b1.P["C"].index.names == ["A", "B", "C"]
    assert b1.P["C"].name == "P(C | A, B)" and b1.P["A"].name == "P(A)"


def test_cpt_dataframe_errors():
    # test_bayes_net.py:265-295
    bn = BayesNet(("A", "B"))
    bn.P["A"] = pd.Series({True: 0.5, False: 0.5})
    bn.P["B"] = pd.DataFrame({"A": [True, True, False, False], "B": [True, False, True, False],
                              "prob": [0.9, 0.1, 0.4, 0.6]})
    with pytest.raises(ValueError, match="must have a 'p' column"):
        bn.prepare()
    bn.P["B"] = pd.DataFrame({"A": [True, True, False, False], "X": [True, False, True, False],
                              "p": [0.9, 0.1, 0.4, 0.6]})
    with pytest.raises(ValueError, match="has columns"):
        bn.prepare()


def test_compiled_tables_follow_sorted_domains():
    bn = examples.grades()
    net = bn._compiled
    g = net.index["Grade"]
    assert net.domains[g] == ["A", "B", "C"]
    assert [net.names[p] for p in net.parents[g]] == ["Difficulty", "Intelligence"]
    # P(Grade | Difficulty=Hard, Intelligence=Smart) = (.5, .3, .2)
    assert np.allclose(net.cpt[g][1, 1], [0.5, 0.3, 0.2])
    # string states
    bn = BayesNet(("Weather", "Mood"))
    bn.P["Weather"] = pd.Series({"Sunny": 0.7, "Rainy": 0.3})
    bn.P["Mood"] = pd.DataFrame({"Weather": ["Sunny", "Sunny", "Rainy", "Rainy"],
                                 "Mood": ["Happy", "Sad", "Happy", "Sad"], "p": [0.9, 0.1, 0.4, 0.6]})
    bn.prepare()
    net = bn._compiled
    assert net.domains[net.index["Weather"]] == ["Rainy", "Sunny"]
    assert np.allclose(net.cpt[net.index["Mood"]], [[0.4, 0.6], [0.9, 0.1]])


def test_query_argument_errors_do_not_need_a_gpu():
    bn = examples.alarm()
    with pytest.raises(ValueError, match="At least one query variable"):
        bn.query(event={})
    with pytest.raises(ValueError, match="cannot be part of the event"):
        bn.query("Alarm", event={"Alarm": True})
    with pytest.raises(ValueError, match="Unknown algorithm"):
        bn.query("Alarm", event={}, algorithm="magic")
    if engine.device_count() == 0:
        for algo in ("gibbs", "likelihood", "rejection"):
            with pytest.raises(engine.EngineError):  # no CPU fallback for the samplers either
                bn.query("Alarm", event={}, algorithm=algo, n_iterations=5)


def test_no_silent_cpu_fallback():
    """Without a GPU the exact path must fail loudly, not compute on the CPU."""
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    bn = examples.alarm()
    with pytest.raises(engine.EngineError):
        bn.query("Burglary", event={"John calls": True, "Mary calls": True})
    with pytest.raises(engine.EngineError):
        bn.query_many("Burglary", events=pd.DataFrame({"John calls": [True], "Mary calls": [False]}))
    with pytest.raises(engine.EngineError):
        bn.query("Burglary", event={"John calls": True}, algorithm="gibbs", n_iterations=10)
    with pytest.raises(engine.EngineError):
        bn.predict_proba({"John calls": True, "Mary calls": False})


def test_library_loads_and_exports_every_declared_symbol():
    lib = engine.load()
    assert lib.sbn_abi_version() == engine.ABI_VERSION
    header = open(os.path.join(ROOT, "include", "sorobn_b200.h")).read()
    declared = set(re.findall(r"\b(sbn_[a-z0-9_]+)\s*\(", header))
    assert declared == set(engine.EXPORTS), declared ^ set(engine.EXPORTS)
    raw = ctypes.CDLL(engine.lib_path())
    for name in declared:
        assert hasattr(raw, name), name
    m = re.search(r"#define SBN_ABI_VERSION (\d+)", header)
    assert int(m.group(1)) == lib.sbn_abi_version()


def test_program_validation_rejects_malformed_programs():
    """sbn_program_create parses and bounds-checks before touching the GPU."""
    from sorobn_b200 import planner

    lib = engine.load()
    bn = examples.alarm()
    net = bn._compiled
    plan = planner.build_plan(net, [net.index["Burglary"]], [net.index["John calls"]])
    blob = np.ascontiguousarray(plan.table_blob)

    def create(words):
        h = ctypes.c_void_p()
        w = np.ascontiguousarray(words, dtype=np.int32)
        rc = lib.sbn_program_create(0, w.ctypes.data, w.size, blob.ctypes.data, blob.size, ctypes.byref(h))
        msg = lib.sbn_last_error().decode()
        if rc == 0:
            lib.sbn_program_destroy(h)
        return rc, msg

    bad = plan.words.copy()
    bad[0] = 123
    assert create(bad)[0] == -1 and "magic" in create(bad)[1]
    bad = plan.words.copy()
    bad[1] = 99
    assert create(bad)[0] == -1
    assert create(plan.words[:-1])[0] == -1  # truncated
    assert create(np.concatenate([plan.words, [0]]))[0] == -1  # trailing
    hdr, tables, slots, steps = __import__("oracle.program_interp", fromlist=["parse"]).parse(plan.words)
    # corrupt a stride so that an input would read past its table
    bad = plan.words.copy()
    bad[-1] = 10_000
    rc, msg = create(bad)
    assert rc == -1 and "past its buffer" in msg
    # a well-formed program fails only because there is no device here (or succeeds on a GPU box)
    rc, msg = create(plan.words)
    assert rc in (0, -4), msg


@pytest.mark.parametrize("make", ALL, ids=lambda f: f.__name__)
def test_fit_partial_fit_and_sample(make):
    # reference check_partial_fit / check_sample_many / check_sample_one (test_bayes_net.py:15-44)
    import copy

    bn = make()
    bn.seed = 1
    one = bn.sample()
    assert isinstance(one, pd.Series) and sorted(one.index) == sorted(bn.nodes)
    for n in (2, 3, 100):
        frame = bn.sample(n)
        assert len(frame) == n and sorted(frame.columns) == sorted(bn.nodes)
    clamp = {bn.nodes[-1]: bn._compiled.domains[len(bn.nodes) - 1][0]}
    assert (bn.sample(50, init=clamp)[bn.nodes[-1]] == clamp[bn.nodes[-1]]).all()

    incremental = copy.deepcopy(bn)
    samples = bn.sample(500)
    bn.fit(samples)
    incremental.P = {}
    for rows in np.array_split(np.arange(len(samples)), 5):
        incremental.partial_fit(samples.iloc[rows])
    for node in bn.P:
        pd.testing.assert_series_equal(bn.P[node], incremental.P[node])
    # the fitted tables are proper CPTs and compile for the device
    for child, parents in bn.parents.items():
        assert np.allclose(bn.P[child].groupby(parents).sum(), 1)
    assert bn._compiled is not None


def test_fit_recovers_the_generating_tables_and_prior_count():
    from sorobn_b200 import examples

    truth = examples.sprinkler(seed=4)
    data = truth.sample(20_000)
    learned = BayesNet(*[(p, c) for c, ps in truth.parents.items() for p in ps]).fit(data)
    for node in truth.P:
        a, b = truth.P[node], learned.P[node].reindex(truth.P[node].index).fillna(0)
        assert np.abs(a - b).max() < 0.03, node
    smooth = BayesNet(*[(p, c) for c, ps in truth.parents.items() for p in ps], prior_count=1).fit(data.iloc[:50])
    assert (smooth.P["Wet grass"] > 0).all()  # every combination got a pseudo-observation


def test_chow_liu_matches_reference_edges():
    """structure.chow_liu against the edges the REAL reference returned on the same seeded
    samples (tests/golden/chow_liu.json), plus the defining properties of the tree."""
    import json

    from sorobn_b200 import structure

    with open(os.path.join(ROOT, "tests", "golden", "chow_liu.json")) as f:
        golden = json.load(f)
    for case in golden["cases"]:
        bn = getattr(examples, case["network"])(seed=case["seed"])
        X = bn.sample(case["n"])
        edges = structure.chow_liu(X, root=case["root"])
        assert sorted(map(tuple, edges)) == sorted(map(tuple, case["edges"])), case["network"]
        # a spanning tree oriented away from the root: n - 1 edges, every node but the root has one parent
        assert len(edges) == len(X.columns) - 1
        children = [c for _, c in edges]
        root = case["root"] if case["root"] is not None else X.columns[0]
        assert sorted(children + [root]) == sorted(X.columns)
    # learning a network from the tree and querying it stays on the normal path
    X = examples.sprinkler(seed=9).sample(4000)
    learned = BayesNet(*structure.chow_liu(X)).fit(X)
    assert learned.is_tree and learned._compiled is not None


def test_out_of_memory_evicts_other_cache_entries_and_retries():
    """A program whose scratch does not fit is retried once after every OTHER cached device object
    has been closed (each owns an arena sized for its largest batch)."""
    from sorobn_b200 import BayesNet, engine

    class FakeProgram:
        def __init__(self, fail_first):
            self.fail_first, self.closed, self.calls = fail_first, False, 0

        def run(self, codes, n):
            self.calls += 1
            if self.fail_first and self.calls == 1:
                raise engine.EngineError("no memory", code=engine.SBN_E_NOMEM)
            return np.zeros((2, n), dtype=np.float32)

        def close(self):
            self.closed = True

        def f32(self):  # a cache entry that is its own float32 program
            return self

    bn = BayesNet(("A", "B"))
    mine, other, sampler = FakeProgram(True), FakeProgram(False), FakeProgram(False)
    bn._engine_cache[("q1",)] = mine
    bn._engine_cache[("q2",)] = other
    bn._engine_cache[("sampler", "q3")] = sampler
    out = bn._run_evicting(mine, np.zeros((1, 4), dtype=np.uint8), 4)
    assert out.shape == (2, 4) and mine.calls == 2 and not mine.closed
    assert other.closed and sampler.closed and list(bn._engine_cache) == [("q1",)]
    # any other engine error is not swallowed
    class Broken(FakeProgram):
        def run(self, codes, n):
            raise engine.EngineError("bad", code=-1)

    with pytest.raises(engine.EngineError):
        bn._run_evicting(Broken(False), np.zeros((1, 4), dtype=np.uint8), 4)


def test_a_device_listed_twice_gets_a_program_per_listing(monkeypatch):
    """`query_many(devices=[0, 0, 0])` runs three threads on one GPU.  A program's scratch arena,
    staging buffers and graph capture serve one caller at a time, so each listing must get its own
    programs; one shared program let the threads free and capture each other's buffers and streams."""
    import threading

    users = {}  # program -> threads that ran it

    class FakeProgram:
        def __init__(self, plan, device=None, f64=False):
            self.Q = plan.Q

        def run(self, codes, n):
            users.setdefault(id(self), set()).add(threading.get_ident())
            return np.full((self.Q, n), 1.0 / self.Q, dtype=np.float32)

        def close(self):
            pass

    monkeypatch.setattr(engine, "Program", FakeProgram)
    bn = examples.build(examples.NETWORKS["asia"])
    ev_vars = ("Smoker", "Dispnea")
    codes = np.zeros((2, 9), dtype=np.uint8)
    post = bn._posterior_codes_multi(("Lung cancer",), ev_vars, codes, np.zeros(9, dtype=bool), [0, 0, 0])
    assert post.shape == (2, 9) and np.allclose(post, 0.5)
    assert len(users) == 3 and all(len(t) == 1 for t in users.values()), users
    keys = [k for k in bn._engine_cache if k[2] == 1 and not k[3]]
    assert len(keys) == 3 and {k[4] for k in keys} == {0, (0, 1), (0, 2)}, keys
