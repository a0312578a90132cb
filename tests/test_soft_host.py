"""The host side of soft evidence (the `likelihoods=` keyword of query, query_many, marginals_many, predict_proba and
predict_log_proba) on the CPU: the device programs are replaced by the CPU interpreter, and only public entry
points are driven, apart from the cache size."""
import numpy as np
import pandas as pd
import pytest

import soft_interp
import soft_oracle
from interpreted_program import InterpretedProgram
from sorobn_b200 import engine, examples, planner, workloads

EV = ["Smoker", "Visit to Asia"]
SOFT = ["Dispnea", "Positive X-ray"]  # sorted: the likelihood column order
QUERY = ("Lung cancer",)


class SoftProgram(InterpretedProgram):
    """InterpretedProgram with `run_soft`; `liks` records the likelihoods of every run."""

    liks = []

    def run_soft(self, codes, lik, n_rows, log_evidence=False):
        self._start(n_rows)
        lik = np.asarray(lik, dtype=self.dtype)
        SoftProgram.liks.append((self.f64, lik.copy()))
        codes = np.asarray(codes, dtype=np.uint8)
        if self.plan.version == planner.VERSION_MARGINALS:
            post = soft_interp.run_marginals(self.plan.words, self.blob, codes, lik, n_rows=n_rows, dtype=self.dtype,
                                             min_total=self._min_total())
            return (post, None) if log_evidence else post
        post, total, log_ev = soft_interp.run(self.plan.words, self.blob, codes, lik, n_rows=n_rows, dtype=self.dtype)
        if self._min_total() is not None:
            low = ~(total >= self._min_total())
            post[:, low], log_ev[low] = np.nan, np.nan
        return (post, log_ev) if log_evidence else post


@pytest.fixture
def interpreted(monkeypatch):
    monkeypatch.setattr(InterpretedProgram, "live", [])
    monkeypatch.setattr(InterpretedProgram, "calls", [])
    monkeypatch.setattr(InterpretedProgram, "flag_below", None)
    monkeypatch.setattr(SoftProgram, "liks", [])
    monkeypatch.setattr(engine, "Program", SoftProgram)
    return SoftProgram


def frame(bn, n, seed):
    net = bn._compiled
    codes = workloads.forward_sample_codes(net, n, seed)
    return pd.DataFrame({c: np.asarray(net.domains[net.index[c]], dtype=object)[codes[net.index[c]]] for c in EV},
                        index=pd.RangeIndex(5, 5 + n, name="row"))


def likelihoods(bn, n, seed):
    rng = np.random.default_rng(seed)
    return {s: rng.random((n, len(bn._compiled.domains[bn._compiled.index[s]]))) * 10.0 ** rng.integers(-3, 3, (n, 1))
            for s in SOFT}


def oracle_rows(bn, X, lik, query):
    net = bn._compiled
    dn = soft_oracle.dense(net)
    post, log_ev = [], []
    for b in range(len(X)):
        hard = {c: X[c].iloc[b] for c in X.columns}
        soft = {s: lik[s][b] for s in lik}
        post.append(soft_oracle.posterior(dn, list(query), hard, soft))
        log_ev.append(soft_oracle.log_evidence(dn, hard, soft))
    return np.array(post), np.array(log_ev)


def test_query_many_and_predict_against_oracle(interpreted):
    bn = examples.asia()
    X = frame(bn, 12, 1)
    lik = likelihoods(bn, 12, 2)
    lik["Dispnea"][3] = 0.0  # an impossible row
    got = bn.query_many(*QUERY, events=X, likelihoods=lik)
    want, log_ev = oracle_rows(bn, X, lik, QUERY)
    assert np.isnan(got.to_numpy()[3]).all()
    ok = np.arange(12) != 3
    np.testing.assert_allclose(got.to_numpy()[ok], want[ok], rtol=2e-6)
    lp = bn.predict_log_proba(X, likelihoods=lik)
    assert lp.iloc[3] == -np.inf
    np.testing.assert_allclose(lp.to_numpy()[ok], log_ev[ok], rtol=1e-6)
    np.testing.assert_allclose(bn.predict_proba(X, likelihoods=lik).to_numpy(), np.exp(lp.to_numpy()), rtol=1e-12)
    # a soft node may be queried
    q = bn.query_many("Dispnea", events=X, likelihoods=lik)
    np.testing.assert_allclose(q.to_numpy()[ok], oracle_rows(bn, X, lik, ("Dispnea",))[0][ok], rtol=2e-6)


def test_marginals_many_against_oracle(interpreted):
    bn = examples.asia()
    X = frame(bn, 6, 3)
    lik = likelihoods(bn, 6, 4)
    got = bn.marginals_many(X, likelihoods=lik)
    for t in got.columns.get_level_values(0).unique():
        want, _ = oracle_rows(bn, X, lik, (t,))
        np.testing.assert_allclose(got[t].to_numpy(), want, rtol=2e-6)


def test_every_accepted_form_gives_the_same_answer(interpreted):
    bn = examples.asia()
    X = frame(bn, 5, 5)
    lik = likelihoods(bn, 5, 6)
    base = bn.query_many(*QUERY, events=X, likelihoods=lik).to_numpy()
    net = bn._compiled
    frames = {s: pd.DataFrame(v[:, ::-1], columns=net.domains[net.index[s]][::-1]) for s, v in lik.items()}
    np.testing.assert_array_equal(bn.query_many(*QUERY, events=X, likelihoods=frames).to_numpy(), base)
    torch = pytest.importorskip("torch")
    as_torch = {s: torch.as_tensor(v) for s, v in lik.items()}
    np.testing.assert_array_equal(bn.query_many(*QUERY, events=X, likelihoods=as_torch).to_numpy(), base)
    # query: a vector, or a {state: weight} dict
    event = {c: X[c].iloc[0] for c in EV}
    one = {s: v[0] for s, v in lik.items()}
    a = bn.query(*QUERY, event=event, likelihoods=one)
    dom = {s: net.domains[net.index[s]] for s in SOFT}
    b = bn.query(*QUERY, event=event, likelihoods={s: dict(zip(dom[s], v)) for s, v in one.items()})
    pd.testing.assert_series_equal(a, b)
    np.testing.assert_allclose(a.to_numpy(), oracle_rows(bn, X.iloc[:1], {s: v[:1] for s, v in lik.items()}, QUERY)[0][0],
                               rtol=1e-12)
    assert InterpretedProgram.calls[-1] == (planner.VERSION, planner.MODE_BATCHED, True, 1)


@pytest.mark.parametrize("bad, match", [
    ({"Dispnea": np.ones((4, 2))}, "shape"),
    ({"Dispnea": np.ones((5, 3))}, "shape"),
    ({"Dispnea": np.full((5, 2), np.nan)}, "finite"),
    ({"Dispnea": np.full((5, 2), np.inf)}, "finite"),
    ({"Dispnea": -np.ones((5, 2))}, "non-negative"),
    ({"Dispnea": pd.DataFrame({"maybe": [1.0] * 5})}, "not states"),
    ({"Smoker": np.ones((5, 2))}, "both hard evidence"),
    ({"nope": np.ones((5, 2))}, "not a node"),
    ({}, "non-empty"),
])
def test_bad_likelihoods_raise(interpreted, bad, match):
    bn = examples.asia()
    X = frame(bn, 5, 7)
    with pytest.raises(ValueError, match=match):
        bn.query_many(*QUERY, events=X, likelihoods=bad)


def test_soft_calls_refuse_other_algorithms_and_devices(interpreted):
    bn = examples.asia()
    X = frame(bn, 5, 8)
    lik = likelihoods(bn, 5, 9)
    with pytest.raises(ValueError, match="exact"):
        bn.query_many(*QUERY, events=X, likelihoods=lik, algorithm="gibbs")
    with pytest.raises(ValueError, match="devices"):
        bn.query_many(*QUERY, events=X, likelihoods=lik, devices=[0, 0])


def test_rescue_reruns_the_flagged_rows_with_their_likelihoods(interpreted, monkeypatch):
    bn = examples.asia()
    net = bn._compiled
    n = 20
    X = frame(bn, n, 10)
    lik = likelihoods(bn, n, 11)
    L = np.concatenate([lik[s] for s in SOFT], axis=1)
    plan = planner.build_plan(net, [net.index[q] for q in QUERY], [net.index[c] for c in EV],
                              soft=[net.index[s] for s in SOFT])
    codes = np.array([[net.domains[net.index[c]].index(x) for x in X[c]] for c in EV], dtype=np.uint8)
    _, total, _ = soft_interp.run(plan.words, plan.table_blob, codes, L, dtype=np.float32)
    below = float(np.sort(total)[12])  # flags the 12 rows of the lowest normalisers: more than 8
    flagged = np.flatnonzero(~(total >= below))
    monkeypatch.setattr(InterpretedProgram, "flag_below", below)
    got = bn.query_many(*QUERY, events=X, likelihoods=lik)
    want, _ = oracle_rows(bn, X, lik, QUERY)
    np.testing.assert_allclose(got.to_numpy(), want, rtol=2e-6)
    np.testing.assert_allclose(got.to_numpy()[flagged], want[flagged], rtol=1e-12)  # settled in float64
    # one float64 re-run on the batched program, with the flagged rows' likelihoods
    f64 = [l for is64, l in SoftProgram.liks if is64]
    assert len(f64) == 1
    np.testing.assert_array_equal(f64[0], L[flagged])
    assert InterpretedProgram.calls[-1] == (planner.VERSION, planner.MODE_BATCHED, True, len(flagged))
    # a few flagged rows go the same way: the single-event programs take no likelihoods
    below = float(np.sort(total)[3])
    monkeypatch.setattr(InterpretedProgram, "flag_below", below)
    bn.query_many(*QUERY, events=X, likelihoods=lik)
    assert InterpretedProgram.calls[-1] == (planner.VERSION, planner.MODE_BATCHED, True, 3)


def test_cache_bound_holds_with_soft_entries(interpreted):
    bn = examples.asia()
    bn.max_cached_programs = 3
    X = frame(bn, 4, 13)
    lik = likelihoods(bn, 4, 14)
    for q in ["Lung cancer", "Tuberculosis", "Bronchitis", "TB or cancer", "Lung cancer"]:
        bn.query_many(q, events=X, likelihoods=lik)
        bn.query_many(q, events=X)
        assert len(bn._engine_cache) <= 3
    live = [p for p in InterpretedProgram.live if not p.closed]
    assert len(live) <= 3 * 2


def golden_check(bn, name, tol):
    """Every case of tests/golden/soft_<name>.json (the reference on virtual-child networks) through `query` and
    `predict_log_proba` with likelihoods."""
    from conftest import load_golden

    g = load_golden(f"soft_{name}")
    assert g["kind"] == "soft_evidence"
    n_log = 0
    for case in g["cases"]:
        event = {k: v for k, v in case["event"]}
        lik = {s: np.asarray(v) for s, v in case["likelihoods"]}
        got = bn.query(*case["query"], event=event, likelihoods=lik)
        want = case["values"]
        assert [list(k) if isinstance(k, tuple) else [k] for k in got.index.tolist()] == case["index"]
        np.testing.assert_allclose(got.to_numpy(), want, rtol=tol)
        if case.get("log_evidence") is not None and event:
            lp = bn.predict_log_proba(event, likelihoods=lik)
            assert abs(lp - case["log_evidence"]) <= tol * max(1.0, abs(case["log_evidence"]))
            n_log += 1
    return n_log


@pytest.mark.parametrize("name", ["alarm", "asia", "grades", "sprinkler"])
def test_reference_goldens(interpreted, name):
    bn = getattr(examples, name)()
    assert golden_check(bn, name, 1e-6) > 0
