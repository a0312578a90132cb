"""The host side of the posterior entry points (query, query_many, marginals, marginals_many, predict_proba) and
of the program cache, on the CPU: the device programs are replaced by the CPU interpreter
(tests/interpreted_program.py).  Only public entry points are driven, apart from the cache size."""
import numpy as np
import pandas as pd
import pytest

from interpreted_program import InterpretedProgram
from oracle import program_interp, ve_oracle
from sorobn_b200 import engine, examples, planner, workloads

EV = ["Dispnea", "Positive X-ray", "Smoker", "Visit to Asia"]  # sorted, as predict_proba orders its columns
QUERY = ("Lung cancer",)


@pytest.fixture
def interpreted(monkeypatch):
    monkeypatch.setattr(InterpretedProgram, "live", [])
    monkeypatch.setattr(InterpretedProgram, "calls", [])
    monkeypatch.setattr(InterpretedProgram, "flag_below", None)
    monkeypatch.setattr(engine, "Program", InterpretedProgram)
    return InterpretedProgram


def frame(bn, n, seed, columns=EV):
    net = bn._compiled
    codes = workloads.forward_sample_codes(net, n, seed)
    return pd.DataFrame({c: np.asarray(net.domains[net.index[c]], dtype=object)[codes[net.index[c]]] for c in columns},
                        index=pd.RangeIndex(10, 10 + n, name="row"))


def encode(bn, X):
    net = bn._compiled
    return np.array([[net.domains[net.index[c]].index(x) for x in X[c]] for c in X.columns], dtype=np.uint8)


def plan_of(bn, kind, X):
    net = bn._compiled
    ev = [net.index[c] for c in X.columns]
    if kind == "marginals":
        targets = sorted(n for n in bn.nodes if n not in X.columns)
        return planner.build_marginals_plan(net, ev, targets=[net.index[t] for t in targets])
    query = QUERY if kind == "posterior" else ()
    return planner.build_plan(net, [net.index[q] for q in query], ev, allow_empty_query=True)


def flagged(bn, kind, X, below):
    """The rows the batched float32 program flags when totals below `below` are out of range."""
    plan, codes = plan_of(bn, kind, X), encode(bn, X)
    if kind == "marginals":
        post = program_interp.run_marginals(plan.words, plan.table_blob, codes, dtype=np.float32, min_total=below)
        return np.flatnonzero(np.isnan(post).any(axis=0))
    _, total = program_interp.run(plan.words, plan.table_blob, codes, dtype=np.float32, return_totals=True)
    return np.flatnonzero(~(total >= below))


def threshold(bn, kind, X, few):
    """A `flag_below` under which 1 to 8 rows (few) or more than 8 but not every row are flagged, and those rows.
    The candidates lie between the rows' float64 levels: P(event), times the smallest non-zero marginal entry for
    a marginals program."""
    level = reference64(bn, "evidence", X)
    if kind == "marginals":
        post = reference64(bn, "marginals", X)
        level = level * np.where(post > 0, post, np.inf).min(axis=0)
    level = np.unique(level)
    for below in np.sqrt(level[1:] * level[:-1]):
        rows = flagged(bn, kind, X, below)
        if (1 <= len(rows) <= 8) if few else (8 < len(rows) < len(X)):
            return below, rows
    raise AssertionError("no threshold gives the wanted number of flagged rows")


def rescue_calls(version, rows):
    """The float64 re-runs of the flagged `rows`: one batched call for more than 8, else one flat call per row."""
    if len(rows) > 8:
        return [(version, planner.MODE_BATCHED, True, len(rows))]
    return [(version, planner.MODE_FLAT, True, 1)] * len(rows)


def reference64(bn, kind, X):
    plan, codes = plan_of(bn, kind, X), encode(bn, X)
    if kind == "marginals":
        return program_interp.run_marginals(plan.words, plan.table_blob64, codes, dtype=np.float64)
    post, total = program_interp.run(plan.words, plan.table_blob64, codes, dtype=np.float64, return_totals=True)
    return total if kind == "evidence" else post


ENTRY = {
    "posterior": (planner.VERSION, lambda bn, X: bn.query_many(*QUERY, events=X).to_numpy().T),
    "marginals": (planner.VERSION_MARGINALS, lambda bn, X: bn.marginals_many(X).to_numpy().T),
    "evidence": (planner.VERSION, lambda bn, X: bn.predict_proba(X).to_numpy()),
}


@pytest.mark.parametrize("few", [True, False], ids=["few", "many"])
@pytest.mark.parametrize("kind", list(ENTRY))
def test_flagged_rows_are_settled_in_float64_by_how_many_there_are(interpreted, kind, few):
    """Rows the float32 program flags are re-run in float64: more than 8 as one batch on the batched plan's
    float64 program, up to 8 one by one on the single-event program."""
    bn = examples.asia()
    # every joint state of the evidence columns, once (few) or three times (many), in a shuffled order
    states = pd.MultiIndex.from_product([[False, True]] * len(EV), names=EV).to_frame(index=False)
    X = pd.concat([states] * (1 if few else 3), ignore_index=True).sample(frac=1.0, random_state=3)
    version, call = ENTRY[kind]
    below, rows = threshold(bn, kind, X, few)
    plain = call(bn, X)
    assert interpreted.calls == [(version, planner.MODE_BATCHED, False, len(X))]
    interpreted.calls.clear()
    interpreted.flag_below = below
    got = call(bn, X)
    assert interpreted.calls == [(version, planner.MODE_BATCHED, False, len(X))] + rescue_calls(version, rows)
    assert not np.isnan(got).any()
    kept = np.setdiff1d(np.arange(len(X)), rows)
    assert np.array_equal(got[..., kept], plain[..., kept])
    np.testing.assert_allclose(got[..., rows], reference64(bn, kind, X)[..., rows], rtol=1e-12, atol=0)


def test_unknown_values_and_impossible_rows(interpreted):
    """A value outside its variable's domain gives a NaN row (0.0 in predict_proba) and is never re-run; a row of
    probability zero is re-run in float64 and stays NaN."""
    bn = examples.asia()
    X = pd.DataFrame({"TB or cancer": [False, "maybe", True, False], "Tuberculosis": [False, False, False, True]})
    post = bn.query_many(*QUERY, events=X)
    assert post.iloc[[1, 3]].isna().all().all() and not post.iloc[[0, 2]].isna().any().any()
    assert interpreted.calls == [(planner.VERSION, planner.MODE_BATCHED, False, 4),
                                 (planner.VERSION, planner.MODE_FLAT, True, 1)]
    marg = bn.marginals_many(X)
    assert marg.iloc[[1, 3]].isna().all().all() and not marg.iloc[[0, 2]].isna().any().any()
    p = bn.predict_proba(X[["Tuberculosis", "TB or cancer"]])
    assert p.iloc[1] == 0.0 and p.iloc[3] == 0.0 and (p.iloc[[0, 2]] > 0).all()
    assert p.name == "P(TB or cancer, Tuberculosis)" and p.index.names == ["TB or cancer", "Tuberculosis"]
    assert bn.predict_log_proba(X[["Tuberculosis", "TB or cancer"]]).iloc[3] == -np.inf


def test_empty_frames_and_frames_without_evidence_columns(interpreted):
    bn = examples.asia()
    empty = frame(bn, 0, 1)
    got = bn.query_many(*QUERY, events=empty)
    assert got.shape == (0, 2) and got.index.equals(empty.index) and list(got.columns) == [False, True]
    assert got.columns.name == "Lung cancer"
    marg = bn.marginals_many(empty)
    assert marg.shape == (0, 8) and marg.columns.names == ["variable", "state"]
    p = bn.predict_proba(empty)
    assert len(p) == 0 and p.dtype == np.float64 and p.name == f"P({', '.join(EV)})"
    # no evidence column: every row is the prior, no row is flagged
    none = pd.DataFrame(index=pd.RangeIndex(3))
    got = bn.query_many(*QUERY, events=none)
    prior = ve_oracle.query(ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes), *QUERY, event={})[1]
    assert got.shape == (3, 2) and np.allclose(got.to_numpy(), prior.reshape(1, -1), rtol=1e-6)
    marg = bn.marginals_many(none)
    assert marg.shape == (3, 16) and np.allclose(marg["Lung cancer"].to_numpy(), prior.reshape(1, -1), rtol=1e-6)


@pytest.mark.parametrize("event", [{"TB or cancer": False}, {"Smoker": True, "Dispnea": False},
                                   {"TB or cancer": False, "Lung cancer": True}, {"Smoker": "maybe"}])
def test_query_and_marginals_of_one_event(interpreted, event):
    """The single-event programs run in float64: states of probability zero are left out, and evidence of
    probability zero or outside the domain gives empty Series."""
    bn = examples.asia()
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    possible = "maybe" not in event.values() and "Lung cancer" not in event
    marginals = bn.marginals(event)
    assert list(marginals) == sorted(n for n in bn.nodes if n not in event)
    for q in ("Tuberculosis", "Bronchitis"):
        got = bn.query(q, event=event)
        assert got.name == f"P({q})" and got.index.name == q
        assert marginals[q].name == got.name and marginals[q].index.equals(got.index)
        if not possible:
            assert len(got) == 0 and got.dtype == np.float64
            continue
        _, want, support = ve_oracle.query(dn, q, event=event)
        states = np.asarray(bn._compiled.domains[bn._compiled.index[q]], dtype=object)[support.reshape(-1)]
        assert list(got.index) == list(states) and (got > 0).all()
        np.testing.assert_allclose(got.to_numpy(), want.reshape(-1)[support.reshape(-1)], rtol=1e-12)
        np.testing.assert_allclose(marginals[q].to_numpy(), got.to_numpy(), rtol=1e-12)
    assert all(f64 for _, _, f64, _ in interpreted.calls)
    assert all(mode == planner.MODE_FLAT and n == 1 for _, mode, _, n in interpreted.calls)


def run_all(bn, X, Xm):
    """Every exact-inference kind once, each with its own programs."""
    out = [bn.query_many(*QUERY, events=X), bn.marginals_many(X), bn.predict_proba(X)]
    out += list(bn.expected_counts(Xm).values())
    out += [bn.sample_many(Xm, n=2, seed=5), bn.mpe_many(Xm), bn.map_many(Xm)]
    out += [bn.query("Bronchitis", event={"Smoker": True})]
    out += list(bn.marginals({"Dispnea": True}).values())
    return out


def test_the_cache_bound_holds_across_every_kind_and_closes_what_it_evicts(interpreted):
    bn = examples.asia()
    X = frame(bn, 40, 2)
    Xm = frame(bn, 40, 3, columns=["Dispnea", "Smoker", "Bronchitis"])
    Xm = Xm.mask(np.random.default_rng(4).random(Xm.shape) < 0.3)
    want = run_all(bn, X, Xm)
    interpreted.live.clear()
    small = examples.asia()
    small.max_cached_programs = 3
    for _ in range(2):
        got = run_all(small, X, Xm)
        assert len(small._engine_cache) <= small.max_cached_programs
        assert all(g.equals(w) for g, w in zip(got, want))
    # one more plan with room for one entry: every other program is closed
    small.max_cached_programs = 1
    small.query_many("Tuberculosis", events=X)
    assert [p.plan.query for p in interpreted.live if not p.closed] == [(small._compiled.index["Tuberculosis"],)]
