"""The host side of soft evidence on counts, EM, samples, MPE and marginal MAP (the likelihoods= keyword of
expected_counts, fit_em, sample_many, mpe_many / mpe and map_many / map) on the CPU: the device programs are
replaced by the CPU replay of their words, and only public entry points are driven."""
import numpy as np
import pandas as pd
import pytest

import em_oracle
import map_oracle
import mpe_oracle
import soft_oracle
import soft_pattern_interp as spi
from oracle import ve_oracle
from sorobn_b200 import engine, examples, workloads
from test_soft_host import SoftProgram

SOFT = "Dispnea"


class PatternProgram(SoftProgram):
    """SoftProgram whose counts, sample, MPE and MAP runs take likelihoods `lik` (numpy or torch), recorded in
    `liks` with the program's precision."""

    def _lik(self, lik):
        # as engine.Program: the float32 MPE and MAP programs take float64 likelihoods
        dtype = np.float64 if self.plan.version in (8, 9) else self.dtype
        lik = np.asarray(lik.cpu().numpy() if hasattr(lik, "cpu") else lik, dtype=dtype)
        PatternProgram.liks.append((self.f64, lik.copy()))
        return lik

    def counts(self, codes, n_rows, lik=None, log_evidence=False):
        if lik is None:
            return super().counts(codes, n_rows)
        self._start(n_rows)
        c, prob, log_ev = spi.run_counts(self.plan.words, self.blob, codes, self._lik(lik), n_rows=n_rows,
                                         dtype=self.dtype, min_total=self._min_total())
        return (c, prob, log_ev) if log_evidence else (c, prob)

    def sample(self, codes, n_rows, n_draws, seed, row_base=0, lik=None, log_evidence=False):
        if lik is None:
            return super().sample(codes, n_rows, n_draws, seed, row_base)
        self._start(n_rows)
        drawn, prob, _, log_ev = spi.run_sample(self.plan.words, self.plan.table_blob64, codes, self._lik(lik),
                                                n_rows=n_rows, n_draws=n_draws, seed=seed, row_base=row_base,
                                                min_total=self._min_total())
        prob = prob.astype(self.dtype)
        return (drawn, prob, log_ev) if log_evidence else (drawn, prob)

    def mpe(self, codes, n_rows, lik=None):
        if lik is None:
            return super().mpe(codes, n_rows)
        self._start(n_rows)
        return spi.run_mpe(self.plan.words, self.plan.table_blob, codes, self._lik(lik), n_rows=n_rows)

    def map(self, codes, n_rows, lik=None):
        return self.mpe(codes, n_rows, lik)


@pytest.fixture
def interpreted(monkeypatch):
    monkeypatch.setattr(PatternProgram, "live", [])
    monkeypatch.setattr(PatternProgram, "calls", [])
    monkeypatch.setattr(PatternProgram, "flag_below", None)
    monkeypatch.setattr(PatternProgram, "liks", [])
    monkeypatch.setattr(engine, "Program", PatternProgram)
    return PatternProgram


def frame(bn, n, seed, cols=("Smoker", "Visit to Asia", "Positive X-ray"), frac=0.35):
    """n rows of asia with the cells of `cols` missing at random (scattered patterns)."""
    net = bn._compiled
    codes = workloads.forward_sample_codes(net, n, seed)
    rng = np.random.default_rng(seed)
    out = {}
    for c in cols:
        vals = np.asarray(net.domains[net.index[c]], dtype=object)[codes[net.index[c]]].copy()
        vals[rng.random(n) < frac] = None
        out[c] = vals
    return pd.DataFrame(out, index=pd.RangeIndex(3, 3 + n, name="row")), codes


def lik_of(n, seed, card=2):
    rng = np.random.default_rng(seed)
    return rng.random((n, card)) * 10.0 ** rng.integers(-3, 3, (n, 1)) + 1e-3


def row_events(X, b, lik):
    return {k: v for k, v in X.iloc[b].items() if v is not None and v == v}, {k: v[b] for k, v in lik.items()}


def test_counts_mpe_map_against_the_oracle_with_scattered_patterns(interpreted):
    bn = examples.asia()
    X, _ = frame(bn, 40, 1)
    lik = {SOFT: lik_of(40, 2), "Tuberculosis": lik_of(40, 3)}
    dn = soft_oracle.dense(bn._compiled)
    counts = bn.expected_counts(X, likelihoods=lik)
    want = {n: 0.0 for n in bn.nodes}
    for b in range(len(X)):
        hard, s = row_events(X, b, lik)
        vnet, event, _ = soft_oracle.virtual(dn, s)
        for node, c in em_oracle.expected_counts(vnet, [{**hard, **event}]).items():
            if node in want:
                want[node] = want[node] + c
    for node in bn.nodes:
        np.testing.assert_allclose(counts[node].to_numpy(), want[node].reshape(-1), rtol=2e-5, atol=1e-9)
    frame_, lp = bn.mpe_many(X, return_log_proba=True, likelihoods=lik)
    mframe, mlp = bn.map_many(X, return_log_proba=True, likelihoods=lik)
    assert list(mframe.columns) == sorted(X.columns)
    for b in range(len(X)):
        hard, s = row_events(X, b, lik)
        vnet, event, log_k = soft_oracle.virtual(dn, s)
        x, L = mpe_oracle.brute_force(vnet, {**hard, **event})
        assert abs(lp.iloc[b] - (L + log_k)) <= 1e-5 * max(1.0, abs(L))
        assert all(frame_.iloc[b][k] == v for k, v in x.items())
        x, L, gap = map_oracle.solve(vnet, {**hard, **event}, [c for c in X.columns if c not in hard])
        assert abs(mlp.iloc[b] - (L + log_k)) <= 1e-5 * max(1.0, abs(L))
        if gap > 1e-4:
            assert all(mframe.iloc[b][k] == v for k, v in x.items())
    # every pattern's program got exactly the likelihood rows of its own rows
    assert sum(len(lk) for f64, lk in interpreted.liks) == 3 * len(X)


def test_torch_and_numpy_likelihoods_agree(interpreted):
    torch = pytest.importorskip("torch")
    bn = examples.asia()
    X, _ = frame(bn, 25, 4)
    lik = lik_of(25, 5)
    t = {SOFT: torch.as_tensor(lik)}
    pd.testing.assert_frame_equal(bn.mpe_many(X, likelihoods=t), bn.mpe_many(X, likelihoods={SOFT: lik}))
    pd.testing.assert_frame_equal(bn.map_many(X, likelihoods=t), bn.map_many(X, likelihoods={SOFT: lik}))
    pd.testing.assert_frame_equal(bn.sample_many(X, 2, seed=1, likelihoods=t),
                                  bn.sample_many(X, 2, seed=1, likelihoods={SOFT: lik}))
    a, b = bn.expected_counts(X, likelihoods=t), bn.expected_counts(X, likelihoods={SOFT: lik})
    for node in bn.nodes:
        pd.testing.assert_series_equal(a[node], b[node])


def test_flagged_rows_rerun_in_float64_with_their_likelihoods(interpreted):
    bn = examples.asia()
    X, _ = frame(bn, 30, 6)
    lik = {SOFT: lik_of(30, 7)}
    want_counts = bn.expected_counts(X, likelihoods=lik)
    want_draws = bn.sample_many(X, 3, seed=9, likelihoods=lik)
    interpreted.flag_below = 0.05  # rows of small P(observed, lik / max) come back NaN from the float32 program
    interpreted.liks.clear()
    got = bn.expected_counts(X, likelihoods=lik)
    f64 = [lk for is64, lk in interpreted.liks if is64]
    assert f64 and sum(len(lk) for lk in f64) < len(X)
    for node in bn.nodes:
        np.testing.assert_allclose(got[node].to_numpy(), want_counts[node].to_numpy(), rtol=1e-5)
    # the rerun rows' likelihoods are theirs: a rerun row is one of the frame's likelihood rows
    rows = {tuple(r) for r in lik[SOFT]}
    assert all(tuple(r) in rows for lk in f64 for r in lk)
    pd.testing.assert_frame_equal(bn.sample_many(X, 3, seed=9, likelihoods=lik), want_draws)


def test_one_hot_is_the_column_and_all_ones_is_no_column(interpreted):
    bn = examples.asia()
    X, codes = frame(bn, 30, 8, cols=("Smoker", "Positive X-ray"))
    net = bn._compiled
    v = net.index[SOFT]
    hot = np.eye(2)[codes[v]] * 0.5
    Xh = X.assign(**{SOFT: np.asarray(net.domains[v], dtype=object)[codes[v]]})
    # counts
    a, b = bn.expected_counts(Xh), bn.expected_counts(X, likelihoods={SOFT: hot})
    for node in bn.nodes:
        np.testing.assert_allclose(b[node].to_numpy(), a[node].to_numpy(), rtol=1e-5, atol=1e-9)
    a, b = bn.expected_counts(X), bn.expected_counts(X, likelihoods={SOFT: np.ones((30, 2))})
    for node in bn.nodes:
        np.testing.assert_allclose(b[node].to_numpy(), a[node].to_numpy(), rtol=1e-5, atol=1e-9)
    # MPE: the soft node is decoded to its one-hot state; log P moves by log 0.5
    fa, la = bn.mpe_many(Xh, return_log_proba=True)
    fb, lb = bn.mpe_many(X, return_log_proba=True, likelihoods={SOFT: hot})
    pd.testing.assert_frame_equal(fb, fa)
    np.testing.assert_allclose(lb, la + np.log(0.5), rtol=1e-6)
    fa, la = bn.mpe_many(X, return_log_proba=True)
    fb, lb = bn.mpe_many(X, return_log_proba=True, likelihoods={SOFT: np.ones((30, 2))})
    pd.testing.assert_frame_equal(fb, fa)
    np.testing.assert_allclose(lb, la, rtol=1e-6)
    # MAP: the soft node is summed out, so one-hot gives the column's MAP states of the other missing cells
    fa, la = bn.map_many(Xh, return_log_proba=True)
    fb, lb = bn.map_many(X, return_log_proba=True, likelihoods={SOFT: hot})
    pd.testing.assert_frame_equal(fb, fa[fb.columns])
    np.testing.assert_allclose(lb, la + np.log(0.5), rtol=1e-6)
    fa, la = bn.map_many(X, return_log_proba=True)
    fb, lb = bn.map_many(X, return_log_proba=True, likelihoods={SOFT: np.ones((30, 2))})
    pd.testing.assert_frame_equal(fb, fa)
    np.testing.assert_allclose(lb, la, rtol=1e-6)
    # sample: one-hot pins the soft node's draws
    draws = bn.sample_many(X, 4, seed=2, likelihoods={SOFT: hot})
    np.testing.assert_array_equal(draws[SOFT].to_numpy(), np.repeat(Xh[SOFT].to_numpy(), 4))


def test_scale_moves_only_the_log_probabilities(interpreted):
    bn = examples.asia()
    X, _ = frame(bn, 20, 10)
    lik = lik_of(20, 11)
    c = 2.0 ** 7  # exact in float32, so the packed slots are the same
    fa, la = bn.mpe_many(X, return_log_proba=True, likelihoods={SOFT: lik})
    fb, lb = bn.mpe_many(X, return_log_proba=True, likelihoods={SOFT: lik * c})
    pd.testing.assert_frame_equal(fa, fb)
    np.testing.assert_allclose(lb - la, np.log(c), rtol=1e-9)
    fa, la = bn.map_many(X, return_log_proba=True, likelihoods={SOFT: lik})
    fb, lb = bn.map_many(X, return_log_proba=True, likelihoods={SOFT: lik * c})
    pd.testing.assert_frame_equal(fa, fb)
    np.testing.assert_allclose(lb - la, np.log(c), rtol=1e-9)
    a, b = bn.expected_counts(X, likelihoods={SOFT: lik}), bn.expected_counts(X, likelihoods={SOFT: lik * c})
    for node in bn.nodes:
        pd.testing.assert_series_equal(a[node], b[node])
    pd.testing.assert_frame_equal(bn.sample_many(X, 2, seed=4, likelihoods={SOFT: lik}),
                                  bn.sample_many(X, 2, seed=4, likelihoods={SOFT: lik * c}))
    # fit_em: the same CPTs, and the log-likelihood moves by n log c
    one, two = examples.asia(), examples.asia()
    one.fit_em(X, max_iter=3, likelihoods={SOFT: lik})
    two.fit_em(X, max_iter=3, likelihoods={SOFT: lik * c})
    np.testing.assert_allclose(np.array(two.em_log_likelihood_) - one.em_log_likelihood_, len(X) * np.log(c), rtol=1e-9)
    for node in one.nodes:
        pd.testing.assert_series_equal(one.P[node], two.P[node])


@pytest.mark.parametrize("c", [1e-50, 1e40])
def test_scales_float32_cannot_hold_decode_as_the_unscaled_likelihoods(interpreted, c):
    bn = examples.asia()
    X, _ = frame(bn, 20, 16)
    lik = lik_of(20, 17)
    for many in (bn.mpe_many, bn.map_many):
        fa, la = many(X, return_log_proba=True, likelihoods={SOFT: lik})
        fb, lb = many(X, return_log_proba=True, likelihoods={SOFT: lik * c})
        pd.testing.assert_frame_equal(fb, fa)
        np.testing.assert_allclose(lb - la, np.log(c), rtol=0, atol=1e-5)
    one = pd.DataFrame({"Smoker": [True, None]})
    base = np.array([[.2, .8], [.9, .1]])
    pd.testing.assert_frame_equal(bn.mpe_many(one, likelihoods={SOFT: base * c}), bn.mpe_many(one, likelihoods={SOFT: base}))


def test_fit_em_log_likelihood_is_that_of_the_observed_cells_and_likelihoods(interpreted):
    bn = examples.asia()
    X, _ = frame(bn, 20, 12)
    lik = {SOFT: lik_of(20, 13)}
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    want = sum(soft_oracle.log_evidence(dn, *row_events(X, b, lik)) for b in range(len(X)))
    bn.fit_em(X, max_iter=1, likelihoods=lik)
    assert abs(bn.em_log_likelihood_[0] - want) <= 1e-5 * abs(want)


def test_map_of_a_pattern_that_observes_nothing_still_has_its_likelihood(interpreted):
    bn = examples.asia()
    X = pd.DataFrame({"Smoker": [None] * 4})
    lik = {SOFT: lik_of(4, 14)}
    frame_, lp = bn.map_many(X, variables=[], return_log_proba=True, likelihoods=lik)
    assert frame_["Smoker"].isna().all()
    dn = soft_oracle.dense(bn._compiled)
    for b in range(4):
        want = soft_oracle.log_evidence(dn, {}, {SOFT: lik[SOFT][b]})
        assert abs(lp.iloc[b] - want) <= 1e-5 * max(1.0, abs(want))
    assert not lp.eq(0).any()


def test_single_events_take_vectors_and_state_dicts(interpreted):
    bn = examples.asia()
    event = {"Smoker": True}
    a = bn.mpe(event, likelihoods={SOFT: [0.2, 0.9]})
    b = bn.mpe(event, likelihoods={SOFT: {False: 0.2, True: 0.9}})
    pd.testing.assert_series_equal(a, b)
    assert bn.map(event, variables=["Lung cancer"], likelihoods={SOFT: np.array([0.9, 0.1])}).index.tolist() == \
        ["Lung cancer", "Smoker"]


def test_refusals_and_cache_keys(interpreted):
    bn = examples.asia()
    X, _ = frame(bn, 10, 15)
    with pytest.raises(ValueError, match="both hard evidence and likelihoods"):
        bn.expected_counts(X, likelihoods={"Smoker": np.ones((10, 2))})
    with pytest.raises(ValueError, match="shape"):
        bn.mpe_many(X, likelihoods={SOFT: np.ones((9, 2))})
    with pytest.raises(ValueError, match="non-negative"):
        bn.map_many(X, likelihoods={SOFT: -np.ones((10, 2))})
    with pytest.raises(ValueError, match="not a node"):
        bn.sample_many(X, likelihoods={"nope": np.ones((10, 2))})
    zero = np.ones((10, 2))
    zero[4] = 0.0  # an all-zero likelihood row: probability zero
    for call in (lambda: bn.expected_counts(X, likelihoods={SOFT: zero}),
                 lambda: bn.sample_many(X, likelihoods={SOFT: zero}),
                 lambda: bn.mpe_many(X, likelihoods={SOFT: zero}),
                 lambda: bn.map_many(X, likelihoods={SOFT: zero}),
                 lambda: bn.fit_em(X, max_iter=1, likelihoods={SOFT: zero})):
        with pytest.raises(ValueError, match="probability zero"):
            call()
    # keys without soft evidence keep their shape; with it, the soft var ids come last before the device
    bn._engine_cache.clear()
    bn.mpe_many(X)
    bn.mpe_many(X, likelihoods={SOFT: np.ones((10, 2))})
    keys = list(bn._engine_cache)
    plain = [k for k in keys if len(k) == 3]
    soft = [k for k in keys if len(k) == 4]
    assert plain and soft and len(plain) + len(soft) == len(keys)
    assert all(k[0] == "mpe" and k[2] == (bn._compiled.index[SOFT],) for k in soft)


def impute_golden_check(bn, name):
    """Every case of tests/golden/soft_impute_<name>.json (the reference's `impute` on virtual-child networks)
    through `map_many` with likelihoods: the imputed cells are the marginal MAP state of the missing ones."""
    from conftest import load_golden

    g = load_golden(f"soft_impute_{name}")
    assert g["kind"] == "soft_impute"
    for case in g["cases"]:
        row = {**{k: v for k, v in case["hard"]}, **{m: None for m in case["missing"]}}
        X = pd.DataFrame([row], columns=sorted(row))
        lik = {s: np.asarray(v)[None, :] for s, v in case["likelihoods"]}
        got = bn.map_many(X, likelihoods=lik).iloc[0]
        assert {m: got[m] for m in case["missing"]} == {m: v for m, v in case["imputed"]}, case
    return len(g["cases"])


@pytest.mark.parametrize("name", ["alarm", "asia", "grades", "sprinkler"])
def test_reference_impute_goldens(interpreted, name):
    assert impute_golden_check(getattr(examples, name)(), name) > 0
