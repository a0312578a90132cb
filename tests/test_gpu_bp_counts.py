"""Expected counts and Bethe-EM by loopy belief propagation on the device (csrc/sbn_bp.cu, version-3 words) against
the exact path and the float64 oracle.

Tolerances come from the float32 replay of the same words (tests/test_bp_counts_plan.py): F32_COUNTS_TOL per row
counted for a count entry, F32_LOGZ_TOL for a row's Bethe log-likelihood (relative beyond 1)."""
import warnings

import numpy as np
import pytest

import bp_counts_oracle
from sorobn_b200 import BayesNet, bp, engine, planner, synthetic
from test_bp_counts_plan import F32_COUNTS_TOL, F32_LOGZ_TOL, counts_graph, dense, dense_counts, evidence_names, sampled
from test_bp_mpe_plan import IMPOSSIBLE_OBSERVED, structural_zero_chain
from test_bp_plan import GRID16_EVIDENCE, LOOPY, WIDE, naive_bayes_spec, near_tol, network
from test_gpu_bp import frame, rows

pytestmark = pytest.mark.gpu


def missing_frame(bn, n, seed, frac=0.3, drop=()):
    """n rows drawn from the network, a fraction `frac` of the cells missing, the `drop` columns removed (latent)."""
    X = frame(bn._compiled, list(bn.nodes), sampled(bn, list(bn.nodes), n, seed))
    X = X.drop(columns=list(drop)).astype(object)
    mask = np.random.default_rng(seed).random(X.shape) < frac
    X = X.mask(mask, None)
    return X


def logz_tol(z):
    return F32_LOGZ_TOL * np.maximum(1.0, np.abs(z))


@pytest.mark.parametrize("name,latent", [("chain12s4", ()), ("naive_bayes", ("C",)), ("chow_liu", ())])
def test_polytrees_equal_the_exact_expected_counts(name, latent):
    bn = network(name)
    X = missing_frame(bn, 3000, seed=1, frac=0.3, drop=latent)
    exact = bn.expected_counts(X)
    got = bn.expected_counts(X, algorithm="bp", damping=0.0, tol=1e-6)
    assert set(got) == set(exact)
    for v in exact:
        assert got[v].index.equals(exact[v].index)
        assert np.allclose(got[v].to_numpy(), exact[v].to_numpy(), rtol=0, atol=F32_COUNTS_TOL * len(X)), v


def test_latent_class_em_follows_the_exact_trajectory():
    spec = naive_bayes_spec()
    truth = synthetic.load(spec, BayesNet)
    X = missing_frame(truth, 4000, seed=4, frac=0.2, drop=("C",))
    start = {n: np.asarray(t) for n, t in truth.cpt_tensors().items()}
    rng = np.random.default_rng(5)
    start = {n: 0.5 * t + 0.5 * rng.dirichlet(np.ones(t.shape[-1]), size=t.shape[:-1]) for n, t in start.items()}
    a = synthetic.load(spec, BayesNet).assign_cpts(start)
    b = synthetic.load(spec, BayesNet).assign_cpts(start)
    a.fit_em(X, max_iter=6, tol=-1.0)
    b.fit_em(X, max_iter=6, tol=-1.0, algorithm="bp", damping=0.0, bp_tol=1e-6)
    assert len(a.em_log_likelihood_) == len(b.em_log_likelihood_) == 6
    la, lb = np.array(a.em_log_likelihood_), np.array(b.em_log_likelihood_)
    assert np.allclose(lb, la, rtol=2e-6, atol=0), (la, lb)
    ta, tb = a.cpt_tensors(), b.cpt_tensors()
    for n in ta:
        assert np.allclose(tb[n].numpy(), ta[n].numpy(), rtol=0, atol=2e-5), n
    for n in a._P_sizes:
        assert np.allclose(np.asarray(b._P_sizes[n]), np.asarray(a._P_sizes[n]), rtol=1e-5)


def test_fully_observed_frame_gives_the_exact_counts_and_log_likelihood():
    bn = network("alarm")
    names = list(bn.nodes)
    codes = sampled(bn, names, 2000, seed=6)
    X = frame(bn._compiled, names, codes)
    exact = bn.expected_counts(X)
    got = bn.expected_counts(X, algorithm="bp")
    for v in exact:
        assert np.array_equal(got[v].to_numpy(), exact[v].to_numpy()), v
    net = bn._compiled
    g = counts_graph(bn, names)
    r = engine.BeliefPropagation(g.words, g.tables)
    _, log_z, iters = r.counts(codes, codes.shape[1], 10, 0.5, 1e-5)
    r.close()
    assert (iters == 0).all()
    want = np.zeros(codes.shape[1])
    for v in range(len(net.names)):
        cpt = np.asarray(net.cpt[v], dtype=np.float32).astype(np.float64)
        want += np.log(cpt[tuple(codes[names.index(net.names[u])] for u in net.scope(v))])
    assert np.allclose(log_z, want, rtol=1e-12, atol=0)
    a, b = network("alarm"), network("alarm")
    a.fit_em(X, max_iter=1)
    b.fit_em(X, max_iter=1, algorithm="bp")
    assert abs(b.em_log_likelihood_[0] - a.em_log_likelihood_[0]) < 1e-6 * abs(a.em_log_likelihood_[0])


def device_vs_oracle(bn, names, codes, n_iterations, damping, tol):
    g = counts_graph(bn, names)
    r = engine.BeliefPropagation(g.words, g.tables)
    got, log_z, iters = r.counts(codes, codes.shape[1], n_iterations, damping, tol)
    r.close()
    want = bp_counts_oracle.run(dense(bn), names, codes, n_iterations, damping, tol)
    assert np.array_equal(np.isnan(log_z), np.isnan(want["log_z"]))
    same = iters == want["iterations"]
    assert not (~same & ~near_tol(want["residual"], iters, want["iterations"], tol, 2e-6)).any()
    ok = same & ~np.isnan(log_z)
    err = np.abs(log_z[ok] - want["log_z"][ok])
    assert (err < logz_tol(want["log_z"][ok])).all(), err.max()
    if same.all():
        counts = dense_counts(bn, g, got)
        for v in bn.nodes:
            assert np.allclose(counts[v], want["counts"][v], rtol=0, atol=F32_COUNTS_TOL * codes.shape[1]), v
    return same


@pytest.mark.parametrize("name", LOOPY + WIDE + ["alarm"])
def test_loopy_networks_match_the_oracle(name):
    bn = network(name)
    names = evidence_names(bn, max(1, len(bn.nodes) // 4), seed=7)
    codes = rows(bn, names, 400, seed=8)  # every 5th row random: some impossible, some dead before the first sweep
    for damping, tol, n_iterations in [(0.5, 0.0, 30), (0.3, 0.0, 6), (0.5, 1e-5, 100)]:
        same = device_vs_oracle(bn, names, codes, n_iterations, damping, tol)
        assert same.mean() > 0.9


def test_grid10x10_matches_the_oracle():
    bn = synthetic.load(synthetic.grid(10, 10, 5), BayesNet)
    names = evidence_names(bn, 30, seed=9)
    codes = sampled(bn, names, 100, seed=10)
    device_vs_oracle(bn, names, codes, 8, 0.5, 0.0)


def test_em_on_the_grid_the_exact_planner_refuses():
    spec = synthetic.grid(16, 16, 3)
    truth = synthetic.load(spec, BayesNet)
    net = truth._compiled
    with pytest.raises(ValueError):
        planner.build_counts_plan(net, tuple(sorted(net.index[e] for e in GRID16_EVIDENCE)))
    n = 4000
    X = frame(net, list(truth.nodes), sampled(truth, list(truth.nodes), n, seed=11)).astype(object)
    rng = np.random.default_rng(12)
    patterns = rng.random((4, X.shape[1])) < 0.3  # four missingness patterns, 30 % of the cells each
    X = X.mask(patterns[rng.integers(0, 4, size=n)], None)
    want = truth.cpt_tensors()
    start = {k: 0.5 * np.asarray(t) + 0.5 * rng.dirichlet(np.ones(3), size=t.shape[:-1]) for k, t in want.items()}
    bn = synthetic.load(spec, BayesNet).assign_cpts(start)

    def error(cpts):
        return float(np.mean([np.abs(np.asarray(cpts[k]) - np.asarray(want[k])).mean() for k in want]))

    before = error(start)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        bn.fit_em(X, max_iter=5, algorithm="bp", n_iterations=50)
    assert len([w for w in caught if issubclass(w.category, RuntimeWarning)]) <= 1
    after = error(bn.cpt_tensors())
    assert after < 0.75 * before, (before, after)
    assert np.isfinite(bn.em_log_likelihood_).all()


@pytest.mark.parametrize("k", range(len(IMPOSSIBLE_OBSERVED)))
def test_dead_rows_raise_as_the_exact_path(k):
    bn = structural_zero_chain()
    X = IMPOSSIBLE_OBSERVED[k]
    with pytest.raises(ValueError) as exact_error:
        bn.expected_counts(X)
    with pytest.raises(ValueError) as bp_error:
        bn.expected_counts(X, algorithm="bp")
    assert str(bp_error.value) == str(exact_error.value)
    with pytest.raises(ValueError):
        bn.fit_em(X, algorithm="bp", max_iter=2)
    names = list(X.columns)
    net = bn._compiled
    codes = np.stack([[net.domains[net.index[c]].index(x) for x in X[c]] for c in names]).astype(np.uint8)
    g = counts_graph(bn, names)
    r = engine.BeliefPropagation(g.words, g.tables)
    _, log_z, iters = r.counts(codes, codes.shape[1], 20, 0.5, 1e-6)
    zero = X.index == "zero"
    assert np.isnan(log_z[zero]).all() and (iters[zero] == 0).all() and not np.isnan(log_z[~zero]).any()


def test_non_converged_rows_warn_once():
    bn = network("grid4x4s3")
    X = missing_frame(bn, 500, seed=13, frac=0.5)
    with pytest.warns(RuntimeWarning, match="did not converge") as caught:
        bn.expected_counts(X, algorithm="bp", n_iterations=1, tol=0.0)
    assert len([w for w in caught if issubclass(w.category, RuntimeWarning)]) == 1
    with pytest.warns(RuntimeWarning, match="did not converge") as caught:
        bn.fit_em(X, algorithm="bp", max_iter=3, tol=-1.0, n_iterations=1, bp_tol=0.0)
    assert len([w for w in caught if issubclass(w.category, RuntimeWarning)]) == 1


def test_determinism_and_chunking(monkeypatch):
    bn = synthetic.load(synthetic.grid(10, 10, 5), BayesNet)
    names = evidence_names(bn, 30, seed=14)
    codes = rows(bn, names, 60_000, seed=15)
    g = counts_graph(bn, names)
    r = engine.BeliefPropagation(g.words, g.tables)
    a = r.counts(codes, codes.shape[1], 10, 0.5, 1e-4)
    b = r.counts(codes, codes.shape[1], 10, 0.5, 1e-4)
    for x, y in zip(a, b):
        assert np.array_equal(x, y, equal_nan=True)
    monkeypatch.setenv("SOROBN_B200_CHUNK_ROWS", "17000")
    c = engine.BeliefPropagation(g.words, g.tables).counts(codes, codes.shape[1], 10, 0.5, 1e-4)
    assert np.array_equal(c[1], a[1], equal_nan=True) and np.array_equal(c[2], a[2])
    assert np.allclose(c[0], a[0], rtol=1e-12, atol=0)
    r.close()


def test_set_tables_and_the_run_calls_refuse_other_words():
    bn = network("asia")
    net = bn._compiled
    g1 = bp.compile_graph(net, [0], [1])
    g2 = bp.compile_mpe_graph(net, [0])
    g3 = bp.compile_counts_graph(net, [0])
    r1, r2, r3 = (engine.BeliefPropagation(g.words, g.tables) for g in (g1, g2, g3))
    codes = np.zeros((1, 4), np.uint8)
    with pytest.raises(engine.EngineError, match="sbn_bp_counts_host"):
        r3.run(codes, 4, 5, 0.5, 1e-5)
    with pytest.raises(engine.EngineError, match="sbn_bp_counts_host"):
        r3.mpe(codes, 4, 5, 0.5, 1e-5)
    with pytest.raises(engine.EngineError, match="sbn_bp_run_host"):
        r1.counts(codes, 4, 5, 0.5, 1e-5)
    with pytest.raises(engine.EngineError, match="sbn_bp_mpe_host"):
        r2.counts(codes, 4, 5, 0.5, 1e-5)
    with pytest.raises(engine.EngineError, match="table floats|floats"):
        r3.set_tables(g3.tables[:-1])
    # new tables of the same size: the counts of a graph compiled with them
    cpts = [np.flip(np.asarray(c, dtype=np.float64), axis=-1) * 0.5 + 0.25 for c in net.cpt]  # binary: rows sum to 1
    flat = np.concatenate([c.reshape(-1) for c in cpts])
    r3.set_tables(flat[g3.perm])
    before = r3.counts(codes, 4, 20, 0.5, 1e-6)
    bn.assign_cpts({name: cpts[v] for v, name in enumerate(net.names)})
    g4 = bp.compile_counts_graph(bn._compiled, [0])
    fresh = engine.BeliefPropagation(g4.words, g4.tables).counts(codes, 4, 20, 0.5, 1e-6)
    for x, y in zip(before, fresh):
        assert np.array_equal(x, y, equal_nan=True)
