"""Loopy belief propagation on the device (csrc/sbn_bp.cu) against the exact path and the float64 oracle.

Tolerances come from the float32 replay of the same words (tests/test_bp_plan.py): F32_BELIEF_TOL for beliefs and
F32_RESIDUAL_NOISE for how far a row's residual may sit from tol when the device and the oracle stop at different
sweeps."""
import warnings

import numpy as np
import pandas as pd
import pytest

import bp_oracle
from oracle import ve_oracle
from sorobn_b200 import BayesNet, bp, engine, planner, synthetic, workloads
from test_bp_plan import (F32_BELIEF_TOL, F32_RESIDUAL_NOISE, GRID16_EVIDENCE, many_children_rows, naive_bayes_spec,
                          near_tol, network)

pytestmark = pytest.mark.gpu


def frame(net, names, codes):
    return pd.DataFrame({e: np.asarray(net.domains[net.index[e]], dtype=object)[codes[i]]
                         for i, e in enumerate(names)}).infer_objects()


def rows(bn, names, n, seed, random_every=5):
    """Codes [n_ev, n]: rows drawn from the network, every `random_every`-th row random (possibly impossible)."""
    net = bn._compiled
    rng = np.random.default_rng(seed)
    codes = workloads.forward_sample_codes(net, n, seed)[[net.index[e] for e in names]]
    for b in range(0, n, random_every):
        codes[:, b] = [rng.integers(net.card[net.index[e]]) for e in names]
    return np.ascontiguousarray(codes)


def evidence_names(bn, k, seed):
    rng = np.random.default_rng(seed)
    return sorted(rng.choice(bn.nodes, size=k, replace=False).tolist())


def device_vs_oracle(bn, names, codes, n_iterations, damping, tol):
    net = bn._compiled
    targets = sorted(v for v in bn.nodes if v not in names)
    g = bp.compile_graph(net, [net.index[e] for e in names], [net.index[t] for t in targets])
    runner = engine.BeliefPropagation(g.words, g.tables)
    got, iters = runner.run(codes, codes.shape[1], n_iterations, damping, tol)
    runner.close()
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    want = bp_oracle.run(dn, names, codes, targets, n_iterations, damping, tol)
    assert np.array_equal(np.isnan(got).any(axis=0), np.isnan(want["beliefs"]).any(axis=0))
    same = iters == want["iterations"]
    assert not (~same & ~near_tol(want["residual"], iters, want["iterations"], tol, F32_RESIDUAL_NOISE)).any()
    # rows that stopped at the same sweep, converged or not (n_iterations + 1: both ran every sweep)
    both = same & ~np.isnan(got).any(axis=0)
    err = float(np.abs(got[:, both] - want["beliefs"][:, both]).max(initial=0.0))
    assert err < F32_BELIEF_TOL, err
    return both, iters


def impossible_last_state(spec):
    """`spec` with the last state of its last node given probability 0 under every parent configuration."""
    v = spec.nodes[-1]
    cpt = spec.cpt[v].copy()
    cpt[..., -1] = 0.0
    spec.cpt[v] = cpt / cpt.sum(axis=-1, keepdims=True)
    return synthetic.load(spec, BayesNet), v


@pytest.mark.parametrize("name", ["chain12s4", "naive_bayes", "chow_liu"])
def test_polytrees_equal_the_exact_marginals(name):
    if name == "chain12s4":
        bn, forced = impossible_last_state(synthetic.chain(12, 4))
    elif name == "naive_bayes":
        bn, forced = impossible_last_state(naive_bayes_spec())
    else:
        bn, forced = network(name), None
    names = evidence_names(bn, max(1, len(bn.nodes) // 3), seed=1)
    if forced is not None and forced not in names:
        names = sorted(names[1:] + [forced])
    codes = rows(bn, names, 10_000, seed=2)
    events = frame(bn._compiled, names, codes)
    exact = bn.marginals_many(events)
    got = bn.marginals_many(events, algorithm="bp", n_iterations=100, damping=0.0, tol=1e-6)
    assert list(got.columns) == list(exact.columns)
    nan_exact, nan_bp = exact.isna().any(axis=1).to_numpy(), got.isna().any(axis=1).to_numpy()
    assert np.array_equal(nan_exact, nan_bp)
    assert nan_exact.any() or forced is None
    assert np.abs(got.to_numpy()[~nan_bp] - exact.to_numpy()[~nan_exact]).max() < 1e-5


@pytest.mark.parametrize("name,n_rows", [("asia", 400), ("alarm", 400), ("sprinkler", 400), ("grades", 400),
                                         ("grid4x4s3", 400), ("grid4x4s10x3", 400), ("grid10x10s5", 200)])
def test_loopy_networks_match_the_oracle(name, n_rows):
    bn = synthetic.load(synthetic.grid(10, 10, 5), BayesNet) if name == "grid10x10s5" else network(name)
    names = evidence_names(bn, max(1, len(bn.nodes) // 4), seed=3)
    codes = rows(bn, names, n_rows, seed=4)
    for damping, tol, n_iterations in [(0.5, 1e-4, 100), (0.0, 1e-5, 30), (0.3, 0.0, 12)]:
        both, _ = device_vs_oracle(bn, names, codes, n_iterations, damping, tol)
        assert both.sum() >= n_rows // 2


def test_grid_the_exact_planner_refuses():
    bn = synthetic.load(synthetic.grid(16, 16, 3), BayesNet)
    names = sorted(GRID16_EVIDENCE)
    net = bn._compiled
    with pytest.raises(ValueError):
        planner.build_marginals_plan(net, [net.index[e] for e in names])  # the targets of marginals_many's default
    codes = rows(bn, names, 500, seed=6, random_every=50)
    both, _ = device_vs_oracle(bn, names, codes, 60, 0.5, 1e-4)
    assert both.sum() >= 400


@pytest.mark.parametrize("name", ["nb60s3", "nb60s10"])
def test_many_children_rescale(name):
    """60 disagreeing observed children: the product of the class variable's messages needs the underflow rescale
    (tests/test_bp_plan.py shows it falls below float32's range), in the narrow and in the wide kernel."""
    bn = network(name)
    dn, names, codes = many_children_rows(bn, 2000, seed=14)
    device_vs_oracle(bn, names, codes, 10, 0.0, 1e-12)
    events = frame(bn._compiled, names, codes)
    got = bn.marginals_many(events, algorithm="bp", n_iterations=10, damping=0.0, tol=1e-12)
    exact = bn.marginals_many(events)
    assert not got.isna().any().any()
    assert np.abs(got.to_numpy() - exact.to_numpy()).max() < 1e-5


def test_chunking_and_determinism():
    bn = synthetic.load(synthetic.grid(10, 10, 5), BayesNet)
    net = bn._compiled
    names = evidence_names(bn, 30, seed=7)
    codes = rows(bn, names, 200_000, seed=8)
    targets = sorted(v for v in bn.nodes if v not in names)
    g = bp.compile_graph(net, [net.index[e] for e in names], [net.index[t] for t in targets])
    assert 200_000 * 2 * g.n_edges * 4 > 1 << 30  # more than one chunk of message state
    runner = engine.BeliefPropagation(g.words, g.tables)
    a, ia = runner.run(codes, 200_000, 20, 0.5, 1e-4)
    b, ib = runner.run(codes, 200_000, 20, 0.5, 1e-4)
    assert np.array_equal(a, b, equal_nan=True) and np.array_equal(ia, ib)
    small = engine.BeliefPropagation(g.words, g.tables)
    for lo in range(0, 200_000, 37_000):
        hi = min(lo + 37_000, 200_000)
        s, si = small.run(np.ascontiguousarray(codes[:, lo:hi]), hi - lo, 20, 0.5, 1e-4)
        assert np.array_equal(s, a[:, lo:hi], equal_nan=True) and np.array_equal(si, ia[lo:hi])


def test_entry_points_agree():
    bn = network("alarm")
    names = evidence_names(bn, 2, seed=9)
    events = frame(bn._compiled, names, rows(bn, names, 300, seed=10)).astype(object)
    events.iloc[3, 0] = "not a state"
    q = next(v for v in bn.nodes if v not in names)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        one = bn.marginals_many(events, variables=[q], algorithm="bp", n_iterations=40)
        every = bn.marginals_many(events, algorithm="bp", n_iterations=40)
        many = bn.query_many(q, events=events, algorithm="bp", n_iterations=40)
    assert np.array_equal(many.to_numpy(), one.to_numpy(), equal_nan=True)
    assert np.isnan(many.iloc[3]).all()
    block = every[q].to_numpy()
    ok = ~np.isnan(block).any(axis=1)
    assert np.abs(many.to_numpy()[ok] - block[ok]).max() < 1e-5
    for b in (0, 1, 2, 5):
        event = {e: events[e].iloc[b] for e in names}
        single = bn.query(q, event=event, algorithm="bp", n_iterations=40)
        row = many.iloc[b]
        assert np.allclose(single.to_numpy(), row[row > 0].to_numpy(), rtol=0, atol=0)
        assert list(single.index) == list(row[row > 0].index)


def test_rows_that_do_not_converge_warn():
    bn = network("grid4x4s3")
    names = evidence_names(bn, 4, seed=11)
    events = frame(bn._compiled, names, rows(bn, names, 50, seed=12))
    with pytest.warns(RuntimeWarning, match="50 of 50 rows did not converge"):
        bn.marginals_many(events, algorithm="bp", n_iterations=2, tol=0.0)
