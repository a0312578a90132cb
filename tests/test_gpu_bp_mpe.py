"""Max-product belief propagation on the device (the max-product instantiations of csrc/sbn_bp.cu) against the exact
MPE and the float64 oracle.

Tolerances come from the float32 replay of the same words (tests/test_bp_mpe_plan.py): decoded states are compared on
rows the oracle settled where its belief margin exceeds MPE_F32_BELIEF_TOL, and stop sweeps may differ where the
residual lies within MPE_F32_RESIDUAL_NOISE of tol."""
import warnings

import numpy as np
import pandas as pd
import pytest

import bp_mpe_oracle
from oracle import ve_oracle
from sorobn_b200 import BayesNet, bp, engine, examples, planner, synthetic, workloads
from test_bp_mpe_plan import (IMPOSSIBLE_OBSERVED, MPE_F32_BELIEF_TOL, MPE_F32_RESIDUAL_NOISE, by_var_order, margins,
                              not_gate, structural_zero_chain, trusted)
from test_bp_plan import GRID16_EVIDENCE, many_children_rows, naive_bayes_spec, near_tol, network
from test_gpu_bp import evidence_names, frame, impossible_last_state, rows

pytestmark = pytest.mark.gpu


def exact_tolerance(exact_lp):
    """1e-5, widened by the float32 rounding of the exact path's max log P (1e-6 of it: -200 on the 60-child rows)."""
    return 1e-5 + 1e-6 * np.abs(exact_lp)


def sampled_rows(bn, names, n, seed):
    """Codes [n_ev, n] of rows drawn from the network: every row has positive probability."""
    net = bn._compiled
    return np.ascontiguousarray(workloads.forward_sample_codes(net, n, seed)[[net.index[e] for e in names]])


def host_log_p(net, g, ev, ev_codes, decoded):
    """sum over every CPT of log(double(float32 entry)) at the observed and decoded codes, per row."""
    full = np.zeros((len(net.names), ev_codes.shape[1]), dtype=np.int64)
    full[list(ev)] = ev_codes
    full[list(g.variables)] = decoded
    total = np.zeros(ev_codes.shape[1])
    with np.errstate(divide="ignore"):
        for v in range(len(net.names)):
            cpt = np.asarray(net.cpt[v], dtype=np.float32).astype(np.float64)
            total += np.log(cpt[tuple(full[u] for u in net.scope(v))])
    return total


def device_vs_oracle(bn, names, codes, n_iterations, damping, tol):
    """Run the device and the oracle on the same rows and check iterations, codes and the score; returns (decoded
    codes [n_var, n], log P, iterations, rows compared) of the device."""
    net = bn._compiled
    ev = [net.index[e] for e in names]
    g = bp.compile_mpe_graph(net, ev)
    runner = engine.BeliefPropagation(g.words, g.tables)
    got, log_p, iters = runner.mpe(codes, codes.shape[1], n_iterations, damping, tol)
    runner.close()
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    want = bp_mpe_oracle.run(dn, names, codes, n_iterations, damping, tol)
    want_codes, want_beliefs = by_var_order(want, net, g)
    assert np.array_equal(np.isnan(log_p), np.isnan(want["log_p"]))
    same = iters == want["iterations"]
    if not same.all():  # (a pattern that observes every node runs no sweep and has no residual to consult)
        assert near_tol(want["residual"], iters, want["iterations"], tol, MPE_F32_RESIDUAL_NOISE)[~same].all()
    live = ~np.isnan(log_p)
    compared = same & live & trusted(want, n_iterations)
    clear = margins(want_beliefs) > MPE_F32_BELIEF_TOL if want_beliefs else np.zeros(got.shape, dtype=bool)
    assert np.array_equal(got[clear & compared], want_codes[clear & compared])
    want_lp = host_log_p(net, g, ev, codes, got)
    finite = live & np.isfinite(want_lp)
    assert np.allclose(log_p[finite], want_lp[finite], rtol=1e-12, atol=0)
    assert np.array_equal(np.isneginf(log_p[live]), np.isneginf(want_lp[live]))
    return got, log_p, iters, compared


def events_of(bn, names, codes):
    return frame(bn._compiled, names, codes)


@pytest.mark.parametrize("name", ["chain12s4", "naive_bayes", "chow_liu"])
def test_polytrees_equal_the_exact_mpe(name):
    if name == "chain12s4":
        bn, forced = impossible_last_state(synthetic.chain(12, 4))
    elif name == "naive_bayes":
        bn, forced = impossible_last_state(naive_bayes_spec())
    else:
        bn, forced = network(name), None
    names = evidence_names(bn, max(1, len(bn.nodes) // 3), seed=1)
    if forced is not None and forced not in names:
        names = sorted(names[1:] + [forced])
    codes = rows(bn, names, 5_000, seed=2)
    events = events_of(bn, names, codes)
    impossible = bn.marginals_many(events).isna().any(axis=1).to_numpy()
    assert impossible.any() or forced is None
    if impossible.any():
        with pytest.raises(ValueError) as exact_error:
            bn.mpe_many(events)
        with pytest.raises(ValueError) as bp_error:
            bn.mpe_many(events, algorithm="bp", damping=0.0, tol=1e-6)
        assert str(bp_error.value) == str(exact_error.value)
    events = events[~impossible]
    exact, exact_lp = bn.mpe_many(events, return_log_proba=True)
    got, got_lp = bn.mpe_many(events, return_log_proba=True, algorithm="bp", damping=0.0, tol=1e-6)
    assert list(got.columns) == list(exact.columns) and got.index.equals(exact.index)
    gap = np.abs(got_lp.to_numpy() - exact_lp.to_numpy())
    assert (gap < exact_tolerance(exact_lp.to_numpy())).all(), gap.max()
    # On a polytree the max-marginals are exact: where every variable's normalised max-marginal leads by more than
    # 1e-3 (well past the float32 rounding of the exact path's log P), the MPE is unique and both paths must find it.
    net = bn._compiled
    g = bp.compile_mpe_graph(net, [net.index[e] for e in names])
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    _, beliefs = by_var_order(bp_mpe_oracle.run(dn, names, codes[:, ~impossible], 100, 0.0, 1e-6), net, g)
    clear = (margins(beliefs) > 1e-3).all(axis=0)
    assert clear.sum() >= len(clear) // 4
    assert got[clear].equals(exact[clear])


@pytest.mark.parametrize("name,n_rows", [("asia", 400), ("alarm", 400), ("sprinkler", 400), ("grades", 400),
                                         ("grid4x4s3", 400), ("grid4x4s10x3", 400), ("grid10x10s5", 200)])
def test_loopy_networks_match_the_oracle(name, n_rows):
    bn = synthetic.load(synthetic.grid(10, 10, 5), BayesNet) if name == "grid10x10s5" else network(name)
    names = evidence_names(bn, max(1, len(bn.nodes) // 4), seed=3)
    codes = sampled_rows(bn, names, n_rows, seed=4)
    exact_lp = bn.mpe_many(events_of(bn, names, codes), return_log_proba=True)[1].to_numpy()
    n_compared = 0
    for damping, tol, n_iterations in [(0.5, 1e-4, 100), (0.0, 1e-5, 30), (0.3, 0.0, 6)]:
        _, log_p, _, compared = device_vs_oracle(bn, names, codes, n_iterations, damping, tol)
        n_compared += compared.sum()
        assert (log_p <= exact_lp + exact_tolerance(exact_lp)).all()
    assert n_compared >= n_rows


def test_grid_the_exact_planner_refuses():
    bn = synthetic.load(synthetic.grid(16, 16, 3), BayesNet)
    names = sorted(GRID16_EVIDENCE)
    net = bn._compiled
    with pytest.raises(ValueError):
        planner.build_mpe_plan(net, tuple(sorted(net.index[e] for e in names)))
    codes = rows(bn, names, 500, seed=6, random_every=50)
    device_vs_oracle(bn, names, codes, 60, 0.5, 1e-4)  # max-product does not settle here: iterations and score
    _, _, _, compared = device_vs_oracle(bn, names, codes, 6, 0.5, 0.0)
    assert compared.sum() >= 400


@pytest.mark.parametrize("name", ["nb60s3", "nb60s10"])
def test_many_children_rescale(name):
    bn = network(name)
    dn, names, codes = many_children_rows(bn, 2000, seed=14)
    got, log_p, _, compared = device_vs_oracle(bn, names, codes, 10, 0.0, 1e-12)
    assert compared.all()
    events = events_of(bn, names, codes)
    frame_bp, lp_bp = bn.mpe_many(events, return_log_proba=True, algorithm="bp", n_iterations=10, damping=0.0,
                                  tol=1e-12)
    frame_exact, lp_exact = bn.mpe_many(events, return_log_proba=True)
    assert (np.abs(lp_bp.to_numpy() - lp_exact.to_numpy()) < exact_tolerance(lp_exact.to_numpy())).all()
    assert (frame_bp["C"] == frame_exact["C"]).mean() > 0.99


@pytest.mark.parametrize("k", range(len(IMPOSSIBLE_OBSERVED)))
def test_impossible_inside_an_observed_family_raises_as_the_exact_path(k):
    bn = structural_zero_chain()
    events = IMPOSSIBLE_OBSERVED[k]
    with pytest.raises(ValueError) as exact_error:
        bn.mpe_many(events)
    with pytest.raises(ValueError) as bp_error:
        bn.mpe_many(events, algorithm="bp")
    assert str(bp_error.value) == str(exact_error.value)
    names = list(events.columns)
    net = bn._compiled
    codes = np.stack([[net.domains[net.index[c]].index(x) for x in events[c]] for c in names]).astype(np.uint8)
    _, log_p, iters, _ = device_vs_oracle(bn, names, codes, 20, 0.5, 1e-6)
    zero = events.index == "zero"
    assert np.isnan(log_p[zero]).all() and (iters[zero] == 0).all() and not np.isnan(log_p[~zero]).any()


def test_chunking_and_determinism():
    bn = synthetic.load(synthetic.grid(10, 10, 5), BayesNet)
    net = bn._compiled
    names = evidence_names(bn, 30, seed=7)
    codes = rows(bn, names, 200_000, seed=8)
    g = bp.compile_mpe_graph(net, [net.index[e] for e in names])
    assert 200_000 * 2 * g.n_edges * 4 > 1 << 30  # more than one chunk of message state
    runner = engine.BeliefPropagation(g.words, g.tables)
    a = runner.mpe(codes, 200_000, 20, 0.5, 1e-4)
    b = runner.mpe(codes, 200_000, 20, 0.5, 1e-4)
    for x, y in zip(a, b):
        assert np.array_equal(x, y, equal_nan=True)
    small = engine.BeliefPropagation(g.words, g.tables)
    for lo in range(0, 200_000, 37_000):
        hi = min(lo + 37_000, 200_000)
        part = small.mpe(np.ascontiguousarray(codes[:, lo:hi]), hi - lo, 20, 0.5, 1e-4)
        for x, y in zip(part, a):
            assert np.array_equal(x, y[..., lo:hi], equal_nan=True)


def test_entry_points_and_edge_cases():
    bn = examples.alarm()
    names = evidence_names(bn, 5, seed=9)
    events = events_of(bn, names, sampled_rows(bn, names, 300, seed=10)).astype(object)
    events.iloc[::7, 1] = None
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        many = bn.mpe_many(events, algorithm="bp", n_iterations=40)
        for b in (0, 1, 7, 20):
            event = {e: events[e].iloc[b] for e in names if events[e].iloc[b] is not None}
            single = bn.mpe(event, algorithm="bp", n_iterations=40)
            assert single.to_dict() == many.iloc[b].to_dict()
    # every node observed: nothing to decode, log P of the row itself
    full = many.iloc[:3].reset_index(drop=True)
    same, lp = bn.mpe_many(full, return_log_proba=True, algorithm="bp")
    _, lp_exact = bn.mpe_many(full, return_log_proba=True)
    assert same.equals(full) and (np.abs(lp.to_numpy() - lp_exact.to_numpy()) < exact_tolerance(lp_exact)).all()
    # a live decode of probability zero
    with pytest.warns(RuntimeWarning, match="2 of 2 rows decoded an explanation of probability zero"):
        _, lp = not_gate().mpe_many(pd.DataFrame({"A": [None, None]}), return_log_proba=True, algorithm="bp")
    assert (lp == -np.inf).all()
    # each run call refuses the other kind's words
    g1 = bp.compile_graph(bn._compiled, [0], [1])
    g2 = bp.compile_mpe_graph(bn._compiled, [0])
    r1, r2 = engine.BeliefPropagation(g1.words, g1.tables), engine.BeliefPropagation(g2.words, g2.tables)
    with pytest.raises(engine.EngineError, match="sbn_bp_mpe_host"):
        r2.run(np.zeros((1, 4), np.uint8), 4, 5, 0.5, 1e-5)
    with pytest.raises(engine.EngineError, match="sbn_bp_run_host"):
        r1.mpe(np.zeros((1, 4), np.uint8), 4, 5, 0.5, 1e-5)
