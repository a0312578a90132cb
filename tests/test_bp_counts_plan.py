"""Expected counts by loopy belief propagation (sorobn_b200/bp.py, "Expected counts") checked on the CPU.

tests/bp_counts_oracle.py restates the semantics in float64 from the dense network: on polytrees its counts must be the
exact expected counts of tests/em_oracle.py and its Bethe log-likelihood the exact log P(observed); on loopy networks
its converged family beliefs must agree with its variable beliefs.  tests/bp_counts_interp.py replays the version-3
words as csrc/sbn_bp.cu executes them: in float64 it must equal the oracle, and its float32 run sets the tolerances of
tests/test_gpu_bp_counts.py."""
import hashlib
import json
import os

import numpy as np
import pandas as pd
import pytest

import bp_counts_interp
import bp_counts_oracle
import em_oracle
from oracle import ve_oracle
from sorobn_b200 import BayesNet, bp, engine, examples, planner, synthetic, workloads
from test_bp_plan import GRID16_EVIDENCE, LOOPY, WIDE, network

# Float32 replay against the float64 oracle, measured by test_float32_replay_sets_the_device_tolerance over the
# networks and settings below: a count entry differs by at most 9.9e-8 per row counted, and a row's log Z_B by at
# most 2.7e-7.  The GPU tests allow about ten times as much.
F32_COUNTS_TOL = 1e-6  # per row counted: |device - oracle| <= F32_COUNTS_TOL * n_rows
F32_LOGZ_TOL = 3e-6

POLYTREES = ["chain12s4", "naive_bayes", "chow_liu"]
SETTINGS = [(0.0, 1e-6, 50), (0.5, 1e-5, 100), (0.3, 0.0, 7), (0.8, 1e-4, 3)]


def dense(bn):
    return ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)


def sampled(bn, names, n, seed):
    """Codes [n_ev, n] of rows drawn from the network: every row has positive probability."""
    net = bn._compiled
    return np.ascontiguousarray(workloads.forward_sample_codes(net, n, seed)[[net.index[e] for e in names]])


def evidence_names(bn, k, seed):
    rng = np.random.default_rng(seed)
    return sorted(rng.choice(bn.nodes, size=k, replace=False).tolist())


def counts_graph(bn, names):
    net = bn._compiled
    return bp.compile_counts_graph(net, [net.index[e] for e in names])


def dense_counts(bn, g, blob_counts):
    """Blob-order counts -> {node: [*parents, node]} by `perm`."""
    net = bn._compiled
    flat = np.zeros(blob_counts.size)
    flat[g.perm] = blob_counts
    offsets, _ = planner.count_layout(net)
    return {name: flat[offsets[v]:offsets[v] + net.cpt[v].size].reshape(net.cpt[v].shape)
            for v, name in enumerate(net.names)}


def row_dicts(dn, names, codes):
    return [{e: dn.domains[e][codes[i, b]] for i, e in enumerate(names)} for b in range(codes.shape[1])]


@pytest.mark.parametrize("name,n_ev", [("chain12s4", 4), ("chain12s4", 0), ("naive_bayes", 3), ("chow_liu", 3),
                                       ("nb60s3", 60)])
def test_oracle_is_exact_on_polytrees(name, n_ev):
    bn = network(name)
    dn = dense(bn)
    names = [v for v in bn.nodes if v != "C"] if name == "nb60s3" else evidence_names(bn, n_ev, seed=1)
    if name == "naive_bayes":
        names = [v for v in names if v != "C"]  # the class stays latent
    n = 8 if name == "nb60s3" else 20
    codes = sampled(bn, names, n, seed=2)
    res = bp_counts_oracle.run(dn, names, codes, 200, 0.0, 1e-13, n_rows=n)
    assert (res["iterations"] <= 200).all()
    rows = row_dicts(dn, names, codes)
    want = em_oracle.expected_counts(dn, rows)
    for v in bn.nodes:
        assert np.allclose(res["counts"][v], want[v], rtol=0, atol=1e-9), v
    for b, row in enumerate(rows):
        lp = np.log(ve_oracle.evidence_probability(dn, row)) if row else 0.0
        assert abs(res["log_z"][b] - lp) < 1e-9 * max(1.0, abs(lp)), (b, res["log_z"][b], lp)


def test_fully_observed_rows_give_the_histogram_and_log_p():
    bn = network("chow_liu")
    dn = dense(bn)
    names = list(bn.nodes)
    codes = sampled(bn, names, 30, seed=3)
    res = bp_counts_oracle.run(dn, names, codes, 10, 0.5, 1e-6)
    assert (res["iterations"] == 0).all()
    rows = row_dicts(dn, names, codes)
    want = em_oracle.expected_counts(dn, rows)
    for v in bn.nodes:
        assert np.array_equal(res["counts"][v], want[v])
    lp = np.log([ve_oracle.evidence_probability(dn, r) for r in rows])
    assert np.allclose(res["log_z"], lp, rtol=1e-12, atol=0)


@pytest.mark.parametrize("name", LOOPY + WIDE)
def test_converged_beliefs_are_marginally_consistent_on_loopy_networks(name):
    bn = network(name)
    dn = dense(bn)
    names = evidence_names(bn, max(1, len(bn.nodes) // 4), seed=4)
    codes = sampled(bn, names, 30, seed=5)
    res = bp_counts_oracle.run(dn, names, codes, 500, 0.5, 1e-12)
    done = (res["iterations"] <= 500) & ~np.isnan(res["log_z"])
    assert done.sum() >= 20
    observed = set(names)
    for v in bn.nodes:
        members = [u for u in dn.scope(v) if u not in observed]
        if not members:
            continue
        fam = res["family"][v][done]
        for i, u in enumerate(members):
            marg = fam.sum(axis=tuple(a + 1 for a in range(len(members)) if a != i))
            assert np.allclose(marg, res["variable"][u][done], rtol=0, atol=1e-8), (v, u)


@pytest.mark.parametrize("name", POLYTREES + LOOPY + WIDE + ["alarm"])
@pytest.mark.parametrize("damping,tol,n_iterations", SETTINGS)
def test_float64_replay_equals_the_oracle(name, damping, tol, n_iterations):
    bn = network(name)
    dn = dense(bn)
    names = evidence_names(bn, max(1, len(bn.nodes) // 4), seed=6)
    codes = np.ascontiguousarray(workloads.forward_sample_codes(bn._compiled, 40, 7)[
        [bn._compiled.index[e] for e in names]])
    rng = np.random.default_rng(8)
    for b in range(0, 40, 5):  # random codes: some rows impossible, some dead before the first sweep
        codes[:, b] = [rng.integers(len(dn.domains[e])) for e in names]
    g = counts_graph(bn, names)
    want = bp_counts_oracle.run(dn, names, codes, n_iterations, damping, tol)
    got, log_z, iters = bp_counts_interp.run(g.words, g.tables64, codes, 40, n_iterations, damping, tol)
    assert np.array_equal(iters, want["iterations"])
    assert np.array_equal(np.isnan(log_z), np.isnan(want["log_z"]))
    assert np.allclose(log_z, want["log_z"], rtol=1e-12, atol=1e-12, equal_nan=True)
    counts = dense_counts(bn, g, got)
    for v in bn.nodes:
        assert np.allclose(counts[v], want["counts"][v], rtol=0, atol=1e-10), v


def test_float32_replay_sets_the_device_tolerance():
    worst_c = worst_z = 0.0
    for name in ["chain12s4", "naive_bayes"] + LOOPY + WIDE + ["alarm"]:
        bn = network(name)
        dn = dense(bn)
        names = evidence_names(bn, max(1, len(bn.nodes) // 4), seed=9)
        codes = sampled(bn, names, 40, seed=10)
        g = counts_graph(bn, names)
        for damping, tol, n_iterations in SETTINGS:
            want = bp_counts_oracle.run(dn, names, codes, n_iterations, damping, 0.0)
            got, log_z, _ = bp_counts_interp.run(g.words, g.tables, codes, 40, n_iterations, damping, 0.0,
                                                 dtype=np.float32)
            assert np.array_equal(np.isnan(log_z), np.isnan(want["log_z"]))
            worst_z = max(worst_z, float(np.nanmax(np.abs(log_z - want["log_z"]), initial=0.0)))
            counts = dense_counts(bn, g, got)
            worst_c = max(worst_c, max(float(np.abs(counts[v] - want["counts"][v]).max()) for v in bn.nodes) / 40)
    assert worst_c < F32_COUNTS_TOL / 5, worst_c
    assert worst_z < F32_LOGZ_TOL / 5, worst_z


@pytest.mark.parametrize("name", ["asia", "alarm", "grid4x4s3", "naive_bayes", "grid4x4s10x3"])
def test_compiler_keeps_every_cpt_and_permutes_the_dense_tables(name):
    bn = network(name)
    net = bn._compiled
    rng = np.random.default_rng(11)
    offsets, n_counts = planner.count_layout(net)
    flat = np.concatenate([np.asarray(c, dtype=np.float64).reshape(-1) for c in net.cpt])
    for n_ev in (0, 1, len(bn.nodes) // 2, len(bn.nodes)):
        ev = sorted(rng.choice(len(bn.nodes), size=n_ev, replace=False).tolist())
        g = bp.compile_counts_graph(net, ev)
        assert int(g.words[1]) == bp.VERSION_COUNTS
        assert g.families == tuple(range(len(net.names)))
        assert g.variables == tuple(v for v in range(len(net.names)) if v not in ev) == g.targets
        assert np.array_equal(np.sort(g.perm), np.arange(n_counts))
        assert np.array_equal(g.tables64, flat[g.perm])
        # the version-2 layout: the words differ from compile_mpe_graph's in the version word alone
        g2 = bp.compile_mpe_graph(net, ev)
        assert np.array_equal(np.delete(g.words, 1), np.delete(g2.words, 1))
        assert np.array_equal(g.tables64, g2.tables64) and g2.perm is None
        w, p = g.words, int(g.words[9])
        zero = 0
        for _ in range(int(w[3])):
            zero += int(w[p + 2]) == 0
            p += 4 + 3 * (int(w[p + 2]) + int(w[p + 3]))
        assert zero == sum(set(net.scope(v)) <= set(ev) for v in range(len(net.names)))


def test_version_1_and_2_words_are_those_of_the_parent():
    with open(os.path.join(os.path.dirname(__file__), "golden", "bp_words_parent.json")) as f:
        want = json.load(f)["sha256"]  # of the parent commit's compile_graph / compile_mpe_graph
    nets = {"asia": examples.asia(), "alarm": examples.alarm(), "grid4x4s10x3": network("grid4x4s10x3")}
    for key, digest in want.items():
        name, kind = key.split("/")
        net = nets[name]._compiled
        n = len(net.names)
        ev = list(range(0, n, 3))
        g = bp.compile_graph(net, ev, [v for v in range(n) if v not in ev]) if kind == "v1" else \
            bp.compile_mpe_graph(net, ev)
        h = hashlib.sha256(np.ascontiguousarray(g.words).tobytes() + np.ascontiguousarray(g.tables64).tobytes())
        assert h.hexdigest() == digest, key


def test_counts_planner_refuses_the_16x16_grid():
    net = synthetic.load(synthetic.grid(16, 16, 3), BayesNet)._compiled
    evidence = tuple(sorted(net.index[e] for e in GRID16_EVIDENCE))
    with pytest.raises(ValueError, match="2\\^31"):
        planner.build_counts_plan(net, evidence)
    g = bp.compile_counts_graph(net, evidence)
    assert len(g.families) == 256 and g.tables.size == 6348 and len(g.variables) == 226


def test_argument_errors_need_no_gpu():
    bn = examples.asia()
    X = pd.DataFrame({"Smoker": [True, False], "Dispnea": [None, True]})
    for kw in ({"damping": 1.0}, {"damping": -0.1}, {"n_iterations": 0}, {"n_iterations": 2.5}, {"tol": -1e-3},
               {"tol": float("nan")}):
        with pytest.raises(ValueError):
            bn.expected_counts(X, algorithm="bp", **kw)
    for kw in ({"damping": 1.0}, {"n_iterations": 0}, {"bp_tol": -1e-3}, {"bp_tol": float("inf")}):
        with pytest.raises(ValueError):
            bn.fit_em(X, algorithm="bp", **kw)
    with pytest.raises(ValueError, match="Unknown algorithm"):
        bn.expected_counts(X, algorithm="loopy")
    with pytest.raises(ValueError, match="Unknown algorithm"):
        bn.fit_em(X, algorithm="loopy")
    lik = {"Lung cancer": np.ones((2, 2))}
    with pytest.raises(ValueError, match="soft evidence"):
        bn.expected_counts(X, algorithm="bp", likelihoods=lik)
    with pytest.raises(ValueError, match="soft evidence"):
        bn.fit_em(X, algorithm="bp", likelihoods=lik)


def test_no_silent_cpu_fallback():
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    bn = examples.asia()
    X = pd.DataFrame({"Smoker": [True, False], "Dispnea": [None, True]})
    with pytest.raises(engine.EngineError):
        bn.expected_counts(X, algorithm="bp")
    with pytest.raises(engine.EngineError):
        bn.fit_em(X, algorithm="bp", max_iter=2)
