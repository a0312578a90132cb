"""Soft evidence on counts, sample, MPE and marginal MAP programs on the GPU (engine.Program.counts / sample / mpe /
map with `lik`, and the likelihoods= keyword of expected_counts, fit_em, sample_many, mpe_many and map_many): the
device against the CPU replay of the words (tests/soft_pattern_interp.py) and the float64 virtual-evidence
oracles (tests/soft_oracle.py with em_oracle, mpe_oracle and map_oracle)."""
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

import em_oracle
import map_oracle
import mpe_oracle
import soft_oracle
import soft_pattern_interp as spi
from oracle import ve_oracle
from sorobn_b200 import engine, examples, planner, workloads

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXAMPLES = ["asia", "alarm", "sprinkler", "grades"]


def lik_for(rng, net, soft, n_rows, zeros=True):
    n_lik = sum(int(net.card[v]) for v in soft)
    lik = rng.random((n_rows, n_lik)) * 10.0 ** rng.integers(-4, 4, size=(n_rows, 1))
    if zeros:
        lik[rng.random(lik.shape) < 0.1] = 0.0
        lik[0] = 0.0
    return lik


def codes_for(net, evidence, n_rows, seed):
    return np.ascontiguousarray(workloads.forward_sample_codes(net, n_rows, seed)[list(evidence)])


def case(net, rng, n_soft=2, n_ev=2):
    """(hard evidence, soft variables, one other variable) of a network with at least n_soft + 2 variables."""
    perm = [int(v) for v in rng.permutation(len(net.names))]
    n_ev = min(n_ev, len(net.names) - n_soft - 1)
    return tuple(sorted(perm[n_soft:n_soft + n_ev])), tuple(perm[:n_soft]), perm[n_soft + n_ev]


def virtual(net, plan, ev, codes, lik):
    dn = soft_oracle.dense(net)
    out = []
    for hard, s in soft_oracle.rows(net, ev, codes, plan.soft, lik):
        vnet, event, log_k = soft_oracle.virtual(dn, s)
        ok = event is not None and ve_oracle.evidence_probability(vnet, {**hard, **event}) > 0
        out.append((vnet, {**hard, **(event or {})}, log_k, ok))
    return out


def grid_case(n_soft, seed):
    w = workloads.grid10x10()
    bn = w.build()
    net = bn._compiled
    rng = np.random.default_rng(seed)
    ev = tuple(net.index[e] for e in w.evidence)  # the order of w.codes' rows
    hidden = [v for v in range(len(net.names)) if v not in ev and net.names[v] not in w.query]
    soft = tuple(int(v) for v in rng.choice(hidden, size=n_soft, replace=False))
    return w, bn, net, ev, soft, rng


# ----------------------------------------------------------------------------- counts and EM
@pytest.mark.parametrize("name", EXAMPLES)
def test_counts_against_the_oracle_bitwise_repeatable(name):
    net = getattr(examples, name)()._compiled
    rng = np.random.default_rng(1)
    offsets, _ = planner.count_layout(net)
    ev, soft, _ = case(net, rng)
    plan = planner.build_pattern_plan(net, "counts", ev, soft=soft)
    B = 96
    codes, lik = codes_for(net, ev, B, 2), lik_for(rng, net, plan.soft, B)
    prog = engine.Program(plan)
    counts, prob, log_ev = prog.counts(codes, B, lik=lik, log_evidence=True)
    again = prog.counts(codes, B, lik=lik)
    assert np.array_equal(again[0], counts) and np.array_equal(again[1], prob, equal_nan=True)
    rows = virtual(net, plan, ev, codes, lik)
    ok = np.array([r[3] for r in rows])
    assert not ok[0] and np.isnan(prob[0]) and np.isnan(log_ev[0])  # the all-zero likelihood row
    assert np.isnan(prob[~ok]).all()
    want = {node: np.zeros(net.cpt[v].shape) for v, node in enumerate(net.names)}
    for b, (vnet, event, log_k, good) in enumerate(rows):
        if not good or np.isnan(prob[b]):
            continue
        for node, c in em_oracle.expected_counts(vnet, [event]).items():
            if node in want:  # the virtual children's families are dropped
                want[node] += c
        le = em_oracle.log_likelihood(vnet, [event]) + log_k
        assert abs(log_ev[b] - le) <= 1e-5 * max(1.0, abs(le))
    n_ok = int((~np.isnan(prob)).sum())
    for v, node in enumerate(net.names):
        got = counts[offsets[v]:offsets[v] + net.cpt[v].size]
        w = want[node].reshape(-1)
        assert np.all(np.abs(got - w) <= 2e-6 * np.abs(w) + 1e-12 * n_ok), (node, np.max(np.abs(got - w)))
        assert abs(got.sum() - n_ok) <= 1e-6 * n_ok  # each family sums to the row count
    # the float64 twin: the same, to 1e-9 against the float64 replay
    p64 = engine.Program(plan, f64=True)
    c64, pr64 = p64.counts(codes, B, lik=lik)
    ref = spi.run_counts(plan.words, plan.table_blob64, codes, lik, n_rows=B)
    np.testing.assert_allclose(c64, ref[0], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(pr64, ref[1], rtol=1e-9)


def _oracle_em(bn, X, latent, lik, iterations):
    """`iterations` EM steps of the float64 oracle, each row with its own virtual child: the CPTs {node: array}."""
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    for _ in range(iterations):
        counts = {v: np.zeros(dn.cpt[v].shape) for v in dn.nodes}
        for b, row in enumerate(X.to_dict("records")):
            vnet, event, _ = soft_oracle.virtual(dn, {latent: lik[b]})
            for node, c in em_oracle.expected_counts(vnet, [{**row, **event}]).items():
                if node in counts:
                    counts[node] += c
        for v in dn.nodes:
            counts[v] = counts[v] + (1.0 if bn.prior_count else 0.0)
            tot = counts[v].sum(axis=-1, keepdims=True)
            with np.errstate(invalid="ignore", divide="ignore"):
                dn.cpt[v] = np.where(tot > 0, counts[v] / tot, 0.0)
    return dn


@pytest.mark.parametrize("name,latent", [("asia", "Lung cancer"), ("alarm", "Alarm")])
def test_fit_em_with_soft_labels_reaches_the_oracle_fixpoint(name, latent):
    bn = getattr(examples, name)()
    net = bn._compiled
    n = 64
    codes = workloads.forward_sample_codes(net, n, 3)
    X = pd.DataFrame({c: np.asarray(net.domains[v], dtype=object)[codes[v]] for v, c in enumerate(net.names) if c != latent})
    # noisy labels of the latent node: 0.8 on the true state
    v = net.index[latent]
    lik = np.full((n, int(net.card[v])), 0.2)
    lik[np.arange(n), codes[v]] = 0.8
    iters = 12
    start = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    want = _oracle_em(bn, X, latent, lik, iters)
    bn.fit_em(X, max_iter=iters, tol=-np.inf, likelihoods={latent: lik})
    assert len(bn.em_log_likelihood_) == iters
    lls = bn.em_log_likelihood_
    assert all(b >= a - 1e-4 * n for a, b in zip(lls, lls[1:]))  # EM never descends (float32 E-steps aside)
    for node in start.nodes:
        # fit_em leaves entries of zero expected count out of P
        got = dict(zip(bn.P[node].index, bn.P[node].to_numpy()))
        keys = pd.MultiIndex.from_product([want.domains[u] for u in want.scope(node)]) if len(want.scope(node)) > 1 \
            else want.domains[node]
        np.testing.assert_allclose([got.get(k, 0.0) for k in keys], want.cpt[node].reshape(-1), atol=2e-5, err_msg=node)
    # the log-likelihood is sum log P(observed, lik), on the scale of the given likelihoods
    fresh = getattr(examples, name)()
    ll = sum(soft_oracle.log_evidence(soft_oracle.dense(fresh._compiled), row, {latent: lik[b]})
             for b, row in enumerate(X.to_dict("records")))
    fresh.fit_em(X, max_iter=1, likelihoods={latent: lik * 3.0})
    assert abs(fresh.em_log_likelihood_[0] - (ll + n * np.log(3.0))) <= 1e-5 * abs(ll)


# ----------------------------------------------------------------------------- sample
def test_sample_follows_the_replay_and_is_invariant_to_grouping_chunking_and_lik_memory():
    torch = pytest.importorskip("torch")
    for name in EXAMPLES:
        net = getattr(examples, name)()._compiled
        rng = np.random.default_rng(7)
        ev, soft, _ = case(net, rng)
        plan = planner.build_pattern_plan(net, "sample", ev, soft=soft)
        B, D, seed = 513, 3, 99
        codes, lik = codes_for(net, ev, B, 4), lik_for(rng, net, plan.soft, B)
        prog = engine.Program(plan)
        drawn, prob, log_ev = prog.sample(codes, B, D, seed, lik=lik, log_evidence=True)
        mine, _, info, _ = spi.run_sample(plan.words, plan.table_blob, codes, lik, n_rows=B, n_draws=D, seed=seed,
                                          dtype=np.float32, given=drawn)
        _, p_ref, _, le_ref = spi.run_sample(plan.words, plan.table_blob64, codes, lik, n_rows=B, seed=seed)
        ok = ~np.isnan(prob)
        assert ok.mean() > 0.8 and not ok[0]
        assert np.all(np.abs(prob[ok] - p_ref[ok]) <= 1e-4 * p_ref[ok])
        assert np.all(np.abs(log_ev[ok] - le_ref[ok]) <= 1e-4 * np.maximum(1.0, np.abs(le_ref[ok])))
        for st in info:
            rows = slice(st["d_first"], st["d_first"] + len(st["cards"]))
            sure = (st["margin"] > 1e-5) & ok[None, :]
            assert sure.mean() > 0.7 * ok.mean()
            assert np.array_equal(drawn[rows][:, sure], mine[rows][:, sure]), name
        # pieces with their row_base, and CUDA-tensor likelihoods, give bitwise the same draws
        parts = [prog.sample(np.ascontiguousarray(codes[:, a:b]), b - a, D, seed, row_base=a, lik=lik[a:b])[0]
                 for a, b in ((0, 100), (100, 101), (101, B))]
        assert np.array_equal(np.concatenate(parts, axis=2), drawn)
        dev, dprob = prog.sample(codes, B, D, seed, lik=torch.as_tensor(lik, device="cuda"))
        assert np.array_equal(dev, drawn) and np.array_equal(dprob, prob, equal_nan=True)


def test_sample_many_draws_follow_row_positions():
    """A row's draws depend on the seed, its position, its pattern and its likelihoods: a prefix of the frame
    draws the same values, whatever the other rows' patterns."""
    bn = examples.asia()
    net = bn._compiled
    n = 300
    codes = workloads.forward_sample_codes(net, n, 5)
    rng = np.random.default_rng(5)
    cols = {}
    for c in ("Smoker", "Visit to Asia", "Positive X-ray"):
        vals = np.asarray(net.domains[net.index[c]], dtype=object)[codes[net.index[c]]].copy()
        vals[rng.random(n) < 0.3] = None
        cols[c] = vals
    X = pd.DataFrame(cols, index=pd.RangeIndex(10, 10 + n))
    lik = {"Dispnea": rng.random((n, 2)) * 10.0 ** rng.integers(-20, 2, (n, 1))}
    a = bn.sample_many(X, n=2, seed=3, likelihoods=lik)
    assert a.shape == (2 * n, len(net.names)) and a.notna().all().all()
    b = bn.sample_many(X.iloc[:120], n=2, seed=3, likelihoods={"Dispnea": lik["Dispnea"][:120]})
    pd.testing.assert_frame_equal(b, a.iloc[:240])
    torch = pytest.importorskip("torch")
    c = bn.sample_many(X, n=2, seed=3, likelihoods={"Dispnea": torch.as_tensor(lik["Dispnea"], device="cuda")})
    pd.testing.assert_frame_equal(c, a)


# ----------------------------------------------------------------------------- MPE and MAP
@pytest.mark.parametrize("kind", ["mpe", "map"])
def test_decode_against_the_replay_and_the_oracle(kind):
    for name in EXAMPLES:
        net = getattr(examples, name)()._compiled
        rng = np.random.default_rng(11)
        ev, soft, m = case(net, rng)
        map_vars = (m, soft[0]) if kind == "map" else None
        plan = planner.build_pattern_plan(net, kind, ev, soft=soft, map_vars=map_vars)
        B = 600
        codes, lik = codes_for(net, ev, B, 6), lik_for(rng, net, plan.soft, B)
        prog = engine.Program(plan)
        decoded, lp = getattr(prog, kind)(codes, B, lik=lik)
        d2, lp2 = getattr(prog, kind)(codes, B, lik=lik)
        assert np.array_equal(d2, decoded) and np.array_equal(lp2, lp)
        ref, rlp = spi.run_mpe(plan.words, plan.table_blob, codes, lik, n_rows=B, dtype=np.float32)
        assert lp[0] == -np.inf and rlp[0] == -np.inf
        assert np.array_equal(lp == -np.inf, rlp == -np.inf)
        fin = lp > -np.inf
        assert np.all(np.abs(lp[fin] - rlp[fin]) <= 4e-6 * np.maximum(1.0, np.abs(rlp[fin]))), name
        differ = np.flatnonzero(fin & (decoded != ref).any(axis=0))
        if kind == "mpe":
            assert not len(differ), name  # max-sum: bitwise the replay's
        else:
            # log-sum-exp: the device's expf / logf and numpy's exp / log differ in the last bits, so a decision may
            # differ from the float32 replay's, but only at a near-tie under the float64 oracle
            assert len(differ) <= 0.01 * fin.sum(), (name, len(differ))
            names = [net.names[v] for v in plan.sampled]
            for b, (vnet, event, _, _) in zip(differ, virtual(net, plan, ev, codes[:, differ], lik[differ])):
                mine = {n: net.domains[v][int(decoded[j, b])] for j, (n, v) in enumerate(zip(names, plan.sampled))}
                theirs = {n: net.domains[v][int(ref[j, b])] for j, (n, v) in enumerate(zip(names, plan.sampled))}
                a, c = map_oracle.log_prob(vnet, event, mine), map_oracle.log_prob(vnet, event, theirs)
                assert abs(a - c) <= 1e-5 * max(1.0, abs(c)), (name, b, a, c)
        for b, (vnet, event, log_k, good) in enumerate(virtual(net, plan, ev, codes[:, :40], lik[:40])):
            if not good:
                assert lp[b] == -np.inf
                continue
            got = {net.names[v]: net.domains[v][int(decoded[j, b])] for j, v in enumerate(plan.sampled)}
            if kind == "mpe":
                try:
                    _, L = mpe_oracle.brute_force(vnet, event)
                except ValueError:
                    _, L = mpe_oracle.max_sum(vnet, event)
                assert abs(mpe_oracle.log_joint(vnet, {**event, **got}) - L) <= 1e-4  # ties aside, the oracle's state
            else:
                x, L, gap = map_oracle.solve(vnet, event, [net.names[v] for v in map_vars])
                if gap > 1e-4:
                    assert got == x, (name, b)
            assert abs(lp[b] - (L + log_k)) <= 2e-5 * max(1.0, abs(L + log_k)), (name, b)


@pytest.mark.parametrize("c", [1e-50, 1e40])
def test_any_finite_scale_decodes_as_the_unscaled_likelihoods(c):
    """MPE and MAP programs are float only: scales float32 cannot hold must still only shift log P by log c."""
    bn = examples.asia()
    X = pd.DataFrame({"Smoker": [True, None]})
    base = np.array([[.2, .8], [.9, .1]])
    for many in (bn.mpe_many, bn.map_many):
        fa, la = many(X, return_log_proba=True, likelihoods={"Dispnea": base})
        fb, lb = many(X, return_log_proba=True, likelihoods={"Dispnea": base * c})
        pd.testing.assert_frame_equal(fb, fa)
        np.testing.assert_allclose(lb - la, np.log(c), rtol=0, atol=1e-5)
    # and a ratio below float32's range keeps its log: the row weights its states by 1e-60 : 1
    net = bn._compiled
    plan = planner.build_pattern_plan(net, "mpe", (net.index["Smoker"],), soft=(net.index["Dispnea"],))
    lik = np.array([[1e-60, 1.0], [1.0, 1e-60]]) * c
    codes = np.array([[0, 1]], dtype=np.uint8)
    decoded, lp = engine.Program(plan).mpe(codes, 2, lik=lik)
    ref, rlp = spi.run_mpe(plan.words, plan.table_blob, codes, lik, n_rows=2, dtype=np.float32)
    assert np.array_equal(decoded, ref) and np.isfinite(lp).all()
    np.testing.assert_allclose(lp, rlp, rtol=4e-6)


def test_map_program_that_observes_and_decodes_nothing():
    """A MAP program with soft evidence, no hard column and no MAP variable: no argmax step, log P(lik) per row."""
    bn = examples.asia()
    net = bn._compiled
    soft = (net.index["Dispnea"], net.index["Smoker"])
    plan = planner.build_pattern_plan(net, "map", (), soft=soft, map_vars=())
    assert plan.sampled == () and not plan.evidence
    rng = np.random.default_rng(31)
    B = 5000  # past the graph threshold
    lik = lik_for(rng, net, plan.soft, B)
    prog = engine.Program(plan)
    decoded, lp = prog.map(np.zeros((0, B), np.uint8), B, lik=lik)
    assert decoded.shape == (0, B) and lp[0] == -np.inf
    dn = soft_oracle.dense(net)
    for b, (_, s) in enumerate(soft_oracle.rows(net, (), np.zeros((0, B), np.uint8)[:, :60], plan.soft, lik[:60])):
        want = soft_oracle.log_evidence(dn, {}, s)
        assert (lp[b] == -np.inf) if want == -np.inf else abs(lp[b] - want) <= 2e-5 * max(1.0, abs(want)), (b, lp[b], want)
    prog.set_graph(0)
    assert np.array_equal(prog.map(np.zeros((0, B), np.uint8), B, lik=lik)[1], lp)
    # through map_many: a pattern that observes nothing and decodes nothing
    X = pd.DataFrame({"Visit to Asia": [None] * 4})
    frame, mlp = bn.map_many(X, variables=[], return_log_proba=True, likelihoods={"Dispnea": lik[1:5, :2]})
    assert frame["Visit to Asia"].isna().all()
    for b in range(4):
        want = soft_oracle.log_evidence(dn, {}, {"Dispnea": lik[1 + b, :2]})
        assert abs(mlp.iloc[b] - want) <= 2e-5 * max(1.0, abs(want))


def test_map_many_and_mpe_many_with_likelihoods():
    bn = examples.asia()
    net = bn._compiled
    n = 50
    codes = workloads.forward_sample_codes(net, n, 8)
    X = pd.DataFrame({c: np.asarray(net.domains[net.index[c]], dtype=object)[codes[net.index[c]]]
                      for c in ("Smoker", "Positive X-ray")})
    X.loc[X.index[::3], "Smoker"] = None
    rng = np.random.default_rng(8)
    lik = {"Dispnea": rng.random((n, 2)), "Tuberculosis": rng.random((n, 2))}
    frame, lp = bn.mpe_many(X, return_log_proba=True, likelihoods=lik)
    assert list(frame.columns) == sorted(net.names) and np.isfinite(lp).all()
    dn = soft_oracle.dense(net)
    for b in range(n):
        row = {k: v for k, v in X.iloc[b].items() if v is not None and v == v}
        vnet, event, log_k = soft_oracle.virtual(dn, {k: v[b] for k, v in lik.items()})
        _, L = mpe_oracle.brute_force(vnet, {**row, **event})
        assert abs(lp.iloc[b] - (L + log_k)) <= 2e-5 * max(1.0, abs(L))
    mframe, mlp = bn.map_many(X, return_log_proba=True, likelihoods=lik)
    assert list(mframe.columns) == ["Positive X-ray", "Smoker"]  # soft nodes summed out by default
    for b in range(n):
        row = {k: v for k, v in X.iloc[b].items() if v is not None and v == v}
        vnet, event, log_k = soft_oracle.virtual(dn, {k: v[b] for k, v in lik.items()})
        x, L, gap = map_oracle.solve(vnet, {**row, **event}, [c for c in X.columns if c not in row])
        assert abs(mlp.iloc[b] - (L + log_k)) <= 2e-5 * max(1.0, abs(L))
        if gap > 1e-4:
            assert all(mframe.iloc[b][k] == v for k, v in x.items())
    with pytest.raises(ValueError, match="both hard evidence and likelihoods"):
        bn.mpe_many(X, likelihoods={"Smoker": np.ones((n, 2))})
    zero = {k: v.copy() for k, v in lik.items()}
    zero["Dispnea"][4] = 0.0
    with pytest.raises(ValueError, match="probability zero"):
        bn.map_many(X, likelihoods=zero)


def test_kernel_census_of_a_soft_mpe_program():
    """A soft MPE run launches the log-domain pack, the max-sum / log-sum-exp step instantiations and the argmax
    step, and nothing else."""
    script = f"""
import sys
sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]
import numpy as np
from kernel_census import census
from sorobn_b200 import engine, planner, workloads
wl = workloads.grid10x10()
net = wl.build()._compiled
observed = tuple(sorted(net.index[e] for e in wl.evidence))
hidden = [v for v in range(len(net.names)) if v not in observed]
plan = planner.build_pattern_plan(net, "mpe", observed, soft=tuple(hidden[:5]))
codes = workloads.forward_sample_codes(net, 1000, 1)[list(observed)]
lik = np.random.default_rng(0).random((1000, sum(int(net.card[v]) for v in plan.soft)))
p = engine.Program(plan, device=0)
class Run:
    def run(self, c, n):
        p.mpe(c, n, lik=lik)
    def set_graph(self, g):
        p.set_graph(g)
print(sorted({{name for name, _ in census(Run(), codes, 1000)}}))
"""
    out = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, check=True).stdout
    names = eval(out.strip().splitlines()[-1])
    assert "sbn_soft_pack_log" in names and "sbn_argmax_step" in names, names
    assert all(n in ("sbn_soft_pack_log", "sbn_argmax_step") or n.endswith(", SbnMaxSum>") or n.endswith(", SbnLogSumExp>")
               for n in names), names


# ----------------------------------------------------------------------------- graph replay and the benchmark grid
def test_graph_replay_reads_new_likelihoods():
    w, bn, net, ev, soft, rng = grid_case(5, 21)
    B = 8192
    codes = w.codes(bn, B, 3)
    for kind in ("mpe", "sample", "counts"):
        plan = planner.build_pattern_plan(net, kind, ev, soft=soft)
        prog = engine.Program(plan)

        def run(lik):
            if kind == "mpe":
                return prog.mpe(codes, B, lik=lik)
            if kind == "sample":
                return prog.sample(codes, B, 1, 5, lik=lik)
            return prog.counts(codes, B, lik=lik)

        a = run(lik_for(rng, net, plan.soft, B, zeros=False))
        lik2 = lik_for(rng, net, plan.soft, B, zeros=False)
        b = run(lik2)
        assert not np.array_equal(a[1], b[1], equal_nan=True), kind
        prog.set_graph(0)
        c = run(lik2)
        for x, y in zip(b, c):
            assert np.array_equal(x, y, equal_nan=True), kind


@pytest.mark.parametrize("n_soft", [1, 5, 10])
def test_benchmark_grid_with_soft_hidden_nodes(n_soft):
    w, bn, net, ev, soft, rng = grid_case(n_soft, 200 + n_soft)
    B = 100_000
    codes = w.codes(bn, B, 9)
    sample_rows = np.array([0, 1, 777, 31337, B - 1])
    for kind in ("mpe", "sample", "counts"):
        plan = planner.build_pattern_plan(net, kind, ev, soft=soft)
        lik = lik_for(rng, net, plan.soft, B, zeros=False)
        prog = engine.Program(plan)
        sub_codes, sub_lik = np.ascontiguousarray(codes[:, sample_rows]), lik[sample_rows]
        if kind == "mpe":
            decoded, lp = prog.mpe(codes, B, lik=lik)
            assert np.isfinite(lp).all()
            ref, rlp = spi.run_mpe(plan.words, plan.table_blob, sub_codes, sub_lik, dtype=np.float32)
            assert np.array_equal(decoded[:, sample_rows], ref)
            assert np.all(np.abs(lp[sample_rows] - rlp) <= 4e-6 * np.maximum(1.0, np.abs(rlp)))
        elif kind == "sample":
            drawn, prob = prog.sample(codes, B, 1, 17, lik=lik)
            ok = ~np.isnan(prob)
            assert ok.mean() > 0.99
            _, p_ref, _, _ = spi.run_sample(plan.words, plan.table_blob64, sub_codes, sub_lik)
            good = ok[sample_rows]
            assert np.all(np.abs(prob[sample_rows][good] - p_ref[good]) <= 1e-4 * p_ref[good])
            # draws of the sampled rows, each a batch of its own at its own row_base
            for r in sample_rows[good]:
                one = prog.sample(np.ascontiguousarray(codes[:, r:r + 1]), 1, 1, 17, row_base=int(r), lik=lik[r:r + 1])[0]
                assert np.array_equal(one[:, :, 0], drawn[:, :, r])
        else:
            counts, prob = prog.counts(codes, B, lik=lik)
            ok = ~np.isnan(prob)
            assert ok.mean() > 0.99
            _, p_ref, _ = spi.run_counts(plan.words, plan.table_blob64, sub_codes, sub_lik)
            good = ok[sample_rows]
            assert np.all(np.abs(prob[sample_rows][good] - p_ref[good]) <= 1e-4 * p_ref[good])
            offsets, _ = planner.count_layout(net)
            for v in range(len(net.names)):
                fam = counts[offsets[v]:offsets[v] + net.cpt[v].size]
                assert abs(fam.sum() - ok.sum()) <= 1e-5 * ok.sum()


def test_entry_points_refuse_the_wrong_programs():
    net = examples.asia()._compiled
    a, c = net.index["Smoker"], net.index["Dispnea"]
    lib = engine.load()
    soft = engine.Program(planner.build_pattern_plan(net, "mpe", (c,), soft=(a,)))
    plain = engine.Program(planner.build_mpe_plan(net, (c,)))
    codes = np.zeros((1, 4), np.uint8)
    with pytest.raises(engine.EngineError, match="sbn_program_mpe_soft_host"):
        soft.mpe(codes, 4)
    with pytest.raises(engine.EngineError, match="sbn_program_mpe_host"):
        plain.mpe(codes, 4, lik=np.ones((4, 0)))
    counts = engine.Program(planner.build_pattern_plan(net, "counts", (c,), soft=(a,)))
    with pytest.raises(engine.EngineError, match="sbn_program_counts_soft_host"):
        counts.counts(codes, 4)
    sample = engine.Program(planner.build_pattern_plan(net, "sample", (c,), soft=(a,)))
    with pytest.raises(engine.EngineError, match="sbn_program_sample_soft_host"):
        sample.sample(codes, 4, 1, 0)
    plain_counts = engine.Program(planner.build_counts_plan(net, (c,)))
    with pytest.raises(engine.EngineError, match="sbn_program_counts_host"):
        plain_counts.counts(codes, 4, lik=np.ones((4, 0)))
    out, lp = np.empty(4, np.uint8), np.empty(4)
    lik = np.ones((4, 2), np.float32)
    assert lib.sbn_program_mpe_soft_host(soft._h, codes.ctypes.data, 4, 4, None, 2, 0, out.ctypes.data, lp.ctypes.data) != 0
    assert lib.sbn_program_mpe_soft_host(soft._h, codes.ctypes.data, 4, 4, lik.ctypes.data, 1, 0, out.ctypes.data,
                                         lp.ctypes.data) != 0  # ld_lik below the likelihood columns
    assert soft.mpe(codes, 4, lik=lik)[1].shape == (4,)  # and the program still works


@pytest.mark.parametrize("name", EXAMPLES)
def test_reference_impute_goldens(name):
    from test_soft_patterns_host import impute_golden_check

    assert impute_golden_check(getattr(examples, name)(), name) > 0
