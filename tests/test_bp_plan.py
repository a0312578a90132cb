"""Loopy belief propagation (sorobn_b200/bp.py) checked on the CPU.

tests/bp_oracle.py restates the algorithm in float64 from the dense network; on polytrees it must give the exact
marginals of ve_oracle, on loopy networks a fixed point.  tests/bp_interp.py replays the compiled words as
csrc/sbn_bp.cu executes them: in float64 it must equal the oracle, and the float32 replay measures how far the
device's arithmetic can drift from it, which sets the tolerances of tests/test_gpu_bp.py."""
import numpy as np
import pandas as pd
import pytest

import bp_interp
import bp_oracle
from oracle import ve_oracle
from sorobn_b200 import BayesNet, bp, engine, examples, planner, structure, synthetic, workloads

# Float32 replay against the float64 oracle, measured by test_float32_replay_sets_the_device_tolerance over the
# networks and settings below: beliefs differ by at most 2.3e-7, and the messages of the first sweeps by at most
# 1.1e-7, so a sweep's residual by at most about that much.  The GPU tests allow about ten times as much.
F32_BELIEF_TOL = 3e-6
F32_RESIDUAL_NOISE = 2e-6

LOOPY = ["asia", "sprinkler", "grades", "grid4x4s3"]
# Networks with variables of more than 8 states: they run the wide kernel instantiation (sbn_bp_kernel<256>)
WIDE = ["grid4x4s10x3"]

# The observed cells of the 16 x 16 grid of 3 states the GPU tests and tools/bp_bench.py run: the last row and the
# rest of the last column, 30 cells.  The exact planner refuses it (test_exact_planner_refuses_the_16x16_grid).
GRID16_EVIDENCE = [f"g15{j:02d}" for j in range(16)] + [f"g{i:02d}15" for i in range(1, 15)]


def naive_bayes_spec(n_children=6, seed=0):
    """Class C with `n_children` binary or ternary features: a polytree."""
    rng = np.random.default_rng(seed)
    spec = synthetic.NetSpec("nb", ["C"] + [f"f{k}" for k in range(n_children)], {}, {"C": 3}, {})
    spec.cpt["C"] = rng.dirichlet(np.ones(3))
    for k in range(n_children):
        name = f"f{k}"
        spec.parents[name] = ["C"]
        spec.n_states[name] = 2 + k % 2
        spec.cpt[name] = rng.dirichlet(np.ones(spec.n_states[name]), size=3)
    return spec


def naive_bayes():
    return synthetic.load(naive_bayes_spec(), BayesNet)


def many_children_spec(n_class, n_children=60, seed=0):
    """Class C of `n_class` states with `n_children` binary children: child k says 1 with probability 0.999 under
    class k mod n_class and 0.001 under every other class.  Given random codes for every child, the children
    disagree, and every state of C gets a product of many small messages, far below float32's range."""
    rng = np.random.default_rng(seed)
    names = [f"f{k:02d}" for k in range(n_children)]
    spec = synthetic.NetSpec(f"nb{n_children}s{n_class}", ["C"] + names, {}, {"C": n_class}, {})
    spec.cpt["C"] = rng.dirichlet(np.ones(n_class))
    for k, name in enumerate(names):
        spec.parents[name] = ["C"]
        spec.n_states[name] = 2
        p1 = np.where(np.arange(n_class) == k % n_class, 0.999, 0.001)
        spec.cpt[name] = np.stack([1.0 - p1, p1], axis=-1)
    return spec


def chow_liu_tree(seed=0):
    data = synthetic.load(synthetic.random_dag(8, 2, 3, seed=seed), BayesNet).sample(2000)
    return BayesNet(*structure.chow_liu(data)).fit(data)


def network(name):
    if name in ("asia", "sprinkler", "grades", "alarm"):
        return getattr(examples, name)()
    if name == "grid4x4s3":
        return synthetic.load(synthetic.grid(4, 4, 3, seed=11), BayesNet)
    if name == "chain12s4":
        return synthetic.load(synthetic.chain(12, 4), BayesNet)
    if name == "naive_bayes":
        return naive_bayes()
    if name == "chow_liu":
        return chow_liu_tree()
    if name == "grid4x4s10x3":
        return synthetic.load(synthetic.grid(4, 4, (10, 3), seed=11), BayesNet)
    if name in ("nb60s3", "nb60s10"):
        return synthetic.load(many_children_spec(int(name[5:])), BayesNet)
    raise KeyError(name)


def setup(bn, n_ev, n, seed):
    """(compiled net, dense net, evidence names, codes [n_ev, n], target names) of random evidence columns, with
    rows drawn from the network and one in five rows given a random (possibly impossible) code."""
    rng = np.random.default_rng(seed)
    net = bn._compiled
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    ev = sorted(rng.choice(len(bn.nodes), size=n_ev, replace=False).tolist())
    codes = workloads.forward_sample_codes(net, n, seed)[ev]
    for b in range(0, n, 5):
        codes[:, b] = [rng.integers(net.card[v]) for v in ev]
    names = [net.names[v] for v in ev]
    targets = sorted(v for v in bn.nodes if v not in names)
    return net, dn, names, np.ascontiguousarray(codes), targets


def graph(net, names, targets):
    return bp.compile_graph(net, [net.index[e] for e in names], [net.index[t] for t in targets])


def exact_marginals(dn, names, codes, targets, b):
    event = {e: dn.domains[e][codes[i, b]] for i, e in enumerate(names)}
    if event and ve_oracle.evidence_probability(dn, event) <= 0:
        return None
    return np.concatenate([ve_oracle.query(dn, t, event=event)[1].reshape(-1) for t in targets])


def near_tol(residual, a, b, tol, eps):
    """Rows whose stop sweeps a and b differ only because the residual at the first of them lies within eps of tol."""
    t = np.minimum(a, b) - 1
    ok = t < residual.shape[1]
    r = np.where(ok, residual[np.arange(len(a)), np.minimum(t, residual.shape[1] - 1)], np.inf)
    return np.abs(r - tol) <= eps


@pytest.mark.parametrize("name", ["chain12s4", "naive_bayes", "chow_liu"])
def test_oracle_is_exact_on_polytrees(name):
    bn = network(name)
    net, dn, names, codes, targets = setup(bn, max(1, len(bn.nodes) // 3), 30, seed=1)
    res = bp_oracle.run(dn, names, codes, targets, 200, 0.0, 1e-14)
    assert (res["iterations"] <= 200).all()
    for b in range(codes.shape[1]):
        want = exact_marginals(dn, names, codes, targets, b)
        if want is None:
            assert np.isnan(res["beliefs"][:, b]).all(), b
            continue
        assert np.allclose(res["beliefs"][:, b], want, rtol=0, atol=1e-10), b


@pytest.mark.parametrize("name", LOOPY)
def test_oracle_converges_to_a_fixed_point_on_loopy_networks(name):
    bn = network(name)
    net, dn, names, codes, targets = setup(bn, max(1, len(bn.nodes) // 4), 20, seed=2)
    tol = 1e-8
    first = bp_oracle.run(dn, names, codes, targets, 300, 0.5, tol)
    done = (first["iterations"] <= 300) & ~np.isnan(first["beliefs"]).any(axis=0)
    assert done.sum() >= 10
    more = bp_oracle.run(dn, names, codes, targets, int(first["iterations"][done].max()) + 1, 0.5, 0.0)
    after = more["residual"][np.flatnonzero(done), first["iterations"][done]]  # the sweep after convergence
    assert (after < tol).all(), after.max()
    assert np.allclose(more["beliefs"][:, done], first["beliefs"][:, done], atol=1e-7)


SETTINGS = [(0.0, 1e-6, 50), (0.5, 1e-5, 100), (0.3, 0.0, 7), (0.8, 1e-4, 3)]


@pytest.mark.parametrize("name", ["chain12s4", "naive_bayes", "chow_liu"] + LOOPY + WIDE + ["alarm"])
@pytest.mark.parametrize("damping,tol,n_iterations", SETTINGS)
def test_float64_replay_equals_the_oracle(name, damping, tol, n_iterations):
    bn = network(name)
    net, dn, names, codes, targets = setup(bn, max(1, len(bn.nodes) // 4), 40, seed=3)
    g = graph(net, names, targets)
    want = bp_oracle.run(dn, names, codes, targets, n_iterations, damping, tol)
    got, iters = bp_interp.run(g.words, g.tables64, codes, codes.shape[1], n_iterations, damping, tol)
    assert np.array_equal(np.isnan(got), np.isnan(want["beliefs"]))
    assert np.allclose(got, want["beliefs"], rtol=0, atol=1e-12, equal_nan=True)
    differ = iters != want["iterations"]
    assert not (differ & ~near_tol(want["residual"], iters, want["iterations"], tol, 1e-9)).any()
    if tol == 0:
        assert (iters[~np.isnan(got).any(axis=0)] == n_iterations + 1).all()


def test_float32_replay_sets_the_device_tolerance():
    worst_b = worst_r = 0.0
    for name in ["chain12s4", "naive_bayes"] + LOOPY + WIDE + ["alarm"]:
        bn = network(name)
        net, dn, names, codes, targets = setup(bn, max(1, len(bn.nodes) // 4), 40, seed=4)
        g = graph(net, names, targets)
        for damping, tol, n_iterations in SETTINGS:
            want = bp_oracle.run(dn, names, codes, targets, n_iterations, damping, 0.0)
            got, iters = bp_interp.run(g.words, g.tables, codes, codes.shape[1], n_iterations, damping, 0.0,
                                       dtype=np.float32)
            assert np.array_equal(np.isnan(got), np.isnan(want["beliefs"]))
            worst_b = max(worst_b, float(np.nanmax(np.abs(got - want["beliefs"]), initial=0.0)))
            # the residual the float32 row sees: from a replay that stops at every sweep count
            for t in range(1, min(n_iterations, 4) + 1):
                _, _, m32 = bp_interp.run(g.words, g.tables, codes, codes.shape[1], t, damping, 0.0, np.float32, True)
                _, _, m64 = bp_interp.run(g.words, g.tables64, codes, codes.shape[1], t, damping, 0.0, np.float64, True)
                ok = ~np.isnan(m64).any(axis=1)
                worst_r = max(worst_r, float(np.abs(m32[ok] - m64[ok]).max(initial=0.0)))
    assert worst_b < F32_BELIEF_TOL / 5, worst_b
    assert worst_r < F32_RESIDUAL_NOISE / 5, worst_r


@pytest.mark.parametrize("name", ["asia", "alarm", "grid4x4s3", "naive_bayes"])
def test_compiler_factors_and_variables(name):
    bn = network(name)
    net = bn._compiled
    rng = np.random.default_rng(5)
    for n_ev in (0, 1, len(bn.nodes) // 2, len(bn.nodes) - 1):
        ev = sorted(rng.choice(len(bn.nodes), size=n_ev, replace=False).tolist())
        free = [v for v in range(len(bn.nodes)) if v not in ev]
        targets = [free[-1]]
        g = bp.compile_graph(net, ev, targets)
        plan = planner.build_marginals_plan(net, ev, targets=targets)
        relevant = set(int(v) for v in plan.tables)
        assert len(g.families) == len(set(g.families))
        observed_families = {v for v in relevant if set(net.scope(v)) <= set(ev)}
        assert set(g.families) == relevant - observed_families
        assert set(g.variables) == relevant - set(ev)
        assert g.Q == int(net.card[targets[0]])


def test_exact_planner_refuses_the_16x16_grid():
    net = synthetic.load(synthetic.grid(16, 16, 3), BayesNet)._compiled
    evidence = [net.index[e] for e in GRID16_EVIDENCE]
    assert len(evidence) == 30
    with pytest.raises(ValueError, match="2\\^31"):
        planner.build_marginals_plan(net, evidence)
    g = bp.compile_graph(net, evidence, [v for v in range(len(net.names)) if v not in evidence])
    assert len(g.families) == 255 and g.Q == 3 * 226  # g1515's family is all observed


def many_children_rows(bn, n, seed):
    """(dense net, child names, random codes [60, n]) of `many_children_spec`'s network, every child observed."""
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    names = [v for v in bn.nodes if v != "C"]
    codes = np.random.default_rng(seed).integers(0, 2, size=(len(names), n)).astype(np.uint8)
    return dn, names, codes


@pytest.mark.parametrize("name", ["nb60s3", "nb60s10"])
def test_rescale_keeps_many_children_in_range(name):
    """A class variable with 60 disagreeing observed children: the product of its messages falls below float32's
    smallest subnormal for every state, so without the rescale the float32 beliefs would be NaN.  With it the float32
    replay stays on the float64 oracle, which equals the exact marginals (a polytree)."""
    bn = network(name)
    dn, names, codes = many_children_rows(bn, 64, seed=13)
    n = codes.shape[1]
    lik = np.stack([np.asarray(dn.cpt[f])[:, codes[k]] for k, f in enumerate(names)])  # [child, class, row]
    log_prod = np.log(lik / lik.sum(axis=1, keepdims=True)).sum(axis=0)
    assert (log_prod.max(axis=0) < np.log(2.0**-149)).all()
    want = bp_oracle.run(dn, names, codes, ["C"], 10, 0.0, 1e-12)
    for b in range(n):
        assert np.allclose(want["beliefs"][:, b], exact_marginals(dn, names, codes, ["C"], b), rtol=0, atol=1e-10)
    net = bn._compiled
    g = graph(net, names, ["C"])
    got64, it64 = bp_interp.run(g.words, g.tables64, codes, n, 10, 0.0, 1e-12)
    assert np.allclose(got64, want["beliefs"], rtol=0, atol=1e-12) and np.array_equal(it64, want["iterations"])
    got32, _ = bp_interp.run(g.words, g.tables, codes, n, 10, 0.0, 1e-12, dtype=np.float32)
    assert not np.isnan(got32).any()
    assert np.abs(got32 - want["beliefs"]).max() < F32_BELIEF_TOL / 5


def test_argument_errors_need_no_gpu():
    bn = examples.asia()
    events = pd.DataFrame({"Smoker": [True, False]})
    for kw in ({"damping": 1.0}, {"damping": -0.1}, {"n_iterations": 0}, {"n_iterations": 2.5}, {"tol": -1e-3},
               {"tol": float("nan")}):
        with pytest.raises(ValueError):
            bn.marginals_many(events, algorithm="bp", **kw)
    with pytest.raises(ValueError, match="Unknown algorithm"):
        bn.marginals_many(events, algorithm="loopy")
    with pytest.raises(ValueError, match="one query variable"):
        bn.query_many("Lung cancer", "Tuberculosis", events=events, algorithm="bp")
    with pytest.raises(ValueError, match="one query variable"):
        bn.query("Lung cancer", "Tuberculosis", event={"Smoker": True}, algorithm="bp")
    with pytest.raises(ValueError, match="bp"):
        bn.query("Lung cancer", event={}, algorithm="magic")
    lik = {"Dispnea": np.ones((2, 2))}
    with pytest.raises(ValueError, match="soft evidence"):
        bn.marginals_many(events, algorithm="bp", likelihoods=lik)
    with pytest.raises(ValueError, match="soft evidence"):
        bn.query_many("Lung cancer", events=events, algorithm="bp", likelihoods=lik)
    with pytest.raises(ValueError, match="devices"):
        bn.query_many("Lung cancer", events=events, algorithm="bp", devices=[0, 1])


def test_no_silent_cpu_fallback():
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    bn = examples.asia()
    with pytest.raises(engine.EngineError):
        bn.marginals_many(pd.DataFrame({"Smoker": [True]}), algorithm="bp")
    with pytest.raises(engine.EngineError):
        bn.query("Lung cancer", event={"Smoker": True}, algorithm="bp")
