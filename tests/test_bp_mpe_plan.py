"""Max-product loopy belief propagation (sorobn_b200/bp.py, "Max-product") checked on the CPU.

tests/bp_mpe_oracle.py restates the semantics in float64 from the dense network; on polytrees its decode must be
the exact MPE of tests/mpe_oracle.py.  tests/bp_mpe_interp.py replays the compiled version-2 words as the
max-product instantiations of csrc/sbn_bp.cu execute them: in float64 it must equal the oracle, and the float32
replay measures how far the device's arithmetic can drift from it, which sets the tolerances of
tests/test_gpu_bp_mpe.py.  The host side of `mpe_many(algorithm="bp")` runs here on the float32 replay."""
import warnings

import numpy as np
import pandas as pd
import pytest

import bp_mpe_interp
import bp_mpe_oracle
import mpe_oracle
from oracle import ve_oracle
from sorobn_b200 import BayesNet, bp, engine, examples, planner, synthetic
from test_bp_plan import near_tol, network, setup

# Float32 replay against the float64 oracle, measured by test_float32_replay_sets_the_device_tolerance over the
# networks and settings below.  On a loopy graph max-product often does not settle: undamped, a 4 x 4 grid's messages
# keep changing by 0.1 a sweep after 50 sweeps, and such a row amplifies rounding (its float32 beliefs drift 5e-4 from
# the oracle's).  On trusted rows (last residual below SETTLED, or at most SHORT sweeps run), normalised beliefs
# differ by at most about 6e-7, and the messages of the first sweeps by at most about 1e-7 on every row.  The GPU
# tests allow about ten times as much: on trusted rows a decoded state is compared where the oracle's belief margin
# (largest minus second largest normalised belief) exceeds MPE_F32_BELIEF_TOL, and stop sweeps may differ where the
# residual lies within MPE_F32_RESIDUAL_NOISE of tol.
MPE_F32_BELIEF_TOL = 6e-6
MPE_F32_RESIDUAL_NOISE = 2e-6
SETTLED = 1e-3
SHORT = 7

LOOPY = ["asia", "alarm", "grid4x4s3", "grid4x4s10x3"]
POLYTREES = ["chain12s4", "naive_bayes", "chow_liu", "barren_ab"]
SETTINGS = [(0.0, 1e-6, 50), (0.5, 1e-5, 100), (0.3, 0.0, 7), (0.8, 1e-4, 3)]


def barren_ab():
    """P(A=0) = 0.6; B | A=0 = (0.5, 0.5), B | A=1 = (0.9, 0.1): the MPE is A=1, B=0 (0.36 > 0.30), and a graph
    without the barren leaf B would decode A=0."""
    bn = BayesNet(("A", "B"))
    bn.P["A"] = pd.Series({0: 0.6, 1: 0.4})
    bn.P["B"] = pd.Series({(0, 0): 0.5, (0, 1): 0.5, (1, 0): 0.9, (1, 1): 0.1})
    return bn.prepare()


def not_gate():
    """A uniform, B = not A: both max-marginals tie exactly, so the first-state decode is A=0, B=0, of probability 0."""
    bn = BayesNet(("A", "B"))
    bn.P["A"] = pd.Series({0: 0.5, 1: 0.5})
    bn.P["B"] = pd.Series({(0, 0): 0.0, (0, 1): 1.0, (1, 0): 1.0, (1, 1): 0.0})
    return bn.prepare()


def structural_zero_chain():
    """A -> B -> C, binary, with P(B=1 | A=1) = 0: A=1, B=1 is impossible inside B's family alone."""
    bn = BayesNet(("A", "B"), ("B", "C"))
    bn.P["A"] = pd.Series({0: 0.3, 1: 0.7})
    bn.P["B"] = pd.Series({(0, 0): 0.4, (0, 1): 0.6, (1, 0): 1.0, (1, 1): 0.0})
    bn.P["C"] = pd.Series({(0, 0): 0.2, (0, 1): 0.8, (1, 0): 0.5, (1, 1): 0.5})
    return bn.prepare()


# rows of structural_zero_chain impossible only inside an observed family: partly observed and every node observed
IMPOSSIBLE_OBSERVED = [pd.DataFrame({"A": [1, 1, 0], "B": [0, 1, 1]}, index=["ok", "zero", "fine"]),
                       pd.DataFrame({"A": [1, 1], "B": [1, 0], "C": [0, 0]}, index=["zero", "ok"])]


def mpe_network(name):
    return barren_ab() if name == "barren_ab" else network(name)


def mpe_graph(net, names):
    return bp.compile_mpe_graph(net, [net.index[e] for e in names])


def by_var_order(res, net, g):
    """The oracle's codes and beliefs in the graph's variable order."""
    order = [res["variables"].index(net.names[v]) for v in g.variables]
    return res["codes"][order], [res["beliefs"][net.names[v]] for v in g.variables]


def last_residual(res):
    """[n] the oracle's residual at the last sweep each row ran (0 for a row that ran none)."""
    r, it = res["residual"], res["iterations"]
    if r.shape[1] == 0:
        return np.zeros(len(it))
    return np.where(it > 0, r[np.arange(len(it)), np.clip(it, 1, r.shape[1]) - 1], 0.0)


def trusted(res, n_iterations):
    """[n] rows of an oracle run whose float32 beliefs stay within the measured drift: settled, or short."""
    return (last_residual(res) < SETTLED) | (np.minimum(res["iterations"], n_iterations) <= SHORT)


def margins(beliefs):
    """[n_var, n] largest minus second largest normalised belief (inf for one state)."""
    out = []
    for b in beliefs:
        s = np.sort(b, axis=1)
        out.append(s[:, -1] - s[:, -2] if b.shape[1] > 1 else np.full(b.shape[0], np.inf))
    return np.array(out)


def joint_log_values(dn, event):
    """log P(x, e) of every joint state of the unobserved nodes (mpe_oracle's dense sum of log CPTs)."""
    union, total = mpe_oracle._add(mpe_oracle._factors(dn, event))
    return np.broadcast_to(total, [len(dn.domains[v]) for v in union]).reshape(-1)


@pytest.mark.parametrize("name", POLYTREES)
def test_oracle_is_the_exact_mpe_on_polytrees(name):
    bn = mpe_network(name)
    if name == "barren_ab":
        dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
        names, codes = [], np.zeros((0, 1), dtype=np.int64)
    else:
        _, dn, names, codes, _ = setup(bn, max(1, len(bn.nodes) // 3), 30, seed=1)
    n = codes.shape[1]
    res = bp_mpe_oracle.run(dn, names, codes, 200, 0.0, 1e-14, n_rows=n)
    assert (res["iterations"] <= 200).all()
    checked = 0
    for b in range(n):
        event = {e: dn.domains[e][codes[i, b]] for i, e in enumerate(names)}
        values = joint_log_values(dn, event)
        best, L = mpe_oracle.brute_force(dn, event)
        if L == -np.inf:
            assert np.isnan(res["log_p"][b]), b
            continue
        assert abs(res["log_p"][b] - L) < 1e-9, b
        top2 = np.sort(values)[-2:]
        if top2[1] - top2[0] > 1e-9:
            got = {v: dn.domains[v][int(res["codes"][j, b])] for j, v in enumerate(res["variables"])}
            assert got == best, b
            checked += 1
    assert checked >= n // 2
    if name == "barren_ab":
        assert dict(zip(res["variables"], res["codes"][:, 0])) == {"A": 1, "B": 0}
        assert res["log_p"][0] == pytest.approx(np.log(0.36), abs=1e-12)


@pytest.mark.parametrize("name", LOOPY)
@pytest.mark.parametrize("damping,tol,n_iterations", SETTINGS)
def test_float64_replay_equals_the_oracle(name, damping, tol, n_iterations):
    bn = mpe_network(name)
    net, dn, names, codes, _ = setup(bn, max(1, len(bn.nodes) // 4), 40, seed=3)
    g = mpe_graph(net, names)
    want = bp_mpe_oracle.run(dn, names, codes, n_iterations, damping, tol)
    got, log_p, iters, _ = bp_mpe_interp.run(g.words, g.tables64, codes, codes.shape[1], n_iterations, damping, tol)
    want_codes, want_beliefs = by_var_order(want, net, g)
    assert np.array_equal(np.isnan(log_p), np.isnan(want["log_p"]))
    differ = iters != want["iterations"]
    assert not (differ & ~near_tol(want["residual"], iters, want["iterations"], tol, 1e-9)).any()
    live = ~np.isnan(log_p) & ~differ
    clear = margins(want_beliefs) > 1e-9  # exact ties (max-product beliefs often tie) may round either way
    assert np.array_equal(got[clear & live], want_codes[clear & live])
    same = live & (got == want_codes).all(axis=0)
    assert same.sum() >= len(same) // 2
    assert np.allclose(log_p[same], want["log_p"][same], rtol=0, atol=1e-12)


def test_float32_replay_sets_the_device_tolerance():
    worst_b = worst_r = 0.0
    for name in ["chain12s4", "naive_bayes"] + LOOPY:
        bn = mpe_network(name)
        net, dn, names, codes, _ = setup(bn, max(1, len(bn.nodes) // 4), 40, seed=4)
        g = mpe_graph(net, names)
        n = codes.shape[1]
        for damping, tol, n_iterations in SETTINGS:
            want = bp_mpe_oracle.run(dn, names, codes, n_iterations, damping, 0.0)
            _, log_p, _, beliefs = bp_mpe_interp.run(g.words, g.tables, codes, n, n_iterations, damping, 0.0,
                                                     dtype=np.float32)
            _, want_beliefs = by_var_order(want, net, g)
            assert np.array_equal(np.isnan(log_p), np.isnan(want["log_p"]))
            ok = trusted(want, n_iterations)
            for b, wb in zip(beliefs, want_beliefs):
                worst_b = max(worst_b, float(np.nanmax(np.abs(b - wb)[ok], initial=0.0)))
            for t in range(1, min(n_iterations, 4) + 1):
                m32 = bp_mpe_interp.run(g.words, g.tables, codes, n, t, damping, 0.0, np.float32, True)[-1]
                m64 = bp_mpe_interp.run(g.words, g.tables64, codes, n, t, damping, 0.0, np.float64, True)[-1]
                ok = ~np.isnan(m64).any(axis=1)
                worst_r = max(worst_r, float(np.abs(m32[ok] - m64[ok]).max(initial=0.0)))
    assert worst_b < MPE_F32_BELIEF_TOL / 5, worst_b
    assert worst_r < MPE_F32_RESIDUAL_NOISE / 5, worst_r


@pytest.mark.parametrize("name", ["asia", "alarm", "grid4x4s3", "naive_bayes"])
def test_compiler_keeps_every_family_and_every_unobserved_node(name):
    bn = mpe_network(name)
    net = bn._compiled
    rng = np.random.default_rng(5)
    n_nodes = len(bn.nodes)
    for n_ev in (0, 1, n_nodes // 2, n_nodes - 1, n_nodes):
        ev = sorted(rng.choice(n_nodes, size=n_ev, replace=False).tolist())
        g = bp.compile_mpe_graph(net, ev)
        w = g.words
        assert int(w[0]) == bp.MAGIC and int(w[1]) == bp.VERSION_MPE == 2
        assert g.families == tuple(range(n_nodes))
        assert g.variables == tuple(v for v in range(n_nodes) if v not in ev)
        assert g.targets == g.variables and g.q_offsets == tuple(range(len(g.variables))) and g.Q == len(g.variables)
        # factor records: 0 members exactly for the all-observed families
        p = int(w[9])
        for v in g.families:
            n_mem = int(w[p + 2])
            assert n_mem == sum(u not in ev for u in net.scope(v))
            p += 4 + 3 * (n_mem + int(w[p + 3]))
        # target records: every variable record in order, q_offset its position
        p, tgt = int(w[10]), int(w[11])
        for k in range(len(g.variables)):
            assert (int(w[tgt + 2 * k]), int(w[tgt + 2 * k + 1])) == (p, k)
            p += 3 + int(w[p + 2])
        observed_only = bp.Graph(w, g.tables, g.tables64, (), (), (), (), 0, 0)
        assert n_ev < n_nodes or observed_only.message_bytes_per_sweep() == 0
        if n_ev == n_nodes:
            assert g.n_edges == 0 and int(w[4]) == 0


def test_the_barren_leaf_stays_in_the_graph():
    net = barren_ab()._compiled
    a, b = net.index["A"], net.index["B"]
    g = bp.compile_mpe_graph(net, [])
    assert g.variables == (a, b) and g.families == (a, b)
    assert bp.compile_graph(net, [], [a]).variables == (a,)  # sum-product prunes it
    codes, log_p, iters, _ = bp_mpe_interp.run(g.words, g.tables64, np.zeros((0, 1)), 1, 50, 0.0, 1e-9)
    assert codes[:, 0].tolist() == [1, 0] and log_p[0] == pytest.approx(np.log(0.36), abs=1e-12)


def test_all_observed_pattern_only_scores():
    bn = examples.asia()
    net = bn._compiled
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    codes = np.zeros((len(net.names), 3), dtype=np.uint8)
    codes[:, 1] = 1
    codes[0, 2] = 1
    g = bp.compile_mpe_graph(net, list(range(len(net.names))))
    assert int(g.words[4]) == 0 and g.n_edges == 0 and g.message_bytes_per_sweep() == 0
    out, log_p, iters, _ = bp_mpe_interp.run(g.words, g.tables64, codes, 3, 10, 0.5, 0.0)
    assert out.shape == (0, 3) and (iters == 0).all()
    for b in range(3):
        assignment = {net.names[v]: net.domains[v][codes[v, b]] for v in range(len(net.names))}
        assert log_p[b] == pytest.approx(mpe_oracle.log_joint(dn, assignment), abs=1e-12)
    names = [net.names[v] for v in range(len(net.names))]
    res = bp_mpe_oracle.run(dn, names, codes, 10, 0.5, 0.0)
    assert (res["iterations"] == 0).all() and np.allclose(res["log_p"], log_p, rtol=0, atol=1e-12)


# ---- the host side of mpe_many(algorithm="bp"), on the float32 replay


class ReplayBP:
    """engine.BeliefPropagation over the float32 replay of the words.  `live` lists every runner created."""

    live = []

    def __init__(self, words, tables, device=None):
        self.words, self.tables = np.asarray(words), np.asarray(tables)
        self.n_ev, self.n_var = int(self.words[2]), int(self.words[4])
        self.closed = False
        ReplayBP.live.append(self)

    def mpe(self, codes, n_rows, n_iterations, damping, tol):
        assert not self.closed
        out, log_p, iters, _ = bp_mpe_interp.run(self.words, self.tables, codes, n_rows, n_iterations, damping, tol,
                                                 dtype=np.float32)
        return out, log_p, iters.astype(np.int32)

    def close(self):
        self.closed = True


@pytest.fixture
def replay(monkeypatch):
    ReplayBP.live = []
    monkeypatch.setattr(engine, "BeliefPropagation", ReplayBP)
    return ReplayBP


def test_patterns_latent_nodes_and_missing_cells(replay):
    bn = examples.asia()
    net = bn._compiled
    events = pd.DataFrame({"Smoker": [True, None, False, None, True], "Dispnea": [True, False, None, None, True],
                           "Visit to Asia": [None, True, False, None, None]}, index=list("abcde"))
    frame, log_p = bn.mpe_many(events, return_log_proba=True, algorithm="bp", n_iterations=60, damping=0.3, tol=1e-7)
    assert list(frame.index) == list("abcde") and list(frame.columns) == sorted(bn.nodes)
    assert list(log_p.index) == list("abcde") and log_p.dtype == np.float64
    assert len(replay.live) == 4  # one runner per missingness pattern: a and e share one
    assert len([k for k in bn._engine_cache if k[0] == "bp_mpe"]) == 4
    for b, label in enumerate(events.index):
        observed = {c: events.loc[label, c] for c in events.columns if events.loc[label, c] is not None}
        for c, value in observed.items():
            assert frame.loc[label, c] == value
        ev = sorted(net.index[c] for c in observed)
        g = bp.compile_mpe_graph(net, ev)
        codes = np.array([[net.domains[v].index(observed[net.names[v]])] for v in ev], dtype=np.uint8).reshape(-1, 1)
        out, lp, _, _ = bp_mpe_interp.run(g.words, g.tables, codes, 1, 60, 0.3, 1e-7, dtype=np.float32)
        for j, v in enumerate(g.variables):
            assert frame.loc[label, net.names[v]] == net.domains[v][out[j, 0]]
        assert log_p[label] == lp[0]
    # the same call again reuses every pattern's runner
    bn.mpe_many(events, algorithm="bp", n_iterations=60, damping=0.3, tol=1e-7)
    assert len(replay.live) == 4


def test_all_observed_rows_and_the_single_event_entry_point(replay):
    bn = examples.asia()
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    full = {v: bn.P[v].index.levels[-1][0] if isinstance(bn.P[v].index, pd.MultiIndex) else bn.P[v].index[0]
            for v in bn.nodes}
    events = pd.DataFrame([full, {"Smoker": True}])
    frame, log_p = bn.mpe_many(events, return_log_proba=True, algorithm="bp")
    assert frame.iloc[0].to_dict() == full
    assert log_p.iloc[0] == pytest.approx(mpe_oracle.log_joint(dn, full), rel=1e-6)
    one = bn.mpe({"Smoker": True}, algorithm="bp")
    assert one.to_dict() == frame.iloc[1].to_dict()


def test_a_dead_row_raises_the_exact_paths_error(replay):
    spec = synthetic.chain(6, 3)
    v = spec.nodes[-1]
    cpt = spec.cpt[v].copy()
    cpt[..., -1] = 0.0
    spec.cpt[v] = cpt / cpt.sum(axis=-1, keepdims=True)
    bn = synthetic.load(spec, BayesNet)
    dom = bn._compiled.domains[bn._compiled.index[v]]
    events = pd.DataFrame({v: [dom[0], dom[-1], dom[1]]}, index=["ok", "impossible", "fine"])
    with pytest.raises(ValueError, match="1 row\\(s\\) have observed cells of probability zero.*'impossible'"):
        bn.mpe_many(events, algorithm="bp")


def test_impossible_inside_an_observed_family_is_dead():
    """A 0-member factor is skipped by the sweep, so its zero never reaches a message: the row is dead before its
    first sweep, in the oracle and the replay alike, as brute force finds it impossible."""
    bn = structural_zero_chain()
    net = bn._compiled
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    for events in IMPOSSIBLE_OBSERVED:
        names = list(events.columns)
        codes = np.stack([[net.domains[net.index[c]].index(x) for x in events[c]] for c in names]).astype(np.uint8)
        n = codes.shape[1]
        g = mpe_graph(net, names)
        want = bp_mpe_oracle.run(dn, names, codes, 20, 0.5, 1e-9)
        for tables in (g.tables64, g.tables):
            got, log_p, iters, _ = bp_mpe_interp.run(g.words, tables, codes, n, 20, 0.5, 1e-9)
            for b, label in enumerate(events.index):
                impossible = mpe_oracle.brute_force(dn, dict(events.loc[label]))[1] == -np.inf
                assert impossible == (label == "zero")
                assert np.isnan(log_p[b]) == np.isnan(want["log_p"][b]) == impossible
                if impossible:
                    assert iters[b] == want["iterations"][b] == 0 and not got[:, b].any()
                else:
                    assert log_p[b] == pytest.approx(want["log_p"][b], abs=1e-6)


@pytest.mark.parametrize("k", range(len(IMPOSSIBLE_OBSERVED)))
def test_impossible_inside_an_observed_family_raises(replay, k):
    with pytest.raises(ValueError, match="1 row\\(s\\) have observed cells of probability zero \\(first: 'zero'\\)"):
        structural_zero_chain().mpe_many(IMPOSSIBLE_OBSERVED[k], algorithm="bp")


def test_warnings_count_zero_probability_decodes_and_unconverged_rows(replay):
    bn = not_gate()
    events = pd.DataFrame({"A": [None, None, None]})
    with pytest.warns(RuntimeWarning, match="3 of 3 rows decoded an explanation of probability zero"):
        frame, log_p = bn.mpe_many(events, return_log_proba=True, algorithm="bp")
    assert (log_p == -np.inf).all() and (frame.to_numpy() == 0).all()
    bn = examples.asia()
    events = pd.DataFrame({"Smoker": [True, False, True, None]})
    with pytest.warns(RuntimeWarning, match="4 of 4 rows did not converge to tol=0 in 2 sweeps"):
        bn.mpe_many(events, algorithm="bp", n_iterations=2, tol=0.0)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        bn.mpe_many(events, algorithm="bp", n_iterations=200)


def test_argument_errors(replay):
    bn = examples.asia()
    events = pd.DataFrame({"Smoker": [True, False]})
    for kw in ({"damping": 1.0}, {"damping": -0.1}, {"n_iterations": 0}, {"n_iterations": 2.5}, {"tol": -1e-3},
               {"tol": float("nan")}):
        with pytest.raises(ValueError):
            bn.mpe_many(events, algorithm="bp", **kw)
        with pytest.raises(ValueError):
            bn.mpe({"Smoker": True}, algorithm="bp", **kw)
    with pytest.raises(ValueError, match="Unknown algorithm"):
        bn.mpe_many(events, algorithm="loopy")
    with pytest.raises(ValueError, match="soft evidence"):
        bn.mpe_many(events, algorithm="bp", likelihoods={"Dispnea": np.ones((2, 2))})
    with pytest.raises(ValueError, match="soft evidence"):
        bn.mpe({"Smoker": True}, algorithm="bp", likelihoods={"Dispnea": [0.5, 0.5]})
    with pytest.raises(ValueError, match="not a state"):
        bn.mpe_many(pd.DataFrame({"Smoker": ["maybe"]}), algorithm="bp")
    assert not replay.live


def test_no_silent_cpu_fallback():
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    bn = examples.asia()
    with pytest.raises(engine.EngineError):
        bn.mpe_many(pd.DataFrame({"Smoker": [True, None]}), algorithm="bp")
    with pytest.raises(engine.EngineError):
        bn.mpe({"Smoker": True}, algorithm="bp")


def test_exact_planner_refuses_the_16x16_mpe():
    from test_bp_plan import GRID16_EVIDENCE

    net = synthetic.load(synthetic.grid(16, 16, 3), BayesNet)._compiled
    evidence = sorted(net.index[e] for e in GRID16_EVIDENCE)
    with pytest.raises(ValueError, match="2\\^31"):
        planner.build_mpe_plan(net, tuple(evidence))
    g = bp.compile_mpe_graph(net, evidence)
    assert len(g.families) == 256 and len(g.variables) == 226
