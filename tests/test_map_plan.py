"""Marginal MAP plans (planner.build_map_plan, version-9 programs) and BayesNet.map_many, checked on the CPU.

tests/map_oracle.py finds the marginal MAP state in float64 without the planner (brute force, and the
argmax of the dense posterior); oracle/program_interp.py executes the serialised words.  The host side of
`map_many` runs with the device programs replaced by the float32 interpreter."""
import json
import os

import numpy as np
import pandas as pd
import pytest

import kernel_corpus
import map_oracle
from conftest import build_network, load_golden
from interpreted_program import InterpretedProgram
from oracle import program_interp, ve_oracle
from sorobn_b200 import engine, examples, planner, workloads

EXAMPLES = ["alarm", "asia", "sprinkler", "grades"]
DENSE = ["grid4x4s3", "chain9s4", "dag20p4s4"]
CORPUS = ["dag9p2s4x1x4x4_seed54_q1-8_e2", "dag14p4s5x8_seed1_zeros_q10-13_e1", "dag8p2s37x3x2_seed3_q0-3_e2",
          "dag16p4s8_seed0_q15_e2", "grid7x7s5_seed39_q48_e18", "dag19p7s3_seed93_q12_e3"]
TOL = 2e-5  # x max(1, |L*|): float32 rounding of a sum of logs
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def network(name):
    if name in EXAMPLES:
        return getattr(examples, name)()._compiled
    if name in DENSE:
        return build_network(load_golden(name))._compiled
    case = next(c for c in kernel_corpus.CASES if c["name"] == name)
    return kernel_corpus.compiled_net(kernel_corpus.make_spec(case))


def dense(net):
    """The oracle's DenseNet of a CompiledNet (CPT axes [*parents, v], parents sorted by name in both)."""
    names = net.names
    dn = ve_oracle.DenseNet(nodes=list(names), parents={names[v]: [names[p] for p in net.parents[v]] for v in range(len(names))},
                            domains={names[v]: list(net.domains[v]) for v in range(len(names))})
    for v in range(len(names)):
        dn.cpt[names[v]] = np.asarray(net.cpt[v], dtype=np.float64)
    return dn


def queries(net, seed, max_map_states=4096):
    """(observed var ids, MAP var ids) pairs: no evidence, some evidence, MAP sets of one to four variables."""
    rng = np.random.default_rng(seed)
    n = len(net.names)
    out = []
    for k_obs in (0, 1, n // 3):
        observed = tuple(sorted(rng.choice(n, size=k_obs, replace=False).tolist()))
        free = [v for v in range(n) if v not in observed]
        for k_map in (1, 2, 4):
            if k_map > len(free):
                continue
            m = tuple(sorted(rng.choice(free, size=k_map, replace=False).tolist()))
            if int(np.prod([int(net.card[v]) for v in m])) <= max_map_states:
                out.append((observed, m))
    return out


def check_rows(net, dn, plan, observed, codes, decoded, log_p, tol, exact=False):
    """Every row: its log-probability is the oracle's L*, and so is log P(decoded state, e); where the oracle's
    best beats the runner-up by more than `tol`, the decoded state is the oracle's."""
    near = 0
    for b in range(codes.shape[1]):
        ev = {net.names[v]: net.domains[v][codes[i, b]] for i, v in enumerate(observed)}
        mv = [net.names[v] for v in plan.sampled]
        x, L, gap = map_oracle.solve(dn, ev, mv)
        mine = {net.names[v]: net.domains[v][decoded[j, b]] for j, v in enumerate(plan.sampled)}
        if L == -np.inf:
            assert log_p[b] == -np.inf
            continue
        t = tol * max(1.0, abs(L))
        assert abs(float(log_p[b]) - L) <= t, (observed, plan.sampled, b, float(log_p[b]), L)
        if gap > t:
            assert mine == x, (observed, plan.sampled, b)
        else:
            assert abs(map_oracle.log_prob(dn, ev, mine) - L) <= t
            near += mine != x
    return near


# ------------------------------------------------------------------------------------- the oracle
@pytest.mark.parametrize("name", EXAMPLES + ["chain9s4"])
def test_dense_query_agrees_with_brute_force(name):
    net = network(name)
    dn = dense(net)
    codes = workloads.forward_sample_codes(net, 3, 1)
    checked = 0
    for observed, m in queries(net, 2):
        mv = [net.names[v] for v in m]
        for b in range(3):
            ev = {net.names[v]: net.domains[v][codes[v, b]] for v in observed}
            xb, Lb, gb = map_oracle.brute_force(dn, ev, mv)
            xd, Ld, gd = map_oracle.dense_query(dn, ev, mv)
            assert abs(Lb - Ld) < 1e-9 and abs(gb - gd) < 1e-9 or (gb == gd == np.inf)
            assert abs(map_oracle.log_prob(dn, ev, xb) - Lb) < 1e-9
            checked += 1
    assert checked > 0


# ------------------------------------------------------------------------------ the interpreter
@pytest.mark.parametrize("name", EXAMPLES + DENSE + CORPUS)
def test_interpreter_finds_the_oracles_state(name):
    """In float64 every row reaches the oracle's L* to 1e-9 (the state itself where the margin is wider); in
    float32, to the float32 rounding of sums of logs."""
    net = network(name)
    dn = dense(net)
    n_rows = 5
    codes_all = workloads.forward_sample_codes(net, n_rows, 5)
    for observed, m in queries(net, 3):
        plan = planner.build_map_plan(net, observed, m)
        assert sorted(plan.sampled) == list(m)
        codes = np.ascontiguousarray(codes_all[list(observed)])
        d64, l64 = program_interp.run_mpe(plan.words, plan.table_blob64, codes, n_rows=n_rows, dtype=np.float64)
        d32, l32 = program_interp.run_mpe(plan.words, plan.table_blob, codes, n_rows=n_rows, dtype=np.float32)
        assert l64.dtype == np.float64 and l32.dtype == np.float32
        if not observed:
            codes = np.zeros((0, n_rows), dtype=np.uint8)
        check_rows(net, dn, plan, observed, codes, d64, l64, 1e-9)
        check_rows(net, dn, plan, observed, codes, d32, l32, TOL)


@pytest.mark.parametrize("name", EXAMPLES)
def test_impute_goldens_are_reproduced(name):
    """The reference's `impute` cases: the MAP variables are the missing cells, nothing is latent.  Where the
    oracle's best beats the runner-up by more than the tolerance the states are equal; at near-ties the
    log-probabilities are."""
    with open(os.path.join(GOLDEN, f"impute_{name}.json")) as f:
        cases = json.load(f)["cases"]
    bn = getattr(examples, name)()
    net = bn._compiled
    dn = dense(net)
    compared = 0
    for case in cases:
        sample = dict((k, v) for k, v in case["sample"])
        filled = dict((k, v) for k, v in case["filled"])
        observed = tuple(sorted(net.index[k] for k, v in sample.items() if v is not None))
        m = tuple(sorted(net.index[k] for k, v in sample.items() if v is None))
        plan = planner.build_map_plan(net, observed, m)
        codes = np.array([[net.domains[v].index(sample[net.names[v]])] for v in observed], dtype=np.uint8).reshape(len(observed), 1)
        for blob, dtype, tol in ((plan.table_blob64, np.float64, 1e-9), (plan.table_blob, np.float32, TOL)):
            d, lp = program_interp.run_mpe(plan.words, blob, codes, n_rows=1, dtype=dtype)
            ev = {k: v for k, v in sample.items() if v is not None}
            mine = {net.names[v]: net.domains[v][d[j, 0]] for j, v in enumerate(plan.sampled)}
            want = {k: filled[k] for k in mine}
            x, L, gap = map_oracle.brute_force(dn, ev, list(mine))
            t = tol * max(1.0, abs(L))
            assert abs(float(lp[0]) - L) <= t
            if gap > t:
                assert mine == want, case
                compared += 1
            else:
                assert abs(map_oracle.log_prob(dn, ev, mine) - map_oracle.log_prob(dn, ev, want)) <= t
    assert compared > 0


def test_an_impossible_row_has_log_probability_minus_infinity():
    bn = examples.sprinkler()
    net = bn._compiled
    observed = tuple(sorted(net.index[c] for c in ("Rain", "Sprinkler", "Wet grass")))
    plan = planner.build_map_plan(net, observed, [net.index["Cloudy"]])
    event = {"Rain": False, "Sprinkler": False, "Wet grass": True}
    codes = np.array([[net.domains[v].index(event[net.names[v]])] for v in observed], dtype=np.uint8)
    for blob, dtype in ((plan.table_blob, np.float32), (plan.table_blob64, np.float64)):
        _, lp = program_interp.run_mpe(plan.words, blob, codes, dtype=dtype)
        assert lp[0] == -np.inf and not np.isnan(lp[0])


# -------------------------------------------------------------------------------- plan structure
def summed_steps_ok(plan, net, observed, m):
    summed = set(plan.order) - set(m)
    assert set(plan.order) <= set(range(len(net.names))) - set(observed)
    k = len(summed)
    assert set(plan.order[:k]) == summed and set(plan.order[k:]) == set(m)  # summed before maximised
    for st in plan.steps:
        if st.kind in (planner.KIND_FLAT, planner.KIND_BATCHED):
            kinds = {e in summed for e in st.elims}
            assert len(kinds) <= 1, "a launch mixes a summed and a maximised variable"
            want = planner.REDUCE_LOGSUMEXP if kinds == {True} else planner.REDUCE_MAX
            assert st.reduce == want
        else:
            assert st.kind == planner.KIND_ARGMAX and set(st.elims) <= set(m)


@pytest.mark.parametrize("name", EXAMPLES + DENSE + CORPUS)
def test_no_bucket_mixes_summed_and_maximised_variables(name):
    net = network(name)
    for observed, m in queries(net, 7):
        plan = planner.build_map_plan(net, observed, m)
        assert plan.version == planner.VERSION_MAP and plan.words[1] == 9 and plan.words[7] == 1
        assert plan.words[10] == len(plan.sampled) == len(m) and sorted(plan.sampled) == list(m)
        summed_steps_ok(plan, net, observed, m)
        argmax = [st for st in plan.steps if st.kind == planner.KIND_ARGMAX]
        assert plan.steps[-len(argmax):] == argmax
        done = set()
        for st in argmax:  # every separator is decoded first, and holds MAP variables only
            assert st.q_offset == len(done)
            for f, _, _ in st.inputs:
                for col, _, _ in f.ev:
                    assert col < len(observed) or plan.sampled[col - len(observed)] in done
                assert set(f.vars) <= set(st.elims) | done
            done |= set(st.elims)
        assert done == set(m)


def test_barren_summed_variables_drop_out():
    """Relevant = MAP variables, evidence and their ancestors: a summed descendant of neither is not planned."""
    net = examples.asia()._compiled
    m = (net.index["Smoker"],)
    plan = planner.build_map_plan(net, (), m)
    assert set(plan.tables) == {net.index["Smoker"]} and plan.order == list(m)
    mpe = planner.build_mpe_plan(net, ())
    assert len(mpe.tables) == len(net.names)


def test_a_map_set_of_every_unobserved_variable_is_the_mpe_plan():
    """Nothing to sum: the same order and steps as the MPE plan, every reduction word 0."""
    for name in ("asia", "alarm", "grid4x4s3", "dag20p4s4"):
        net = network(name)
        observed = (0, len(net.names) - 1)
        hidden = tuple(v for v in range(len(net.names)) if v not in observed)
        mpe = planner.build_mpe_plan(net, observed)
        mp = planner.build_map_plan(net, observed, hidden)
        assert mp.order == mpe.order and mp.sampled == mpe.sampled
        assert all(st.reduce == planner.REDUCE_MAX for st in mp.steps)
        hdr, _, _, steps = program_interp.parse(mp.words)
        stripped = list(mp.words[:planner.HEADER_WORDS + 2 * hdr["n_tables"] + 2 * hdr["n_slots"]])
        p = len(stripped)
        w = [int(x) for x in mp.words]
        for st in steps:
            n_in, n_axes, n_elim = w[p + 1], w[p + 3], w[p + 4]
            stripped += w[p:p + 5]
            extra = w[p + 5]
            p += 6
            if st["kind"] == planner.KIND_ARGMAX:
                stripped.append(extra)
            size = n_axes + n_elim
            for _ in range(n_in):
                size += 4 + 3 * w[p + size + 3] + n_elim + n_axes
            stripped += w[p:p + size]
            p += size
        assert p == len(w)
        stripped[1] = 8
        assert np.array_equal(np.asarray(stripped, dtype=np.int32), mpe.words)
        assert np.array_equal(mp.table_blob, mpe.table_blob)


def test_versions_4_to_8_have_no_reduction_word():
    for name in ("asia", "alarm", "grid4x4s3"):
        net = network(name)
        assert planner.build_plan(net, [1], [0]).words[1] == 4
        mpe = planner.build_mpe_plan(net, [0])
        assert mpe.words[1] == 8 and len(mpe.words) == len(planner.build_sample_plan(net, [0]).words)


def test_a_given_order_must_sum_first():
    net = examples.asia()._compiled
    m = (net.index["Lung cancer"],)
    observed = (net.index["Dispnea"],)
    plan = planner.build_map_plan(net, observed, m)
    bad = list(m) + [v for v in plan.order if v not in m]
    with pytest.raises(ValueError, match="before any MAP variable"):
        planner.build_map_plan(net, observed, m, order=bad)
    assert planner.build_map_plan(net, observed, m, order=plan.order).order == plan.order


def test_refusals():
    net = examples.asia()._compiled
    with pytest.raises(ValueError, match="cannot be part of the event"):
        planner.build_map_plan(net, [0], [0])
    with pytest.raises(ValueError, match="duplicate"):
        planner.build_map_plan(net, [0], [1, 1])
    with pytest.raises(ValueError, match="nothing to compute"):
        planner.build_map_plan(net, [], [])


def test_bounds_are_those_of_the_mpe_plan(monkeypatch):
    net = examples.asia()._compiled
    planner.build_map_plan(net, [0], [1, 2])
    monkeypatch.setattr(planner, "SAMPLE_MAX_CARD", 1)
    with pytest.raises(ValueError, match="uint8"):
        planner.build_map_plan(net, [0], [1, 2])
    monkeypatch.undo()
    monkeypatch.setattr(planner, "MAX_Z", 1)
    with pytest.raises(ValueError, match="draws from at most 1"):
        planner.build_map_plan(net, [0], [1, 2])


def test_a_constrained_order_past_the_axes_is_refused_naming_the_bucket(monkeypatch):
    """Summing a hub first joins its neighbours into one factor; past the kernel's axes the plan is refused."""
    net = network("grid4x4s3")
    m = tuple(range(1, len(net.names)))  # everything but variable 0 is MAP
    planner.build_map_plan(net, (), m)
    monkeypatch.setattr(planner, "MAX_AXES", 1)
    with pytest.raises(ValueError, match=r"the bucket of \['.*'\]: a factor over"):
        planner.build_map_plan(net, (), m)


def test_benchmark_grid_plan_counts():
    wl = workloads.grid10x10()
    net = wl.build()._compiled
    observed = tuple(sorted(net.index[e] for e in wl.evidence))
    hidden = [v for v in range(len(net.names)) if v not in observed]
    m = tuple(hidden[::5])
    plan = planner.build_map_plan(net, observed, m)
    kinds = [st.kind for st in plan.steps]
    assert kinds.count(planner.KIND_ARGMAX) >= 1 and len(plan.sampled) == len(m)
    assert any(st.reduce == planner.REDUCE_LOGSUMEXP for st in plan.steps if st.kind == planner.KIND_BATCHED)
    summed_steps_ok(plan, net, observed, m)


# --------------------------------------------------------------------- map_many on the interpreter
@pytest.fixture
def interpreted(monkeypatch):
    InterpretedProgram.live = []
    monkeypatch.setattr(engine, "Program", InterpretedProgram)
    return InterpretedProgram


def frame(bn, n, seed, frac, latent=()):
    net = bn._compiled
    codes = workloads.forward_sample_codes(net, n, seed)
    rng = np.random.default_rng(seed + 1)
    cols = {}
    for v, name in enumerate(net.names):
        if name in latent:
            continue
        values = np.asarray(net.domains[v], dtype=object)[codes[v]]
        values[rng.random(n) < frac] = None
        cols[name] = values
    return pd.DataFrame(cols, index=pd.RangeIndex(100, 100 + n, name="row"))


def check_frame(bn, X, got, log_p, variables=None):
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    for b in range(len(X)):
        ev = {c: X[c].iloc[b] for c in X.columns if pd.notna(X[c].iloc[b])}
        mv = [c for c in X.columns if pd.isna(X[c].iloc[b])] if variables is None else [v for v in variables if v not in ev]
        row = got.iloc[b]
        assert all(row[c] == v for c, v in ev.items())  # observed cells are copied through
        mine = {c: row[c] for c in mv}
        x, L, gap = map_oracle.solve(dn, ev, mv)
        t = TOL * max(1.0, abs(L))
        assert abs(log_p.iloc[b] - L) <= t and abs(map_oracle.log_prob(dn, ev, mine) - L) <= t, b
        others = [c for c in got.columns if c not in ev and c not in mv]
        assert all(pd.isna(row[c]) for c in others)  # summed out: still missing


def test_map_many_with_missing_cells_and_a_latent_node(interpreted):
    bn = examples.asia()
    bn.max_cached_programs = 4
    X = frame(bn, 80, 3, 0.3, latent=["Tuberculosis"])
    got, log_p = bn.map_many(X, return_log_proba=True)
    assert list(got.columns) == sorted(X.columns) and got.index.equals(X.index) and log_p.index.equals(X.index)
    assert log_p.dtype == np.float64 and not got.isna().any().any()
    assert all(got[c].dtype == bool for c in got.columns)
    assert len(bn._engine_cache) <= bn.max_cached_programs
    check_frame(bn, X, got, log_p)
    assert bn.map_many(X).equals(got)


def test_map_many_with_listed_variables(interpreted):
    bn = examples.alarm()
    X = frame(bn, 40, 8, 0.3, latent=["Burglary"])
    variables = ["Burglary", "Alarm"]
    got, log_p = bn.map_many(X, variables=variables, return_log_proba=True)
    assert list(got.columns) == sorted(set(X.columns) | set(variables))
    assert not got["Burglary"].isna().any() and not got["Alarm"].isna().any()
    check_frame(bn, X, got, log_p, variables)
    keys = [k for k in bn._engine_cache if k[0] == "map"]
    assert keys and all(set(k[2]) <= {bn._compiled.index[v] for v in variables} for k in keys)


def test_map_agrees_with_impute_many(interpreted, monkeypatch):
    bn = examples.grades()
    X = frame(bn, 60, 4, 0.4)
    got = bn.map_many(X)
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    for b in range(len(X)):
        sample = {c: (None if pd.isna(X[c].iloc[b]) else X[c].iloc[b]) for c in X.columns}
        missing = [c for c, v in sample.items() if v is None]
        if not missing or len(missing) == len(sample):
            continue
        ev = {c: v for c, v in sample.items() if v is not None}
        _, L, gap = map_oracle.solve(dn, ev, missing)
        if gap > TOL * max(1.0, abs(L)):
            want = ve_oracle.impute(dn, sample)
            assert all(got[c].iloc[b] == want[c] for c in missing), b


def test_map_of_one_event_and_errors(interpreted):
    bn = examples.asia()
    got = bn.map({"Dispnea": True, "Smoker": False, "Lung cancer": None})
    assert isinstance(got, pd.Series) and list(got.index) == ["Dispnea", "Lung cancer", "Smoker"]
    assert got["Dispnea"] == True and got["Smoker"] == False  # noqa: E712
    both = bn.map({"Dispnea": True}, variables=["Lung cancer", "Tuberculosis"])
    assert list(both.index) == ["Dispnea", "Lung cancer", "Tuberculosis"]
    sprinkler = examples.sprinkler()
    X = pd.DataFrame({"Rain": [False, True], "Sprinkler": [False, True], "Wet grass": [True, True], "Cloudy": [None, None]})
    with pytest.raises(ValueError, match="probability zero"):
        sprinkler.map_many(X)
    with pytest.raises(ValueError, match="not a state"):
        sprinkler.map_many(pd.DataFrame({"Rain": ["maybe"]}))
    with pytest.raises(ValueError, match="not nodes"):
        sprinkler.map_many(X.iloc[:1], variables=["Sunny"])
    empty = sprinkler.map_many(X.iloc[:0])
    assert empty.shape == (0, 4) and list(empty.columns) == sorted(X.columns)


def test_the_map_pattern_programs_are_keyed_by_their_variables(monkeypatch):
    class FakeProgram:
        def __init__(self, plan, device=None, f64=False):
            self.plan = plan

        def close(self):
            pass

    monkeypatch.setattr(engine, "Program", FakeProgram)
    bn = examples.asia()
    a = bn._pattern_runner("map", (0,), (1,))
    assert a.plan.version == planner.VERSION_MAP and bn._pattern_runner("map", (0,), (1,)) is a
    assert bn._pattern_runner("map", (0,), (1, 2)) is not a
    assert bn._pattern_runner("mpe", (0,)).plan.version == planner.VERSION_MPE
