"""MPE plans (planner.build_mpe_plan, version-8 programs) and BayesNet.mpe_many, checked on the CPU.

tests/mpe_oracle.py finds the most probable explanation in float64 without the planner (brute force,
and dense max-sum elimination with a traceback); oracle/program_interp.py executes the serialised words.
The host side of `mpe_many` runs with the device programs replaced by the float32 interpreter, which
follows the kernels' arithmetic exactly."""
import numpy as np
import pandas as pd
import pytest

import mpe_oracle
from conftest import build_network, load_golden
from interpreted_program import InterpretedProgram
from oracle import program_interp, ve_oracle
from sorobn_b200 import engine, examples, planner, workloads

EXAMPLES = ["alarm", "asia", "sprinkler", "grades"]
DENSE = ["grid4x4s3", "chain9s4", "dag20p4s4"]


def network(name):
    if name in EXAMPLES:
        return getattr(examples, name)()
    return build_network(load_golden(name))


def oracle_net(bn):
    return ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)


def hidden_states(dn, event):
    return int(np.prod([len(dn.domains[v]) for v in dn.nodes if v not in event], dtype=np.int64))


def patterns(n_vars, seed):
    """Observed var ids: none, every node, and a few in between (the others latent)."""
    rng = np.random.default_rng(seed)
    out = [(), tuple(range(n_vars))]
    for k in (1, n_vars // 3, n_vars - 1):
        out.append(tuple(sorted(rng.choice(n_vars, size=k, replace=False).tolist())))
    return out


def explanation(net, plan, observed, codes, decoded, b):
    """{node: value} of every node: the row's observed cells and the decoded rest."""
    a = {net.names[v]: net.domains[v][codes[i, b]] for i, v in enumerate(observed)}
    a.update({net.names[v]: net.domains[v][decoded[j, b]] for j, v in enumerate(plan.sampled)})
    return a


# ------------------------------------------------------------------------------------- the oracle
@pytest.mark.parametrize("name", EXAMPLES + DENSE)
def test_max_sum_elimination_agrees_with_brute_force(name):
    bn = network(name)
    dn = oracle_net(bn)
    net = bn._compiled
    checked = 0
    for observed in patterns(len(net.names), 1):
        codes = workloads.forward_sample_codes(net, 4, 2)
        for b in range(4):
            ev = {net.names[v]: net.domains[v][codes[v, b]] for v in observed}
            x, L = mpe_oracle.max_sum(dn, ev)
            assert abs(mpe_oracle.log_joint(dn, {**ev, **x}) - L) < 1e-9
            if hidden_states(dn, ev) <= mpe_oracle.BRUTE_MAX:
                xb, Lb = mpe_oracle.brute_force(dn, ev)
                assert abs(Lb - L) < 1e-9 and abs(mpe_oracle.log_joint(dn, {**ev, **xb}) - L) < 1e-9
                checked += 1
    assert checked > 0


# ------------------------------------------------------------------------------ the interpreter
@pytest.mark.parametrize("name", EXAMPLES + DENSE)
def test_interpreter_finds_the_oracles_explanation(name):
    """In float64 every row's explanation reaches the oracle's maximum L* and its log-probability is L*, to
    1e-9; in float32, to the float32 rounding of a sum of logs."""
    bn = network(name)
    dn = oracle_net(bn)
    net = bn._compiled
    n_rows = 6
    codes_all = workloads.forward_sample_codes(net, n_rows, 5)
    for observed in patterns(len(net.names), 3):
        plan = planner.build_mpe_plan(net, observed)
        codes = np.ascontiguousarray(codes_all[list(observed)])
        d64, l64 = program_interp.run_mpe(plan.words, plan.table_blob64, codes, n_rows=n_rows, dtype=np.float64)
        d32, l32 = program_interp.run_mpe(plan.words, plan.table_blob, codes, n_rows=n_rows, dtype=np.float32)
        assert l64.dtype == np.float64 and l32.dtype == np.float32
        for b in range(n_rows):
            ev = {net.names[v]: net.domains[v][codes[i, b]] for i, v in enumerate(observed)}
            x, L = mpe_oracle.max_sum(dn, ev)
            assert abs(l64[b] - L) < 1e-9, (observed, b)
            assert abs(mpe_oracle.log_joint(dn, explanation(net, plan, observed, codes, d64, b)) - L) < 1e-9
            tol = 2e-5 * max(1.0, abs(L))
            assert abs(float(l32[b]) - L) < tol
            assert abs(mpe_oracle.log_joint(dn, explanation(net, plan, observed, codes, d32, b)) - L) < tol
            if len(observed) == len(net.names):
                assert abs(l64[b] - mpe_oracle.log_joint(dn, ev)) < 1e-9  # nothing to decode: log P(row)


def test_an_impossible_row_has_log_probability_minus_infinity():
    bn = examples.sprinkler()
    net = bn._compiled
    observed = tuple(sorted(net.index[c] for c in ("Rain", "Sprinkler", "Wet grass")))
    plan = planner.build_mpe_plan(net, observed)
    # neither rain nor the sprinkler, and yet wet grass
    event = {"Rain": False, "Sprinkler": False, "Wet grass": True}
    codes = np.array([[net.domains[v].index(event[net.names[v]])] for v in observed], dtype=np.uint8)
    assert mpe_oracle.max_sum(oracle_net(bn), event)[1] == -np.inf
    for blob, dtype in ((plan.table_blob, np.float32), (plan.table_blob64, np.float64)):
        _, lp = program_interp.run_mpe(plan.words, blob, codes, dtype=dtype)
        assert lp[0] == -np.inf


# -------------------------------------------------------------------------------- plan structure
def test_every_unobserved_node_is_decoded_once_after_its_separator():
    for name in EXAMPLES + DENSE:
        net = network(name)._compiled
        for observed in ((0, len(net.names) - 1), ()):
            plan = planner.build_mpe_plan(net, observed)
            assert plan.version == planner.VERSION_MPE and plan.words[1] == 8 and plan.words[7] == 1
            assert sorted(plan.sampled) == [v for v in range(len(net.names)) if v not in observed]
            assert plan.words[10] == len(plan.sampled) and plan.words[11] == 0
            argmax = [st for st in plan.steps if st.kind == planner.KIND_ARGMAX]
            assert plan.steps[-len(argmax):] == argmax  # the argmax steps run last
            assert all(st.kind in (planner.KIND_FLAT, planner.KIND_BATCHED) for st in plan.steps[:-len(argmax)])
            done = set()
            for st in argmax:
                assert st.q_offset == len(done) and tuple(plan.sampled[st.q_offset:st.q_offset + len(st.elims)]) == st.elims
                for f, _, _ in st.inputs:
                    for col, _, _ in f.ev:
                        assert col < len(observed) or plan.sampled[col - len(observed)] in done
                    assert set(f.vars) <= set(st.elims) | done
                done |= set(st.elims)
            assert done == set(plan.sampled)


def test_a_pattern_with_no_hidden_variable_is_planned():
    net = examples.asia()._compiled
    plan = planner.build_mpe_plan(net, tuple(range(len(net.names))))
    assert plan.sampled == () and plan.words[10] == 0
    assert not any(st.kind == planner.KIND_ARGMAX for st in plan.steps)


def test_tables_are_shipped_as_logs():
    net = examples.sprinkler()._compiled
    sample = planner.build_sample_plan(net, [0])
    mpe = planner.build_mpe_plan(net, [0])
    with np.errstate(divide="ignore"):
        want = np.log(sample.table_blob64)
    assert np.array_equal(mpe.table_blob64, want)
    assert np.array_equal(mpe.table_blob, want.astype(np.float32))
    assert np.isneginf(mpe.table_blob[sample.table_blob64 == 0]).all()


def test_a_decode_step_past_the_bounds_is_refused_as_by_the_sample_plan(monkeypatch):
    net = examples.asia()._compiled
    planner.build_mpe_plan(net, [0])
    monkeypatch.setattr(planner, "SAMPLE_MAX_CARD", 1)
    with pytest.raises(ValueError, match="uint8"):
        planner.build_mpe_plan(net, [0])
    monkeypatch.undo()
    monkeypatch.setattr(planner, "SAMPLE_MAX_TERMS", 1)
    with pytest.raises(ValueError, match="gathers at most 1"):
        planner.build_mpe_plan(net, [0])
    monkeypatch.undo()
    monkeypatch.setattr(planner, "MAX_Z", 1)
    with pytest.raises(ValueError, match="draws from at most 1"):
        planner.build_mpe_plan(net, [0])


def test_version_4_to_7_words_are_unchanged_by_the_mpe_planner():
    """The older programs keep their version numbers, and an MPE program is a sample program's words with
    version 8 and kind 5 in place of 7 and 4."""
    for name in ("asia", "alarm", "grid4x4s3"):
        net = network(name)._compiled
        assert planner.build_plan(net, [1], [0]).words[1] == 4
        assert planner.build_marginals_plan(net, [0]).words[1] == 5
        assert planner.build_counts_plan(net, [0]).words[1] == 6
        sample = planner.build_sample_plan(net, [0]).words
        mpe = planner.build_mpe_plan(net, [0]).words
        assert sample[1] == 7 and mpe[1] == 8 and len(sample) == len(mpe)
        diff = np.flatnonzero(sample != mpe)
        assert diff[0] == 1 and (sample[diff[1:]] == planner.KIND_SAMPLE).all() and (mpe[diff[1:]] == planner.KIND_ARGMAX).all()
        assert len(diff) - 1 == sum(st.kind == planner.KIND_ARGMAX for st in planner.build_mpe_plan(net, [0]).steps)


def test_benchmark_grid_plan_counts():
    wl = workloads.grid10x10()
    net = wl.build()._compiled
    observed = tuple(sorted(net.index[e] for e in wl.evidence))
    plan = planner.build_mpe_plan(net, observed)
    kinds = [st.kind for st in plan.steps]
    assert (len(plan.evidence), len(plan.sampled)) == (30, 70)
    assert (kinds.count(planner.KIND_BATCHED), kinds.count(planner.KIND_FLAT), kinds.count(planner.KIND_ARGMAX)) == (47, 20, 66)
    assert plan.bytes_per_row() == 157_216 and plan.scratch_floats_per_row() == 19_367
    assert plan.bytes_per_row() == planner.build_sample_plan(net, observed).bytes_per_row(n_draws=1)


# --------------------------------------------------------------------- mpe_many on the interpreter
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


def check_rows(bn, X, got, log_p):
    dn = oracle_net(bn)
    for b in range(len(X)):
        ev = {c: X[c].iloc[b] for c in X.columns if pd.notna(X[c].iloc[b])}
        row = got.iloc[b].to_dict()
        assert all(row[c] == v for c, v in ev.items())  # observed cells are copied through
        _, L = mpe_oracle.max_sum(dn, ev)
        tol = 2e-5 * max(1.0, abs(L))
        assert abs(mpe_oracle.log_joint(dn, row) - L) < tol and abs(log_p.iloc[b] - L) < tol, b


def test_more_patterns_than_cached_programs(interpreted):
    bn = examples.asia()
    bn.max_cached_programs = 4
    X = frame(bn, 120, 3, 0.3, latent=["Tuberculosis"])
    assert len(bn._count_patterns(X)) > 3 * bn.max_cached_programs
    got, log_p = bn.mpe_many(X, return_log_proba=True)
    assert len(bn._engine_cache) <= bn.max_cached_programs
    assert list(got.columns) == sorted(bn.nodes) and got.index.equals(X.index) and log_p.index.equals(X.index)
    assert log_p.dtype == np.float64 and not got.isna().any().any()
    assert all(got[c].dtype == bool for c in got.columns)  # inferred, as sample_many
    check_rows(bn, X, got, log_p)
    assert bn.mpe_many(X).equals(got)


def test_alarm_with_missing_cells_and_a_latent_node(interpreted):
    bn = examples.alarm()
    X = frame(bn, 40, 8, 0.3, latent=[bn.nodes[0]])
    got, log_p = bn.mpe_many(X, return_log_proba=True)
    check_rows(bn, X, got, log_p)


def test_all_observed_rows_get_log_p_of_the_row(interpreted):
    bn = examples.asia()
    X = frame(bn, 30, 4, 0.0)
    got, log_p = bn.mpe_many(X, return_log_proba=True)
    dn = oracle_net(bn)
    assert got.equals(X[sorted(X.columns)].infer_objects())
    for b in range(len(X)):
        want = mpe_oracle.log_joint(dn, X.iloc[b].to_dict())
        assert abs(log_p.iloc[b] - want) < 2e-5 * max(1.0, abs(want))


def test_mpe_of_one_event(interpreted):
    bn = examples.asia()
    event = {"Dispnea": True, "Smoker": False}
    got = bn.mpe(event)
    assert isinstance(got, pd.Series) and list(got.index) == sorted(bn.nodes)
    assert got["Dispnea"] == True and got["Smoker"] == False  # noqa: E712
    want, _ = mpe_oracle.max_sum(oracle_net(bn), event)
    assert abs(mpe_oracle.log_joint(oracle_net(bn), got.to_dict()) - mpe_oracle.log_joint(oracle_net(bn), {**event, **want})) < 1e-5


def test_errors_and_an_empty_frame(interpreted):
    bn = examples.sprinkler()
    X = pd.DataFrame({"Rain": [False, True], "Sprinkler": [False, True], "Wet grass": [True, True]})
    with pytest.raises(ValueError, match="probability zero"):
        bn.mpe_many(X)
    with pytest.raises(ValueError, match="not a state"):
        bn.mpe_many(pd.DataFrame({"Rain": ["maybe"]}))
    empty = bn.mpe_many(X.iloc[:0])
    assert empty.shape == (0, len(bn.nodes)) and list(empty.columns) == sorted(bn.nodes)
    got, log_p = bn.mpe_many(X.iloc[:0], return_log_proba=True)
    assert got.shape == (0, len(bn.nodes)) and len(log_p) == 0


def test_the_mpe_pattern_programs_share_the_pattern_cache(monkeypatch):
    class FakeProgram:
        def __init__(self, plan, device=None, f64=False):
            self.plan = plan

        def close(self):
            pass

    monkeypatch.setattr(engine, "Program", FakeProgram)
    bn = examples.asia()
    mpe = bn._pattern_runner("mpe", (0,))
    assert mpe.plan.version == planner.VERSION_MPE and bn._pattern_runner("mpe", (0,)) is mpe
    assert bn._pattern_runner("sample", (0,)) is not mpe and bn._pattern_runner("sample", (0,)).plan.version == planner.VERSION_SAMPLE
