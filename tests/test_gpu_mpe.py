"""The most probable explanation on the device (BayesNet.mpe_many, the max-sum step kernels and
sbn_argmax_step), against the float32 interpreter bit for bit (oracle/program_interp.py) and the float64 oracle
(tests/mpe_oracle.py)."""
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

import mpe_oracle
from conftest import ROOT
from oracle import program_interp, ve_oracle
from sorobn_b200 import engine, examples, planner, workloads
from test_gpu_sample import networks

pytestmark = pytest.mark.gpu

ROWS = [1, 2, 127, 128, 129, 513]
ORACLE_ROWS = 160  # rows per network held to the float64 oracle
TOL = 2e-5  # x max(1, |L*|): a near-tie under float32 rounding


def dense(net):
    """The oracle's DenseNet of a CompiledNet (CPT axes [*parents, v], parents sorted by name in both)."""
    names = net.names
    dn = ve_oracle.DenseNet(nodes=list(names), parents={names[v]: [names[p] for p in net.parents[v]] for v in range(len(names))},
                            domains={names[v]: list(net.domains[v]) for v in range(len(names))})
    for v in range(len(names)):
        dn.cpt[names[v]] = np.asarray(net.cpt[v], dtype=np.float64)
    return dn


def test_codes_and_log_probabilities_equal_the_float32_interpreter_bitwise():
    for name, net, observed, codes in networks():
        plan = planner.build_mpe_plan(net, observed)
        program = engine.Program(plan, device=0)
        for n_rows in ROWS:
            c = np.ascontiguousarray(codes[:, :n_rows])
            got, lp = program.mpe(c, n_rows)
            want, wlp = program_interp.run_mpe(plan.words, plan.table_blob, c, n_rows=n_rows, dtype=np.float32)
            assert np.array_equal(got, want), (name, n_rows)
            assert lp.dtype == np.float32 and np.array_equal(lp.view(np.uint32), wlp.view(np.uint32)), (name, n_rows)
        program.close()


def test_graph_path_and_chunks_equal_the_interpreter():
    """4,096 rows and more replay a captured graph; plain launches and pieces give the same bits."""
    bn = examples.asia()
    net = bn._compiled
    observed = (0, 3, len(net.names) - 1)
    plan = planner.build_mpe_plan(net, observed)
    n = 6000
    codes = np.ascontiguousarray(workloads.forward_sample_codes(net, n, 4)[list(observed)])
    program = engine.Program(plan, device=0)
    got, lp = program.mpe(codes, n)
    want, wlp = program_interp.run_mpe(plan.words, plan.table_blob, codes, dtype=np.float32)
    assert np.array_equal(got, want) and np.array_equal(lp, wlp)
    again = program.mpe(codes, n)
    assert np.array_equal(again[0], got) and np.array_equal(again[1].view(np.uint32), lp.view(np.uint32))
    program.set_graph(False)
    plain = program.mpe(codes, n)
    assert np.array_equal(plain[0], got) and np.array_equal(plain[1], lp)
    program.set_graph(True)
    pieces = [program.mpe(np.ascontiguousarray(codes[:, a:a + 4096]), min(4096, n - a)) for a in range(0, n, 4096)]
    assert np.array_equal(np.concatenate([p[0] for p in pieces], axis=1), got)
    # no evidence at all: one max log P for every row, broadcast from an evidence-independent slot
    free = engine.Program(planner.build_mpe_plan(net, ()), device=0)
    d, l = free.mpe(np.zeros((0, 5000), dtype=np.uint8), 5000)
    wd, wl = program_interp.run_mpe(free.plan.words, free.plan.table_blob, np.zeros((0, 1), dtype=np.uint8), n_rows=1)
    assert (d == wd).all() and (l == wl[0]).all()


def test_explanations_against_the_float64_oracle():
    near_ties = checked = 0
    for name, net, observed, codes in networks():
        plan = planner.build_mpe_plan(net, observed)
        n_rows = min(ORACLE_ROWS, codes.shape[1])
        c = np.ascontiguousarray(codes[:, :n_rows])
        got, lp = engine.Program(plan, device=0).mpe(c, n_rows)
        if name == "grid10x10":  # too wide for the dense oracle: the float64 interpreter is the reference
            d64, l64 = program_interp.run_mpe(plan.words, plan.table_blob64, c, dtype=np.float64)
            assert np.all(np.abs(lp - l64) <= TOL * np.maximum(1.0, np.abs(l64)))
            near_ties += int((got != d64).any(axis=0).sum())
            checked += n_rows
            continue
        dn = dense(net)
        for b in range(n_rows):
            ev = {net.names[v]: net.domains[v][c[i, b]] for i, v in enumerate(observed)}
            x, L = mpe_oracle.max_sum(dn, ev)
            tol = TOL * max(1.0, abs(L))
            assert abs(float(lp[b]) - L) <= tol, (name, b)
            mine = {net.names[v]: net.domains[v][got[j, b]] for j, v in enumerate(plan.sampled)}
            if mine != x:
                assert abs(mpe_oracle.log_joint(dn, {**ev, **mine}) - L) <= tol, (name, b)
                near_ties += 1
            checked += 1
    print(f"\n{near_ties} near-tie(s) of {checked} rows")


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
    return pd.DataFrame(cols)


def runner_up_gap(dn, event):
    """L* minus the second-largest log P(x, e) over the unobserved joint (inf if it has one state)."""
    hidden = [v for v in dn.nodes if v not in event]
    shape = [len(dn.domains[v]) for v in hidden]
    logs = np.zeros(shape)
    for v in dn.nodes:
        scope = dn.scope(v)
        idx = tuple(dn.domains[u].index(event[u]) if u in event else slice(None) for u in scope)
        with np.errstate(divide="ignore"):
            t = np.log(dn.cpt[v][idx])
        free = [u for u in scope if u not in event]
        t = np.transpose(t, np.argsort([hidden.index(u) for u in free])) if free else t
        logs = logs + t.reshape([len(dn.domains[u]) if u in free else 1 for u in hidden])
    flat = np.sort(logs.reshape(-1))
    return np.inf if flat.size < 2 else flat[-1] - flat[-2]


@pytest.mark.parametrize("name", ["asia", "alarm"])
def test_mpe_many_matches_the_oracle_and_impute_many(name):
    bn = getattr(examples, name)()
    bn.device = 0
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    # missing cells and a latent node
    X = frame(bn, 300, 5, 0.3, latent=[bn.nodes[1]])
    got, log_p = bn.mpe_many(X, return_log_proba=True)
    assert list(got.columns) == sorted(bn.nodes) and got.index.equals(X.index)
    for b in range(len(X)):
        ev = {c: X[c].iloc[b] for c in X.columns if pd.notna(X[c].iloc[b])}
        _, L = mpe_oracle.max_sum(dn, ev)
        tol = TOL * max(1.0, abs(L))
        assert abs(mpe_oracle.log_joint(dn, got.iloc[b].to_dict()) - L) <= tol and abs(log_p.iloc[b] - L) <= tol
    # every node a column: where the maximum is unique by more than the tolerance, impute_many fills the same cells
    Y = frame(bn, 300, 6, 0.3)
    filled = bn.impute_many(Y)
    got = bn.mpe_many(Y)
    compared = 0
    for b in range(len(Y)):
        ev = {c: Y[c].iloc[b] for c in Y.columns if pd.notna(Y[c].iloc[b])}
        _, L = mpe_oracle.max_sum(dn, ev)
        if runner_up_gap(dn, ev) > TOL * max(1.0, abs(L)):
            assert all(got[c].iloc[b] == filled[c].iloc[b] for c in Y.columns), b
            compared += 1
    assert compared > 150
    # all observed: log P(row), as predict_log_proba
    Z = frame(bn, 50, 7, 0.0)
    _, lz = bn.mpe_many(Z, return_log_proba=True)
    want = np.asarray(bn.predict_log_proba(Z), dtype=np.float64)
    assert np.all(np.abs(lz.to_numpy() - want) <= TOL * np.maximum(1.0, np.abs(want)))


def test_two_runs_are_bitwise_equal_and_errors_raise():
    wl = workloads.grid10x10()
    bn = wl.build(device=0)
    events = wl.events(2000, seed=3, bn=bn)
    a, la = bn.mpe_many(events, return_log_proba=True)
    b, lb = bn.mpe_many(events, return_log_proba=True)
    assert a.equals(b) and np.array_equal(la.to_numpy(), lb.to_numpy())
    sprinkler = examples.sprinkler()
    sprinkler.device = 0
    with pytest.raises(ValueError, match="probability zero"):
        sprinkler.mpe_many(pd.DataFrame({"Rain": [False], "Sprinkler": [False], "Wet grass": [True]}))
    with pytest.raises(ValueError, match="not a state"):
        sprinkler.mpe_many(pd.DataFrame({"Rain": ["maybe"]}))


def test_the_abi_refuses_other_programs_by_return_code():
    net = examples.asia()._compiled
    lib = engine.load()
    mpe = engine.Program(planner.build_mpe_plan(net, [0]), device=0)
    sample = engine.Program(planner.build_sample_plan(net, [0]), device=0)
    other = engine.Program(planner.build_plan(net, [1], [0]), device=0)
    codes = np.zeros((1, 4), dtype=np.uint8)
    out = np.zeros((7, 4), dtype=np.uint8)
    lp = np.zeros(4, dtype=np.float32)
    for prog in (sample, other):
        assert lib.sbn_program_mpe_host(prog._h, codes.ctypes.data, 4, 4, out.ctypes.data, lp.ctypes.data) != 0
    post = np.zeros((2, 4), dtype=np.float32)
    assert lib.sbn_program_run_host(mpe._h, codes.ctypes.data, 4, 4, post.ctypes.data, 4) != 0
    assert lib.sbn_program_evidence_host(mpe._h, codes.ctypes.data, 4, 4, lp.ctypes.data) != 0
    cnt = np.zeros(16, dtype=np.float64)
    assert lib.sbn_program_counts_host(mpe._h, codes.ctypes.data, 4, 4, cnt.ctypes.data, cnt.size, lp.ctypes.data) != 0
    assert lib.sbn_program_sample_host(mpe._h, codes.ctypes.data, 4, 4, 1, 1, 0, out.ctypes.data, lp.ctypes.data) != 0
    with pytest.raises(engine.EngineError, match="float32 only"):
        engine.Program(mpe.plan, device=0, f64=True)
    decoded, p = mpe.mpe(codes, 4)  # and the program still works
    assert decoded.shape == (7, 4) and np.isfinite(p).all()


def test_kernel_census_shows_only_the_max_sum_kernels():
    """An MPE run launches the max-sum instantiations of the plain batched kernel and the argmax step, and
    nothing else, whatever the program's switches."""
    script = f"""
import sys
sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]
from kernel_census import census
from sorobn_b200 import engine, planner, workloads
wl = workloads.grid10x10()
net = wl.build()._compiled
observed = tuple(sorted(net.index[e] for e in wl.evidence))
plan = planner.build_mpe_plan(net, observed)
codes = workloads.forward_sample_codes(net, 1000, 1)[list(observed)]
p = engine.Program(plan, device=0)
for mode in (1, 7, 9, 11):
    p.set_tiled(mode)
class Run:
    def run(self, c, n):
        p.mpe(c, n)
    def set_graph(self, g):
        p.set_graph(g)
print(sorted({{name for name, _ in census(Run(), codes, 1000)}}))
"""
    out = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, check=True).stdout
    names = eval(out.strip().splitlines()[-1])
    assert "sbn_argmax_step" in names and any(n.startswith("sbn_step_batched<") for n in names), names
    assert all(n == "sbn_argmax_step" or (n.startswith("sbn_step_batched<") and n.endswith(", SbnMaxSum>")) for n in names), names
