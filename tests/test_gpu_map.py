"""Marginal MAP on the device (BayesNet.map_many, the log-sum-exp and max-sum step kernels and sbn_argmax_step),
against the float32 replay of the words (oracle/program_interp.py) and the float64 oracle (tests/map_oracle.py)."""
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

import map_oracle
from conftest import ROOT
from oracle import program_interp, ve_oracle
from sorobn_b200 import engine, examples, planner, workloads
from test_gpu_sample import networks

pytestmark = pytest.mark.gpu

ROWS = [1, 2, 127, 128, 129, 513]
RTOL = 4e-6  # device against the float32 replay: x max(1, |r|) (expf / logf differ from numpy's in the last bits)
TOL = 2e-5  # against the float64 oracle: a near-tie under float32 rounding


def dense(net):
    names = net.names
    dn = ve_oracle.DenseNet(nodes=list(names), parents={names[v]: [names[p] for p in net.parents[v]] for v in range(len(names))},
                            domains={names[v]: list(net.domains[v]) for v in range(len(names))})
    for v in range(len(names)):
        dn.cpt[names[v]] = np.asarray(net.cpt[v], dtype=np.float64)
    return dn


def map_sets(net, observed, seed):
    """MAP sets of one, two and four unobserved variables (their joint small enough for the dense oracle)."""
    rng = np.random.default_rng(seed)
    free = [v for v in range(len(net.names)) if v not in observed]
    out = []
    for k in (1, 2, 4):
        if k <= len(free):
            m = tuple(sorted(rng.choice(free, size=k, replace=False).tolist()))
            if int(np.prod([int(net.card[v]) for v in m])) <= 4096:
                out.append(m)
    return out


def test_log_values_match_the_replay_and_decisions_the_oracle():
    """Entry-wise |device - replay| <= 4e-6 max(1, |replay|) on every row's log-probability.  Where the device
    decodes another state than the replay, the oracle shows a near-tie: that state's log P is L* too."""
    differ = checked = 0
    for name, net, observed, codes in networks():
        dn = dense(net) if name != "grid10x10" else None
        for m in map_sets(net, observed, 1):
            plan = planner.build_map_plan(net, observed, m)
            program = engine.Program(plan, device=0)
            for n_rows in ROWS:
                c = np.ascontiguousarray(codes[:, :n_rows])
                got, lp = program.map(c, n_rows)
                want, wlp = program_interp.run_mpe(plan.words, plan.table_blob, c, n_rows=n_rows, dtype=np.float32)
                assert lp.dtype == np.float32 and got.shape == want.shape
                fin = np.isfinite(wlp)
                assert np.array_equal(np.isfinite(lp), fin), (name, m, n_rows)
                assert np.all(np.abs(lp[fin].astype(np.float64) - wlp[fin]) <= RTOL * np.maximum(1.0, np.abs(wlp[fin]))), (name, m)
                rows = np.flatnonzero((got != want).any(axis=0))
                differ += len(rows)
                checked += n_rows
                if dn is None:  # too wide for the oracle: a differing decision is a rare near-tie
                    assert len(rows) <= max(1, n_rows // 100), (name, m, n_rows, len(rows))
                for b in rows if dn is not None else ():
                    ev = {net.names[v]: net.domains[v][c[i, b]] for i, v in enumerate(observed)}
                    mine = {net.names[v]: net.domains[v][got[j, b]] for j, v in enumerate(plan.sampled)}
                    _, L, gap = map_oracle.solve(dn, ev, [net.names[v] for v in plan.sampled])
                    t = TOL * max(1.0, abs(L))
                    assert gap <= t and abs(map_oracle.log_prob(dn, ev, mine) - L) <= t, (name, m, b)
            program.close()
    print(f"\n{differ} row(s) of {checked} decode a near-tie differently from the replay")


def test_the_impute_goldens_are_reproduced():
    import json

    for name in ("alarm", "asia", "sprinkler", "grades"):
        with open(os.path.join(ROOT, "tests", "golden", f"impute_{name}.json")) as f:
            cases = json.load(f)["cases"]
        bn = getattr(examples, name)()
        bn.device = 0
        dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
        X = pd.DataFrame([dict(c["sample"]) for c in cases])
        got, log_p = bn.map_many(X, return_log_proba=True)
        compared = 0
        for b, case in enumerate(cases):
            sample, filled = dict(case["sample"]), dict(case["filled"])
            ev = {k: v for k, v in sample.items() if v is not None}
            missing = [k for k, v in sample.items() if v is None]
            x, L, gap = map_oracle.brute_force(dn, ev, missing)
            t = TOL * max(1.0, abs(L))
            assert abs(log_p.iloc[b] - L) <= t
            mine = {k: got[k].iloc[b] for k in missing}
            if gap > t:
                assert mine == {k: filled[k] for k in missing}, (name, b)
                compared += 1
            else:
                assert abs(map_oracle.log_prob(dn, ev, mine) - L) <= t
        assert compared > 0


def missing_frame(net, n, seed, k_missing, n_patterns=None):
    """n forward samples with exactly `k_missing` random cells blanked per row (every node a column), drawn from
    `n_patterns` missingness patterns (None: every row its own)."""
    codes = workloads.forward_sample_codes(net, n, seed)
    rng = np.random.default_rng(seed + 1)
    cols = {name: np.asarray(net.domains[v], dtype=object)[codes[v]] for v, name in enumerate(net.names)}
    X = pd.DataFrame(cols)
    blank = np.argsort(rng.random((n if n_patterns is None else n_patterns, len(net.names))), axis=1)[:, :k_missing]
    if n_patterns is not None:
        blank = blank[rng.integers(0, n_patterns, size=n)]
    mask = np.zeros((n, len(net.names)), dtype=bool)
    np.put_along_axis(mask, blank, True, axis=1)
    return X.mask(pd.DataFrame(mask, columns=X.columns))


@pytest.mark.parametrize("k_missing", [1, 2, 3, 4])
def test_map_many_agrees_with_impute_many_on_alarm(k_missing):
    bn = examples.alarm()
    bn.device = 0
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    X = missing_frame(bn._compiled, 400, 10 + k_missing, k_missing)
    got, log_p = bn.map_many(X, return_log_proba=True)
    filled = bn.impute_many(X)
    assert list(got.columns) == sorted(X.columns) and got.index.equals(X.index) and not got.isna().any().any()
    compared = 0
    for b in range(len(X)):
        ev = {c: X[c].iloc[b] for c in X.columns if pd.notna(X[c].iloc[b])}
        missing = [c for c in X.columns if c not in ev]
        _, L, gap = map_oracle.brute_force(dn, ev, missing)
        t = TOL * max(1.0, abs(L))
        assert abs(log_p.iloc[b] - L) <= t
        if gap > t:
            assert all(got[c].iloc[b] == filled[c].iloc[b] for c in missing), b
            compared += 1
    assert compared > len(X) // 2


def test_twelve_or_more_missing_cells_per_row():
    """Past what impute_many can hold: 14 or more missing cells of the benchmark grid (at least 2 states each)
    are 16,384 or more joint states per row, 5^14 = 6.1e9 at 5 states.  Ten nodes have no column and are summed
    out.  Against the float64 replay of the same words."""
    wl = workloads.grid10x10()
    bn = wl.build(device=0)
    net = bn._compiled
    latent = [net.names[v] for v in range(5, len(net.names), 10)]
    X = missing_frame(net, 3000, 21, 24, n_patterns=6).drop(columns=latent)
    assert (X.isna().sum(axis=1) >= 14).all()
    got, log_p = bn.map_many(X, return_log_proba=True)
    assert not got.isna().any().any() and np.isfinite(log_p.to_numpy()).all()
    groups = bn._count_patterns(X)
    assert len(groups) == 6
    for ev, rows, codes in groups:
        m = tuple(sorted(net.index[c] for c in X.columns if net.index[c] not in ev))
        plan = planner.build_map_plan(net, ev, m)
        d64, l64 = program_interp.run_mpe(plan.words, plan.table_blob64, codes, n_rows=len(rows), dtype=np.float64)
        assert np.all(np.abs(log_p.to_numpy()[rows] - l64) <= TOL * np.maximum(1.0, np.abs(l64)))


def test_two_runs_are_bitwise_equal():
    wl = workloads.grid10x10()
    bn = wl.build(device=0)
    events = wl.events(2000, seed=3, bn=bn)
    variables = [n for n in bn.nodes if n not in events.columns][::7]
    a, la = bn.map_many(events, variables=variables, return_log_proba=True)
    b, lb = bn.map_many(events, variables=variables, return_log_proba=True)
    assert a.equals(b) and np.array_equal(la.to_numpy().view(np.uint64), lb.to_numpy().view(np.uint64))


@pytest.mark.parametrize("n", [4095, 4096, 4097, 150_000])
def test_row_counts_around_the_graph_threshold_and_large_batches(n):
    """Below 4,096 rows a chunk runs as plain launches, from 4,096 on it replays a captured graph; a large batch
    equals its pieces of 4,096 rows."""
    net = examples.asia()._compiled
    observed = (0, 3, len(net.names) - 1)
    m = (1, 4)
    plan = planner.build_map_plan(net, observed, m)
    codes = np.ascontiguousarray(workloads.forward_sample_codes(net, n, 4)[list(observed)])
    program = engine.Program(plan, device=0)
    got, lp = program.map(codes, n)
    if n < 10_000:
        want, wlp = program_interp.run_mpe(plan.words, plan.table_blob, codes, dtype=np.float32)
        assert np.array_equal(got, want)
        assert np.all(np.abs(lp - wlp) <= RTOL * np.maximum(1.0, np.abs(wlp)))
    pieces = [program.map(np.ascontiguousarray(codes[:, a:a + 4096]), min(4096, n - a)) for a in range(0, n, 4096)]
    assert np.array_equal(np.concatenate([p[0] for p in pieces], axis=1), got)
    assert np.array_equal(np.concatenate([p[1] for p in pieces]), lp)
    program.set_graph(False)
    plain = program.map(codes, n)
    assert np.array_equal(plain[0], got) and np.array_equal(plain[1], lp)
    program.close()


def test_map_agrees_with_map_many_and_errors_raise():
    bn = examples.asia()
    bn.device = 0
    X = pd.DataFrame([{"Dispnea": True, "Smoker": None, "Lung cancer": None},
                      {"Dispnea": False, "Smoker": True, "Lung cancer": None}])
    many = bn.map_many(X)
    for b in range(len(X)):
        one = bn.map({k: (None if pd.isna(v) else v) for k, v in X.iloc[b].items()})
        assert one.to_dict() == many.iloc[b].to_dict()
    with_vars = bn.map_many(X, variables=["Tuberculosis"])
    assert bn.map({"Dispnea": True}, variables=["Tuberculosis"])["Tuberculosis"] == with_vars["Tuberculosis"].iloc[0]
    sprinkler = examples.sprinkler()
    sprinkler.device = 0
    with pytest.raises(ValueError, match="probability zero"):
        sprinkler.map_many(pd.DataFrame({"Rain": [False], "Sprinkler": [False], "Wet grass": [True], "Cloudy": [None]}))
    with pytest.raises(ValueError, match="not a state"):
        sprinkler.map_many(pd.DataFrame({"Rain": ["maybe"]}))
    map_prog = engine.Program(planner.build_map_plan(bn._compiled, [0], [1]), device=0)
    with pytest.raises(engine.EngineError, match="float32 only"):
        engine.Program(map_prog.plan, device=0, f64=True)
    lib = engine.load()
    codes = np.zeros((1, 4), dtype=np.uint8)
    post = np.zeros((2, 4), dtype=np.float32)
    assert lib.sbn_program_run_host(map_prog._h, codes.ctypes.data, 4, 4, post.ctypes.data, 4) != 0
    out = np.zeros((1, 4), dtype=np.uint8)
    lp = np.zeros(4, dtype=np.float32)
    assert lib.sbn_program_sample_host(map_prog._h, codes.ctypes.data, 4, 4, 1, 1, 0, out.ctypes.data, lp.ctypes.data) != 0
    decoded, p = map_prog.map(codes, 4)  # and the program still works
    assert decoded.shape == (1, 4) and np.isfinite(p).all()
    map_prog.close()


def test_kernel_census_shows_both_log_sum_exp_instantiations():
    """A marginal MAP run launches the log-sum-exp and max-sum instantiations of the plain batched kernel, the
    log-sum-exp flat kernel (at program creation) and the argmax step, and nothing else."""
    script = f"""
import sys
sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]
from kernel_census import census
from sorobn_b200 import engine, planner, workloads
wl = workloads.grid10x10()
net = wl.build()._compiled
observed = tuple(sorted(net.index[e] for e in wl.evidence))
hidden = [v for v in range(len(net.names)) if v not in observed]
plan = planner.build_map_plan(net, observed, hidden[::9])
lse = {{st.kind for st in plan.steps if st.kind in (0, 1) and st.reduce == planner.REDUCE_LOGSUMEXP}}
assert lse == {{0, 1}}, lse
codes = workloads.forward_sample_codes(net, 1000, 1)[list(observed)]
class Run:
    # the program is created inside the profiled run: its evidence-independent steps run at creation
    def run(self, c, n):
        p = engine.Program(plan, device=0)
        for mode in (1, 7, 9, 11):
            p.set_tiled(mode)
        p.set_graph(False)
        p.map(c, n)
        p.close()
    def set_graph(self, g):
        pass
print(sorted({{name for name, _ in census(Run(), codes, 1000)}}))
"""
    out = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, check=True).stdout
    names = eval(out.strip().splitlines()[-1])
    assert "sbn_argmax_step" in names, names
    assert "sbn_step_flat<float, SbnLogSumExp>" in names, names
    assert any(n.startswith("sbn_step_batched<") and n.endswith(", SbnLogSumExp>") for n in names), names
    allowed = ("sbn_argmax_step",)
    for n in names:
        assert n in allowed or n.endswith(", SbnLogSumExp>") or n.endswith(", SbnMaxSum>"), names
