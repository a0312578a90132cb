"""The expanding product contracted by its consumer (`sbn_contract_kernel`, pair kind 2 of `csrc/sbn_pair.cu`).

Step 1 multiplies two batched factors and sums out one variable (an expanding product, no tables); step 2
multiplies its output M with one more batched factor C and sums out one or more variables.  The pair runs as
one launch and M never reaches memory.  Hand-built programs (tests/pair_programs.py `build`) cover the
benchmark grid's shape (M x C rounded, then summed), 4-state variables, a step 2 that keeps two axes of M (M and
C on different sides of the consumer's tile: one fused fma), and a C that carries an output variable M lacks, in
both axis orders.  Per case and row count: the output equals the program with one launch per step bit for
bit, 128-row pieces equal the whole batch bit for bit, the roles are 2 / 3, the census shows the kernel, and
sampled rows match the float64 interpreter.  Two refusals (a table, an evidence gather in step 2) stay two
launches.  On the benchmark grid at 100,007 rows the pair is steps 63 / 64 and launches once.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import pair_programs as pp
from oracle import program_interp
from test_gpu_kernel_variants import check_row

pytestmark = pytest.mark.gpu

RTOL = 1e-6
ROW_COUNTS = (1, 31, 257, 5003)
KERNEL = "sbn_contract_kernel"
GRID_ROWS = 100_007


def _case(name, a, b, c, mid, elim, out, card=None, c_table=None, roles=(1, 1, 1, 2, 3)):
    """A (over `a` and e0, e0 = 1 impossible), B (over `b` and e1), C (over `c` and e0) per row; then
    step 1: M[mid] = sum_j A B, step 2: O[out] = sum_elim M C.  `c_table`: step 2 multiplies M with this
    table (name -> spec) instead of the batched C."""
    card = {**dict(a=5, b=5, c=5, j=5, z=5, w=5, e0=3, e1=4), **(card or {})}
    tables = {"SA": (f"{a} e0", {}, {"e0": 1}), "SB": f"{b} e1", "SC": f"{c} e0"}
    steps = [(1, "A", "SA", "", a), (1, "B", "SB", "", b), (1, "C", "SC", "", c)]
    second = "C"
    if c_table is not None:
        tables = {"SA": tables["SA"], "SB": tables["SB"], "TC": c_table}
        steps, second = steps[:2], "TC"
    steps += [(1, "M", "A B", "j", mid), (1, "O", f"M {second}", elim, out)]
    used = {v for t in tables.values() for v in (t if isinstance(t, str) else t[0]).split()}
    return dict(name=name, card={k: v for k, v in card.items() if k in used}, ev=["e0", "e1"], tables=tables, steps=steps,
                slots={}, roles=list(roles))


CASES = [
    _case("grid_shape", "a j b", "c z j", "a b c", "a c b z", "a b c", "z"),
    _case("card4", "a j b", "c z j", "a b c", "a c b z", "a b c", "z", card=dict(a=4, b=4, c=4, j=4, z=4)),
    _case("keeps_two_axes", "a j b", "c z j w", "a b c", "a c b z w", "a b c", "z w", card=dict(w=2)),
    _case("c_carries_w", "a j b", "c z j", "a b w", "a c b z", "a b c", "z w", card=dict(w=3)),
    _case("c_carries_w_first", "a j b", "c z j", "a b w", "a c b z", "a b c", "w z", card=dict(w=3)),
]
REFUSED = [
    _case("refuse_table", "a j b", "c z j", "a b c", "a c b z", "a b c", "z", c_table="a b c", roles=(1, 1, 1, 1)),
    _case("refuse_evidence_gather", "a j b", "c z j", "a b c", "a c b z", "a b c", "z", c_table="a b c e1",
          roles=(1, 1, 1, 1)),
]


_CENSUS_SCRIPT = f"""
import json, os, sys, tempfile
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile
import pair_programs as pp
import test_gpu_contract_pair as T
from sorobn_b200 import engine, planner, workloads

out = {{}}
runs = []
for case in T.CASES + T.REFUSED:
    built = pp.build(case)
    runs.append((case["name"], engine.Program(built.plan), pp.evidence_rows(built, 257, seed=1), 257))
wl = workloads.grid10x10()
bn = wl.build()
net = bn._compiled
plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
runs.append(("grid", engine.Program(plan), wl.codes(bn, {GRID_ROWS}, seed=5), {GRID_ROWS}))
for _, prog, codes, n in runs:
    prog.set_graph(False)
    prog.run(codes, n)
torch.cuda.synchronize()
for name, prog, codes, n in runs:
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        prog.run(codes, n)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    out[name] = sum(1 for ev in trace.get("traceEvents", []) if ev.get("cat") == "kernel" and "{KERNEL}" in ev.get("name", ""))
json.dump(out, sys.stdout)
"""


@pytest.fixture(scope="module")
def launches():
    """Launches of the contraction kernel in one run of each case (257 rows) and of the grid, in a fresh
    interpreter."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, "-c", _CENSUS_SCRIPT], capture_output=True, text=True, env=env, cwd=here,
                         timeout=1800)
    assert res.returncode == 0, res.stderr[-3000:]
    return json.loads(res.stdout)


def _interp(built, codes, cols):
    uniq, inv = pp.unique_rows(np.ascontiguousarray(codes[:, cols]))
    want = program_interp.run(built.plan.words, built.plan.table_blob64, uniq, n_rows=uniq.shape[1])
    return want[:, inv]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_contract_pair_matches_the_single_launches(case, launches):
    from sorobn_b200 import engine

    built = pp.build(case)
    prog, pieces = engine.Program(built.plan), engine.Program(built.plan)
    assert prog.step_roles().tolist() == case["roles"]
    assert prog.info()["pairs"] == 1
    assert launches[case["name"]] == 1
    codes = pp.evidence_rows(built, max(ROW_COUNTS), seed=1)
    for n in ROW_COUNTS:
        sub = np.ascontiguousarray(codes[:, :n])
        out = prog.run(sub, n).copy()
        prog.set_tiled(10)
        single = prog.run(sub, n).copy()
        prog.set_tiled(11)
        assert np.array_equal(out, single, equal_nan=True), n
        got = [pieces.run(np.ascontiguousarray(sub[:, lo:lo + 128]), min(128, n - lo)) for lo in range(0, n, 128)]
        assert np.array_equal(np.concatenate(got, axis=1), out, equal_nan=True), n
        cols = np.unique(np.linspace(0, n - 1, min(n, 48)).astype(np.int64))
        want = _interp(built, sub, cols)
        for k, b in enumerate(cols):
            check_row(out[:, b], want[:, k], RTOL)
    prog.close()
    pieces.close()


@pytest.mark.parametrize("case", REFUSED, ids=lambda c: c["name"])
def test_contract_pair_refusals_stay_two_launches(case, launches):
    from sorobn_b200 import engine

    built = pp.build(case)
    prog = engine.Program(built.plan)
    assert prog.step_roles().tolist() == case["roles"]
    assert prog.info()["pairs"] == 0
    assert launches[case["name"]] == 0
    codes = pp.evidence_rows(built, 257, seed=1)
    out = prog.run(codes, 257)
    want = _interp(built, codes, np.arange(257))
    for b in range(257):
        check_row(out[:, b], want[:, b], RTOL)
    prog.close()


def test_contract_pair_on_the_benchmark_grid(launches):
    from oracle import ve_oracle
    from sorobn_b200 import engine, planner, workloads

    wl = workloads.grid10x10()
    bn = wl.build()
    net = bn._compiled
    plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
    prog = engine.Program(plan)
    roles = prog.step_roles()
    assert roles[63] == 2 and roles[64] == 3, roles
    # every other pair as before: one expanding product fused with its consumer, paired frontier steps
    assert (roles == 4).sum() == (roles == 5).sum() == 1
    assert (roles == 2).sum() == (roles == 3).sum() == prog.info()["pairs"] - 1
    assert launches["grid"] == 1
    codes = wl.codes(bn, GRID_ROWS, seed=5)
    out = prog.run(codes, GRID_ROWS)
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    order = [net.names[v] for v in plan.order]
    for b in (0, 1, GRID_ROWS // 3, GRID_ROWS // 2, GRID_ROWS - 2, GRID_ROWS - 1):
        ev = {v: net.domains[net.index[v]][codes[i, b]] for i, v in enumerate(wl.evidence)}
        want = ve_oracle.query(dn, *wl.query, event=ev, order=order)[1].reshape(-1)
        check_row(out[:, b], want, RTOL)
    prog.close()
