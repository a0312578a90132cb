"""The row-block expanding product (csrc/sbn_triple_rows.cu) on batches large enough to take it.

It replaces `sbn_triple_kernel` for the fused expanding product + contraction only when the batch has at
least 2 x SMs blocks of 16 rows and each operand's share of one row's combinations is one box (one digit of at
most one axis beside p and the two loop axes, 8 to 25 combinations).  Small batches, such as the 2048-row pieces
below, stay on `sbn_triple_kernel`.  Here: the kernel must run where it is claimed and nowhere else, its output
must be bitwise equal to the same batch run in pieces (the two kernels do the same fp32 operations in the same
order), the step roles and program info must not depend on the batch, and a sample of rows must match the
float64 oracle.  Every row count is ragged (not a multiple of 16).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import kernel_census
import pair_programs as pp
from oracle import program_interp, ve_oracle
from test_gpu_kernel_variants import check_row

pytestmark = pytest.mark.gpu

RTOL = 1e-6
PIECE = 2048  # 128 row blocks: below the threshold on any GPU with at least 64 SMs
GRID_ROWS = 100_007
ROWS_KERNEL = "sbn_triple_rows_kernel"
TRIPLE_KERNEL = "sbn_triple_kernel"
# the TRIPLE_CASES whose combinations of untouched axes the row-block kernel covers (15 and 12 of them); the others
# have fewer than 8 combinations, or more than 25 with two untouched axes in A
COVERED = {"triple_g5_r1", "triple_g1_r2"}


def _grid():
    from sorobn_b200 import planner, workloads

    wl = workloads.grid10x10()
    bn = wl.build()
    net = bn._compiled
    plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
    return wl, bn, net, plan


def _row_counts(n_sms):
    """Ragged counts just above the threshold and with several row blocks per CTA."""
    return (2 * n_sms * 16 + 5, 20_011)


def _census_main():
    """Run in a fresh interpreter (after many profiler sessions in one process the profiler stops recording):
    prints {"<program>:<rows>": [expanding-product kernel names]} for every run the tests below make."""
    import torch

    from sorobn_b200 import engine

    runs, keys = [], []
    wl, bn, _, plan = _grid()
    codes = wl.codes(bn, GRID_ROWS, seed=13)
    for n in (GRID_ROWS, PIECE):
        runs.append((engine.Program(plan), np.ascontiguousarray(codes[:, :n]), n))
        keys.append(f"grid:{n}")
    for n in _row_counts(torch.cuda.get_device_properties(0).multi_processor_count):
        for case in pp.TRIPLE_CASES:
            built = pp.build(case)
            codes = pp.evidence_rows(built, n, seed=3)
            for m in (n, PIECE):
                runs.append((engine.Program(built.plan), np.ascontiguousarray(codes[:, :m]), m))
                keys.append(f"{case['name']}:{m}")
    seen = kernel_census.census_many(runs)
    json.dump({k: [name.split("<")[0] for name, _ in s if name.startswith((ROWS_KERNEL, TRIPLE_KERNEL))]
               for k, s in zip(keys, seen)}, sys.stdout)


@pytest.fixture(scope="module")
def census():
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, "-c", "import test_gpu_triple_rows as t; t._census_main()"], capture_output=True,
                         text=True, env=env, cwd=here, timeout=1800)
    assert res.returncode == 0, res.stderr[-3000:]
    return json.loads(res.stdout)


def same_shape_info(a, b):
    keep = lambda d: {k: v for k, v in d.items() if k not in ("reserved_rows", "launches")}  # noqa: E731
    return keep(a.info()) == keep(b.info())


def run_pieces(program, codes, n):
    return np.concatenate([program.run(np.ascontiguousarray(codes[:, lo:lo + PIECE]), min(PIECE, n - lo))
                           for lo in range(0, n, PIECE)], axis=1)


def test_triple_rows_full_size_grid(census):
    """The benchmark grid (10x10, 5 states) at 100,007 rows: steps 34 + 35 (`3125 <- B625 x B625`, then
    `625 <- sum_25 B625 x B3125`) run as one row-block launch, 25 combinations per row."""
    from sorobn_b200 import engine

    wl, bn, net, plan = _grid()
    n = GRID_ROWS
    codes = wl.codes(bn, n, seed=13)
    assert census[f"grid:{n}"] == [ROWS_KERNEL]
    assert census[f"grid:{PIECE}"] == [TRIPLE_KERNEL]
    big = engine.Program(plan)
    out = big.run(codes, n)
    small = engine.Program(plan)
    assert np.array_equal(run_pieces(small, codes, n), out)
    assert big.step_roles().tolist() == small.step_roles().tolist()
    assert ((big.step_roles() == 4).sum(), (big.step_roles() == 5).sum()) == (1, 1)
    assert same_shape_info(big, small)

    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    order = [net.names[v] for v in plan.order]
    worst = 0.0
    for b in list(range(0, n, n // 12)) + [n - 1]:
        ev = {v: int(net.domains[net.index[v]][codes[i, b]]) for i, v in enumerate(wl.evidence)}
        want = ve_oracle.query(dn, *wl.query, event=ev, order=order)[1].reshape(-1)
        pos = want > 0
        assert (out[~pos, b] == 0).all()
        worst = max(worst, float(np.max(np.abs(out[pos, b] - want[pos]) / want[pos])))
    assert worst < RTOL, worst


@pytest.mark.parametrize("case", pp.TRIPLE_CASES, ids=pp.case_id)
def test_triple_rows_hand_built_programs(case, census):
    """Each hand-built triple program just above the threshold (and with several row blocks per CTA): the cases
    the row-block kernel covers take it and match their pieces bitwise and the float64 interpreter; the others
    stay on sbn_triple_kernel."""
    import torch

    from sorobn_b200 import engine

    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    built = pp.build(case)
    plan = built.plan
    big = engine.Program(plan)
    small = engine.Program(plan)
    for n in _row_counts(n_sms):
        codes = pp.evidence_rows(built, n, seed=3)
        want_kernel = ROWS_KERNEL if case["name"] in COVERED else TRIPLE_KERNEL
        assert census[f"{case['name']}:{n}"] == [want_kernel], case["branch"]
        assert census[f"{case['name']}:{PIECE}"] == [TRIPLE_KERNEL]
        out = big.run(codes, n).copy()
        assert np.array_equal(run_pieces(small, codes, n), out, equal_nan=True), n
        assert big.step_roles().tolist() == small.step_roles().tolist() == case["roles"]
        assert same_shape_info(big, small)
        uniq, inv = pp.unique_rows(codes)
        want = program_interp.run(plan.words, plan.table_blob64, uniq, n_rows=uniq.shape[1])
        for k in range(uniq.shape[1]):
            b = int(np.flatnonzero(inv == k)[-1])
            check_row(out[:, b], want[:, k], RTOL)
    big.close()
    small.close()
