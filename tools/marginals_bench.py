"""Marginals of every unobserved variable: one marginals program against one program per variable.

Workload: the benchmark grid (10x10, 5 states, 30 observed nodes), forward-sampled rows.  Both
sides run on resident evidence codes (device pointers, `Program.run_device`): the single marginals
program (planner.build_marginals_plan) and the 70 per-variable programs (planner.build_plan) run
back to back on the same rows.  After warm-up the two are timed alternately with CUDA events,
several repetitions; the median is reported with the algorithmic bytes per row of both plans and
the achieved GB/s.  The two answers are checked to agree to 1e-6 on every row.

    python tools/marginals_bench.py [--rows 100000] [--reps 7] [--out results/marginals_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_limits():
    try:
        res = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30)
        return res.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--group", type=int, default=10, help="per-variable programs alive at once")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from sorobn_b200 import engine, planner, workloads

    wl = workloads.grid10x10()
    bn = wl.build(device=0)
    net = bn._compiled
    ev_ids = [net.index[e] for e in wl.evidence]
    n = args.rows
    codes = wl.codes(bn, n, seed=1)

    mplan = planner.build_marginals_plan(net, ev_ids)
    mprog = engine.Program(mplan, device=0)
    qplans = [planner.build_plan(net, [t], ev_ids) for t in mplan.targets]

    dev = torch.device("cuda:0")
    d_ev = torch.from_numpy(np.ascontiguousarray(codes)).to(dev)
    d_m = torch.empty((mplan.Q, n), dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream(dev)
    sp = stream.cuda_stream

    def timed(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        return a.elapsed_time(b)

    def run_marginals():
        mprog.run_device(d_ev.data_ptr(), n, n, d_m.data_ptr(), n, sp)

    # Each per-variable program owns scratch for its batch (about 4 GB at 100k grid rows), so the 70 do
    # not fit the device at once: they are timed in groups that do, each group alternating with the
    # marginals program; the per-variable time is the sum of the groups' medians.
    tm, tq_groups, worst = [], [], 0.0
    for _ in range(args.warmup):
        run_marginals()
    for g0 in range(0, len(qplans), args.group):
        plans = qplans[g0:g0 + args.group]
        progs = [engine.Program(p, device=0) for p in plans]
        outs = [torch.empty((p.Q, n), dtype=torch.float32, device=dev) for p in plans]

        def run_group():
            for prog, out in zip(progs, outs):
                prog.run_device(d_ev.data_ptr(), n, n, out.data_ptr(), n, sp)

        for _ in range(args.warmup):
            run_group()
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            tm.append(timed(run_marginals))
            times.append(timed(run_group))
        tq_groups.append(times)
        got = d_m[5 * g0:5 * (g0 + len(plans))].double()
        want = torch.cat(outs).double()
        assert bool(torch.isfinite(got).all())
        worst = max(worst, float((got - want).abs().max()))  # posteriors: absolute difference
        for prog in progs:
            prog.close()
        del outs
    assert worst < 1e-6, worst
    tq = [float(x) for x in np.sum(np.array(tq_groups), axis=0)]
    ms_m = float(np.median(tm))
    ms_q = float(np.sum([np.median(t) for t in tq_groups]))

    bpr_m = mplan.bytes_per_row()
    bpr_q = sum(p.bytes_per_row() for p in qplans)
    result = {
        "workload": "grid10x10, 5 states, 30 observed, 70 targets",
        "rows": n,
        "gpu (name, power limit, max SM clock)": gpu_limits(),
        "marginals_ms_median": round(ms_m, 3),
        "per_variable_ms_median": round(ms_q, 3),
        "speedup": round(ms_q / ms_m, 2),
        "marginals_ms_all": [round(t, 3) for t in tm],
        "per_variable_ms_all": [round(t, 3) for t in tq],
        "marginals_bytes_per_row": bpr_m,
        "per_variable_bytes_per_row": bpr_q,
        "marginals_GBps": round(bpr_m * n / (ms_m * 1e-3) / 1e9, 1),
        "per_variable_GBps": round(bpr_q * n / (ms_q * 1e-3) / 1e9, 1),
        "launches_marginals": sum(1 for st in mplan.steps if st.kind != planner.KIND_FLAT),
        "launches_per_variable": sum(sum(1 for st in p.steps if st.kind != planner.KIND_FLAT) + 1 for p in qplans),
        "max_err_vs_per_variable": worst,
    }
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
