"""Time the most probable explanation on the benchmark grid (10x10, 5 states): 100k forward-sampled rows
with the grid's evidence columns observed and the other 70 variables decoded.

One call = one `Program.mpe` of the whole batch on the MPE program (codes in, max-sum upward pass on the
plain batched kernel, argmax steps, decoded codes and max log P(x, e) out, synchronised).  The sample
program of the same evidence columns at n = 1 (`Program.sample`) is timed alternately with it, in the
same process, as the yardstick: both run an upward pass of the same shape, the sample program's on the
tuned sum-product kernels.  Medians of several rounds, their spread (min .. max) and rows per second are
printed with the card's name and power limit.

A second part times `BayesNet.mpe_many` end to end (grouping, one device call per missingness pattern,
the result frame) on Alarm with 30 % of the cells missing.

    python tools/mpe_bench.py [--rounds 7] [--rows 100000] [--alarm-rows 100000] [--out results/mpe_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_limits():
    try:
        res = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30)
        return res.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def spread(ts):
    ms = [t * 1e3 for t in ts]
    return f"{np.median(ms):.2f} ms (min {min(ms):.2f}, max {max(ms):.2f})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--alarm-rows", type=int, default=100_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from sorobn_b200 import engine, planner, workloads

    results = {"gpu": gpu_limits(), "rows": args.rows}
    print("gpu:", results["gpu"], flush=True)
    wl = workloads.grid10x10()
    bn = wl.build(device=0)
    net = bn._compiled
    observed = [net.index[e] for e in wl.evidence]
    n = args.rows
    codes = np.ascontiguousarray(wl.codes(bn, n, seed=1)[np.argsort(observed)])
    mplan = planner.build_mpe_plan(net, sorted(observed))
    splan = planner.build_sample_plan(net, sorted(observed))
    mprog, sprog = engine.Program(mplan, device=0), engine.Program(splan, device=0)
    for _ in range(2):  # warm-up: reservation, graph capture
        mprog.mpe(codes, n)
        sprog.sample(codes, n, 1, seed=1)
    tm, ts = [], []
    for r in range(args.rounds):
        tm.append(timed(lambda: mprog.mpe(codes, n)))
        ts.append(timed(lambda: sprog.sample(codes, n, 1, seed=r)))
    m, s = float(np.median(tm)), float(np.median(ts))
    results["grid"] = dict(mpe_ms=m * 1e3, mpe_ms_all=[t * 1e3 for t in tm], sample_ms=s * 1e3,
                           sample_ms_all=[t * 1e3 for t in ts], mpe_rows_per_s=n / m, sample_rows_per_s=n / s,
                           decoded=len(mplan.sampled), bytes_per_row=mplan.bytes_per_row())
    print(f"grid, {n} rows, {len(mplan.sampled)} variables decoded ({mplan.bytes_per_row()} algorithmic B/row):\n"
          f"  mpe            {spread(tm)} per call, {n / m / 1e6:.2f} M rows/s\n"
          f"  sample (n = 1) {spread(ts)} per call, {n / s / 1e6:.2f} M rows/s", flush=True)

    import pandas as pd

    from sorobn_b200 import examples

    alarm = examples.alarm(device=0)
    anet = alarm._compiled
    k = args.alarm_rows
    acodes = workloads.forward_sample_codes(anet, k, 3)
    X = pd.DataFrame({name: np.asarray(anet.domains[v], dtype=object)[acodes[v]] for v, name in enumerate(anet.names)})
    X = X.mask(np.random.default_rng(4).random(X.shape) < 0.3)
    patterns = len(alarm._count_patterns(X))
    alarm.mpe_many(X)  # warm-up: plans, programs
    t = [timed(lambda: alarm.mpe_many(X)) for _ in range(args.rounds)]
    med = float(np.median(t))
    results["alarm"] = dict(rows=k, patterns=patterns, mpe_many_ms=med * 1e3, mpe_many_ms_all=[x * 1e3 for x in t],
                            rows_per_s=k / med)
    print(f"alarm, {k} rows, 30 % of the cells missing, {patterns} patterns: mpe_many {spread(t)}, "
          f"{k / med / 1e6:.2f} M rows/s", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
