"""Time one E-step of expectation-maximisation (`BayesNet.expected_counts`: every missingness pattern's
counts program, plus the host's grouping and reduction) on two workloads:

* grid: the benchmark grid (10x10, 5 states), 100k forward-sampled rows; 3 columns latent and 2 more
  missing in 20 % of the rows (4 patterns);
* asia: the Asia network, 1M rows, one column missing in 30 % of the rows.

Two parts are timed separately with a synchronised host clock (the counts path ends in a device
synchronise), after warm-up: encoding the frame and grouping its rows by pattern (host only), and the
E-step proper (every pattern's counts program: codes in, kernels, counts and probabilities out, plus
the host's sum over patterns).  Medians of several calls are printed with the card's name and power
limit and the algorithmic bytes per row of every pattern's plan (planner.Plan.bytes_per_row).

    python tools/em_bench.py [--reps 5] [--out results/em_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_limits():
    try:
        res = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30)
        return res.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def rows(bn, n, seed, latent, missing, frac):
    from sorobn_b200 import workloads

    net = bn._compiled
    codes = workloads.forward_sample_codes(net, n, seed)
    rng = np.random.default_rng(seed + 1)
    cols = {}
    for v, name in enumerate(net.names):
        if name in latent:
            continue
        values = np.asarray(net.domains[v], dtype=object)[codes[v]]
        if name in missing:
            values[rng.random(n) < frac] = None
        cols[name] = values
    return pd.DataFrame(cols)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from sorobn_b200 import examples, planner, workloads

    results = {"gpu": gpu_limits()}
    print("gpu:", results["gpu"], flush=True)
    wl = workloads.grid10x10()
    grid = wl.build(device=0)
    names = sorted(grid.nodes)
    X_grid = rows(grid, 100_000, 1, latent=names[:3], missing=names[3:5], frac=0.2)
    asia = examples.asia(device=0)
    X_asia = rows(asia, 1_000_000, 2, latent=(), missing=("Smoker",), frac=0.3)
    for label, bn, X in (("grid_100k", grid, X_grid), ("asia_1m", asia, X_asia)):
        groups = bn._count_patterns(X)
        net = bn._compiled
        per_pattern = [(len(rows_), planner.build_counts_plan(net, ev).bytes_per_row()) for ev, rows_, _ in groups]
        _, n_counts = planner.count_layout(net)
        for _ in range(args.warmup):
            bn.expected_counts(X)
        host, estep = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            groups = bn._count_patterns(X)
            t1 = time.perf_counter()
            bn._e_step(X, groups, lambda k, ev: bn._pattern_runner("counts", ev), n_counts)
            t2 = time.perf_counter()
            host.append(t1 - t0)
            estep.append(t2 - t1)
        h, med = float(np.median(host)), float(np.median(estep))
        n = len(X)
        bytes_row = sum(r * b for r, b in per_pattern) / n
        results[label] = dict(rows=n, patterns=len(groups), encode_median_s=h, encode_s=host, estep_median_s=med,
                              estep_s=estep, rows_per_s=n / med, bytes_per_row=bytes_row,
                              pattern_rows_and_bytes=per_pattern, gb_per_s=n * bytes_row / med / 1e9)
        print(f"{label}: {len(groups)} patterns; encode + group {h * 1e3:.1f} ms; E-step median {med * 1e3:.1f} ms "
              f"({n / med / 1e6:.2f} M rows/s), {bytes_row:.0f} algorithmic B/row ({n * bytes_row / med / 1e9:.2f} GB/s); "
              f"per pattern (rows, B/row) {per_pattern}", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
