"""Time marginal MAP (`BayesNet.map_many`) against `impute_many`, which answers the same question through the
dense posterior over the joint of a row's missing cells.

* Alarm (5 binary nodes), 100k forward-sampled rows with exactly 2, then 4, random cells missing per row:
  `map_many` and `impute_many` of the same frame, timed alternately in the same process.
* The benchmark grid (10x10, 5 states), 100k rows with 24 of its 100 cells missing (from 8 missingness
  patterns) and 10 nodes without a column (summed out): `map_many` alone.  One row's missing cells have
  5^24 = 6e16 joint states, which `impute_many` cannot hold.

Each call is end to end: grouping, one device call per missingness pattern (codes in, decoded codes and
log-probabilities out, synchronised) and the result frame; the programs are planned and created by a
warm-up call first.  Medians of several rounds, their spread (min .. max) and rows per second are printed
with the card's name, power limit and largest SM clock.

    python tools/map_bench.py [--rounds 5] [--rows 100000] [--out results/map_bench.json]
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
    return f"{np.median(ms):.1f} ms (min {min(ms):.1f}, max {max(ms):.1f})"


def missing_frame(net, n, seed, k_missing, n_patterns=None):
    """n forward samples with exactly `k_missing` random cells missing per row, from `n_patterns` patterns
    (None: every row draws its own)."""
    import pandas as pd

    from sorobn_b200 import workloads

    codes = workloads.forward_sample_codes(net, n, seed)
    rng = np.random.default_rng(seed + 1)
    X = pd.DataFrame({name: np.asarray(net.domains[v], dtype=object)[codes[v]] for v, name in enumerate(net.names)})
    blank = np.argsort(rng.random((n if n_patterns is None else n_patterns, len(net.names))), axis=1)[:, :k_missing]
    if n_patterns is not None:
        blank = blank[rng.integers(0, n_patterns, size=n)]
    mask = np.zeros((n, len(net.names)), dtype=bool)
    np.put_along_axis(mask, blank, True, axis=1)
    return X.mask(pd.DataFrame(mask, columns=X.columns))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from sorobn_b200 import examples, workloads

    n = args.rows
    results = {"gpu": gpu_limits(), "rows": n}
    print("gpu:", results["gpu"], flush=True)

    alarm = examples.alarm(device=0)
    for k in (2, 4):
        X = missing_frame(alarm._compiled, n, 10 + k, k)
        patterns = len(alarm._count_patterns(X))
        alarm.map_many(X)  # warm-up: plans, programs, graphs
        alarm.impute_many(X)
        tm, ti = [], []
        for _ in range(args.rounds):
            tm.append(timed(lambda: alarm.map_many(X)))
            ti.append(timed(lambda: alarm.impute_many(X)))
        m, i = float(np.median(tm)), float(np.median(ti))
        results[f"alarm_{k}_missing"] = dict(patterns=patterns, map_many_ms=m * 1e3, map_many_ms_all=[t * 1e3 for t in tm],
                                             impute_many_ms=i * 1e3, impute_many_ms_all=[t * 1e3 for t in ti],
                                             map_rows_per_s=n / m, impute_rows_per_s=n / i)
        print(f"alarm, {n} rows, {k} missing cells per row, {patterns} patterns:\n"
              f"  map_many    {spread(tm)}, {n / m / 1e6:.2f} M rows/s\n"
              f"  impute_many {spread(ti)}, {n / i / 1e6:.2f} M rows/s", flush=True)

    wl = workloads.grid10x10()
    bn = wl.build(device=0)
    net = bn._compiled
    latent = [net.names[v] for v in range(5, len(net.names), 10)]
    X = missing_frame(net, n, 21, 24, n_patterns=8).drop(columns=latent)
    least = int(X.isna().sum(axis=1).min())
    patterns = len(bn._count_patterns(X))
    bn.map_many(X)  # warm-up
    tm = [timed(lambda: bn.map_many(X)) for _ in range(args.rounds)]
    m = float(np.median(tm))
    results["grid_many_missing"] = dict(patterns=patterns, least_missing=least, latent=len(latent), map_many_ms=m * 1e3,
                                        map_many_ms_all=[t * 1e3 for t in tm], map_rows_per_s=n / m)
    print(f"grid10x10, {n} rows, at least {least} missing cells per row, {len(latent)} latent nodes, {patterns} patterns:\n"
          f"  map_many    {spread(tm)}, {n / m / 1e6:.2f} M rows/s (impute_many: the joint does not fit)", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
