"""Time exact posterior sampling on the benchmark grid (10x10, 5 states): 100k forward-sampled rows with
the grid's evidence columns observed and the other 70 variables drawn, n = 1 and n = 8 draws per row.

One call = one `Program.sample` of the whole batch on the float32 sample program (codes in, upward pass,
sample steps, drawn codes and P(observed) out, synchronised).  The marginals program of the same
evidence columns (`Program.run`, posteriors out) is timed alternately with it, in the same process, as
the yardstick: both run the same upward pass.  Medians of several rounds are printed with the card's
name and power limit, the draws per second and the algorithmic bytes per row (planner.Plan.bytes_per_row).

A second part times `BayesNet.sample_many` end to end (grouping, device calls, the result frame) on Asia
with "Smoker" missing in 30 % of `--scattered-rows` rows, twice: with the missing rows scattered through the
frame, and with the same rows sorted by pattern.  A row's random stream is its position in the frame, so
`sample_many` makes one device call per run of consecutive rows of one pattern: the scattered frame costs
one call per run, the sorted one a call per pattern.

    python tools/sample_bench.py [--rounds 5] [--rows 100000] [--scattered-rows 100000] [--out results/sample_bench.json]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--scattered-rows", type=int, default=100_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from sorobn_b200 import engine, planner, workloads

    results = {"gpu": gpu_limits(), "rows": args.rows}
    print("gpu:", results["gpu"], flush=True)
    wl = workloads.grid10x10()
    bn = wl.build(device=0)
    net = bn._compiled
    observed = [net.index[e] for e in wl.evidence]
    codes = wl.codes(bn, args.rows, seed=1)
    n = args.rows
    splan = planner.build_sample_plan(net, sorted(observed))
    scodes = np.ascontiguousarray(codes[np.argsort(observed)])
    mplan = planner.build_marginals_plan(net, observed)
    sprog, mprog = engine.Program(splan, device=0), engine.Program(mplan, device=0)
    mout = np.empty((mprog.Q, n), dtype=np.float32)
    for n_draws in (1, 8):
        for _ in range(2):  # warm-up: reservation, graph capture
            sprog.sample(scodes, n, n_draws, seed=1)
            mprog.run(codes, n, out=mout)
        ts, tm = [], []
        for r in range(args.rounds):
            ts.append(timed(lambda: sprog.sample(scodes, n, n_draws, seed=r)))
            tm.append(timed(lambda: mprog.run(codes, n, out=mout)))
        s, m = float(np.median(ts)), float(np.median(tm))
        b = splan.bytes_per_row(n_draws)
        results[f"n{n_draws}"] = dict(sample_ms=s * 1e3, sample_ms_all=[t * 1e3 for t in ts], marginals_ms=m * 1e3,
                                      marginals_ms_all=[t * 1e3 for t in tm], draws_per_s=n * n_draws / s,
                                      bytes_per_row=b, marginals_bytes_per_row=mplan.bytes_per_row())
        print(f"n={n_draws}: sample {s * 1e3:.2f} ms per call ({n * n_draws / s / 1e6:.2f} M draws/s, {b} algorithmic "
              f"B/row); marginals program {m * 1e3:.2f} ms ({mplan.bytes_per_row()} B/row)", flush=True)
    import pandas as pd

    from sorobn_b200 import examples

    asia = examples.asia(device=0)
    anet = asia._compiled
    m = args.scattered_rows
    acodes = workloads.forward_sample_codes(anet, m, 3)
    X = pd.DataFrame({name: np.asarray(anet.domains[v], dtype=object)[acodes[v]] for v, name in enumerate(anet.names)})
    X.loc[np.random.default_rng(4).random(m) < 0.3, "Smoker"] = None
    frames = {"scattered": X, "sorted": X.iloc[np.argsort(X["Smoker"].isna().to_numpy(), kind="stable")]}
    for label, frame in frames.items():
        calls = sum(int(np.count_nonzero(np.diff(rows) != 1)) + 1 for _, rows, _ in asia._count_patterns(frame))
        asia.sample_many(frame, n=1, seed=0)  # warm-up: plans, programs
        t = [timed(lambda: asia.sample_many(frame, n=1, seed=r)) for r in range(args.rounds)]
        med = float(np.median(t))
        results[f"asia_{label}"] = dict(rows=m, device_calls=calls, sample_many_ms=med * 1e3,
                                        sample_many_ms_all=[x * 1e3 for x in t], rows_per_s=m / med)
        print(f"asia {label}, {m} rows, {calls} device calls: sample_many {med * 1e3:.1f} ms ({m / med / 1e6:.2f} M rows/s)",
              flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
