"""Time posteriors with soft evidence (`engine.Program.run_soft`) against the same programs with hard evidence only.

* Asia, 1M rows: P(Lung cancer | Visit to Asia, Smoker) with hard evidence only, against the same with
  likelihoods on Dispnea and Positive X-ray, from host memory and from a CUDA tensor.
* The benchmark grid (10x10, 5 states), 100k rows: its 30 hard columns, against the same plus likelihoods on 1, 5
  and 10 hidden nodes.

Each call is one host-path run (codes and likelihoods in, posteriors out, synchronised) on a program created and
warmed up first.  Medians of several rounds and their spread (min .. max), rows per second and the algorithmic HBM
bytes per row (`Plan.bytes_per_row`) are printed, and the pack kernel's share of a soft run from a separate
torch.profiler run, with the card's name, power limit and largest SM clock.

    python tools/soft_bench.py [--rounds 7] [--out results/soft_bench.json]
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


def timed(fn, rounds):
    fn()  # warm-up: scratch, graph capture
    ts = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return ts


def report(name, plan, n, ts):
    ms = np.array(ts) * 1e3
    row = dict(case=name, rows=n, ms_median=float(np.median(ms)), ms_min=float(ms.min()), ms_max=float(ms.max()),
               rows_per_s=float(n / np.median(ts)), bytes_per_row=int(plan.bytes_per_row()))
    print(f"{name:44s} {row['ms_median']:9.2f} ms ({row['ms_min']:.2f} .. {row['ms_max']:.2f})  "
          f"{row['rows_per_s'] / 1e6:8.2f} M rows/s  {row['bytes_per_row']:6d} B/row", flush=True)
    return row


def pack_share(prog, codes, lik, n):
    """(pack kernel ms, every kernel's ms) of one soft run, from torch.profiler's CUDA activities."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        prog.run_soft(codes, lik, n)
        torch.cuda.synchronize()
    pack = total = 0.0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            t = e.device_time / 1e3
            total += t
            pack += t if "sbn_soft_pack" in e.name else 0.0
    return pack, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    from sorobn_b200 import engine, examples, planner, workloads

    print("GPU:", gpu_limits(), flush=True)
    rows = []
    rng = np.random.default_rng(0)

    # Asia, 1M rows
    bn = examples.asia()
    net = bn._compiled
    n = 1_000_000
    allc = workloads.forward_sample_codes(net, n, 1)
    ev = [net.index["Visit to Asia"], net.index["Smoker"]]
    q = [net.index["Lung cancer"]]
    soft = [net.index["Dispnea"], net.index["Positive X-ray"]]
    codes = np.ascontiguousarray(allc[ev])
    hard_plan = planner.build_plan(net, q, ev)
    soft_plan = planner.build_plan(net, q, ev, soft=soft)
    lik = rng.random((n, 4))
    hard = engine.Program(hard_plan)
    prog = engine.Program(soft_plan)
    lik_dev = torch.as_tensor(lik, dtype=torch.float32, device="cuda")
    rows.append(report("asia 1M: 2 hard columns", hard_plan, n, timed(lambda: hard.run(codes, n), args.rounds)))
    rows.append(report("asia 1M: + 2 soft nodes, host likelihoods", soft_plan, n,
                       timed(lambda: prog.run_soft(codes, lik, n), args.rounds)))
    rows.append(report("asia 1M: + 2 soft nodes, CUDA likelihoods", soft_plan, n,
                       timed(lambda: prog.run_soft(codes, lik_dev, n), args.rounds)))
    pack, total = pack_share(prog, codes, lik_dev, n)
    print(f"  pack kernel: {pack:.3f} ms of {total:.3f} ms of kernels ({100 * pack / total:.1f} %)", flush=True)
    rows[-1]["pack_ms"], rows[-1]["kernel_ms"] = pack, total
    hard.close()
    prog.close()

    # the benchmark grid, 100k rows
    w = workloads.grid10x10()
    bn = w.build()
    net = bn._compiled
    n = 100_000
    codes = w.codes(bn, n, 2)
    q = [net.index[x] for x in w.query]
    ev = [net.index[e] for e in w.evidence]
    hidden = [v for v in range(len(net.names)) if v not in set(ev) | set(q)]
    hard_plan = planner.build_plan(net, q, ev)
    hard = engine.Program(hard_plan)
    rows.append(report("grid 100k: 30 hard columns", hard_plan, n, timed(lambda: hard.run(codes, n), args.rounds)))
    hard.close()
    for k in (1, 5, 10):
        soft = [int(v) for v in rng.choice(hidden, size=k, replace=False)]
        plan = planner.build_plan(net, q, ev, soft=soft)
        prog = engine.Program(plan)
        lik = rng.random((n, 5 * k))
        rows.append(report(f"grid 100k: + {k} soft nodes, host likelihoods", plan, n,
                           timed(lambda: prog.run_soft(codes, lik, n), args.rounds)))
        pack, total = pack_share(prog, codes, lik, n)
        print(f"  pack kernel: {pack:.3f} ms of {total:.3f} ms of kernels ({100 * pack / total:.1f} %)", flush=True)
        rows[-1]["pack_ms"], rows[-1]["kernel_ms"] = pack, total
        prog.close()

    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(gpu=gpu_limits(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
