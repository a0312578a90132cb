"""Time MPE, sampling and expected counts with soft evidence (`engine.Program.mpe / sample / counts` with `lik`)
against the same programs with hard evidence only.

* The benchmark grid (10x10, 5 states), 100k rows, its 30 hard columns: `Program.mpe`, `Program.sample` at n = 1
  and `Program.counts` with likelihoods on 0, 1, 5 and 10 hidden nodes.
* Asia, 1M rows, Visit to Asia and Smoker observed: `Program.counts` with likelihoods on Dispnea and Positive
  X-ray, from host memory and from a CUDA tensor.

Each call is one host-path run (codes and likelihoods in, outputs back, synchronised) on a program created and
warmed up first.  Medians of several rounds and their spread (min .. max) and rows per second are printed, and the
pack kernel's share of the kernel time of one run from a separate torch.profiler run, with the card's name, power
limit and largest SM clock.

    python tools/soft_decode_bench.py [--rounds 7] [--out results/soft_decode_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.soft_bench import gpu_limits, timed  # noqa: E402


def report(name, n, ts):
    ms = np.array(ts) * 1e3
    row = dict(case=name, rows=n, ms_median=float(np.median(ms)), ms_min=float(ms.min()), ms_max=float(ms.max()),
               rows_per_s=float(n / np.median(ts)))
    print(f"{name:52s} {row['ms_median']:9.2f} ms ({row['ms_min']:.2f} .. {row['ms_max']:.2f})  "
          f"{row['rows_per_s'] / 1e6:8.2f} M rows/s", flush=True)
    return row


def pack_share(fn):
    """(pack kernel ms, every kernel's ms) of one run of `fn`, from torch.profiler's CUDA activities."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
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

    # the benchmark grid, 100k rows
    w = workloads.grid10x10()
    bn = w.build()
    net = bn._compiled
    n = 100_000
    codes = w.codes(bn, n, 2)
    ev = [net.index[e] for e in w.evidence]
    hidden = [v for v in range(len(net.names)) if v not in set(ev)]
    for k in (0, 1, 5, 10):
        soft = [int(v) for v in rng.choice(hidden, size=k, replace=False)]
        lik = rng.random((n, 5 * k)) + 0.01 if k else None
        kw = dict(lik=lik) if k else {}
        for kind in ("mpe", "sample", "counts"):
            plan = planner.build_pattern_plan(net, kind, ev, soft=soft)
            prog = engine.Program(plan)
            if kind == "mpe":
                fn = lambda: prog.mpe(codes, n, **kw)  # noqa: E731
            elif kind == "sample":
                fn = lambda: prog.sample(codes, n, 1, 7, **kw)  # noqa: E731
            else:
                fn = lambda: prog.counts(codes, n, **kw)  # noqa: E731
            rows.append(report(f"grid 100k {kind}: {k} soft nodes", n, timed(fn, args.rounds)))
            if k:
                pack, total = pack_share(fn)
                print(f"  pack kernel: {pack:.3f} ms of {total:.3f} ms of kernels ({100 * pack / total:.2f} %)",
                      flush=True)
                rows[-1]["pack_ms"], rows[-1]["kernel_ms"] = pack, total
            prog.close()

    # Asia counts, 1M rows: host against CUDA-tensor likelihoods
    bn = examples.asia()
    net = bn._compiled
    n = 1_000_000
    allc = workloads.forward_sample_codes(net, n, 1)
    ev = [net.index["Visit to Asia"], net.index["Smoker"]]
    soft = [net.index["Dispnea"], net.index["Positive X-ray"]]
    codes = np.ascontiguousarray(allc[ev])
    lik = rng.random((n, 4)) + 0.01
    lik_dev = torch.as_tensor(lik, dtype=torch.float32, device="cuda")
    hard_plan = planner.build_counts_plan(net, ev)
    hard = engine.Program(hard_plan)
    rows.append(report("asia 1M counts: 2 hard columns", n, timed(lambda: hard.counts(codes, n), args.rounds)))
    hard.close()
    prog = engine.Program(planner.build_pattern_plan(net, "counts", ev, soft=soft))
    rows.append(report("asia 1M counts: + 2 soft nodes, host likelihoods", n,
                       timed(lambda: prog.counts(codes, n, lik=lik), args.rounds)))
    rows.append(report("asia 1M counts: + 2 soft nodes, CUDA likelihoods", n,
                       timed(lambda: prog.counts(codes, n, lik=lik_dev), args.rounds)))
    pack, total = pack_share(lambda: prog.counts(codes, n, lik=lik_dev))
    print(f"  pack kernel: {pack:.3f} ms of {total:.3f} ms of kernels ({100 * pack / total:.2f} %)", flush=True)
    rows[-1]["pack_ms"], rows[-1]["kernel_ms"] = pack, total
    prog.close()

    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(gpu=gpu_limits(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
