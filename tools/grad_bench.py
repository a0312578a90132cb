"""Time the forward and backward passes of `BayesNet.log_likelihood` against one counts call on the same rows.

Workloads:

* grid: the benchmark grid (10x10, 5 states), 100k forward-sampled rows, the 30 evidence columns of the
  benchmark hard (the other nodes latent), with 0 or 5 latent nodes carrying soft evidence;
* asia: the Asia network, 1M rows, one column missing in 30 % of the rows.

Per workload and rep, alternated in one process: forward (the CPTs as torch tensors that require grad, the
rows pre-encoded with `encode_rows`), backward (`.sum().backward()`), and `Program.counts` of every pattern
on the same codes.  Every timing ends in a device synchronise (the host paths synchronise).  Medians and
ranges are printed with the card's name and power limit, read in the same run.

    python tools/grad_bench.py [--reps 5] [--out results/grad_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from em_bench import gpu_limits, rows  # noqa: E402


def workload_rows(label, seed=1):
    from sorobn_b200 import examples, workloads

    if label.startswith("grid"):
        wl = workloads.grid10x10()
        bn = wl.build(device=0)
        ev = list(wl.evidence)
        latent = [n for n in bn.nodes if n not in set(ev)]
        X = rows(bn, 100_000, seed, latent=latent, missing=(), frac=0.0)
        n_soft = int(label.split("_soft")[1]) if "_soft" in label else 0
        lik = None
        if n_soft:
            rng = np.random.default_rng(seed)
            lik = {n: rng.random((len(X), len(bn._compiled.domains[bn._compiled.index[n]]))) + 0.05
                   for n in sorted(latent)[:n_soft]}
        return bn, X, lik
    bn = examples.asia(device=0)
    return bn, rows(bn, 1_000_000, seed + 1, latent=(), missing=("Smoker",), frac=0.3), None


def stats(xs):
    return dict(median_ms=1e3 * float(np.median(xs)), min_ms=1e3 * float(np.min(xs)), max_ms=1e3 * float(np.max(xs)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    results = {"gpu": gpu_limits()}
    print("gpu:", results["gpu"], flush=True)
    for label in ("grid_100k_soft0", "grid_100k_soft5", "asia_1m"):
        bn, X, lik = workload_rows(label)
        enc = bn.encode_rows(X)
        cpts = {k: v.clone().requires_grad_(True) for k, v in bn.cpt_tensors().items() if bool((v > 0).all())}
        runners = [bn._pattern_runner("counts", ev, soft=()) for ev, _, _ in enc.groups] if lik is None else None
        fwd, bwd, cnt = [], [], []
        for rep in range(args.reps + 1):  # rep 0 warms every shape up
            t0 = time.perf_counter()
            lp = bn.log_likelihood(enc, cpts=cpts, likelihoods=lik)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            lp.sum().backward()
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if runners is not None:
                for r, (ev, rr, codes) in zip(runners, enc.groups):
                    r.f32().counts(codes, len(rr))
            t3 = time.perf_counter()
            if rep:
                fwd.append(t1 - t0)
                bwd.append(t2 - t1)
                cnt.append(t3 - t2)
        res = dict(rows=len(X), patterns=len(enc.groups), soft=0 if lik is None else len(lik), forward=stats(fwd),
                   backward=stats(bwd))
        if runners is not None:
            res["counts"] = stats(cnt)
        results[label] = res
        print(label, json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
