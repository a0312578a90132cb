"""Cost of belief-propagation expected counts on the device (csrc/sbn_bp.cu, version-3 words).

For 100k rows of grid10x10s5 (30 cells observed) and of the 16 x 16 grid of 3 states (its last row and column
observed), prints one JSON line each with:
  * readout_ms: the family-belief readout and the count reduction over one sweep, t(counts, 1 sweep) - t(marginals,
    1 sweep) of the same rows, host clocks around calls that end in a stream synchronise (median of 5);
  * estep_ms: one E-step at the defaults (n_iterations 100, damping 0.5, tol 1e-5), as each iteration of
    `fit_em(algorithm="bp")` runs it;
  * exact_ms (10 x 10 grid only): `expected_counts` by elimination on the same frame.
The card's name and power limit come first.  Usage: python tools/bp_em_bench.py [--rows N]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from sorobn_b200 import BayesNet, bp, engine, synthetic, workloads  # noqa: E402

GRID16_EVIDENCE = [f"g15{j:02d}" for j in range(16)] + [f"g{i:02d}15" for i in range(1, 15)]


def median_ms(f, reps=5):
    f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


def kernel_ms(f):
    """{kernel: device ms} of one call of `f` by torch.profiler (sweep, readout and reduction apart; the host clocks
    above also count the marginals call's download of its beliefs, which the counts call does not have)."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    f()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "sbn_bp" in e.name:
            key = e.name.split("(")[0].split("<")[0].replace("void ", "")
            out[key] = round(out.get(key, 0.0) + e.device_time / 1e3, 3)
    return out


def case(label, bn, names, n, exact):
    net = bn._compiled
    ev = [net.index[e] for e in names]
    codes = np.ascontiguousarray(workloads.forward_sample_codes(net, n, 1)[ev])
    g1 = bp.compile_graph(net, ev, [v for v in range(len(net.names)) if v not in ev])
    g3 = bp.compile_counts_graph(net, ev)
    r1 = engine.BeliefPropagation(g1.words, g1.tables)
    r3 = engine.BeliefPropagation(g3.words, g3.tables)
    t_marg = median_ms(lambda: r1.run(codes, n, 1, 0.5, 0.0))
    t_cnt = median_ms(lambda: r3.counts(codes, n, 1, 0.5, 0.0))
    t_estep = median_ms(lambda: r3.counts(codes, n, 100, 0.5, 1e-5), reps=3)
    _, _, iters = r3.counts(codes, n, 100, 0.5, 1e-5)
    kern = kernel_ms(lambda: r3.counts(codes, n, 1, 0.5, 0.0))
    out = {"case": label, "rows": n, "table_floats": int(g3.tables.size), "marginals_1sweep_ms": round(t_marg, 3),
           "counts_1sweep_ms": round(t_cnt, 3), "readout_ms": round(t_cnt - t_marg, 3),
           "estep_ms": round(t_estep, 2), "mean_sweeps": round(float(np.minimum(iters, 100).mean()), 2),
           "kernels_1sweep_ms": kern}
    if exact:
        X = pd.DataFrame({e: np.asarray(net.domains[v], dtype=object)[codes[i]] for i, (e, v) in
                          enumerate(zip(names, ev))}).infer_objects()
        out["exact_ms"] = round(median_ms(lambda: bn.expected_counts(X), reps=3), 2)
    r1.close()
    r3.close()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000)
    args = ap.parse_args()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        card = "unknown"
    print(json.dumps({"card": card}), flush=True)
    grid10 = synthetic.load(synthetic.grid(10, 10, 5), BayesNet)
    names = sorted(np.random.default_rng(0).choice(grid10.nodes, size=30, replace=False).tolist())
    case("grid10x10s5", grid10, names, args.rows, exact=True)
    grid16 = synthetic.load(synthetic.grid(16, 16, 3), BayesNet)
    case("grid16x16s3", grid16, sorted(GRID16_EVIDENCE), args.rows, exact=False)


if __name__ == "__main__":
    main()
