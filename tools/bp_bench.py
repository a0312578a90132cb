"""Time loopy belief propagation on the device (csrc/sbn_bp.cu).

Workloads: the benchmark's 10x10 grid with 5 states (30 observed cells, `workloads.grid10x10`), and a 16x16 grid
with 3 states observed on its last row and the rest of its last column (30 cells), which the exact planner refuses
(checked here: `planner.build_marginals_plan` must raise).  Each runs 100k evidence rows with tol=0, so that every
row runs exactly the sweeps asked for.  Reported per workload:
  * ms per sweep: (t(1 + N sweeps) - t(1 sweep)) / N, each t the best of `--repeat` host-clock timings of
    `BeliefPropagation.run` after one warm-up call.  A call ends in a stream synchronise, and the evidence upload,
    the message initialisation, the belief readout and the download are the same in both calls, so the difference
    is the device time of N sweeps;
  * the bytes of message state one sweep accesses (`bp.Graph.message_bytes_per_sweep`, computed from the compiled
    words) and the rate that gives;
  * the whole call with N sweeps, and, on the 10x10 grid, exact `marginals_many` of the same targets on the same rows.
The card's name and power limit are read in the same run.

    python tools/bp_bench.py [--rows 100000] [--sweeps 20] [--repeat 3] [--out FILE]
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

from sorobn_b200 import BayesNet, bp, engine, planner, synthetic, workloads  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(engine.default_device())], capture_output=True, text=True, timeout=60).stdout
        name, power = [s.strip() for s in out.strip().split(",")]
        return name, power
    except Exception as exc:  # the timing itself needs the GPU, not nvidia-smi
        return f"unknown ({exc})", "unknown"


def best(fn, repeat):
    fn()
    times = []
    for _ in range(repeat):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return min(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--sweeps", type=int, default=20)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    if engine.device_count() == 0:
        raise SystemExit("bp_bench needs a GPU")
    name, power = card()
    wl = workloads.grid10x10()
    ev16 = tuple(sorted([f"g15{j:02d}" for j in range(16)] + [f"g{i:02d}15" for i in range(1, 15)]))
    cases = [("grid10x10s5", wl.spec, wl.evidence), ("grid16x16s3", synthetic.grid(16, 16, 3), ev16)]
    results = []
    for label, spec, evidence in cases:
        bn = synthetic.load(spec, BayesNet)
        net = bn._compiled
        ev = [net.index[e] for e in evidence]
        targets = sorted(v for v in bn.nodes if v not in evidence)
        try:
            planner.build_marginals_plan(net, ev)
            exact_plans = True
        except ValueError:
            exact_plans = False
        if label == "grid16x16s3" and exact_plans:
            raise SystemExit("the exact planner plans the 16x16 workload: it no longer shows what BP is for")
        g = bp.compile_graph(net, ev, [net.index[t] for t in targets])
        codes = np.ascontiguousarray(workloads.forward_sample_codes(net, args.rows, seed=1)[ev])
        runner = engine.BeliefPropagation(g.words, g.tables)
        t = best(lambda: runner.run(codes, args.rows, 1 + args.sweeps, 0.5, 0.0), args.repeat)
        t1 = best(lambda: runner.run(codes, args.rows, 1, 0.5, 0.0), args.repeat)
        runner.close()
        ms_sweep = 1e3 * (t - t1) / args.sweeps
        nbytes = g.message_bytes_per_sweep() * args.rows
        row = {"workload": label, "rows": args.rows, "sweeps": args.sweeps, "factors": len(g.families),
               "variables": len(g.variables), "message_floats_per_row": 2 * g.n_edges,
               "exact_planner": "plans" if exact_plans else "refuses",
               "ms_per_call": round(1e3 * t, 3), "ms_per_call_1_sweep": round(1e3 * t1, 3),
               "ms_per_sweep": round(ms_sweep, 4),
               "message_bytes_per_sweep": int(nbytes), "message_GB_per_s": round(nbytes / (ms_sweep * 1e-3) / 1e9, 1)}
        if label == "grid10x10s5":
            events = pd.DataFrame({e: np.asarray(net.domains[net.index[e]], dtype=object)[codes[i]]
                                   for i, e in enumerate(evidence)}).infer_objects()
            row["exact_marginals_many_ms"] = round(1e3 * best(lambda: bn.marginals_many(events), args.repeat), 1)
        results.append(row)
        print(json.dumps(row), flush=True)
    summary = {"gpu": name, "power_limit": power, "results": results}
    print(json.dumps(summary))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
