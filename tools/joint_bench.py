"""Per-row joint posteriors on the GPU (BayesNet.joint_marginals_many / planner.build_joint_plan): time per call and
output bytes, next to what a user computes otherwise.  Prints one JSON object per workload, with the card's name and
power limit.

  grid    10x10 grid, 5 states, 100k rows, the 30 hard columns of bench.py's workload, every family: one joint
          program, against one expected_counts program of the same pattern (the same passes, reduced over the rows)
  alarm   the Alarm example, 100k rows, 30 % missing in every column (5 columns): joint_marginals_many of every
          family, end to end through pandas, against expected_counts of the same frame
  per-family  the Alarm rows without a missing cell through what exists without joint programs: one query_many
          program per family, P(family | the columns outside it) (query_many takes no missing cells)

    python tools/joint_bench.py [--rows N] [--reps K]
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

from sorobn_b200 import engine, examples, planner, workloads  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(fn, reps):
    fn()  # warm-up: program creation, reservation, graph capture
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts)), float(np.min(ts))


def grid(rows, reps):
    wl = workloads.grid10x10()
    bn = wl.build()
    net = bn._compiled
    ev = tuple(sorted(net.index[v] for v in wl.evidence))
    codes = np.ascontiguousarray(workloads.forward_sample_codes(net, rows, 9)[list(ev)])
    jp = planner.build_joint_plan(net, ev)
    cp = planner.build_counts_plan(net, ev)
    joint, counts = engine.Program(jp), engine.Program(cp)
    try:
        tj = timed(lambda: joint.joint(codes, rows), reps)
        tc = timed(lambda: counts.counts(codes, rows), reps)
    finally:
        joint.close()
        counts.close()
    return dict(workload="grid10x10 families", rows=rows, Q=jp.Q, output_bytes_per_row=4 * jp.Q,
                algorithmic_bytes_per_row=jp.bytes_per_row(), joint_s=tj[0], joint_min_s=tj[1],
                expected_counts_s=tc[0], expected_counts_min_s=tc[1])


def alarm_frame(bn, rows):
    net = bn._compiled
    codes = workloads.forward_sample_codes(net, rows, 4)
    rng = np.random.default_rng(4)
    out = {}
    for v, name in enumerate(net.names):
        vals = np.asarray(net.domains[v], dtype=object)[codes[v]].copy()
        vals[rng.random(rows) < 0.3] = None
        out[name] = vals
    return pd.DataFrame(out)


def alarm(rows, reps):
    bn = examples.alarm()
    X = alarm_frame(bn, rows)
    tj = timed(lambda: bn.joint_marginals_many(X), reps)
    tc = timed(lambda: bn.expected_counts(X), reps)
    # the alternative: one query_many program per family, on the rows without a missing cell
    full = X.dropna()
    net = bn._compiled

    def per_family():
        for v in range(len(net.names)):
            family = [net.names[u] for u in net.scope(v)]
            bn.query_many(*family, events=full[[c for c in X.columns if c not in family]])

    tq = timed(per_family, reps)
    return dict(workload="alarm families, 30% missing", rows=rows, patterns=int(X.isna().drop_duplicates().shape[0]),
                joint_marginals_many_s=tj[0], expected_counts_s=tc[0],
                per_family_query_many_s=tq[0], per_family_rows=len(full), per_family_programs=len(net.names))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    gpu = card()
    for fn in (grid, alarm):
        res = fn(args.rows, args.reps)
        res["gpu"] = gpu
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
