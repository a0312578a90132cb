"""Time constraint-based structure learning on the device (structure.pc_cpdag over engine.Tally.tests,
csrc/sbn_tally.cu) level by level, against host counting and reduction.

Workload: `synthetic.random_dag(40, 3, (2, 3, 4))`, 40 columns of 2 to 4 states, sampled with `BayesNet.sample`
at N rows (1M and 10M by default), seeded.  The search runs once with a recording tester to collect the batch of
every level (what `pc_cpdag` sends), then, per level, with a synchronised host clock (every tally call ends in a
device synchronise) after a warm-up call:

  (a) `Tally.tests` (G^2) of the level's batch: words in, count + test kernels, three doubles per test out; the
      median of --reps calls, in calls of at most structure._BATCH_ENTRIES table entries as pc_cpdag sends them;
  (b) the code bytes the count plan must read (tools/structure_bench.plan_code_bytes: N bytes per staged column
      of every shared group, N per member of a table on the global path) and their rate;
  (c) for levels 0 and 1, the same tests on the host: np.bincount of each table and a numpy G^2 / dof / scipy
      gammaincc reduction, timed once over the first --host-tests tests of the batch and scaled to the batch.

Also `pc_cpdag` end to end (encoding, upload, every level).  Printed with the GPU's name, power limit and maximum
SM clock, read in the same run.  Without a usable GPU the first device call raises.

    python tools/pc_bench.py [--rows 1000000 10000000] [--reps 3] [--out results/pc_bench.json]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

import numpy as np
from scipy.special import gammaincc

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from structure_bench import HBM_BYTES_PER_S, gpu_limits, plan_code_bytes, timed  # noqa: E402


def host_tests(codes, cards, ids):
    """(statistic, dof, p) of every test on the host: np.bincount of the table, then a numpy G^2 reduction."""
    out = []
    for t in ids:
        flat = np.zeros(codes.shape[1], dtype=np.int64)
        size = 1
        for v in t:
            flat += codes[v].astype(np.int64) * size
            size *= cards[v]
        tab = np.bincount(flat, minlength=size).reshape(-1, cards[t[1]], cards[t[0]]).astype(np.float64)
        nx, ny = tab.sum(axis=1)[:, None, :], tab.sum(axis=2)[:, :, None]
        nz = tab.sum(axis=(1, 2))[:, None, None]
        cell = tab > 0
        stat = 2.0 * float(np.sum(tab[cell] * np.log((tab * nz)[cell] / (nx * ny)[cell])))
        a, b = (tab.sum(axis=1) > 0).sum(axis=1), (tab.sum(axis=2) > 0).sum(axis=1)
        dof = int(np.sum(np.where(nz[:, 0, 0] > 0, (a - 1) * (b - 1), 0)))
        out.append((stat, dof, float(gammaincc(dof / 2, stat / 2)) if dof > 0 and stat > 0 else 1.0))
    return out


def run(X, reps, host_n, alpha):
    from sorobn_b200 import engine, structure

    n = len(X)
    columns, codes, cards = structure._encode(X)
    index = {c: i for i, c in enumerate(columns)}
    tally = engine.Tally(codes, cards)
    levels = []
    try:
        def recorder(tests):
            ids = [[index[x], index[y], *(index[g] for g in given)] for x, y, given in tests]
            levels.append(ids)
            return structure._device_tests(tally, ids, "g2")[:, 2]

        res = structure.pc_search(columns, cards, recorder, alpha)
        rows = []
        for level, ids in enumerate(levels):
            structure._device_tests(tally, ids, "g2")  # warm-up
            t = timed(lambda: structure._device_tests(tally, ids, "g2"), reps)
            entries = sum(math.prod(cards[v] for v in i) for i in ids)
            code_bytes, groups = plan_code_bytes(ids, cards, n)
            med = float(np.median(t))
            row = dict(level=level, tests=len(ids), table_entries=entries, groups=groups, code_bytes=code_bytes,
                       tally_tests_s=t, median_s=med, code_bytes_per_s=code_bytes / med,
                       share_of_hbm_peak=code_bytes / med / HBM_BYTES_PER_S, host_s="not measured")
            if level <= 1:
                k = min(len(ids), host_n)
                (h,) = timed(lambda: host_tests(codes, cards, ids[:k]), 1)
                row.update(host_s=h * len(ids) / k, host_tests_timed=k)
            rows.append(row)
            host = "not measured" if row["host_s"] == "not measured" else \
                f"{row['host_s'] * 1e3:,.0f} ms (from {row['host_tests_timed']} tests)"
            print(f"  level {level}: {len(ids)} tests, {entries:,} table entries, {groups} group(s), "
                  f"{code_bytes / 1e6:.1f} MB of codes; Tally.tests {med * 1e3:.2f} ms "
                  f"({code_bytes / med / 1e9:.1f} GB/s of codes); host bincount + numpy {host}", flush=True)
    finally:
        tally.close()
    structure.pc_cpdag(X, alpha=alpha)
    e2e = timed(lambda: structure.pc_cpdag(X, alpha=alpha), reps)
    print(f"  pc_cpdag end to end {np.median(e2e) * 1e3:.1f} ms: {len(res.directed)} directed and "
          f"{len(res.undirected)} undirected edges", flush=True)
    return dict(rows=n, levels=rows, pc_cpdag_s=e2e, pc_cpdag_median_s=float(np.median(e2e)),
                directed=res.directed, undirected=res.undirected)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[1_000_000, 10_000_000])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-tests", type=int, default=40)
    ap.add_argument("--alpha", type=float, default=0.05)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from sorobn_b200 import BayesNet, synthetic

    results = {"gpu": gpu_limits(), "runs": []}
    print("gpu:", results["gpu"], flush=True)
    dag40 = synthetic.load(synthetic.random_dag(40, 3, (2, 3, 4), seed=args.seed), BayesNet, seed=args.seed)
    for n in args.rows:
        X = dag40.sample(n)
        print(f"dag40 N={n:,}:", flush=True)
        results["runs"].append(run(X, args.reps, args.host_tests, args.alpha))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1, default=str)


if __name__ == "__main__":
    main()
