"""Time score-based structure learning on the device (structure.family_scores / hill_climb over
engine.Tally, csrc/sbn_tally.cu) against host counting.

Workloads, N rows each (1M and 10M by default), sampled with `BayesNet.sample`, seeded:

* alarm: `examples.alarm()`, 5 binary columns: 20 ordered pair families of 4 entries (the warp-vote path);
* dag40: `synthetic.random_dag(40, 3, (2, 3, 4))`, 40 columns of 2 to 4 states: 1,560 ordered pair families in
  one group, the wide case the grouping is for;
* skew5: codes drawn directly, 40 columns of 5 states, the 1,560 pair families of 25 entries (the
  warp-aggregated path), once uniform and once with 95 % of every column in state 0 (hot bins).

Timed with a synchronised host clock (every tally call ends in a device synchronise), after a warm-up call of each
shape:

  (a) the BIC scores of all ordered pair families (child, (parent,)): `Tally.scores` alone (count + score
      kernels, the family words in, one double per family out), and `family_scores` end to end (encoding the
      frame, uploading the codes, scoring);
  (b) a full `hill_climb(max_parents=3)`, end to end;
  (c) the same pair tables counted on the host with np.bincount over the encoded codes (one call: the host is
      slow), for comparison.

skew5 times (a) `Tally.scores` only.  Printed with the GPU's name and power limit: the code bytes the count plan
must read (for every group of families counted together, N bytes per staged column with more than one state) and
the achieved code bytes/s of `Tally.scores` against the H100 SXM data sheet's 3.35 TB/s.  Without a usable GPU the
first device call raises.

    python tools/structure_bench.py [--rows 1000000 10000000] [--reps 3] [--out results/structure_bench.json]
"""
from __future__ import annotations

import argparse
import itertools
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12
STAGE_COLUMNS = 64  # kMaxStage of csrc/sbn_tally.cu


def gpu_limits():
    try:
        res = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30)
        return res.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def plan_code_bytes(families, cards, n_rows):
    """(code bytes the count plan reads, shared groups): the families packed in order into groups as
    sbn_tally.cu packs them (tables within TALLY_SMEM_BINS together, at most STAGE_COLUMNS staged columns, a
    family counted on the global path closing the group before it), N bytes per staged column of a group, and N
    per member column of a family on the global path."""
    from sorobn_b200 import engine

    total, groups, bins, staged = 0, 0, 0, set()
    for fam in families:
        size = math.prod(cards[v] for v in fam)
        cols = {v for v in fam if cards[v] > 1}
        if size > engine.TALLY_SMEM_BINS:
            total += (len(staged) + len(cols)) * n_rows
            bins, staged = 0, set()
            continue
        if not bins or bins + size > engine.TALLY_SMEM_BINS or len(staged | cols) > STAGE_COLUMNS:
            total += len(staged) * n_rows
            groups, bins, staged = groups + 1, 0, set()
        bins += size
        staged |= cols
    return total + len(staged) * n_rows, groups


def timed(fn, reps):
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.append(time.perf_counter() - t0)
    return out


def pair_ids(n_cols):
    return [[c, p] for p, c in itertools.permutations(range(n_cols), 2)]


def time_tally(codes, cards, ids, reps):
    from sorobn_b200 import engine

    tally = engine.Tally(codes, cards)
    try:
        tally.scores(ids, "bic")  # warm-up
        return timed(lambda: tally.scores(ids, "bic"), reps)
    finally:
        tally.close()


def run_frame(label, X, reps):
    from sorobn_b200 import structure

    n = len(X)
    columns, codes, cards = structure._encode(X)
    ids = pair_ids(len(columns))
    pairs = [(columns[c], (columns[p],)) for c, p in ids]
    code_bytes, groups = plan_code_bytes(ids, cards, n)
    kernel = time_tally(codes, cards, ids, reps)
    structure.family_scores(X, pairs)
    scores_e2e = timed(lambda: structure.family_scores(X, pairs), reps)
    edges = structure.hill_climb(X, max_parents=3)
    climb = timed(lambda: structure.hill_climb(X, max_parents=3), reps)
    host = timed(lambda: [np.bincount(codes[c].astype(np.int64) + cards[c] * codes[p].astype(np.int64),
                                      minlength=cards[c] * cards[p]) for c, p in ids], 1)
    med = {k: float(np.median(v)) for k, v in
           (("tally_scores", kernel), ("family_scores", scores_e2e), ("hill_climb", climb), ("host_bincount", host))}
    rate = code_bytes / med["tally_scores"]
    print(f"{label} N={n:,}: {len(ids)} pair families in {groups} group(s), {code_bytes / 1e6:.1f} MB of codes; "
          f"Tally.scores {med['tally_scores'] * 1e3:.2f} ms ({rate / 1e9:.1f} GB/s of codes, "
          f"{rate / HBM_BYTES_PER_S:.3f} of 3.35 TB/s); family_scores end to end {med['family_scores'] * 1e3:.1f} ms; "
          f"hill_climb {med['hill_climb'] * 1e3:.1f} ms ({len(edges)} items); "
          f"host bincount {med['host_bincount'] * 1e3:.1f} ms", flush=True)
    return dict(workload=label, rows=n, columns=len(columns), pair_families=len(ids), groups=groups,
                code_bytes=code_bytes, median_s=med, tally_scores_s=kernel, family_scores_s=scores_e2e,
                hill_climb_s=climb, host_bincount_s=host, code_bytes_per_s=rate,
                share_of_hbm_peak=rate / HBM_BYTES_PER_S, items=edges)


def run_skew(n, reps, seed):
    rng = np.random.default_rng(seed)
    cards = [5] * 40
    ids = pair_ids(len(cards))
    code_bytes, groups = plan_code_bytes(ids, cards, n)
    out = dict(workload="skew5", rows=n, columns=len(cards), pair_families=len(ids), groups=groups,
               code_bytes=code_bytes)
    for label, hot in (("uniform", 0.0), ("skewed", 0.95)):
        codes = rng.integers(0, 5, (len(cards), n), dtype=np.uint8)
        codes[rng.random((len(cards), n)) < hot] = 0
        ts = time_tally(codes, cards, ids, reps)
        out[label] = dict(tally_scores_s=ts, median_s=float(np.median(ts)))
    print(f"skew5 N={n:,}: {len(ids)} pair families of 25 entries in {groups} group(s), {code_bytes / 1e6:.1f} MB "
          f"of codes; Tally.scores uniform {out['uniform']['median_s'] * 1e3:.2f} ms, 95 % in state 0 "
          f"{out['skewed']['median_s'] * 1e3:.2f} ms", flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[1_000_000, 10_000_000])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from sorobn_b200 import BayesNet, examples, synthetic

    results = {"gpu": gpu_limits(), "runs": []}
    print("gpu:", results["gpu"], flush=True)
    dag40 = synthetic.load(synthetic.random_dag(40, 3, (2, 3, 4), seed=args.seed), BayesNet, seed=args.seed)
    for n in args.rows:
        results["runs"].append(run_frame("alarm", examples.alarm(seed=args.seed).sample(n), args.reps))
        results["runs"].append(run_frame("dag40", dag40.sample(n), args.reps))
        results["runs"].append(run_skew(n, args.reps, args.seed))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1, default=str)


if __name__ == "__main__":
    main()
