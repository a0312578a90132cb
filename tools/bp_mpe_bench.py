"""Time max-product belief propagation on the device (the max-product instantiations of csrc/sbn_bp.cu).

Workloads, as in tools/bp_bench.py: the benchmark's 10x10 grid with 5 states (30 observed cells,
`workloads.grid10x10`), and a 16x16 grid with 3 states observed on its last row and the rest of its last column
(30 cells), which the exact MPE planner refuses (checked here: `planner.build_mpe_plan` must raise).  Each runs 100k
evidence rows with tol=0 and damping 0.5, so that every row runs exactly the sweeps asked for.  Reported per
workload:
  * ms per sweep: (t(1 + N sweeps) - t(1 sweep)) / N, each t the best of `--repeat` host-clock timings of
    `BeliefPropagation.mpe` after one warm-up call.  A call ends in a stream synchronise, and the evidence upload,
    the message initialisation, the decode, the score and the download are the same in both calls, so the
    difference is the device time of N sweeps;
  * the bytes of message state one sweep accesses (`bp.Graph.message_bytes_per_sweep`) and the rate that gives;
  * the whole call with N sweeps.
On the 10x10 grid only, exact `mpe_many` runs on the same rows: its time, and for the timed BP call (1 + N sweeps,
tol 0) and for `mpe_many(algorithm="bp")` at its defaults (100 sweeps, damping 0.5, tol 1e-5; its time and the rows
that did not converge) the fraction of rows whose BP decode equals the exact MPE and the median and largest gap
exact log P - BP log P.  The card's name and power limit are read in the same run.

    python tools/bp_mpe_bench.py [--rows 100000] [--sweeps 20] [--repeat 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import warnings

import numpy as np
import pandas as pd

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bp_bench import best, card  # noqa: E402
from sorobn_b200 import BayesNet, bp, engine, planner, synthetic, workloads  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--sweeps", type=int, default=20)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    if engine.device_count() == 0:
        raise SystemExit("bp_mpe_bench needs a GPU")
    name, power = card()
    wl = workloads.grid10x10()
    ev16 = tuple(sorted([f"g15{j:02d}" for j in range(16)] + [f"g{i:02d}15" for i in range(1, 15)]))
    cases = [("grid10x10s5", wl.spec, wl.evidence), ("grid16x16s3", synthetic.grid(16, 16, 3), ev16)]
    results = []
    for label, spec, evidence in cases:
        bn = synthetic.load(spec, BayesNet)
        net = bn._compiled
        ev = [net.index[e] for e in evidence]
        try:
            planner.build_mpe_plan(net, tuple(sorted(ev)))
            exact_plans = True
        except ValueError:
            exact_plans = False
        if label == "grid16x16s3" and exact_plans:
            raise SystemExit("the exact MPE planner plans the 16x16 workload: it no longer shows what BP is for")
        g = bp.compile_mpe_graph(net, ev)
        codes = np.ascontiguousarray(workloads.forward_sample_codes(net, args.rows, seed=1)[ev])
        runner = engine.BeliefPropagation(g.words, g.tables)
        t = best(lambda: runner.mpe(codes, args.rows, 1 + args.sweeps, 0.5, 0.0), args.repeat)
        t1 = best(lambda: runner.mpe(codes, args.rows, 1, 0.5, 0.0), args.repeat)
        decoded, log_p, _ = runner.mpe(codes, args.rows, 1 + args.sweeps, 0.5, 0.0)
        runner.close()
        ms_sweep = 1e3 * (t - t1) / args.sweeps
        nbytes = g.message_bytes_per_sweep() * args.rows
        row = {"workload": label, "rows": args.rows, "sweeps": args.sweeps, "factors": len(g.families),
               "variables": len(g.variables), "message_floats_per_row": 2 * g.n_edges,
               "exact_mpe_planner": "plans" if exact_plans else "refuses",
               "ms_per_call": round(1e3 * t, 3), "ms_per_call_1_sweep": round(1e3 * t1, 3),
               "ms_per_sweep": round(ms_sweep, 4),
               "message_bytes_per_sweep": int(nbytes), "message_GB_per_s": round(nbytes / (ms_sweep * 1e-3) / 1e9, 1),
               "log_p_neg_inf_rows": int(np.isneginf(log_p).sum())}
        if label == "grid10x10s5":
            events = pd.DataFrame({e: np.asarray(net.domains[net.index[e]], dtype=object)[codes[i]]
                                   for i, e in enumerate(evidence)}).infer_objects()
            row["exact_mpe_many_ms"] = round(1e3 * best(lambda: bn.mpe_many(events), args.repeat), 1)
            exact, exact_lp = bn.mpe_many(events, return_log_proba=True)
            exact_codes = np.stack([pd.Index(net.domains[v]).get_indexer(exact[net.names[v]]) for v in g.variables])

            def quality(prefix, codes_bp, lp_bp):
                gap = exact_lp.to_numpy().astype(np.float64) - lp_bp
                row[f"{prefix}decode_equals_exact_fraction"] = round(float((exact_codes == codes_bp).all(axis=0).mean()), 4)
                row[f"{prefix}log_p_gap_median"] = round(float(np.median(gap)), 5)
                row[f"{prefix}log_p_gap_max"] = round(float(np.max(gap)), 5)

            quality("", decoded, log_p)
            with warnings.catch_warnings(record=True) as caught:
                warnings.simplefilter("always", RuntimeWarning)
                t0 = time.perf_counter()
                frame, lp_default = bn.mpe_many(events, return_log_proba=True, algorithm="bp")
                row["default_mpe_many_bp_first_call_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
            row["default_warnings"] = [str(w.message) for w in caught]
            quality("default_", np.stack([pd.Index(net.domains[v]).get_indexer(frame[net.names[v]])
                                          for v in g.variables]), lp_default.to_numpy())
        results.append(row)
        print(json.dumps(row), flush=True)
    summary = {"gpu": name, "power_limit": power, "results": results}
    print(json.dumps(summary))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
