"""Where a marginals program's time goes: per-step device time (CUDA events between launches, one
run) of the benchmark grid's marginals program, summed by step kind (upward / downward messages
are kind 1, readouts kind 2).

    python tools/marginals_profile.py [--rows 100000]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000)
    args = ap.parse_args()
    import torch

    from sorobn_b200 import engine, planner, workloads

    wl = workloads.grid10x10()
    bn = wl.build(device=0)
    net = bn._compiled
    plan = planner.build_marginals_plan(net, [net.index[e] for e in wl.evidence])
    prog = engine.Program(plan, device=0)
    n = args.rows
    d_ev = torch.from_numpy(np.ascontiguousarray(wl.codes(bn, n, seed=1))).cuda()
    d_out = torch.empty((plan.Q, n), dtype=torch.float32, device="cuda")
    sp = torch.cuda.current_stream().cuda_stream
    prog.profile(d_ev.data_ptr(), n, n, d_out.data_ptr(), n, sp)  # warm-up
    ms = prog.profile(d_ev.data_ptr(), n, n, d_out.data_ptr(), n, sp)
    by_kind = {}
    for st, t in zip(plan.steps, ms[:-1]):
        by_kind[st.kind] = by_kind.get(st.kind, 0.0) + float(t)
    readouts = sorted(((float(t), st.cx, len(st.inputs)) for st, t in zip(plan.steps, ms[:-1]) if st.kind == 2), reverse=True)
    print(json.dumps({"rows": n, "ms_by_kind": {str(k): round(v, 3) for k, v in by_kind.items()},
                      "total_ms": round(float(ms[:-1].sum()), 3),
                      "slowest_readouts_(ms, joint_states, inputs)": [(round(a, 3), b, c) for a, b, c in readouts[:5]]}))


if __name__ == "__main__":
    main()
