"""A/B of the expanding product's two kernels (csrc/sbn_triple_rows.cu: persistent CTAs fed by a TMA ring, against
csrc/sbn_pair.cu's sbn_triple_kernel) on one workload and batch, device-resident codes.  The two alternate
(SOROBN_B200_TRIPLE_ROWS=1 / 0, read at every launch; the graph is re-captured after each switch), each round
times 10 replays after 3 warm-ups with CUDA events and takes the per-launch profile; the fused triple launch and,
for reference, the other launches over 300 us are printed per round.  The outputs of the two must be bitwise equal.
   python tools/triple_ab.py grid10x10 [rows] [rounds]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from sorobn_b200 import engine, planner, workloads  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "grid10x10"
wl = workloads.WORKLOADS[name]()
rows = int(sys.argv[2]) if len(sys.argv) > 2 else wl.default_rows
rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 3
bn = wl.build()
net = bn._compiled
plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
prog = engine.Program(plan)
prog.reserve(rows)
roles = prog.step_roles()
triple = [int(i) for i in np.flatnonzero((roles == 4) | (roles == 5))]
print(f"{name} rows={rows} triple launch at step(s) {triple} (roles 4/5)  info={prog.info()}")
codes = wl.codes(bn, rows, seed=1000)
d_ev = torch.from_numpy(codes).cuda()
d_out = torch.empty((prog.Q, rows), dtype=torch.float32, device="cuda")
stream = torch.cuda.current_stream().cuda_stream
arms = (("rows", "1"), ("triple", "0"))
res, step_ms, triple_us = {}, {}, {label: [] for label, _ in arms}
for rnd in range(rounds):
    for label, env in arms:
        os.environ["SOROBN_B200_TRIPLE_ROWS"] = env
        prog.set_tiled(11)  # drops the captured graph: the next run captures the kernel this arm selects
        for _ in range(3):
            prog.run_device(d_ev.data_ptr(), rows, rows, d_out.data_ptr(), rows, stream)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(10):
            prog.run_device(d_ev.data_ptr(), rows, rows, d_out.data_ptr(), rows, stream)
        e.record()
        torch.cuda.synchronize()
        res[label] = d_out.cpu().numpy().copy()
        prog.profile(d_ev.data_ptr(), rows, rows, d_out.data_ptr(), rows, stream)
        ms = prog.profile(d_ev.data_ptr(), rows, rows, d_out.data_ptr(), rows, stream)
        step_ms[label] = ms
        us = [float(ms[i]) * 1000 for i in triple]
        triple_us[label].append(sum(us))
        print(f"round {rnd} {label:7s} {s.elapsed_time(e) / 10:8.3f} ms/step  triple launch us: "
              + " ".join(f"{i}:{u:.0f}" for i, u in zip(triple, us)))
os.environ.pop("SOROBN_B200_TRIPLE_ROWS")
for label, _ in arms:
    v = triple_us[label]
    print(f"{label:7s} triple launch us: median {np.median(v):.0f}  min {min(v):.0f}  max {max(v):.0f}")
    print(f"{label:7s} launches over 300 us:", " ".join(f"{i}:{float(x) * 1000:.0f}" for i, x in enumerate(step_ms[label][:-1])
                                                       if x > 0.3))
print("outputs bitwise equal:", bool(np.array_equal(res["rows"], res["triple"], equal_nan=True)))
