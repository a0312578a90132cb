"""Which step-kernel variants a program launches, as observed on the GPU.

`census(program, codes, n_rows)` runs `Program.run` once under `torch.profiler` (CUDA activities,
graph replay off, so that every launch is recorded as its own kernel) and returns the demangled
names of the kernels that ran.  The template arguments in those names are the variant, for
example `sbn_pair_kernel<2, 1>` or `sbn_step_tiled<1, 1, 1, 0, 5, 2, 5, false, false>`.  What ran is
read from the device's own record, so the census cannot drift from the dispatch code.

`variants(names)` turns those names into the coverage items of tests/kernel_corpus.py.
"""
from __future__ import annotations

import json
import os
import re
import tempfile

_KERNEL = re.compile(r"\b(sbn_\w+?)(?:<([^()]*)>)?\(")


def census(program, codes, n_rows):
    """Kernel launches of one `program.run(codes, n_rows)`: a sorted list of (name, block y)."""
    return census_many([(program, codes, n_rows)])[0]


def census_many(runs, per_session=10):
    """`census` of several (program, codes, n_rows) runs, `per_session` runs per profiler session
    (a long session can lose activity records).  Each run ends in a device synchronise and is
    followed by a marker kernel from torch, so the kernels between two markers, in device time
    order, belong to one run."""
    if len(runs) > per_session:
        return [s for lo in range(0, len(runs), per_session) for s in census_many(runs[lo:lo + per_session], per_session)]
    import torch
    from torch.profiler import ProfilerActivity, profile

    marker = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    for program, _, _ in runs:
        program.set_graph(False)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for program, codes, n_rows in runs:
            program.run(codes, n_rows)
            marker.add_(1.0)
            torch.cuda.synchronize()
    for program, _, _ in runs:
        program.set_graph(True)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    kernels = sorted((ev for ev in trace.get("traceEvents", []) if ev.get("cat") == "kernel"), key=lambda ev: ev["ts"])
    out = [set() for _ in runs]
    k = 0
    for ev in kernels:
        m = _KERNEL.search(ev.get("name", ""))
        if m is None:  # the marker: the next run starts
            k += 1
            continue
        assert k < len(runs), "kernel launched after the last run"
        block = ev.get("args", {}).get("block", [0, 1, 1])
        name = m.group(1) + (f"<{m.group(2)}>" if m.group(2) is not None else "")
        out[k].add((name, int(block[1])))
    assert k == len(runs), f"{k} markers for {len(runs)} runs: the profiler did not record every kernel"
    return [sorted(s) for s in out]


def _targs(s):
    return tuple(a.strip() for a in s.split(","))


def variants(launches):
    """Coverage items (strings) of a census.  Tiled: the input combination, tile edge, preload
    width, slab and several-eliminated-variables flags; batched: inputs and preload width; pairs:
    the two coefficient modes; triples: the group axis (the CTA's second block dimension); the join
    kernel: its input combination; the readout of marginals programs: element type and accumulator
    count, `marginal<float,2>` ... `marginal<double,8>`.

    The log-domain instantiations (MPE and marginal MAP programs) carry their policy as a trailing
    template argument and get items of their own, never a sum-product one: `batched N_IN=k SbnMaxSum`,
    `batched N_IN=k SbnLogSumExp`, `flat<float> SbnMaxSum`, `flat<float> SbnLogSumExp`, and `argmax`
    for the decode step."""
    out = set()
    for name, block_y in launches:
        m = re.match(r"(\w+)(?:<(.*)>)?$", name)
        kernel, targs = m.group(1), _targs(m.group(2)) if m.group(2) else ()
        if kernel == "sbn_step_batched" and len(targs) == 3:
            out.add(f"batched N_IN={targs[0]} {targs[2]}")
        elif kernel == "sbn_step_flat" and len(targs) == 2:
            out.add(f"flat<{targs[0]}> {targs[1]}")
        elif kernel == "sbn_argmax_step":
            out.add("argmax")
        elif kernel == "sbn_step_tiled":
            nu, na, nb, nc, t, _v, cx, slab, mx = targs
            combo = f"({nu},{na},{nb},{nc})"
            if slab == "true":
                out.add(f"slab NU={nu} T={t} CX={cx}")
                continue
            out.add(f"tiled {combo}")
            if mx == "true":
                out.add(f"tiled MX cx_inner={cx}")
                out.add(f"tiled {combo} T={t} CX={cx} MX")
            else:
                out.add(f"tiled T={t} CX={cx}")
                out.add(f"tiled {combo} T={t} CX={cx}")
            if nc != "0":
                out.add(f"tiled C-side T={t}")
        elif kernel == "sbn_step_batched":
            n_in, cx = targs
            out.add(f"batched N_IN={n_in}")
            out.add(f"batched CX={cx}")
        elif kernel == "sbn_step_batched_f64":
            out.add("batched_f64")
        elif kernel == "sbn_step_flat":
            out.add(f"flat<{targs[0]}>")
        elif kernel == "sbn_pair_kernel":
            out.add(f"pair ({targs[0]},{targs[1]})")
        elif kernel == "sbn_triple_kernel":
            out.add(f"triple group={block_y}")
        elif kernel == "sbn_join_kernel":
            out.add("join ({},{},{})".format(*targs))
        elif kernel == "sbn_marginal_step":
            out.add(f"marginal<{targs[0]},{targs[1]}>")
    return out
