"""CPU interpreter of marginals programs (version 5; TEST INFRASTRUCTURE, not product).

`oracle/program_interp.py` executes the version-4 programs of `planner.build_plan`.  This module
parses the words of `planner.build_marginals_plan` -- the same layout plus the kind-2 readout step
(see the planner's module docstring) -- and executes them with numpy in float64 or float32, so the
whole bucket-tree plan (upward messages, downward messages, readouts, slot reuse) is checked
without a GPU.  Each target's segment is normalised on its own, with the engine's rule for rows
out of range (NaN when the total or the smallest non-zero entry is below `min_total`).
"""
from __future__ import annotations

import numpy as np

MAGIC = 0x53424E31
HEADER_WORDS = 12
READOUT_RUN = 32  # joint states a readout sums in the program's type before a float64 add (SBN_MARG_PART)


def parse(words):
    w = [int(x) for x in np.asarray(words).tolist()]
    assert w[0] == MAGIC, "bad magic"
    assert w[1] == 5, f"version {w[1]}: not a marginals program"
    hdr = dict(version=w[1], mode=w[2], n_ev=w[3], n_tables=w[4], n_slots=w[5], n_steps=w[6], Q=w[7],
               post_slot=w[8], post_batched=w[9])
    p = HEADER_WORDS
    tables = [(w[p + 2 * i], w[p + 2 * i + 1]) for i in range(hdr["n_tables"])]
    p += 2 * hdr["n_tables"]
    slots = [(w[p + 2 * i], w[p + 2 * i + 1]) for i in range(hdr["n_slots"])]
    p += 2 * hdr["n_slots"]
    steps = []
    for _ in range(hdr["n_steps"]):
        kind, n_in, out_slot, n_axes, n_elim = w[p:p + 5]
        p += 5
        q_offset = None
        if kind == 2:
            q_offset = w[p]
            p += 1
        cards = w[p:p + n_axes]
        p += n_axes
        ecards = w[p:p + n_elim]
        p += n_elim
        ins = []
        for _ in range(n_in):
            is_slot, buf, batched, n_ev = w[p:p + 4]
            p += 4
            ev = [tuple(w[p + 3 * k:p + 3 * k + 3]) for k in range(n_ev)]
            p += 3 * n_ev
            estrides = w[p:p + n_elim]
            p += n_elim
            strides = w[p:p + n_axes]
            p += n_axes
            ins.append(dict(is_slot=is_slot, buf=buf, batched=batched, estrides=estrides, ev=ev, strides=strides))
        steps.append(dict(kind=kind, out_slot=out_slot, q_offset=q_offset, cards=cards, ecards=ecards, inputs=ins))
    assert p == len(w), (p, len(w))
    return hdr, tables, slots, steps


def run(words, table_blob, ev_codes, n_rows=None, dtype=np.float64, min_total=None, readout_acc=None):
    """Execute the program.  ev_codes: uint8 [n_ev, B].  Returns the posterior [Q, B], every target's
    segment normalised per row (NaN for a row whose segment is out of range).

    `readout_acc` is the accumulator type of the readouts (kind 2), which sum joint states without the
    MAX_Z bound of the other steps.  By default it is float64, as in the readout kernel
    (sbn_marginal.cuh): the products are summed in `dtype` over runs of READOUT_RUN joint states, the
    partial sums in float64; the segment total, the range rule and the division are float64, and the
    result is rounded once to `dtype` (a target of more than 8 states, which the kernel reads in passes,
    has its raw sums rounded to `dtype` before the division too).  `readout_acc=np.float32` is a single
    float32 accumulator throughout, in the kernel's summation order."""
    hdr, tables, slots, steps = parse(words)
    if min_total is None:
        min_total = 1e-30 if dtype == np.float32 else 1e-290
    if readout_acc is None:
        readout_acc = np.float64
    ev_codes = np.asarray(ev_codes, dtype=np.uint8)
    if hdr["n_ev"]:
        ev_codes = ev_codes.reshape(hdr["n_ev"], -1)
        B = ev_codes.shape[1]
    else:
        B = 1 if n_rows is None else int(n_rows)
    if hdr["mode"] == 0:
        assert B == 1, "flat programs take exactly one evidence row"
    blob = np.asarray(table_blob, dtype=dtype)
    tabs = [blob[o:o + s] for o, s in tables]
    bufs = [None] * len(slots)
    post = np.full((hdr["Q"], B), np.nan, dtype=dtype)
    written = np.zeros(hdr["Q"], dtype=bool)

    for st in steps:
        cards = st["cards"]
        n_out = int(np.prod(cards, dtype=np.int64)) if cards else 1
        digits, rem = [], np.arange(n_out, dtype=np.int64)
        for c in cards:
            digits.append(rem % c)
            rem = rem // c
        assert all(not (i["is_slot"] and i["buf"] == st["out_slot"]) for i in st["inputs"]), "output aliases an input"
        per_row = st["kind"] in (1, 2) or hdr["mode"] == 0
        rows = B if per_row else 1
        acc_t = readout_acc if st["kind"] == 2 else dtype
        acc = np.zeros((n_out, rows), dtype=acc_t)
        cx = int(np.prod(st["ecards"], dtype=np.int64)) if st["ecards"] else 1
        for x in range(cx):
            xd, rem_x = [], x
            for c in st["ecards"]:
                xd.append(rem_x % c)
                rem_x //= c
            prod = np.ones((n_out, rows), dtype=dtype)
            for inp in st["inputs"]:
                off = np.zeros(n_out, dtype=np.int64)
                for d, s in zip(digits, inp["strides"]):
                    off += d * s
                off = off + sum(d * s for d, s in zip(xd, inp["estrides"]))
                evoff = np.zeros(rows, dtype=np.int64)
                for col, s, c in inp["ev"]:
                    evoff = evoff + np.minimum(ev_codes[col, :rows].astype(np.int64), c - 1) * s
                src = bufs[inp["buf"]] if inp["is_slot"] else tabs[inp["buf"]]
                if inp["batched"]:
                    assert inp["is_slot"] and src.ndim == 2 and not inp["ev"]
                    vals = src[off][:, :rows]
                else:
                    vals = src.reshape(-1)[off[:, None] + evoff[None, :]]
                prod = (prod * vals).astype(dtype)
            if acc_t == dtype:
                acc = (acc + prod).astype(acc_t)
            else:  # partial sums in dtype over runs of READOUT_RUN joint states
                part = prod if x % READOUT_RUN == 0 else (part + prod).astype(dtype)
                if x % READOUT_RUN == READOUT_RUN - 1 or x == cx - 1:
                    acc = acc + part.astype(acc_t)
        if st["kind"] == 2:
            if acc.shape[1] != B:
                acc = np.repeat(acc, B, axis=1)
            total = np.zeros(B, dtype=acc_t)
            for s in range(n_out):  # in state order, as the kernel
                total = (total + acc[s]).astype(acc_t)
            lo = np.where(acc > 0, acc, np.inf).min(axis=0)
            raw = acc.astype(dtype).astype(acc_t) if n_out > 8 else acc
            with np.errstate(invalid="ignore", divide="ignore"):
                ok = (total >= min_total) & (lo >= min_total)
                seg = np.where(ok[None, :], raw / total[None, :], np.nan).astype(dtype)
            q0 = st["q_offset"]
            post[q0:q0 + n_out] = seg
            assert not written[q0:q0 + n_out].any(), "two readouts write one posterior entry"
            written[q0:q0 + n_out] = True
        elif st["kind"] == 1:
            bufs[st["out_slot"]] = acc
        else:
            assert rows == 1
            bufs[st["out_slot"]] = acc.reshape(-1)
    assert written.all(), "a posterior entry is never written"
    return post


# A float32 readout writes NaN for a row whose total P(e), or smallest non-zero entry P(e) * p, is below
# min_total = 1e-30 (the engine re-runs such rows in float64).  A NaN segment is put down to that rule
# where the float64 answer puts either below 1e-29, a margin for float32 rounding on the way.
RANGE_RULE_F32 = 1e-29


def segment_starts(plan):
    """First posterior entry of every target's segment (targets in plan order)."""
    return np.cumsum([0] + [int(plan._card[t]) for t in plan.targets[:-1]])


def check_posterior(got, want, starts, p_event=None):
    """A marginals posterior `got` [Q, B] against the float64 answer `want`, target segment by segment
    (`starts`: segment_starts): rows `want` gives NaN (impossible evidence) must be NaN throughout;
    elsewhere every entry is finite, and exact zeros stay exactly 0.  With `p_event` ([B], the float64
    P(e) of every row: float32 runs), a segment that is NaN throughout is accepted where the float32
    range rule explains it; any other NaN fails.  Returns (worst relative error of the non-zero
    entries, number of segments accepted as NaN)."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    impossible = np.isnan(want).all(axis=0)
    assert np.isnan(got[:, impossible]).all(), f"rows {np.flatnonzero(impossible)}: impossible evidence, not NaN"
    got, want = got[:, ~impossible], want[:, ~impossible]
    rows = np.flatnonzero(~impossible)
    assert np.isfinite(want).all(), "the reference has a NaN on a possible row"
    nan_got = np.isnan(got)
    all_nan = np.logical_and.reduceat(nan_got, starts, axis=0)  # [n_segments, B]
    any_nan = np.logical_or.reduceat(nan_got, starts, axis=0)
    bad = np.argwhere(any_nan & ~all_nan)
    assert not len(bad), f"(segment, row) {[(int(s), int(rows[b])) for s, b in bad[:5]]}: partly NaN"
    flagged = 0
    if all_nan.any():
        assert p_event is not None, f"(segment, row) {[(int(s), int(rows[b])) for s, b in np.argwhere(all_nan)[:5]]}: NaN"
        p_e = np.asarray(p_event, dtype=np.float64)[~impossible]
        lo = np.minimum.reduceat(np.where(want > 0, want, np.inf), starts, axis=0) * p_e[None, :]
        unexplained = all_nan & ~((p_e[None, :] < RANGE_RULE_F32) | (lo < RANGE_RULE_F32))
        assert not unexplained.any(), \
            f"(segment, row) {[(int(s), int(rows[b])) for s, b in np.argwhere(unexplained)[:5]]}: NaN within float32 range"
        flagged = int(all_nan.sum())
    keep = ~np.repeat(all_nan, np.diff(np.append(starts, got.shape[0])), axis=0)
    zero = keep & (want == 0)
    assert (got[zero] == 0).all(), f"entries (q, row) {[(int(q), int(rows[b])) for q, b in np.argwhere(zero & (got != 0))[:5]]}: not 0"
    pos = keep & (want > 0)
    err = np.zeros_like(want)
    err[pos] = np.abs(got[pos] - want[pos]) / want[pos]
    return float(err.max(initial=0.0)), flagged
