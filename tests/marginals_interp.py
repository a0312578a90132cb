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


def run(words, table_blob, ev_codes, n_rows=None, dtype=np.float64, min_total=None):
    """Execute the program.  ev_codes: uint8 [n_ev, B].  Returns the posterior [Q, B], every target's
    segment normalised per row (NaN for a row whose segment is out of range)."""
    hdr, tables, slots, steps = parse(words)
    if min_total is None:
        min_total = 1e-30 if dtype == np.float32 else 1e-290
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
        acc = np.zeros((n_out, rows), dtype=dtype)
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
            acc = (acc + prod).astype(dtype)
        if st["kind"] == 2:
            if acc.shape[1] != B:
                acc = np.repeat(acc, B, axis=1)
            total = acc.sum(axis=0, dtype=dtype)
            lo = np.where(acc > 0, acc, np.inf).min(axis=0)
            with np.errstate(invalid="ignore", divide="ignore"):
                ok = (total >= min_total) & (lo >= min_total)
                seg = np.where(ok[None, :], acc / total[None, :], np.nan).astype(dtype)
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
