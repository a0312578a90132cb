"""CPU interpreter of counts programs (version 6; TEST INFRASTRUCTURE, not product).

It parses the words of `planner.build_counts_plan` -- the version-5 layout plus the kind-3 count step
(see the planner's module docstring) -- and executes them with numpy in float64 or float32, so the
whole counts plan (bucket choice, keys, strides, offsets, slot reuse) is checked without a GPU.
Arithmetic follows the count kernel (csrc/sbn_count.cuh): products in the program's type, summed in
that type over runs of READOUT_RUN joint states and then in float64; each contribution is divided by
the row's P(observed) in float64.  A row whose P(observed) is below `min_total` (or zero / NaN) adds
nothing and its probability comes back NaN.
"""
from __future__ import annotations

import numpy as np

MAGIC = 0x53424E31
HEADER_WORDS = 12
READOUT_RUN = 32  # SBN_MARG_PART


def parse(words):
    w = [int(x) for x in np.asarray(words).tolist()]
    assert w[0] == MAGIC, "bad magic"
    assert w[1] == 6, f"version {w[1]}: not a counts program"
    hdr = dict(version=w[1], mode=w[2], n_ev=w[3], n_tables=w[4], n_slots=w[5], n_steps=w[6], Q=w[7],
               p_slot=w[8], p_batched=w[9], n_counts=w[10])
    p = HEADER_WORDS
    tables = [(w[p + 2 * i], w[p + 2 * i + 1]) for i in range(hdr["n_tables"])]
    p += 2 * hdr["n_tables"]
    slots = [(w[p + 2 * i], w[p + 2 * i + 1]) for i in range(hdr["n_slots"])]
    p += 2 * hdr["n_slots"]
    steps = []
    for _ in range(hdr["n_steps"]):
        kind, n_in, out_slot, n_axes, n_elim = w[p:p + 5]
        p += 5
        st = dict(kind=kind, out_slot=out_slot)
        if kind == 3:
            st["c_offset"], n_key = w[p], w[p + 1]
            p += 2
            st["key"] = [tuple(w[p + 3 * k:p + 3 * k + 3]) for k in range(n_key)]
            p += 3 * n_key
            st["cstrides"] = w[p:p + n_axes]
            p += n_axes
        else:
            assert kind in (0, 1), f"kind {kind} in a counts program"
        st["cards"] = w[p:p + n_axes]
        p += n_axes
        st["ecards"] = w[p:p + n_elim]
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
        st["inputs"] = ins
        steps.append(st)
    assert p == len(w), (p, len(w))
    return hdr, tables, slots, steps


def _digits(n, cards):
    out, rem = [], np.arange(n, dtype=np.int64)
    for c in cards:
        out.append(rem % c)
        rem = rem // c
    return out


def run(words, table_blob, ev_codes, n_rows=None, dtype=np.float64, min_total=None):
    """Execute the program.  ev_codes: uint8 [n_ev, B].  Returns (counts float64 [n_counts],
    P(observed) [B] in `dtype`, NaN for a row out of range)."""
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
    counts = np.zeros(hdr["n_counts"], dtype=np.float64)
    written = np.zeros(hdr["n_counts"], dtype=np.int64)
    prob = None

    def evoff(axes, rows):
        off = np.zeros(rows, dtype=np.int64)
        for col, s, c in axes:
            off = off + np.minimum(ev_codes[col, :rows].astype(np.int64), c - 1) * s
        return off

    for st in steps:
        cards = st["cards"]
        n_out = int(np.prod(cards, dtype=np.int64)) if cards else 1
        digits = _digits(n_out, cards)
        assert all(not (i["is_slot"] and i["buf"] == st["out_slot"]) for i in st["inputs"]), "output aliases an input"
        count = st["kind"] == 3
        if count and prob is None:  # P(observed): the header's slot, written by the steps before
            src = bufs[hdr["p_slot"]]
            assert src is not None, "P(observed) is read before it is written"
            p_row = (src[0] if hdr["p_batched"] else np.repeat(src.reshape(-1)[:1], B)).astype(np.float64)
            with np.errstate(invalid="ignore"):
                ok = p_row >= min_total
            prob = np.where(ok, p_row, np.nan).astype(dtype)
        per_row = st["kind"] in (1, 3) or hdr["mode"] == 0
        rows = B if per_row else 1
        acc_t = np.float64 if count else dtype
        acc = np.zeros((n_out, rows), dtype=acc_t)
        cx = int(np.prod(st["ecards"], dtype=np.int64)) if st["ecards"] else 1
        if count and not st["inputs"]:
            acc[:] = 1.0
        for x in range(cx if st["inputs"] else 0):
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
                src = bufs[inp["buf"]] if inp["is_slot"] else tabs[inp["buf"]]
                if inp["batched"]:
                    assert inp["is_slot"] and src.ndim == 2 and not inp["ev"]
                    vals = src[off][:, :rows]
                else:
                    vals = src.reshape(-1)[off[:, None] + evoff(inp["ev"], rows)[None, :]]
                prod = (prod * vals).astype(dtype)
            if not count:
                acc = (acc + prod).astype(acc_t)
            else:  # partial sums in dtype over runs of READOUT_RUN joint states
                part = prod if x % READOUT_RUN == 0 else (part + prod).astype(dtype)
                if x % READOUT_RUN == READOUT_RUN - 1 or x == cx - 1:
                    acc = acc + part.astype(acc_t)
        if count:
            if acc.shape[1] != B:
                acc = np.repeat(acc, B, axis=1)
            if st["inputs"]:
                with np.errstate(invalid="ignore", divide="ignore"):
                    acc = acc * (1.0 / prob.astype(np.float64))[None, :]
            key = evoff(st["key"], B)
            coff = np.zeros(n_out, dtype=np.int64)
            for d, s in zip(digits, st["cstrides"]):
                coff += d * s
            idx = st["c_offset"] + coff[:, None] + key[None, :]
            ok_rows = ~np.isnan(prob)
            np.add.at(counts, idx[:, ok_rows].reshape(-1), acc[:, ok_rows].reshape(-1))
            _mark(written, st, coff)
        elif st["kind"] == 1:
            bufs[st["out_slot"]] = acc
        else:
            assert rows == 1
            bufs[st["out_slot"]] = acc.reshape(-1)
    assert (written == 1).all(), "a count-table entry is not covered by exactly one count step"
    return counts, prob


def _mark(written, st, coff):
    """Every entry of the family's table: the output states times every key value."""
    keys = np.zeros(1, dtype=np.int64)
    for _, s, c in st["key"]:
        keys = (keys[:, None] + np.arange(c, dtype=np.int64)[None, :] * s).reshape(-1)
    idx = st["c_offset"] + (coff[:, None] + keys[None, :]).reshape(-1)
    np.add.at(written, idx, 1)
