"""CPU interpreter of sample programs (version 7; TEST INFRASTRUCTURE, not product).

It parses the words of `planner.build_sample_plan` -- the upward pass in the version-4 step layout,
then the kind-4 sample steps (see the planner's module docstring) -- and executes them with numpy in
float64 or float32.  The sample steps follow the kernel's arithmetic (csrc/sbn_sample.cuh) exactly:

* w_z = product of the input entries in input order, in the program's type, multiplies only;
* total and the cumulative sums = float64 sums of w_z in z order;
* u = ((w0 >> 5) * 2^26 + (w1 >> 6)) * 2^-53 from Philox-4x32-10 with key (seed lo, seed hi) and
  counter (sample-step index, draw, row lo, row hi), row = row_base + position in the batch;
* the draw is the first z with cum_z > u * total, else the last z with w_z > 0 (else 0).

A row whose P(observed), or any step's total, is below `min_total` (or zero / NaN) comes back with
P(observed) NaN.  `given` (drawn codes [n_sampled, n_draws, B], e.g. the device's) replaces the
interpreter's own earlier draws in every gather, so each step can be checked on its own.
"""
from __future__ import annotations

import numpy as np

from oracle.sampler_replay import philox4x32

MAGIC = 0x53424E31
HEADER_WORDS = 12
KIND_SAMPLE = 4


def parse(words):
    w = [int(x) for x in np.asarray(words).tolist()]
    assert w[0] == MAGIC, "bad magic"
    assert w[1] == 7, f"version {w[1]}: not a sample program"
    hdr = dict(version=w[1], mode=w[2], n_ev=w[3], n_tables=w[4], n_slots=w[5], n_steps=w[6], Q=w[7],
               p_slot=w[8], p_batched=w[9], n_sampled=w[10])
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
        if kind == KIND_SAMPLE:
            assert n_axes == 0 and out_slot == -1
            st["d_first"] = w[p]
            p += 1
        else:
            assert kind in (0, 1), f"kind {kind} in a sample program"
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


def uniforms(seed, k, n_draws, rows):
    """[n_draws, len(rows)] float64 uniforms of sample step k (rows: global row indices)."""
    seed = int(seed) & (2**64 - 1)
    rows = np.asarray(rows, dtype=np.uint64)
    d = np.repeat(np.arange(n_draws, dtype=np.uint32)[:, None], len(rows), axis=1)
    lo = np.broadcast_to((rows & np.uint64(0xFFFFFFFF)).astype(np.uint32), d.shape)
    hi = np.broadcast_to((rows >> np.uint64(32)).astype(np.uint32), d.shape)
    out = philox4x32([np.full(d.shape, k, dtype=np.uint32), d, lo, hi], (seed & 0xFFFFFFFF, seed >> 32))
    w0, w1 = out[0].astype(np.uint64), out[1].astype(np.uint64)
    return ((w0 >> np.uint64(5)).astype(np.float64) * 2.0**26 + (w1 >> np.uint64(6)).astype(np.float64)) * 2.0**-53


def run(words, table_blob, ev_codes, n_rows=None, n_draws=1, seed=0, row_base=0, dtype=np.float64, min_total=None,
        given=None):
    """Execute the program.  ev_codes: uint8 [n_ev, B].  Returns (drawn uint8 [n_sampled, n_draws, B],
    P(observed) [B] in `dtype`, NaN for a flagged row, per-step list of dicts with `d_first`, `cards`,
    `cond` (the float64 normalised conditional [cz, n_draws, B]) and `margin` (|u * total - nearest
    cumulative sum| / total [n_draws, B]))."""
    hdr, tables, slots, steps = parse(words)
    if min_total is None:
        min_total = 1e-30 if dtype == np.float32 else 1e-290
    n_ev = hdr["n_ev"]
    ev_codes = np.asarray(ev_codes, dtype=np.uint8)
    if n_ev:
        ev_codes = ev_codes.reshape(n_ev, -1)
        B = ev_codes.shape[1]
    else:
        B = 1 if n_rows is None else int(n_rows)
    D = int(n_draws)
    blob = np.asarray(table_blob, dtype=dtype)
    tabs = [blob[o:o + s] for o, s in tables]
    bufs = [None] * len(slots)
    drawn = np.zeros((hdr["n_sampled"], D, B), dtype=np.uint8)
    src_codes = drawn if given is None else np.asarray(given, dtype=np.uint8).reshape(drawn.shape)
    flagged = np.zeros(B, dtype=bool)
    info = []

    def evoff(axes, rows):
        off = np.zeros(rows, dtype=np.int64)
        for col, s, c in axes:
            off = off + np.minimum(ev_codes[col, :rows].astype(np.int64), c - 1) * s
        return off

    def termoff(axes):  # [D, B]: observed columns and earlier draws
        off = np.zeros((D, B), dtype=np.int64)
        for col, s, c in axes:
            codes = ev_codes[col][None, :] if col < n_ev else src_codes[col - n_ev]
            off = off + np.minimum(codes.astype(np.int64), c - 1) * s
        return off

    k_sample = 0
    for st in steps:
        if st["kind"] == KIND_SAMPLE:
            ecards = st["ecards"]
            cz = int(np.prod(ecards, dtype=np.int64))
            zd = _digits(cz, ecards)
            w = np.empty((cz, D, B), dtype=dtype)
            for z in range(cz):
                prod = None
                for inp in st["inputs"]:
                    off = termoff(inp["ev"]) + sum(int(d[z]) * s for d, s in zip(zd, inp["estrides"]))
                    src = bufs[inp["buf"]] if inp["is_slot"] else tabs[inp["buf"]]
                    if inp["batched"]:
                        vals = src[off, np.arange(B)[None, :]]
                    else:
                        vals = src.reshape(-1)[off]
                    prod = vals.astype(dtype) if prod is None else (prod * vals).astype(dtype)
                w[z] = prod if prod is not None else dtype(1)
            w64 = w.astype(np.float64)
            cum = np.cumsum(w64, axis=0)  # sequential float64 sums in z order
            total = cum[-1]
            u = uniforms(seed, k_sample, D, row_base + np.arange(B))
            thr = u * total
            with np.errstate(invalid="ignore"):
                above = cum > thr[None]
                bad = ~(total >= min_total)
            first = np.where(above.any(axis=0), above.argmax(axis=0), -1)
            pos = w64 > 0
            last_pos = np.where(pos.any(axis=0), cz - 1 - pos[::-1].argmax(axis=0), 0)
            pick = np.where(first >= 0, first, last_pos)
            for j, d in enumerate(zd):
                drawn[st["d_first"] + j] = d[pick].astype(np.uint8)
            flagged |= bad.any(axis=0)
            with np.errstate(invalid="ignore", divide="ignore"):
                cond = w64 / total[None]
                margin = np.min(np.abs(cum - thr[None]), axis=0) / total
            info.append(dict(d_first=st["d_first"], cards=tuple(ecards), cond=cond, margin=margin))
            k_sample += 1
            continue
        cards = st["cards"]
        n_out = int(np.prod(cards, dtype=np.int64)) if cards else 1
        digits = _digits(n_out, cards)
        assert all(not (i["is_slot"] and i["buf"] == st["out_slot"]) for i in st["inputs"]), "output aliases an input"
        rows = B if st["kind"] == 1 else 1
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
                src = bufs[inp["buf"]] if inp["is_slot"] else tabs[inp["buf"]]
                if inp["batched"]:
                    assert inp["is_slot"] and src.ndim == 2 and not inp["ev"]
                    vals = src[off][:, :rows]
                else:
                    vals = src.reshape(-1)[off[:, None] + evoff(inp["ev"], rows)[None, :]]
                prod = (prod * vals).astype(dtype)
            acc = (acc + prod).astype(dtype)
        if st["kind"] == 1:
            bufs[st["out_slot"]] = acc
        else:
            bufs[st["out_slot"]] = acc.reshape(-1)
    src = bufs[hdr["p_slot"]]
    p_row = (src[0] if hdr["p_batched"] else np.repeat(src.reshape(-1)[:1], B)).astype(np.float64)
    with np.errstate(invalid="ignore"):
        ok = (p_row >= min_total) & ~flagged
    prob = np.where(ok, p_row, np.nan).astype(dtype)
    return drawn, prob, info
