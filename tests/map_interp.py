"""CPU interpreter of marginal MAP programs (version 9; TEST INFRASTRUCTURE, not product).

It parses the words of `planner.build_map_plan` -- the version-8 words plus a reduction word on every
kind-0 / kind-1 step (see the planner's module docstring) -- and executes them with numpy on the program's
log tables, in float32 or float64:

* a kind-0 / kind-1 entry first adds its inputs for every eliminated joint state x, in input order,
  ((0 + in_0) + in_1) + ..., every addition rounded to the program's type, as the kernels do;
* reduction 0 takes the maximum of those terms (from -inf), as an MPE program; reduction 1 takes
  m + log(sum_x exp(t_x - m)) with m = max_x t_x, and -inf when m is -inf.  In float32 this follows the
  online form of the kernel's SbnLogSumExp: the running maximum and the sum rescaled when it grows.  The
  device's expf / logf and numpy's differ in the last bits, so device and replay agree to a few ulp, not
  bitwise;
* an argmax step's weight w(z) is the sum of its inputs, and the pick is the first z (first variable
  fastest) with the largest w(z), as in tests/mpe_interp.py;
* the log-probability of a row is its posterior slot, as the upward pass left it.
"""
from __future__ import annotations

import numpy as np

MAGIC = 0x53424E31
HEADER_WORDS = 12
KIND_ARGMAX = 5
REDUCE_MAX, REDUCE_LOGSUMEXP = 0, 1


def parse(words):
    w = [int(x) for x in np.asarray(words).tolist()]
    assert w[0] == MAGIC, "bad magic"
    assert w[1] == 9, f"version {w[1]}: not a marginal MAP program"
    hdr = dict(version=w[1], mode=w[2], n_ev=w[3], n_tables=w[4], n_slots=w[5], n_steps=w[6], Q=w[7],
               p_slot=w[8], p_batched=w[9], n_decoded=w[10])
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
        if kind == KIND_ARGMAX:
            assert n_axes == 0 and out_slot == -1
            st["d_first"] = w[p]
        else:
            assert kind in (0, 1), f"kind {kind} in a marginal MAP program"
            st["reduce"] = w[p]
            assert st["reduce"] in (REDUCE_MAX, REDUCE_LOGSUMEXP)
        p += 1
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


class _LogSumExp:
    """The online log-sum-exp of the kernels (SbnLogSumExp): running maximum m and sum s of exp(t - m)."""

    def __init__(self, shape, dtype):
        self.dtype = dtype
        self.m = np.full(shape, -np.inf, dtype=dtype)
        self.s = np.zeros(shape, dtype=dtype)

    def add(self, t):
        with np.errstate(invalid="ignore", over="ignore"):
            up = t > self.m
            live = ~up & (t > -np.inf)
            grown = (self.s * np.exp(self.m - t) + self.dtype(1)).astype(self.dtype)
            kept = (self.s + np.exp(t - self.m)).astype(self.dtype)
        self.s = np.where(up, grown, np.where(live, kept, self.s)).astype(self.dtype)
        self.m = np.where(up, t, self.m).astype(self.dtype)

    def finish(self):
        with np.errstate(divide="ignore", invalid="ignore"):
            out = (self.m + np.log(self.s)).astype(self.dtype)
        return np.where(self.m == -np.inf, self.dtype(-np.inf), out).astype(self.dtype)


def run(words, table_blob, ev_codes, n_rows=None, dtype=np.float32):
    """Execute the program on its log tables (`plan.table_blob` for float32, `plan.table_blob64` for
    float64).  ev_codes: uint8 [n_ev, B].  Returns (decoded codes uint8 [n_decoded, B],
    max_{x_MAP} log P(x_MAP, e) [B] in `dtype`, -inf for a row of probability zero)."""
    hdr, tables, slots, steps = parse(words)
    n_ev = hdr["n_ev"]
    ev_codes = np.asarray(ev_codes, dtype=np.uint8)
    if n_ev:
        ev_codes = ev_codes.reshape(n_ev, -1)
        B = ev_codes.shape[1]
    else:
        B = 1 if n_rows is None else int(n_rows)
    blob = np.asarray(table_blob, dtype=dtype)
    tabs = [blob[o:o + s] for o, s in tables]
    bufs = [None] * len(slots)
    decoded = np.zeros((hdr["n_decoded"], B), dtype=np.uint8)
    zero, minus_inf = dtype(0), dtype(-np.inf)

    def evoff(axes, rows):
        off = np.zeros(rows, dtype=np.int64)
        for col, s, c in axes:
            off = off + np.minimum(ev_codes[col, :rows].astype(np.int64), c - 1) * s
        return off

    def termoff(axes):  # [B]: observed columns and earlier decoded variables
        off = np.zeros(B, dtype=np.int64)
        for col, s, c in axes:
            codes = ev_codes[col] if col < n_ev else decoded[col - n_ev]
            off = off + np.minimum(codes.astype(np.int64), c - 1) * s
        return off

    for st in steps:
        if st["kind"] == KIND_ARGMAX:
            ecards = st["ecards"]
            cz = int(np.prod(ecards, dtype=np.int64))
            zd = _digits(cz, ecards)
            w = np.empty((cz, B), dtype=dtype)
            for z in range(cz):
                acc = np.full(B, zero, dtype=dtype)
                for inp in st["inputs"]:
                    off = termoff(inp["ev"]) + sum(int(d[z]) * s for d, s in zip(zd, inp["estrides"]))
                    src = bufs[inp["buf"]] if inp["is_slot"] else tabs[inp["buf"]]
                    vals = src[off, np.arange(B)] if inp["batched"] else src.reshape(-1)[off]
                    acc = (acc + vals).astype(dtype)
                w[z] = acc
            pick = np.argmax(w, axis=0)  # the first maximum: a later z wins only by a strict >
            for j, d in enumerate(zd):
                decoded[st["d_first"] + j] = d[pick].astype(np.uint8)
            continue
        cards = st["cards"]
        n_out = int(np.prod(cards, dtype=np.int64)) if cards else 1
        digits = _digits(n_out, cards)
        assert all(not (i["is_slot"] and i["buf"] == st["out_slot"]) for i in st["inputs"]), "output aliases an input"
        rows = B if st["kind"] == 1 else 1
        lse = st["reduce"] == REDUCE_LOGSUMEXP
        acc = _LogSumExp((n_out, rows), dtype) if lse else np.full((n_out, rows), minus_inf, dtype=dtype)
        cx = int(np.prod(st["ecards"], dtype=np.int64)) if st["ecards"] else 1
        for x in range(cx):
            xd, rem_x = [], x
            for c in st["ecards"]:
                xd.append(rem_x % c)
                rem_x //= c
            term = np.full((n_out, rows), zero, dtype=dtype)
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
                term = (term + vals).astype(dtype)
            if lse:
                acc.add(term)
            else:
                acc = np.maximum(acc, term)
        out = acc.finish() if lse else acc
        bufs[st["out_slot"]] = out if st["kind"] == 1 else out.reshape(-1)
    src = bufs[hdr["p_slot"]]
    log_p = (src[0] if hdr["p_batched"] else np.repeat(src.reshape(-1)[:1], B)).astype(dtype)
    return decoded, log_p
