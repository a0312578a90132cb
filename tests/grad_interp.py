"""CPU replay of gradient programs (version 10; TEST INFRASTRUCTURE).

A gradient program is a counts program whose count steps are weighted per row, plus one derivative readout
(kind 6) per soft variable (planner module docstring).  `parse` reads its words; the steps then run on
`oracle.program_interp`'s executor, whose kind-0 / kind-1 contraction, gathers and run-wise readout sums are
the kernels', and the likelihood slots are filled by `soft_interp.soft_pack`, as the device's pack fills them.

`run_grad` follows csrc/sbn_count.cuh (weighted) and csrc/sbn_deriv.cuh: a count contribution is multiplied
by w_b / P_b in float64, a fully observed family adds w_b, a readout is divided by P_b in float64, and a row
whose P(observed) is out of range adds nothing and reads NaN.  `forward=True` runs only `forward_steps`, the
closure of P(observed), as the forward call does.
"""
from __future__ import annotations

import numpy as np

import soft_interp
from oracle import program_interp as pi

KIND_DERIV = 6
VERSION_GRAD = 10


def parse(words):
    """(header, tables, slots, soft section [(slot, card)], steps) of a version-10 program."""
    w = [int(x) for x in np.asarray(words).tolist()]
    assert w[0] == pi.MAGIC and w[1] == VERSION_GRAD, "not a gradient program"
    hdr = dict(version=10, mode=w[2], n_ev=w[3], n_tables=w[4], n_slots=w[5], n_steps=w[6], Q=w[7], post_slot=w[8],
               post_batched=w[9], n_counts=w[10], n_soft=w[11])
    p = pi.HEADER_WORDS

    def take(n):
        nonlocal p
        p += n
        return w[p - n:p]

    def terms(n):
        return [tuple(take(3)) for _ in range(n)]

    tables = [tuple(take(2)) for _ in range(hdr["n_tables"])]
    slots = [tuple(take(2)) for _ in range(hdr["n_slots"])]
    soft = [tuple(take(2)) for _ in range(hdr["n_soft"])]
    steps = []
    for _ in range(hdr["n_steps"]):
        kind, n_in, out_slot, n_axes, n_elim = take(5)
        assert kind in (pi.KIND_FLAT, pi.KIND_BATCHED, pi.KIND_COUNT, KIND_DERIV), f"kind {kind} in a gradient program"
        st = dict(kind=kind, out_slot=out_slot, reduce=pi.REDUCE_SUM)
        if kind == KIND_DERIV:
            st["q_offset"], = take(1)
            assert out_slot == -1 and n_axes == 1
        elif kind == pi.KIND_COUNT:
            st["c_offset"], n_key = take(2)
            st["key"] = terms(n_key)
            st["cstrides"] = take(n_axes)
        st["cards"] = take(n_axes)
        st["ecards"] = take(n_elim)
        st["inputs"] = []
        for _ in range(n_in):
            is_slot, buf, batched, n_ev = take(4)
            st["inputs"].append(dict(is_slot=is_slot, buf=buf, batched=batched, ev=terms(n_ev), estrides=take(n_elim),
                                     strides=take(n_axes)))
        steps.append(st)
    assert p == len(w), (p, len(w))
    return hdr, tables, slots, soft, steps


def _program(words, table_blob, ev_codes, n_rows, dtype):
    """program_interp's executor over the parsed words (its own parser knows versions 4 to 9)."""
    hdr, tables, slots, soft, steps = parse(words)
    prog = pi._Program.__new__(pi._Program)
    prog.hdr, prog.steps = hdr, steps
    prog.n_ev = hdr["n_ev"]
    prog.ev = np.asarray(ev_codes, dtype=np.uint8)
    if prog.n_ev:
        prog.ev = prog.ev.reshape(prog.n_ev, -1)
        prog.B = prog.ev.shape[1]
    else:
        prog.B = int(n_rows)
    prog.dtype = dtype
    prog.unit, prog.combine = dtype(1), np.multiply
    blob = np.asarray(table_blob, dtype=dtype)
    prog.tabs = [blob[o:o + s] for o, s in tables]
    prog.bufs = [None] * len(slots)
    return prog, soft


def run_grad(words, table_blob, ev_codes, weights=None, lik=None, n_rows=None, dtype=np.float64, min_total=None,
             forward_steps=None):
    """Execute a gradient program.  `lik` [B, n_lik] (programs with soft variables), `weights` [B] float64.

    Backward (weights given): (weighted counts [n_counts], derivative readouts [n_lik, B] in `dtype` (NaN on
    flagged rows), P(observed, lik / max) [B] in `dtype`, sum log(max) [B]).  Forward (`forward_steps`, the
    plan's, and no weights): (P(observed, lik / max) [B], sum log(max) [B])."""
    prog, soft = _program(words, table_blob, ev_codes, n_rows, dtype)
    min_total = pi._min_total(min_total, dtype)
    B = prog.B
    if soft:
        packed, log_max = soft_interp.soft_pack(soft, lik, dtype)
        for (slot, _), vals in zip(soft, packed):
            prog.bufs[slot] = vals
    else:
        log_max = np.zeros(B)
    if forward_steps is not None:
        keep = set(forward_steps)
        for i, st in enumerate(prog.steps):
            assert st["kind"] in (0, 1) or i not in keep
            if i in keep:
                prog.contract(st)
        return pi._p_observed(prog, min_total), log_max
    w = np.asarray(weights, dtype=np.float64).reshape(B)
    counts = np.zeros(prog.hdr["n_counts"], dtype=np.float64)
    deriv = np.full((prog.hdr["Q"] - 1, B), np.nan, dtype=dtype)
    prob = None
    for st in prog.steps:
        if st["kind"] in (0, 1):
            prog.contract(st)
            continue
        if prob is None:
            prob = pi._p_observed(prog, min_total)
        ok = ~np.isnan(prob)
        p64 = prob.astype(np.float64)
        if st["kind"] == KIND_DERIV:
            acc = prog.sum(st, B, np.float64, runs=True)
            with np.errstate(invalid="ignore", divide="ignore"):
                val = acc / p64[None, :]
            q0 = st["q_offset"] - 1
            deriv[q0:q0 + acc.shape[0]] = np.where(ok[None, :], val, np.nan).astype(dtype)
            continue
        n_out = int(np.prod(st["cards"], dtype=np.int64))
        if st["inputs"]:
            acc = prog.sum(st, B, np.float64, runs=True)
            with np.errstate(invalid="ignore", divide="ignore"):
                acc = acc * (w / p64)[None, :]
        else:
            acc = np.repeat(w[None, :], n_out, axis=0)
        coff = np.zeros(n_out, dtype=np.int64)
        for d, s in zip(pi._digits(n_out, st["cards"]), st["cstrides"]):
            coff += d * s
        idx = st["c_offset"] + coff[:, None] + prog.offsets(st["key"], (B,))[None, :]
        np.add.at(counts, idx[:, ok].reshape(-1), acc[:, ok].reshape(-1))
    return counts, deriv, prob, log_max
