"""CPU replay of joint programs (version 11; TEST INFRASTRUCTURE).

A joint program is a counts program whose count steps are per-row readouts (kind 7; planner module docstring).
`parse` reads its words; the steps then run on `oracle.program_interp`'s executor, whose kind-0 / kind-1
contraction, gathers and run-wise readout sums are the kernels', and the likelihood slots are filled by
`soft_interp.soft_pack`, as the device's pack fills them.

`run_joint` follows csrc/sbn_count.cuh (`sbn_joint_step`): the products of a readout are summed in the
program's type over runs of READOUT_RUN joint states, then in float64; each entry is divided by the row's
P(observed) in float64 and rounded once to the program's type; a row whose P(observed) is out of range reads
NaN throughout.
"""
from __future__ import annotations

import numpy as np

import soft_interp
from oracle import program_interp as pi

KIND_JOINT = 7
VERSION_JOINT = 11


def parse(words):
    """(header, tables, slots, soft section [(slot, card)], steps) of a version-11 program."""
    w = [int(x) for x in np.asarray(words).tolist()]
    assert w[0] == pi.MAGIC and w[1] == VERSION_JOINT, "not a joint program"
    hdr = dict(version=11, mode=w[2], n_ev=w[3], n_tables=w[4], n_slots=w[5], n_steps=w[6], Q=w[7], post_slot=w[8],
               post_batched=w[9], n_soft=w[11])
    assert w[2] == 1 and w[10] == 0, "bad joint header"
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
        assert kind in (pi.KIND_FLAT, pi.KIND_BATCHED, KIND_JOINT), f"kind {kind} in a joint program"
        st = dict(kind=kind, out_slot=out_slot, reduce=pi.REDUCE_SUM)
        if kind == KIND_JOINT:
            st["q_offset"], = take(1)
            assert out_slot == -1 and n_axes >= 1 and n_in >= 1
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


def run_joint(words, table_blob, ev_codes, lik=None, n_rows=None, dtype=np.float64, min_total=None):
    """Execute a joint program.  `lik` [B, n_lik] for a program with soft variables.  Returns (output [Q, B] in
    `dtype`, NaN on flagged rows; P(observed, lik / max) [B] in `dtype`, NaN where flagged; sum log(max) [B])."""
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
    min_total = pi._min_total(min_total, dtype)
    B = prog.B
    if soft:
        packed, log_max = soft_interp.soft_pack(soft, lik, dtype)
        for (slot, _), vals in zip(soft, packed):
            prog.bufs[slot] = vals
    else:
        log_max = np.zeros(B)
    out = np.full((hdr["Q"], B), np.nan, dtype=dtype)
    written = np.zeros(hdr["Q"], dtype=np.int64)
    prob = None
    for st in prog.steps:
        if st["kind"] != KIND_JOINT:
            prog.contract(st)
            continue
        if prob is None:  # P(observed): the header's slot, written by the steps before
            prob = pi._p_observed(prog, min_total)
        acc = prog.sum(st, B, np.float64, runs=True)
        with np.errstate(invalid="ignore", divide="ignore"):
            val = acc / prob.astype(np.float64)[None, :]
        q0 = st["q_offset"]
        out[q0:q0 + acc.shape[0]] = np.where(np.isnan(prob)[None, :], np.nan, val).astype(dtype)
        written[q0:q0 + acc.shape[0]] += 1
    assert (written == 1).all(), "an output row is not written by exactly one joint step"
    if prob is None:
        prob = pi._p_observed(prog, min_total)
    return out, prob, log_max
