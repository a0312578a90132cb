"""CPU interpreter of the device programs, versions 4 to 9 (TEST INFRASTRUCTURE, not product).

`sorobn_b200.planner` serialises every plan into int32 words that `csrc/sbn_api.cu` parses and runs on the
GPU (the layout is in the planner's module docstring).  This module parses the very same words with numpy
and executes them element by element, in float64 (checker) or float32 (to predict the device's rounding),
so the planner's strides, evidence gathers, bucket readouts and slot reuse are checked without a GPU.  The
version-4 posterior must equal `oracle.ve_oracle.query` (the restatement of
/root/reference/sorobn/bayes_net.py:739-794) row by row.

The arithmetic follows the kernels, operation for operation:

* a kind-0 / kind-1 entry combines its inputs for every eliminated joint state x (first variable fastest)
  in input order, every operation rounded to the program's type: a product from 1 (versions 4 to 7, the
  sum-product semiring) or a sum ((0 + in_0) + in_1) + ... (versions 8 and 9, on log tables).  It then
  reduces over x: a sum in the program's type (versions 4 to 7), a maximum from -inf (version 8, and the
  reduction word 0 of version 9), or the online log-sum-exp of SbnLogSumExp (reduction word 1 of version 9:
  the running maximum and the sum rescaled when it grows; the device's expf / logf and numpy's differ in
  the last bits, so that one agrees to a few ulp, not bitwise);
* a readout (kind 2, version 5) and a count step (kind 3, version 6) sum their products in the program's
  type over runs of READOUT_RUN joint states, then in float64 (csrc/sbn_marginal.cuh, csrc/sbn_count.cuh);
* a sample step (kind 4, version 7) draws z with probability w(z) / sum_z w(z), w(z) the product of its
  inputs, from the Philox stream of csrc/sbn_sample.cuh: the first z with cum(z) > u * total (float64
  sums in z order), else the last z with w(z) > 0 (else 0);
* an argmax step (kind 5, versions 8 and 9) picks the first z with the largest w(z), w(z) the sum of its
  inputs from 0 (csrc/sbn_mpe.cuh), so the device agrees bit for bit.

Only tests import this; the product never does.
"""
from __future__ import annotations

import numpy as np

from oracle.sampler_replay import philox4x32

MAGIC = 0x53424E31
HEADER_WORDS = 12
READOUT_RUN = 32  # joint states a readout or count step sums in the program's type before a float64 add (SBN_MARG_PART)
KIND_FLAT, KIND_BATCHED, KIND_MARGINAL, KIND_COUNT, KIND_SAMPLE, KIND_ARGMAX = range(6)
REDUCE_MAX, REDUCE_LOGSUMEXP = 0, 1  # the reduction words of version 9
REDUCE_SUM = 2  # the reduction of every kind-0 / kind-1 step of versions 4 to 7 (not a program word)
KINDS = {4: (0, 1), 5: (0, 1, 2), 6: (0, 1, 3), 7: (0, 1, 4), 8: (0, 1, 5), 9: (0, 1, 5)}


def parse(words):
    """(header, tables, slots, steps) of a program of any version."""
    w = [int(x) for x in np.asarray(words).tolist()]
    assert w[0] == MAGIC, "bad magic"
    version = w[1]
    assert version in KINDS, f"version {version}: not a program version"
    hdr = dict(version=version, mode=w[2], n_ev=w[3], n_tables=w[4], n_slots=w[5], n_steps=w[6], Q=w[7],
               post_slot=w[8], post_batched=w[9])
    if version == 6:
        hdr["n_counts"] = w[10]
    elif version >= 7:
        hdr["n_decoded"] = w[10]
    p = HEADER_WORDS

    def take(n):
        nonlocal p
        p += n
        return w[p - n:p]

    def terms(n):  # n (col stride card) triples
        return [tuple(take(3)) for _ in range(n)]

    tables = [tuple(take(2)) for _ in range(hdr["n_tables"])]
    slots = [tuple(take(2)) for _ in range(hdr["n_slots"])]
    steps = []
    for _ in range(hdr["n_steps"]):
        kind, n_in, out_slot, n_axes, n_elim = take(5)
        assert kind in KINDS[version], f"kind {kind} in a version-{version} program"
        st = dict(kind=kind, out_slot=out_slot)
        if kind == KIND_MARGINAL:
            st["q_offset"], = take(1)
        elif kind == KIND_COUNT:
            st["c_offset"], n_key = take(2)
            st["key"] = terms(n_key)
            st["cstrides"] = take(n_axes)
        elif kind in (KIND_SAMPLE, KIND_ARGMAX):
            assert n_axes == 0 and out_slot == -1
            st["d_first"], = take(1)
        elif version == 9:
            st["reduce"], = take(1)
            assert st["reduce"] in (REDUCE_MAX, REDUCE_LOGSUMEXP)
        else:
            st["reduce"] = REDUCE_MAX if version == 8 else REDUCE_SUM
        st["cards"] = take(n_axes)
        st["ecards"] = take(n_elim)
        st["inputs"] = []
        for _ in range(n_in):
            is_slot, buf, batched, n_ev = take(4)
            st["inputs"].append(dict(is_slot=is_slot, buf=buf, batched=batched, ev=terms(n_ev), estrides=take(n_elim),
                                     strides=take(n_axes)))
        steps.append(st)
    assert p == len(w), (p, len(w))
    return hdr, tables, slots, steps


def _digits(n, cards):
    """Mixed-radix digits of 0 .. n - 1, the first card fastest."""
    out, rem = [], np.arange(n, dtype=np.int64)
    for c in cards:
        out.append(rem % c)
        rem = rem // c
    return out


def _min_total(min_total, dtype):
    if min_total is not None:
        return min_total
    return 1e-30 if dtype == np.float32 else 1e-290


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


class _Program:
    """One execution of a program: its parsed words, tables, slots and evidence codes [n_ev, B]."""

    def __init__(self, words, table_blob, ev_codes, n_rows, dtype, versions):
        self.hdr, tables, slots, self.steps = parse(words)
        assert self.hdr["version"] in versions, f"version {self.hdr['version']}: not a version-{versions} program"
        self.n_ev = self.hdr["n_ev"]
        self.ev = np.asarray(ev_codes, dtype=np.uint8)
        if self.n_ev:
            self.ev = self.ev.reshape(self.n_ev, -1)
            self.B = self.ev.shape[1]
        else:
            self.B = 1 if n_rows is None else int(n_rows)
        if self.hdr["mode"] == 0:
            assert self.B == 1, "flat programs take exactly one evidence row"
        self.dtype = dtype
        log = self.hdr["version"] >= 8  # MPE and marginal MAP programs run on log tables
        self.unit, self.combine = (dtype(0), np.add) if log else (dtype(1), np.multiply)
        blob = np.asarray(table_blob, dtype=dtype)
        self.tabs = [blob[o:o + s] for o, s in tables]
        self.bufs = [None] * len(slots)

    def source(self, inp):
        return self.bufs[inp["buf"]] if inp["is_slot"] else self.tabs[inp["buf"]]

    def offsets(self, terms, shape, decided=None):
        """sum of min(code, card - 1) * stride over (col stride card) terms, [..., rows]: col < n_ev reads the
        observed column, col >= n_ev the earlier decision `decided[col - n_ev]`."""
        off = np.zeros(shape, dtype=np.int64)
        for col, s, c in terms:
            codes = self.ev[col, :shape[-1]] if col < self.n_ev else decided[col - self.n_ev]
            off = off + np.minimum(codes.astype(np.int64), c - 1) * s
        return off

    def terms(self, st, rows):
        """The term [n_out, rows] of every eliminated joint state x of a kind-0 to kind-3 step."""
        n_out = int(np.prod(st["cards"], dtype=np.int64))
        digits = _digits(n_out, st["cards"])
        assert all(not (i["is_slot"] and i["buf"] == st["out_slot"]) for i in st["inputs"]), "output aliases an input"
        gathers = []  # (input, source, offset of x = 0)
        for inp in st["inputs"]:
            src = self.source(inp)
            off = np.zeros(n_out, dtype=np.int64)
            for d, s in zip(digits, inp["strides"]):
                off += d * s
            if inp["batched"]:
                assert inp["is_slot"] and src.ndim == 2 and not inp["ev"]
            else:
                src, off = src.reshape(-1), off[:, None] + self.offsets(inp["ev"], (rows,))[None, :]
            gathers.append((inp, src, off))
        cx = int(np.prod(st["ecards"], dtype=np.int64))
        xds = _digits(cx, st["ecards"])
        for x in range(cx):
            term = np.full((n_out, rows), self.unit, dtype=self.dtype)
            for inp, src, off in gathers:
                off = off + sum(int(d[x]) * s for d, s in zip(xds, inp["estrides"]))
                vals = src[off][:, :rows] if inp["batched"] else src[off]
                term = self.combine(term, vals).astype(self.dtype)
            yield term

    def sum(self, st, rows, acc_t, runs):
        """Sum of the terms in `acc_t`; with `runs`, in the program's type over runs of READOUT_RUN joint states,
        each run then added in `acc_t`."""
        cx = int(np.prod(st["ecards"], dtype=np.int64))
        acc = np.zeros((int(np.prod(st["cards"], dtype=np.int64)), rows), dtype=acc_t)
        for x, t in enumerate(self.terms(st, rows)):
            if not runs:
                acc = (acc + t).astype(acc_t)
                continue
            part = t if x % READOUT_RUN == 0 else (part + t).astype(self.dtype)
            if x % READOUT_RUN == READOUT_RUN - 1 or x == cx - 1:
                acc = acc + part.astype(acc_t)
        return acc

    def contract(self, st):
        """A kind-0 / kind-1 step: the reduction of its terms into its output slot."""
        rows = self.B if st["kind"] == KIND_BATCHED else 1
        if st["reduce"] == REDUCE_SUM:
            out = self.sum(st, rows, self.dtype, runs=False)
        elif st["reduce"] == REDUCE_MAX:
            out = np.full((int(np.prod(st["cards"], dtype=np.int64)), rows), -np.inf, dtype=self.dtype)
            for t in self.terms(st, rows):
                out = np.maximum(out, t)
        else:
            lse = _LogSumExp((int(np.prod(st["cards"], dtype=np.int64)), rows), self.dtype)
            for t in self.terms(st, rows):
                lse.add(t)
            out = lse.finish()
        self.bufs[st["out_slot"]] = out if st["kind"] == KIND_BATCHED else out.reshape(-1)

    def weights(self, st, decided):
        """A kind-4 / kind-5 step's digits of z and w(z) [cz, D, B]: its inputs combined in input order, gathered
        at the row's observed columns and its earlier decisions `decided` [n_decoded, D, B]."""
        D, B = decided.shape[1], self.B
        cz = int(np.prod(st["ecards"], dtype=np.int64))
        zd = _digits(cz, st["ecards"])
        gathers = [(inp, self.source(inp), self.offsets(inp["ev"], (D, B), decided)) for inp in st["inputs"]]
        w = np.empty((cz, D, B), dtype=self.dtype)
        for z in range(cz):
            acc = np.full((D, B), self.unit, dtype=self.dtype)
            for inp, src, off in gathers:
                off = off + sum(int(d[z]) * s for d, s in zip(zd, inp["estrides"]))
                vals = src[off, np.arange(B)] if inp["batched"] else src.reshape(-1)[off]
                acc = self.combine(acc, vals).astype(self.dtype)
            w[z] = acc
        return zd, w

    def post_rows(self):
        """The posterior slot's value of every row [B]."""
        src = self.bufs[self.hdr["post_slot"]]
        assert src is not None, "the posterior slot is read before it is written"
        return src[0] if self.hdr["post_batched"] else np.repeat(src.reshape(-1)[:1], self.B)


def _p_observed(prog, min_total, flagged=None):
    """P(observed) of every row in the program's type, NaN below `min_total` (or zero / NaN) or where flagged."""
    p_row = prog.post_rows().astype(np.float64)
    with np.errstate(invalid="ignore"):
        ok = p_row >= min_total
    if flagged is not None:
        ok &= ~flagged
    return np.where(ok, p_row, np.nan).astype(prog.dtype)


def run(words, table_blob, ev_codes, n_rows=None, dtype=np.float64, return_totals=False):
    """Execute a posterior program (version 4).  ev_codes: uint8 array [n_ev, B] (n_rows gives B when
    there are no evidence columns).  Returns the normalised posterior [Q, B] (state-major, like the C-ABI's
    output), and with `return_totals` the normaliser P(event) of every row (sbn_program_evidence_host)."""
    prog = _Program(words, table_blob, ev_codes, n_rows, dtype, (4,))
    assert not prog.n_ev or n_rows is None or n_rows == prog.B
    for st in prog.steps:
        prog.contract(st)
    post = prog.bufs[prog.hdr["post_slot"]]
    if post.ndim == 1:
        post = np.repeat(post[:, None], prog.B, axis=1)
    post = post[:prog.hdr["Q"]]
    total = post.sum(axis=0, keepdims=True, dtype=dtype)
    with np.errstate(invalid="ignore", divide="ignore"):
        normalised = (post / total).astype(dtype)
    if return_totals:
        return normalised, total.reshape(-1)
    return normalised


def run_marginals(words, table_blob, ev_codes, n_rows=None, dtype=np.float64, min_total=None, readout_acc=None):
    """Execute a marginals program (version 5).  Returns the posterior [Q, B], every target's segment
    normalised per row: NaN for a row whose segment total, or smallest non-zero entry, is below `min_total`.

    `readout_acc` is the accumulator type of the readouts (kind 2), which sum joint states without the
    MAX_Z bound of the other steps.  By default it is float64, as in the readout kernel: the products are
    summed in `dtype` over runs of READOUT_RUN joint states, the partial sums in float64; the segment total
    (in state order), the range rule and the division are float64, and the result is rounded once to `dtype`
    (a target of more than 8 states, which the kernel reads in passes, has its raw sums rounded to `dtype`
    before the division too).  `readout_acc=np.float32` is a single float32 accumulator throughout, in the
    kernel's summation order."""
    prog = _Program(words, table_blob, ev_codes, n_rows, dtype, (5,))
    min_total = _min_total(min_total, dtype)
    acc_t = np.float64 if readout_acc is None else readout_acc
    B = prog.B
    post = np.full((prog.hdr["Q"], B), np.nan, dtype=dtype)
    written = np.zeros(prog.hdr["Q"], dtype=bool)
    for st in prog.steps:
        if st["kind"] != KIND_MARGINAL:
            prog.contract(st)
            continue
        acc = prog.sum(st, B, acc_t, runs=acc_t != dtype)
        n_out = acc.shape[0]
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
    assert written.all(), "a posterior entry is never written"
    return post


def run_counts(words, table_blob, ev_codes, n_rows=None, dtype=np.float64, min_total=None):
    """Execute a counts program (version 6).  Returns (counts float64 [n_counts], P(observed) [B] in `dtype`,
    NaN for a row out of range).  Each count step's contribution is divided by the row's P(observed) in
    float64; a row out of range adds nothing."""
    prog = _Program(words, table_blob, ev_codes, n_rows, dtype, (6,))
    min_total = _min_total(min_total, dtype)
    B = prog.B
    counts = np.zeros(prog.hdr["n_counts"], dtype=np.float64)
    written = np.zeros(prog.hdr["n_counts"], dtype=np.int64)
    prob = None
    for st in prog.steps:
        if st["kind"] != KIND_COUNT:
            prog.contract(st)
            continue
        if prob is None:  # P(observed): the header's slot, written by the steps before
            prob = _p_observed(prog, min_total)
        n_out = int(np.prod(st["cards"], dtype=np.int64))
        if st["inputs"]:
            acc = prog.sum(st, B, np.float64, runs=True)
            with np.errstate(invalid="ignore", divide="ignore"):
                acc = acc * (1.0 / prob.astype(np.float64))[None, :]
        else:  # a family with no unobserved member: each row adds 1
            acc = np.ones((n_out, B), dtype=np.float64)
        coff = np.zeros(n_out, dtype=np.int64)
        for d, s in zip(_digits(n_out, st["cards"]), st["cstrides"]):
            coff += d * s
        idx = st["c_offset"] + coff[:, None] + prog.offsets(st["key"], (B,))[None, :]
        ok_rows = ~np.isnan(prob)
        np.add.at(counts, idx[:, ok_rows].reshape(-1), acc[:, ok_rows].reshape(-1))
        # every entry of the family's table: the output states times every key value
        keys = np.zeros(1, dtype=np.int64)
        for _, s, c in st["key"]:
            keys = (keys[:, None] + np.arange(c, dtype=np.int64)[None, :] * s).reshape(-1)
        np.add.at(written, st["c_offset"] + (coff[:, None] + keys[None, :]).reshape(-1), 1)
    assert (written == 1).all(), "a count-table entry is not covered by exactly one count step"
    return counts, prob


def uniforms(seed, k, n_draws, rows):
    """[n_draws, len(rows)] float64 uniforms of sample step k (rows: global row indices):
    u = ((w0 >> 5) * 2^26 + (w1 >> 6)) * 2^-53 from Philox-4x32-10 with key (seed lo, seed hi) and counter
    (k, draw, row lo, row hi)."""
    seed = int(seed) & (2**64 - 1)
    rows = np.asarray(rows, dtype=np.uint64)
    d = np.repeat(np.arange(n_draws, dtype=np.uint32)[:, None], len(rows), axis=1)
    lo = np.broadcast_to((rows & np.uint64(0xFFFFFFFF)).astype(np.uint32), d.shape)
    hi = np.broadcast_to((rows >> np.uint64(32)).astype(np.uint32), d.shape)
    out = philox4x32([np.full(d.shape, k, dtype=np.uint32), d, lo, hi], (seed & 0xFFFFFFFF, seed >> 32))
    w0, w1 = out[0].astype(np.uint64), out[1].astype(np.uint64)
    return ((w0 >> np.uint64(5)).astype(np.float64) * 2.0**26 + (w1 >> np.uint64(6)).astype(np.float64)) * 2.0**-53


def run_sample(words, table_blob, ev_codes, n_rows=None, n_draws=1, seed=0, row_base=0, dtype=np.float64,
               min_total=None, given=None):
    """Execute a sample program (version 7).  Returns (drawn uint8 [n_decoded, n_draws, B], P(observed) [B] in
    `dtype`, NaN for a row whose P(observed) or any step's total is below `min_total` (or zero / NaN), per-step
    list of dicts with `d_first`, `cards`, `cond` (the float64 normalised conditional [cz, n_draws, B]) and
    `margin` (|u * total - nearest cumulative sum| / total [n_draws, B])).  The row of batch position b is
    row_base + b.  `given` (drawn codes [n_decoded, n_draws, B], e.g. the device's) replaces the interpreter's
    own earlier draws in every gather, so each step can be checked on its own."""
    prog = _Program(words, table_blob, ev_codes, n_rows, dtype, (7,))
    min_total = _min_total(min_total, dtype)
    D, B = int(n_draws), prog.B
    drawn = np.zeros((prog.hdr["n_decoded"], D, B), dtype=np.uint8)
    decided = drawn if given is None else np.asarray(given, dtype=np.uint8).reshape(drawn.shape)
    flagged = np.zeros(B, dtype=bool)
    info = []
    for st in prog.steps:
        if st["kind"] != KIND_SAMPLE:
            prog.contract(st)
            continue
        zd, w = prog.weights(st, decided)
        w64 = w.astype(np.float64)
        cum = np.cumsum(w64, axis=0)  # sequential float64 sums in z order
        total = cum[-1]
        thr = uniforms(seed, len(info), D, row_base + np.arange(B)) * total
        with np.errstate(invalid="ignore"):
            above = cum > thr[None]
            bad = ~(total >= min_total)
        first = np.where(above.any(axis=0), above.argmax(axis=0), -1)
        pos = w64 > 0
        last_pos = np.where(pos.any(axis=0), len(w) - 1 - pos[::-1].argmax(axis=0), 0)
        pick = np.where(first >= 0, first, last_pos)
        for j, d in enumerate(zd):
            drawn[st["d_first"] + j] = d[pick].astype(np.uint8)
        flagged |= bad.any(axis=0)
        with np.errstate(invalid="ignore", divide="ignore"):
            cond = w64 / total[None]
            margin = np.min(np.abs(cum - thr[None]), axis=0) / total
        info.append(dict(d_first=st["d_first"], cards=tuple(st["ecards"]), cond=cond, margin=margin))
    return drawn, _p_observed(prog, min_total, flagged), info


def run_mpe(words, table_blob, ev_codes, n_rows=None, dtype=np.float32):
    """Execute an MPE (version 8) or marginal MAP (version 9) program on its log tables (`plan.table_blob` for
    float32, `plan.table_blob64` for float64).  Returns (decoded codes uint8 [n_decoded, B], the row's
    max log P(x, e) -- max_{x_MAP} log P(x_MAP, e) for version 9 -- [B] in `dtype`, -inf for a row of
    probability zero), the latter as the upward pass left it in the posterior slot."""
    prog = _Program(words, table_blob, ev_codes, n_rows, dtype, (8, 9))
    decoded = np.zeros((prog.hdr["n_decoded"], 1, prog.B), dtype=np.uint8)
    for st in prog.steps:
        if st["kind"] != KIND_ARGMAX:
            prog.contract(st)
            continue
        zd, w = prog.weights(st, decoded)
        pick = np.argmax(w, axis=0)  # the first maximum: a later z wins only by a strict >
        for j, d in enumerate(zd):
            decoded[st["d_first"] + j] = d[pick].astype(np.uint8)
    return decoded[:, 0], prog.post_rows().astype(dtype)


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
