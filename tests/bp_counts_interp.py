"""CPU replay of compiled expected-counts words (version 3 of the sorobn_b200/bp.py layout), in float64 or float32.

It executes what csrc/sbn_bp.cu executes: the sum-product sweep of `tests/bp_interp.py` over version-3 words (0-member
factors skipped by the sweep, the dead-before-the-first-sweep rule), then sbn_bp_counts_kernel's readout in double
from the messages of the messages' type: per row the variable terms, then per factor in blob order S = sum p and
H = sum p (log f - log p) over its configurations (first member fastest, p = f prod nu), log Z_B += H / S + log S, and
the counts p / S added into the blob-order table.  The float32 replay is close to, though not bitwise, the device,
and sets the tolerances of tests/test_gpu_bp_counts.py."""
from __future__ import annotations

import numpy as np

from bp_interp import _product, _records
from sorobn_b200 import bp


def run(words, tables, codes, n_rows, n_iterations, damping, tol, dtype=np.float64):
    """(counts float64 [n_table_floats] in blob order, log Z_B float64 [n_rows] (NaN for a dead row), iterations int
    [n_rows]) of the words on uint8 codes [n_ev, n_rows]."""
    w = np.asarray(words, dtype=np.int64)
    assert int(w[0]) == bp.MAGIC and int(w[1]) == bp.VERSION_COUNTS
    dt = np.dtype(dtype).type
    tab = np.asarray(tables, dtype=dt)
    n, E = int(n_rows), int(w[5])
    codes = np.asarray(codes, dtype=np.int64).reshape(-1, n)
    factors, variables, _ = _records(w)
    lam, keep = dt(damping), dt(1) - dt(damping)
    mu = np.zeros((n, E), dtype=dt)
    nu = np.zeros((n, E), dtype=dt)
    bases = []
    dead = np.zeros(n, dtype=bool)
    for off, mem, ax in factors:
        for c, _, e in mem:
            mu[:, e:e + c] = nu[:, e:e + c] = dt(1) / dt(c)
        base = np.full(n, off, dtype=np.int64)
        for col, stride, c in ax:
            base += np.minimum(codes[col], c - 1) * stride
        bases.append(base)
        if not mem:
            dead |= ~(tab[base] > 0)
    plans = []
    for (off, mem, ax), base in zip(factors, bases):
        per = []
        for i, (c, si, e) in enumerate(mem):
            others = [u for u in range(len(mem)) if u != i]
            n_other = int(np.prod([mem[u][0] for u in others], dtype=np.int64))
            rem = np.arange(n_other)
            idx = np.zeros(n_other, dtype=np.int64)
            digits = []
            for u in others:
                cu = mem[u][0]
                digits.append((mem[u][2], rem % cu))
                idx += (rem % cu) * mem[u][1]
                rem = rem // cu
            per.append((c, si, e, idx, digits))
        plans.append((base, per))

    none = not variables
    iters = np.where(dead | none, 0, n_iterations + 1).astype(np.int64)
    active = ~dead & (not none)
    with np.errstate(all="ignore"):
        for t in range(1, n_iterations + 1):
            rows = np.flatnonzero(active)
            if not len(rows):
                break
            r = np.zeros(len(rows), dtype=dt)
            d = np.zeros(len(rows), dtype=bool)
            for base, per in plans:
                for c, si, e, idx, digits in per:
                    prod = np.ones((len(rows), len(idx)), dtype=dt)
                    for eu, xu in digits:
                        prod = prod * nu[rows][:, eu + xu]
                    ent = tab[base[rows, None, None] + idx[None, :, None] + si * np.arange(c)[None, None, :]]
                    s = np.cumsum(ent * prod[:, :, None], axis=1, dtype=dt)[:, -1, :]
                    S = np.cumsum(s, axis=1, dtype=dt)[:, -1]
                    d |= ~(S > 0)
                    old = mu[rows, e:e + c]
                    new = keep * (s / S[:, None]) + lam * old
                    r = np.maximum(r, np.abs(new - old).max(axis=1))
                    mu[rows, e:e + c] = new
            if not d.all():
                mrows = mu[rows]
                for c, edges in variables:
                    for k, e in enumerate(edges):
                        p, S = _product(mrows, edges, k, c, len(rows))
                        d |= ~(S > 0)
                        nu[rows, e:e + c] = (p / S[:, None]).astype(dt)
            stop = d | (r < dt(tol))
            iters[rows[stop]] = t
            dead[rows[d]] = True
            active[rows[stop]] = False

        # readout, in double from the stored messages (a row's messages stop changing when it stops)
        log_z = np.zeros(n)
        for c, edges in variables:
            p, S = _product(mu, edges, -1, c, n)
            dead |= ~(S > 0)
            b = p / S[:, None]
            log_z += (len(edges) - 1) * np.where(b > 0, b * np.log(np.where(b > 0, b, 1.0)), 0.0).sum(axis=1)
        terms = []
        for (off, mem, ax), base in zip(factors, bases):
            if not mem:
                log_z += np.log(tab[base].astype(np.float64))
                terms.append(None)
                continue
            T = int(np.prod([c for c, _, _ in mem]))
            j = np.arange(T)
            p = tab[base[:, None] + j[None, :]].astype(np.float64)
            rem = j.copy()
            for c, _, e in mem:
                p = p * nu[:, e + rem % c].astype(np.float64)
                rem = rem // c
            S = np.cumsum(p, axis=1)[:, -1]
            f = tab[base[:, None] + j[None, :]].astype(np.float64)
            pos = p > 0
            H = np.cumsum(np.where(pos, p * (np.log(np.where(pos, f, 1.0)) - np.log(np.where(pos, p, 1.0))), 0.0),
                          axis=1)[:, -1]
            dead |= ~(S > 0)
            log_z += H / S + np.log(S)
            terms.append((p, S))
        log_z[dead] = np.nan
        counts = np.zeros(int(w[8]))
        live = ~dead
        for (off, mem, ax), base, term in zip(factors, bases, terms):
            if term is None:
                np.add.at(counts, base[live], 1.0)
                continue
            p, S = term
            T = p.shape[1]
            np.add.at(counts, base[live][:, None] + np.arange(T)[None, :], p[live] / S[live, None])
    return counts, log_z, iters
