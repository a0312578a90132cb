"""CPU replay of compiled belief-propagation words (sorobn_b200/bp.py layout), in float64 or float32.

It executes what csrc/sbn_bp.cu executes, record by record, vectorised over the evidence rows: the same table
offsets, the same message entries, the same stop rules and the same underflow rescale.  Sums over configurations
run in the kernel's order (first configuration first); the float32 replay is therefore close to, though not
bitwise, the device, and sets the tolerance of the GPU tests."""
from __future__ import annotations

import numpy as np

from sorobn_b200 import bp

TINY, RESCALE = 2.0**-32, 2.0**64


def _records(w):
    n_fac, n_var, n_tgt = int(w[3]), int(w[4]), int(w[6])
    p, factors = int(w[9]), []
    for _ in range(n_fac):
        off, n_mem, n_evax = int(w[p + 1]), int(w[p + 2]), int(w[p + 3])
        mem = [tuple(int(x) for x in w[p + 4 + 3 * i:p + 7 + 3 * i]) for i in range(n_mem)]
        ax = [tuple(int(x) for x in w[p + 4 + 3 * n_mem + 3 * k:p + 7 + 3 * n_mem + 3 * k]) for k in range(n_evax)]
        factors.append((off, mem, ax))
        p += 4 + 3 * (n_mem + n_evax)
    variables, at = [], {}
    for _ in range(n_var):
        c, deg = int(w[p + 1]), int(w[p + 2])
        at[p] = len(variables)
        variables.append((c, [int(e) for e in w[p + 3:p + 3 + deg]]))
        p += 3 + deg
    targets = [(at[int(w[p + 2 * k])], int(w[p + 2 * k + 1])) for k in range(n_tgt)]
    return factors, variables, targets


def _product(mu, edges, skip, c, n):
    """The kernel's bp_product: in float64 whatever the messages' type, rescaled by 2^64 when its largest entry
    falls below 2^-32; (product, sum)."""
    p = np.ones((n, c), dtype=np.float64)
    for k, e in enumerate(edges):
        if k == skip:
            continue
        p = p * mu[:, e:e + c].astype(np.float64)
        low = p.max(axis=1) < TINY
        if low.any():
            p[low] *= RESCALE
    return p, np.cumsum(p, axis=1)[:, -1]


def run(words, tables, codes, n_rows, n_iterations, damping, tol, dtype=np.float64, messages=False):
    """(beliefs [Q, n_rows] of `dtype`, iterations int [n_rows]) of the words on uint8 codes [n_ev, n_rows]; with
    `messages` also the final mu [n_rows, E]."""
    w = np.asarray(words, dtype=np.int64)
    assert int(w[0]) == bp.MAGIC and int(w[1]) == bp.VERSION
    dt = np.dtype(dtype).type
    tab = np.asarray(tables, dtype=dt)
    n, E, Q = int(n_rows), int(w[5]), int(w[7])
    codes = np.asarray(codes, dtype=np.int64).reshape(-1, n)
    factors, variables, targets = _records(w)
    lam, keep = dt(damping), dt(1) - dt(damping)
    mu = np.zeros((n, E), dtype=dt)
    nu = np.zeros((n, E), dtype=dt)
    for off, mem, ax in factors:
        for c, _, e in mem:
            mu[:, e:e + c] = nu[:, e:e + c] = dt(1) / dt(c)
    # per factor: row table bases, and per member the others' configurations (kernel order: first member fastest)
    plans = []
    for off, mem, ax in factors:
        base = np.full(n, off, dtype=np.int64)
        for col, stride, c in ax:
            base += np.minimum(codes[col], c - 1) * stride
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

    iters = np.full(n, n_iterations + 1, dtype=np.int64)
    active = np.ones(n, dtype=bool)
    dead = np.zeros(n, dtype=bool)
    frozen = np.zeros((n, E), dtype=dt)
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
            frozen[rows[stop]] = mu[rows[stop]]
            active[rows[stop]] = False
        frozen[active] = mu[active]
        out = np.zeros((Q, n), dtype=dt)
        for v, q in targets:
            c, edges = variables[v]
            p, S = _product(frozen, edges, -1, c, n)
            dead |= ~(S > 0)
            out[q:q + c] = (p / S[:, None]).astype(dt).T
        out[:, dead] = np.nan
    return (out, iters, frozen) if messages else (out, iters)
