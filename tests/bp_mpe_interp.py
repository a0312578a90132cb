"""CPU replay of compiled max-product words (sorobn_b200/bp.py, version 2), in float64 or float32.

It executes what the max-product instantiations of csrc/sbn_bp.cu execute, record by record, vectorised over the
evidence rows: the sweep of tests/bp_interp.py with a max in step 1 and 0-member factors skipped, then the decode
from the double belief products and the score over every factor.  A max does not depend on its order, so step 1
differs from the device only in the rounding of the normalisation and damping; the float32 replay sets the
tolerances of tests/test_gpu_bp_mpe.py."""
from __future__ import annotations

import numpy as np

from bp_interp import _product, _records
from sorobn_b200 import bp


def run(words, tables, codes, n_rows, n_iterations, damping, tol, dtype=np.float64, messages=False):
    """(codes uint8 [n_var, n_rows], log P float64 [n_rows], iterations int [n_rows], beliefs [(float64 [n_rows,
    card])] normalised per variable) of the words on uint8 codes [n_ev, n_rows]; with `messages` also the final mu
    [n_rows, E]."""
    w = np.asarray(words, dtype=np.int64)
    assert int(w[0]) == bp.MAGIC and int(w[1]) == bp.VERSION_MPE
    dt = np.dtype(dtype).type
    tab = np.asarray(tables, dtype=dt)
    n, E = int(n_rows), int(w[5])
    codes = np.asarray(codes, dtype=np.int64).reshape(-1, n)
    factors, variables, targets = _records(w)
    assert [v for v, _ in targets] == list(range(len(variables)))
    lam, keep = dt(damping), dt(1) - dt(damping)
    mu = np.zeros((n, E), dtype=dt)
    nu = np.zeros((n, E), dtype=dt)
    bases = []
    for off, mem, ax in factors:
        for c, _, e in mem:
            mu[:, e:e + c] = nu[:, e:e + c] = dt(1) / dt(c)
        base = np.full(n, off, dtype=np.int64)
        for col, stride, c in ax:
            base += np.minimum(codes[col], c - 1) * stride
        bases.append(base)
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

    # an all-observed family at an entry of probability 0: dead before the first sweep, 0 recorded
    dead = np.zeros(n, dtype=bool)
    for (off, mem, ax), base in zip(factors, bases):
        if not mem:
            dead |= ~(tab[base] > 0)
    iters = np.where(dead | (not variables), 0, n_iterations + 1).astype(np.int64)
    active = ~dead & bool(variables)
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
                    s = np.maximum((ent * prod[:, :, None]).max(axis=1), dt(0))
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
        out = np.zeros((len(variables), n), dtype=np.uint8)
        code_at = {}  # edge -> the decoded code of its variable
        beliefs = []
        for j, (c, edges) in enumerate(variables):
            p, S = _product(frozen, edges, -1, c, n)
            dead |= ~(S > 0)
            beliefs.append(p / S[:, None])
            out[j] = np.argmax(p, axis=1)
            for e in edges:
                code_at[e] = out[j].astype(np.int64)
        log_p = np.zeros(n)
        for (off, mem, ax), base in zip(factors, bases):
            idx = base.copy()
            for c, si, e in mem:
                idx += code_at[e] * si
            log_p += np.log(tab[idx].astype(np.float64))
    out[:, dead] = 0
    log_p[dead] = np.nan
    for b in beliefs:
        b[dead] = np.nan
    return (out, log_p, iters, beliefs, frozen) if messages else (out, log_p, iters, beliefs)
