"""Float64 oracle of max-product loopy belief propagation (the "Max-product" semantics in sorobn_b200/bp.py).

Built from the dense network of `ve_oracle.dense_from_pandas` by node name, not from the compiled words: every CPT
is a factor (one whose members are all observed only enters the score) and every unobserved node a variable.
Vectorised over evidence rows: every message is an [n_rows, card] array, and a row that stopped (converged or met a
zero sum) keeps the beliefs and sweep count it stopped with while the other rows go on."""
from __future__ import annotations

import numpy as np


def _tables(dn, evidence, codes, n):
    """[(members, table [n, *member cards])] of every CPT, its evidence axes indexed by the rows' codes."""
    ev = {name: np.asarray(codes[i], dtype=np.int64) for i, name in enumerate(evidence)}
    factors = []
    for v in dn.nodes:
        scope = list(dn.scope(v))
        members = [u for u in scope if u not in ev]
        evax = [u for u in scope if u in ev]
        t = np.transpose(np.asarray(dn.cpt[v], dtype=np.float64), [scope.index(u) for u in evax + members])
        if evax:
            t = t[tuple(np.minimum(ev[u], len(dn.domains[u]) - 1) for u in evax)]  # [n, *members]
        else:
            t = np.broadcast_to(t, (n, *t.shape))
        factors.append((members, t))
    return factors


def _normalise(p):
    s = p.sum(axis=1, keepdims=True)
    return p / s, ~(s[:, 0] > 0)


def run(dn, evidence, codes, n_iterations, damping, tol, n_rows=None):
    """Max-product BP of every row of `codes` (int [n_ev, n_rows], columns of `evidence` names).

    Returns a dict: variables (the unobserved node names, in `dn.nodes` order), codes int [n_var, n_rows] (0 for a
    dead row), log_p float64 [n_rows] (NaN for a dead row), iterations int [n_rows], beliefs {name: float64
    [n_rows, card]} normalised (NaN for a dead row), residual float64 [n_rows, sweeps run]."""
    codes = np.asarray(codes)
    n = codes.shape[1] if len(evidence) else int(n_rows)
    factors = _tables(dn, evidence, codes if len(evidence) else np.zeros((0, n), np.int64), n)
    variables = [v for v in dn.nodes if v not in evidence]
    card = {v: len(dn.domains[v]) for v in dn.nodes}
    adj = {v: [] for v in variables}
    for f, (members, _) in enumerate(factors):
        for i, u in enumerate(members):
            adj[u].append((f, i))
    mu = {(f, i): np.full((n, card[u]), 1.0 / card[u]) for f, (m, _) in enumerate(factors) for i, u in enumerate(m)}
    nu = {k: v.copy() for k, v in mu.items()}

    def belief_products():
        out = {}
        for v in variables:
            p = np.ones((n, card[v]))
            for k in adj[v]:
                p = p * mu[k]
            out[v] = p
        return out

    frozen = {v: np.zeros((n, card[v])) for v in variables}
    # a family with every member observed, at an entry of probability 0: dead before any sweep, recording 0
    dead = np.zeros(n, dtype=bool)
    for members, table in factors:
        if not members:
            dead |= ~(table > 0)
    iterations = np.where(dead | (not variables), 0, n_iterations + 1).astype(np.int64)
    active = ~dead & bool(variables)
    residuals = []
    with np.errstate(all="ignore"):
        for t in range(1, n_iterations + 1):
            if not active.any():
                break
            d = np.zeros(n, dtype=bool)
            r = np.zeros(n)
            new_mu = {}
            for f, (members, table) in enumerate(factors):
                for i in range(len(members)):
                    x = np.array(table, dtype=np.float64)
                    for u in range(len(members)):
                        if u != i:
                            shape = [n] + [1] * len(members)
                            shape[u + 1] = card[members[u]]
                            x = x * nu[(f, u)].reshape(shape)
                    others = tuple(a + 1 for a in range(len(members)) if a != i)
                    s = np.maximum(x.max(axis=others), 0.0) if others else x
                    m, z = _normalise(s)
                    d |= z
                    new = (1.0 - damping) * m + damping * mu[(f, i)]
                    r = np.maximum(r, np.abs(new - mu[(f, i)]).max(axis=1))
                    new_mu[(f, i)] = new
            mu = new_mu
            for v in variables:
                for k in adj[v]:
                    p = np.ones((n, card[v]))
                    for g in adj[v]:
                        if g != k:
                            p = p * mu[g]
                    nu[k], z = _normalise(p)
                    d |= z
            residuals.append(r)
            stop = active & (d | (r < tol))
            if stop.any():
                products = belief_products()
                for v in variables:
                    frozen[v][stop] = products[v][stop]
                iterations[stop] = t
                dead |= stop & d
                active &= ~stop
        if active.any():
            products = belief_products()
            for v in variables:
                frozen[v][active] = products[v][active]
        beliefs, out = {}, np.zeros((len(variables), n), dtype=np.int64)
        for j, v in enumerate(variables):
            beliefs[v], z = _normalise(frozen[v])
            dead |= z
            out[j] = np.argmax(frozen[v], axis=1)
        log_p = np.zeros(n)
        for members, table in factors:
            entry = table[(np.arange(n), *[out[variables.index(u)] for u in members])]
            log_p += np.log(entry)
    out[:, dead] = 0
    log_p[dead] = np.nan
    for v in variables:
        beliefs[v][dead] = np.nan
    residual = np.stack(residuals, axis=1) if residuals else np.zeros((n, 0))
    return {"variables": variables, "codes": out, "log_p": log_p, "iterations": iterations, "beliefs": beliefs,
            "residual": residual}
