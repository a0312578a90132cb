"""Float64 oracle of loopy belief propagation (the semantics in sorobn_b200/bp.py's docstring).

Built from the dense network of `ve_oracle.dense_from_pandas` by node name, not from the compiled words: its own
relevant set, factors and message bookkeeping.  Vectorised over evidence rows: every message is an [n_rows, card]
array, and a row that stopped (converged or met a zero sum) keeps the beliefs and sweep count it stopped with while
the other rows go on."""
from __future__ import annotations

import numpy as np


def _factors(dn, evidence, codes, targets):
    """(factors [(family, members, table [n, *member cards])], variables, {var: [(factor index, member index)]})."""
    ev = {name: np.asarray(codes[i], dtype=np.int64) for i, name in enumerate(evidence)}
    relevant = {*targets, *evidence}
    for v in list(relevant):
        relevant |= dn.ancestors(v)
    n = codes.shape[1] if len(evidence) else None
    factors = []
    for v in dn.nodes:
        if v not in relevant:
            continue
        scope = list(dn.scope(v))
        members = [u for u in scope if u not in ev]
        if not members:
            continue
        evax = [u for u in scope if u in ev]
        t = np.transpose(np.asarray(dn.cpt[v], dtype=np.float64), [scope.index(u) for u in evax + members])
        if evax:
            t = t[tuple(np.minimum(ev[u], len(dn.domains[u]) - 1) for u in evax)]  # [n, *members]
        else:
            t = np.broadcast_to(t, (n if n is not None else 1, *t.shape))
        factors.append((v, members, t))
    variables = [v for v in dn.nodes if v in relevant and v not in ev]
    adj = {v: [] for v in variables}
    for f, (_, members, _) in enumerate(factors):
        for i, u in enumerate(members):
            adj[u].append((f, i))
    return factors, variables, adj


def _normalise(p):
    s = p.sum(axis=1, keepdims=True)
    return p / s, ~(s[:, 0] > 0)


def run(dn, evidence, codes, targets, n_iterations, damping, tol, n_rows=None):
    """Belief propagation of every row of `codes` (int [n_ev, n_rows], columns of `evidence` names).

    Returns a dict: beliefs float64 [Q, n_rows] (targets sorted by name, states in domain order; NaN for a row that
    met a zero sum), iterations int [n_rows] (bp.py rule 3 / 4), residual float64 [n_rows, sweeps run] (the largest
    damped-message change of each sweep)."""
    codes = np.asarray(codes)
    n = codes.shape[1] if len(evidence) else int(n_rows)
    targets = sorted(targets)
    factors, variables, adj = _factors(dn, evidence, codes if len(evidence) else np.zeros((0, n), np.int64), targets)
    card = {v: len(dn.domains[v]) for v in dn.nodes}
    mu = {(f, i): np.full((n, card[u]), 1.0 / card[u]) for f, (_, m, _) in enumerate(factors) for i, u in enumerate(m)}
    nu = {k: v.copy() for k, v in mu.items()}

    def beliefs():
        out, dead = [], np.zeros(n, dtype=bool)
        for t in targets:
            p = np.ones((n, card[t]))
            for k in adj[t]:
                p = p * mu[k]
            b, z = _normalise(p)
            out.append(b)
            dead |= z
        out = np.concatenate(out, axis=1).T
        out[:, dead] = np.nan
        return out

    Q = sum(card[t] for t in targets)
    result = np.full((Q, n), np.nan)
    iterations = np.full(n, n_iterations + 1, dtype=np.int64)
    active = np.ones(n, dtype=bool)
    residuals = []
    with np.errstate(all="ignore"):
        for t in range(1, n_iterations + 1):
            dead = np.zeros(n, dtype=bool)
            r = np.zeros(n)
            new_mu = {}
            for f, (_, members, table) in enumerate(factors):
                for i in range(len(members)):
                    x = np.array(table, dtype=np.float64)
                    for u in range(len(members)):
                        if u != i:
                            shape = [x.shape[0]] + [1] * len(members)
                            shape[u + 1] = card[members[u]]
                            x = x * nu[(f, u)].reshape(shape)
                    s = x.sum(axis=tuple(a + 1 for a in range(len(members)) if a != i))
                    s = np.broadcast_to(s, (n, s.shape[1]))
                    m, z = _normalise(s)
                    dead |= z
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
                    dead |= z
            residuals.append(r)
            stop = active & (dead | (r < tol))
            if stop.any():
                result[:, stop] = beliefs()[:, stop]
                result[:, stop & dead] = np.nan
                iterations[stop] = t
                active &= ~stop
            if not active.any():
                break
        if active.any():
            result[:, active] = beliefs()[:, active]
    return {"beliefs": result, "iterations": iterations, "residual": np.stack(residuals, axis=1)}
