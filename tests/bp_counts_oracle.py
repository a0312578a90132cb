"""Float64 oracle of belief-propagation expected counts (sorobn_b200/bp.py, "Expected counts").

Built from the dense network of `ve_oracle.dense_from_pandas` by node name, not from the compiled words: every CPT a
factor (0-member ones kept), every unobserved node a variable, its own message bookkeeping.  Vectorised over evidence
rows; a row that stopped keeps the messages it stopped with while the other rows go on.  The family beliefs, the Bethe
log-likelihood and the counts are then formed term by term as the docstring writes them."""
from __future__ import annotations

import numpy as np


def _normalise(p):
    s = p.sum(axis=1, keepdims=True)
    return p / s, ~(s[:, 0] > 0)


def run(dn, evidence, codes, n_iterations, damping, tol, n_rows=None):
    """Belief propagation and its readout for every row of `codes` (int [n_ev, n_rows], columns of `evidence` names).

    Returns a dict: counts {node: float64 [*parents, node]} summed over the live rows, log_z float64 [n_rows] (NaN for
    a dead row), iterations int [n_rows], family {node: [n_rows, *unobserved member cards]} beliefs (scope order),
    variable {node: [n_rows, card]} beliefs and residual [n_rows, sweeps run]."""
    codes = np.asarray(codes, dtype=np.int64)
    n = codes.shape[1] if len(evidence) else int(n_rows)
    ev = {name: codes[i] for i, name in enumerate(evidence)}
    card = {v: len(dn.domains[v]) for v in dn.nodes}
    factors = []  # (family, members, evidence axes, table [n, *member cards])
    dead = np.zeros(n, dtype=bool)
    for v in dn.nodes:
        scope = list(dn.scope(v))
        members = [u for u in scope if u not in ev]
        evax = [u for u in scope if u in ev]
        t = np.transpose(np.asarray(dn.cpt[v], dtype=np.float64), [scope.index(u) for u in evax + members])
        t = t[tuple(ev[u] for u in evax)] if evax else np.broadcast_to(t, (n, *t.shape))
        if not members:
            dead |= ~(t > 0)
        factors.append((v, members, evax, t))
    variables = [v for v in dn.nodes if v not in ev]
    adj = {v: [] for v in variables}
    for f, (_, members, _, _) in enumerate(factors):
        for i, u in enumerate(members):
            adj[u].append((f, i))
    mu = {(f, i): np.full((n, card[u]), 1.0 / card[u]) for f, (_, m, _, _) in enumerate(factors) for i, u in enumerate(m)}
    nu = {k: x.copy() for k, x in mu.items()}
    iterations = np.zeros(n, dtype=np.int64) if not variables else np.where(dead, 0, n_iterations + 1)
    active = ~dead if variables else np.zeros(n, dtype=bool)
    fmu = {k: x.copy() for k, x in mu.items()}
    fnu = {k: x.copy() for k, x in nu.items()}
    residuals = []
    with np.errstate(all="ignore"):
        for t in range(1, n_iterations + 1):
            if not active.any():
                break
            z = np.zeros(n, dtype=bool)
            r = np.zeros(n)
            new_mu = {}
            for f, (_, members, _, table) in enumerate(factors):
                for i in range(len(members)):
                    x = np.array(table, dtype=np.float64)
                    for u in range(len(members)):
                        if u != i:
                            shape = [n] + [1] * len(members)
                            shape[u + 1] = card[members[u]]
                            x = x * nu[(f, u)].reshape(shape)
                    s = x.sum(axis=tuple(a + 1 for a in range(len(members)) if a != i))
                    m, zz = _normalise(s)
                    z |= zz
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
                    nu[k], zz = _normalise(p)
                    z |= zz
            residuals.append(r)
            stop = active & (z | (r < tol))
            dead |= stop & z
            iterations[stop] = t
            for k in mu:
                fmu[k][stop] = mu[k][stop]
                fnu[k][stop] = nu[k][stop]
            active &= ~stop
        for k in mu:
            fmu[k][active] = mu[k][active]
            fnu[k][active] = nu[k][active]

        # readout
        log_z = np.zeros(n)
        variable = {}
        for v in variables:
            p = np.ones((n, card[v]))
            for k in adj[v]:
                p = p * fmu[k]
            b, zz = _normalise(p)
            dead |= zz
            variable[v] = b
            blogb = np.where(b > 0, b * np.log(np.where(b > 0, b, 1.0)), 0.0).sum(axis=1)
            log_z += (len(adj[v]) - 1) * blogb
        family = {}
        for f, (v, members, evax, table) in enumerate(factors):
            if not members:
                log_z += np.log(table)
                continue
            x = np.array(table, dtype=np.float64)
            for i, u in enumerate(members):
                shape = [n] + [1] * len(members)
                shape[i + 1] = card[u]
                x = x * fnu[(f, i)].reshape(shape)
            s = x.reshape(n, -1).sum(axis=1)
            dead |= ~(s > 0)
            b = x / s.reshape([n] + [1] * len(members))
            family[v] = b
            pos = b > 0
            term = np.where(pos, b * (np.log(np.where(pos, table, 1.0)) - np.log(np.where(pos, b, 1.0))), 0.0)
            log_z += term.reshape(n, -1).sum(axis=1)
        log_z[dead] = np.nan

        counts = {}
        live = ~dead
        for f, (v, members, evax, table) in enumerate(factors):
            scope = list(dn.scope(v))
            c = np.zeros(np.shape(dn.cpt[v]))
            ct = np.transpose(c, [scope.index(u) for u in evax + members])  # a view
            idx = tuple(ev[u][live] for u in evax)
            value = family[v][live] if members else np.ones(int(live.sum()))
            if evax:
                np.add.at(ct, idx, value)
            else:
                ct += value.sum(axis=0)
            counts[v] = c
    return {"counts": counts, "log_z": log_z, "iterations": iterations, "family": family, "variable": variable,
            "residual": np.stack(residuals, axis=1) if residuals else np.zeros((n, 0))}
