"""Float64 ground truth for soft (likelihood, virtual) evidence, without the planner.

Pearl's virtual evidence: a likelihood lambda_v over the states of v is a binary child c_v of v with
P(c_v = 1 | v = x) = lambda_v(x) / K_v, K_v = max lambda_v, observed at c_v = 1.  The posterior of every other
variable given (e, c = 1) is P(. | e, lambda), and P(e, lambda) = P(e, c = 1) * prod_v K_v.  This module builds
that network on `oracle.ve_oracle.DenseNet` for one row at a time and asks the oracle's `query` and
`evidence_probability`.
"""
from __future__ import annotations

import copy

import numpy as np

from oracle import ve_oracle


def dense(net):
    """The oracle's DenseNet of a planner.CompiledNet (CPT axes [*parents, v], parents sorted by name in both)."""
    names = net.names
    dn = ve_oracle.DenseNet(nodes=list(names), parents={names[v]: [names[p] for p in net.parents[v]] for v in range(len(names))},
                            domains={names[v]: list(net.domains[v]) for v in range(len(names))})
    for v in range(len(names)):
        dn.cpt[names[v]] = np.asarray(net.cpt[v], dtype=np.float64)
    return dn


def virtual(dn, soft):
    """(network with one virtual child per soft variable, the event that observes every child, log prod K_v, or
    None when a likelihood is all zeros: the row is impossible).  `soft` maps a node to its likelihood over the
    node's domain."""
    out = copy.copy(dn)
    out.nodes, out.parents, out.domains, out.cpt = list(dn.nodes), dict(dn.parents), dict(dn.domains), dict(dn.cpt)
    event, log_k = {}, 0.0
    for node, lam in soft.items():
        lam = np.asarray(lam, dtype=np.float64)
        k = float(lam.max())
        if not k > 0:
            return out, None, None
        child = f"__soft__{node}"
        out.nodes.append(child)
        out.parents[child] = [node]
        out.domains[child] = [0, 1]
        out.cpt[child] = np.stack([1.0 - lam / k, lam / k], axis=-1)
        event[child] = 1
        log_k += np.log(k)
    return out, event, log_k


def posterior(dn, query, hard, soft):
    """P(query | hard, soft) as a flat float64 vector, query variables sorted by name (the first slowest),
    states in domain order; NaN throughout for an impossible row."""
    size = int(np.prod([len(dn.domains[q]) for q in query]))
    net, event, _ = virtual(dn, soft)
    if event is None:
        return np.full(size, np.nan)
    _, values, _ = ve_oracle.query(net, *query, event={**hard, **event})
    return np.asarray(values, dtype=np.float64).reshape(-1)


def log_evidence(dn, hard, soft):
    """log P(hard, soft): -inf for an impossible row."""
    net, event, log_k = virtual(dn, soft)
    if event is None:
        return -np.inf
    p = ve_oracle.evidence_probability(net, {**hard, **event})
    return float(np.log(p)) + log_k if p > 0 else -np.inf


def rows(net, evidence, codes, soft, lik):
    """(hard event, soft likelihoods) of every row: `evidence` var ids with their uint8 codes [n_ev, B], `soft`
    var ids (likelihood column order) with `lik` [B, sum of cards]."""
    names = net.names
    out = []
    for b in range(lik.shape[0]):
        hard = {names[v]: net.domains[v][int(codes[i, b])] for i, v in enumerate(evidence)}
        s, c0 = {}, 0
        for v in soft:
            c = int(net.card[v])
            s[names[v]] = lik[b, c0:c0 + c]
            c0 += c
        out.append((hard, s))
    return out
