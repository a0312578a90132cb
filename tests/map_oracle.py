"""Float64 oracle of marginal MAP (TEST INFRASTRUCTURE, independent of the planner).

For a DenseNet (`oracle.ve_oracle`), an event {node: value} and MAP variables M (none of them observed),
the marginal MAP state is the joint state x* of M that maximises P(x_M, e) = sum over every other node
of P(x, e); L* = log P(x*, e).

* `brute_force` enumerates the joint of every unobserved node (up to BRUTE_MAX states), sums the others
  out and takes the argmax over M;
* `dense_query` takes the argmax of `ve_oracle.query`'s dense posterior over M (the posterior of
  `impute`), for networks too wide to enumerate but with a small MAP joint;
* `log_prob` is log P(x_M, e) of one assignment of M, the yardstick for near-ties.

Each returns (x*, L*, gap), gap = L* minus the log-probability of the runner-up joint state of M (inf when
M has a single joint state).  Ties go to the first maximum in each one's own enumeration, which need not be
the device's: compare near-ties through `log_prob`.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import ve_oracle

BRUTE_MAX = 2**20


def _log(a):
    with np.errstate(divide="ignore"):
        return np.log(np.asarray(a, dtype=np.float64))


def log_prob(net, event: dict, x_map: dict) -> float:
    """log P(x_map, event), every other node summed out (-inf for an impossible state)."""
    full = {**event, **x_map}
    if not full:
        return 0.0
    return float(_log(ve_oracle.evidence_probability(net, full)))


def _gap(flat_logs):
    s = np.sort(np.asarray(flat_logs).reshape(-1))
    return np.inf if s.size < 2 else float(s[-1] - s[-2])


def brute_force(net, event: dict, map_vars):
    """(x* {node: value}, L*, gap) by enumerating the joint of every unobserved node."""
    map_vars = list(map_vars)
    hidden = [v for v in net.nodes if v not in event]
    shape = [len(net.domains[v]) for v in hidden]
    if math.prod(shape) > BRUTE_MAX:
        raise ValueError("too many joint states to enumerate")
    logs = np.zeros(shape)
    for v in net.nodes:
        scope = net.scope(v)
        idx = tuple(net.domains[u].index(event[u]) if u in event else slice(None) for u in scope)
        t = _log(net.cpt[v][idx])
        free = [u for u in scope if u not in event]
        if free:
            t = np.transpose(t, np.argsort([hidden.index(u) for u in free]))
        logs = logs + t.reshape([len(net.domains[u]) if u in free else 1 for u in hidden])
    summed = tuple(i for i, v in enumerate(hidden) if v not in map_vars)
    with np.errstate(divide="ignore", invalid="ignore"):
        m = np.max(logs, axis=summed, keepdims=True) if summed else logs
        m_safe = np.where(np.isfinite(m), m, 0.0)
        marg = (np.log(np.sum(np.exp(logs - m_safe), axis=summed, keepdims=True)) + m_safe) if summed else logs
        marg = np.where(m == -np.inf, -np.inf, marg)
    kept = [v for v in hidden if v in map_vars]
    marg = marg.reshape([len(net.domains[v]) for v in kept])
    vals = np.transpose(marg, [kept.index(v) for v in map_vars]) if map_vars else marg
    best = np.unravel_index(int(np.argmax(vals)), vals.shape)
    return ({v: net.domains[v][int(i)] for v, i in zip(map_vars, best)}, float(vals.max()), _gap(vals))


def dense_query(net, event: dict, map_vars):
    """(x*, L*, gap) from the dense posterior over the MAP variables (`ve_oracle.query`)."""
    if not map_vars:
        return {}, log_prob(net, event, {}), np.inf
    p_e = ve_oracle.evidence_probability(net, event) if event else 1.0
    names, values, _ = ve_oracle.query(net, *map_vars, event=event)
    logs = _log(values) + _log(p_e)
    best = np.unravel_index(int(np.argmax(values)), values.shape)
    return {n: net.domains[n][int(i)] for n, i in zip(names, best)}, float(logs.max()), _gap(logs)


def solve(net, event: dict, map_vars):
    """`brute_force` where the unobserved joint is small enough, else `dense_query`."""
    hidden = [v for v in net.nodes if v not in event]
    if math.prod(len(net.domains[v]) for v in hidden) <= BRUTE_MAX:
        return brute_force(net, event, map_vars)
    return dense_query(net, event, map_vars)
