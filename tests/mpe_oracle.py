"""Float64 oracle of the most probable explanation (TEST INFRASTRUCTURE, independent of the planner).

For a DenseNet (`oracle.ve_oracle`) and an event {node: value}, the MPE is the joint state x* of every
node outside the event that maximises P(x, e); L* = log P(x*, e).

* `brute_force` enumerates the joint of the unobserved nodes (up to BRUTE_MAX states);
* `max_sum` is dense max-sum variable elimination (min-fill order, `ve_oracle.min_fill_order`) with a
  traceback, for networks whose joint is too large to enumerate;
* `log_joint` is log P(x, e) of one full assignment, the yardstick for near-ties.

Ties go to the first maximum in each one's own enumeration, which need not be the device's: compare
assignments through `log_joint`.
"""
from __future__ import annotations

import numpy as np

from oracle import ve_oracle

BRUTE_MAX = 2**20


def _log(a):
    with np.errstate(divide="ignore"):
        return np.log(np.asarray(a, dtype=np.float64))


def _index(net, node, value):
    return net.domains[node].index(value)


def log_joint(net, assignment: dict) -> float:
    """log P(assignment) for a value of every node (-inf for an impossible one)."""
    total = 0.0
    for node in net.nodes:
        idx = tuple(_index(net, u, assignment[u]) for u in net.scope(node))
        total += float(_log(net.cpt[node][idx]))
    return total


def _factors(net, event):
    """The log CPTs with the observed axes sliced away: [(vars, values)]."""
    out = []
    for node in net.nodes:
        scope = net.scope(node)
        idx = tuple(_index(net, u, event[u]) if u in event else slice(None) for u in scope)
        out.append((tuple(u for u in scope if u not in event), _log(net.cpt[node][idx])))
    return out


def _expand(vars_, values, union):
    perm = sorted(range(len(vars_)), key=lambda i: union.index(vars_[i]))
    vals = np.transpose(values, perm)
    shape = [1] * len(union)
    for i in perm:
        shape[union.index(vars_[i])] = values.shape[i]
    return vals.reshape(shape)


def _add(factors):
    union = []
    for vs, _ in factors:
        union += [v for v in vs if v not in union]
    union = tuple(union)
    total = np.zeros([1] * len(union))
    for vs, vals in factors:
        total = total + _expand(vs, vals, union)
    return union, total


def brute_force(net, event: dict):
    """(x* {node: value} of the unobserved nodes, L*) by enumerating their joint."""
    hidden = tuple(sorted(v for v in net.nodes if v not in event))
    size = int(np.prod([len(net.domains[v]) for v in hidden], dtype=np.int64))
    if size > BRUTE_MAX:
        raise ValueError(f"{size} joint states: too many to enumerate")
    union, total = _add(_factors(net, event))  # every unobserved node is an axis: its own CPT mentions it
    assert set(union) == set(hidden)
    if not hidden:
        return {}, float(total.reshape(()))
    total = np.broadcast_to(total, [len(net.domains[v]) for v in union])
    vals = np.transpose(total, [union.index(v) for v in hidden])
    best = np.unravel_index(int(np.argmax(vals)), vals.shape)
    return {v: net.domains[v][int(i)] for v, i in zip(hidden, best)}, float(vals.max())


def max_sum(net, event: dict):
    """(x*, L*) by dense max-sum variable elimination with a traceback."""
    factors = _factors(net, event)
    hidden = [v for v in net.nodes if v not in event]
    order = ve_oracle.min_fill_order([vs for vs, _ in factors], hidden, {v: len(net.domains[v]) for v in net.nodes})
    trace = []  # (x, vars of the bucket's sum, values)
    for x in order:
        bucket = [f for f in factors if x in f[0]]
        factors = [f for f in factors if x not in f[0]]
        union, total = _add(bucket)
        total = np.broadcast_to(total, [len(net.domains[v]) for v in union])
        trace.append((x, union, total))
        ax = union.index(x)
        factors.append((tuple(v for v in union if v != x), total.max(axis=ax)))
    L = float(sum(float(np.asarray(vals).reshape(())) for _, vals in factors))
    idx = {}
    for x, union, total in reversed(trace):
        sel = tuple(slice(None) if v == x else idx[v] for v in union)
        idx[x] = int(np.argmax(total[sel]))
    return {v: net.domains[v][i] for v, i in idx.items()}, L
