"""Float64 oracle of expected counts and EM steps (TEST INFRASTRUCTURE, not product).

Built on `oracle.ve_oracle`: for every row and every node v, the unobserved members M_v of v's
family get `ve_oracle.query(M_v | the row's observed cells)`, placed at the row's codes of the
observed members; a family the row observes completely gets a histogram entry of 1.  Identical rows
are evaluated once and weighted by their multiplicity.

It sits next to the tests rather than inside `oracle/ve_oracle.py` and uses only that module's public
functions (`query`, `evidence_probability`).  So `ve_oracle`, to which the goldens and every existing
parity test are pinned, is unchanged, and this oracle shares no code with the planner or the engine.
"""
from __future__ import annotations

import numpy as np

from oracle import ve_oracle


def _distinct(rows):
    """[(row dict, multiplicity)], missing cells (None / NaN) dropped from the dicts."""
    out = {}
    for r in rows:
        obs = tuple(sorted(((k, v) for k, v in r.items() if v is not None and v == v), key=lambda kv: str(kv[0])))
        out[obs] = out.get(obs, 0) + 1
    return [(dict(k), n) for k, n in out.items()]


def _p(net, row):
    return ve_oracle.evidence_probability(net, row) if row else 1.0


def expected_counts(net: ve_oracle.DenseNet, rows):
    """{node: float64 ndarray [*parents, node]}: sum over `rows` (dicts node -> value; a missing key,
    None or NaN is unobserved) of P(family | observed cells).  Raises ValueError for a row of
    probability zero."""
    counts = {v: np.zeros(net.cpt[v].shape) for v in net.nodes}
    for row, mult in _distinct(rows):
        if _p(net, row) <= 0:
            raise ValueError(f"row {row!r} has probability zero")
        for v in net.nodes:
            scope = net.scope(v)
            M = [u for u in scope if u not in row]
            index = tuple(net.domains[u].index(row[u]) if u in row else slice(None) for u in scope)
            if not M:
                counts[v][index] += mult
                continue
            names, values, _ = ve_oracle.query(net, *M, event=row)
            values = np.transpose(values, [list(names).index(u) for u in M])  # scope order
            counts[v][index] += mult * values
    return counts


def log_likelihood(net: ve_oracle.DenseNet, rows):
    return float(sum(n * np.log(_p(net, r)) for r, n in _distinct(rows)))


def em_step(net: ve_oracle.DenseNet, rows, prior_count=None):
    """(next DenseNet, log-likelihood of `rows` under `net`): one E-step and M-step.  Parent
    configurations with zero expected count get an all-zero CPT row."""
    counts = expected_counts(net, rows)
    out = ve_oracle.DenseNet(nodes=list(net.nodes), parents=dict(net.parents), domains=dict(net.domains))
    for v in net.nodes:
        c = counts[v] + (1.0 if prior_count else 0.0)
        tot = c.sum(axis=-1, keepdims=True)
        with np.errstate(invalid="ignore", divide="ignore"):
            out.cpt[v] = np.where(tot > 0, c / tot, 0.0)
    return out, log_likelihood(net, rows)
