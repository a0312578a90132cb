"""CPU oracle for the exact-inference hot path (TEST INFRASTRUCTURE, not product).

This is a dense float64 numpy restatement of the reference's variable
elimination (`/root/reference/sorobn/bayes_net.py`).  The reference keeps every
factor as a pandas Series with a (Multi)Index and multiplies with an index join
and sums out with a groupby; here a factor is a dense ndarray with one axis per
variable, multiplication is a broadcast product and sum-out is `ndarray.sum`.
The arithmetic (which numbers get multiplied and added) is the same, only the
container differs, so results agree to float64 rounding.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s CPU-baseline /
`--impl reference` legs may import this module.  The product path
(`sorobn_b200`) never does: it fails loudly when the CUDA library is missing.

Parity pinning: `oracle/gen_golden.py` runs the real reference (imported from
/root/reference in the build container) on the example and synthetic networks,
writes `tests/golden/*.json`, and `tests/test_oracle_golden.py` checks this
module against those vectors (and against the reference's doctest values).

Sparse-vs-dense note: the reference drops zero-probability rows before every
product (`pointwise_mul(..., keep_zeros=False)`, bayes_net.py:253-256), so a row
is present in a reference factor iff its dense value is > 0.  `query` therefore
also returns the support mask (dense value > 0) so callers can compare the index
of the reference's answer as well as its values.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

__all__ = [
    "DenseNet",
    "Factor",
    "sum_out",
    "pointwise_mul_two",
    "pointwise_mul",
    "variable_elimination",
    "query",
    "evidence_probability",
    "dense_from_pandas",
    "min_fill_order",
]


@dataclass
class Factor:
    """A dense factor: `values` has one axis per entry of `vars` (same order)."""

    vars: tuple
    values: np.ndarray

    def __post_init__(self):
        assert self.values.ndim == len(self.vars), (self.vars, self.values.shape)


@dataclass
class DenseNet:
    """Dense mirror of `BayesNet.P` after `prepare()` (bayes_net.py:327-371).

    cpt[node] has axes [*parents[node], node]; parents are sorted (bayes_net.py:312)
    and each axis follows `domains[var]`, which is sorted like `sort_index`
    (bayes_net.py:366) sorts the level values.
    """

    nodes: list
    parents: dict
    domains: dict
    cpt: dict = field(default_factory=dict)

    def ancestors(self, node):
        # bayes_net.py:373-378
        out = set()
        stack = list(self.parents.get(node, ()))
        while stack:
            p = stack.pop()
            if p not in out:
                out.add(p)
                stack.extend(self.parents.get(p, ()))
        return out

    def scope(self, node):
        return (*self.parents.get(node, ()), node)


def sum_out(factor: Factor, *variables) -> Factor:
    """Marginalise `variables` out of `factor` (bayes_net.py:54-103: groupby the
    remaining index levels and sum)."""
    axes = tuple(factor.vars.index(v) for v in variables)
    keep = tuple(v for v in factor.vars if v not in variables)
    return Factor(keep, factor.values.sum(axis=axes))


def pointwise_mul_two(left: Factor, right: Factor) -> Factor:
    """Product of two factors (bayes_net.py:106-250).

    The reference joins the two indexes on their common level names and multiplies
    the aligned values; with no common name it takes the outer product
    (bayes_net.py:234-238).  Dense: broadcast both to the union scope.
    The union keeps left's variables first, then right's new ones, which is the
    level order the pandas join produces; the order is irrelevant to the values.
    """
    union = tuple(left.vars) + tuple(v for v in right.vars if v not in left.vars)

    def expand(f: Factor):
        # permute f's axes into union order and insert singleton axes elsewhere
        perm = sorted(range(len(f.vars)), key=lambda i: union.index(f.vars[i]))
        vals = np.transpose(f.values, perm)
        shape = [1] * len(union)
        for i in perm:
            shape[union.index(f.vars[i])] = f.values.shape[i]
        return vals.reshape(shape)

    return Factor(union, expand(left) * expand(right))


def pointwise_mul(factors) -> Factor:
    """functools.reduce(pointwise_mul_two, ...) as bayes_net.py:253-256.  The
    `cdt[cdt > 0]` filter there only removes rows whose value is zero; densely
    those rows stay and carry 0."""
    factors = list(factors)
    out = factors[0]
    for f in factors[1:]:
        out = pointwise_mul_two(out, f)
    return out


def min_fill_order(scopes, hidden, cards):
    """Greedy min-fill elimination order over `hidden` for the factor scopes given.

    The reference eliminates in Python-set iteration order (bayes_net.py:779),
    which is arbitrary; the answer does not depend on the order.  Ties are broken
    by smaller resulting factor, then by position in `hidden` (deterministic).
    """
    hidden = list(hidden)
    adj = {}
    for sc in scopes:
        for a in sc:
            adj.setdefault(a, set()).update(b for b in sc if b != a)
    for h in hidden:
        adj.setdefault(h, set())
    order = []
    remaining = list(hidden)
    while remaining:
        best = None
        for pos, v in enumerate(remaining):
            nb = list(adj[v])
            fill = 0
            for i in range(len(nb)):
                ai = adj[nb[i]]
                for j in range(i + 1, len(nb)):
                    if nb[j] not in ai:
                        fill += 1
            size = 1
            for u in nb:
                size *= cards[u]
            key = (fill, size, pos)
            if best is None or key < best[0]:
                best = (key, v)
        v = best[1]
        nb = adj.pop(v)
        for a in nb:
            adj[a].discard(v)
            adj[a].update(b for b in nb if b != a)
        remaining.remove(v)
        order.append(v)
    return order


def variable_elimination(net: DenseNet, query_vars, event: dict, order=None) -> Factor:
    """bayes_net.py:739-794, densely.

    Returns the normalised posterior as a Factor over the query variables (in the
    order the elimination leaves them; use `query` for the sorted public form).
    """
    query_vars = tuple(query_vars)
    # bayes_net.py:763-766 -- relevant = query + event + all their ancestors
    relevant = {*query_vars, *event}
    for node in list(relevant):
        relevant |= net.ancestors(node)
    hidden = relevant - {*query_vars, *event}

    # bayes_net.py:768-776 -- one factor per relevant node, filtered by the event.
    # The reference keeps the event level with its single value; densely the axis
    # is indexed away, which is what `droplevel` does at the end (bayes_net.py:791).
    factors = []
    for node in sorted(relevant, key=net.nodes.index):
        scope = net.scope(node)
        vals = net.cpt[node]
        keep = []
        index = []
        for v in scope:
            if v in event:
                index.append(net.domains[v].index(event[v]))
            else:
                index.append(slice(None))
                keep.append(v)
        factors.append(Factor(tuple(keep), np.asarray(vals[tuple(index)], dtype=np.float64)))

    if order is None:
        cards = {v: len(net.domains[v]) for v in net.nodes}
        order = min_fill_order([f.vars for f in factors], sorted(hidden, key=net.nodes.index), cards)
    assert set(order) == hidden

    # bayes_net.py:778-786 -- sum out each hidden variable from the product of the
    # factors that mention it
    for node in order:
        touching = [f for f in factors if node in f.vars]
        factors = [f for f in factors if node not in f.vars]
        prod = pointwise_mul(touching)
        factors.append(sum_out(prod, node))

    # bayes_net.py:788-794 -- multiply what is left and normalise
    posterior = pointwise_mul(factors)
    total = posterior.values.sum()
    with np.errstate(invalid="ignore", divide="ignore"):  # P(event) == 0 -> NaN (reference: empty answer)
        return Factor(posterior.vars, posterior.values / total)


def evidence_probability(net: DenseNet, event: dict) -> float:
    """P(event): what `predict_proba` (bayes_net.py:934-962) looks up in the full joint after
    marginalising the unobserved variables.  Computed by eliminating every non-event variable
    among the event's ancestors (the others sum to one)."""
    relevant = set(event)
    for node in list(relevant):
        relevant |= net.ancestors(node)
    factors = []
    for node in sorted(relevant, key=net.nodes.index):
        scope = net.scope(node)
        index = tuple(net.domains[v].index(event[v]) if v in event else slice(None) for v in scope)
        factors.append(Factor(tuple(v for v in scope if v not in event), np.asarray(net.cpt[node][index], dtype=np.float64)))
    hidden = relevant - set(event)
    cards = {v: len(net.domains[v]) for v in net.nodes}
    for node in min_fill_order([f.vars for f in factors], sorted(hidden, key=net.nodes.index), cards):
        touching = [f for f in factors if node in f.vars]
        factors = [f for f in factors if node not in f.vars]
        factors.append(sum_out(pointwise_mul(touching), node))
    return float(pointwise_mul(factors).values)


def query(net: DenseNet, *query_vars, event: dict, order=None):
    """`BayesNet.query(..., algorithm="exact")` (bayes_net.py:796-875).

    Returns (vars, values, support): `vars` are the query variables sorted like
    `answer.reorder_levels(sorted(answer.index.names))` (bayes_net.py:872-873),
    `values` the dense posterior over them (axes follow the sorted domains, i.e.
    `sort_index`, bayes_net.py:875), `support` the mask of rows the reference
    would return (dense value > 0).
    """
    if not query_vars:
        raise ValueError("At least one query variable has to be specified")
    for q in query_vars:
        if q in event:
            raise ValueError("A query variable cannot be part of the event")
    post = variable_elimination(net, query_vars, event, order=order)
    sorted_vars = tuple(sorted(post.vars))
    perm = [post.vars.index(v) for v in sorted_vars]
    values = np.transpose(post.values, perm)
    return sorted_vars, values, values > 0


def dense_from_pandas(P: dict, parents: dict, nodes: list) -> DenseNet:
    """Build a DenseNet from prepared pandas CPTs (`BayesNet.P` after `prepare()`).

    Each Series has index levels [*parents[node], node] (bayes_net.py:360-365).
    Missing parent/child combinations (possible after `fit`) become zeros.
    """
    values_seen = {}
    for node, series in P.items():
        names = list(series.index.names)
        for lvl, name in enumerate(names):
            values_seen.setdefault(name, set()).update(series.index.get_level_values(lvl).unique().tolist())
    domains = {v: sorted(vals) for v, vals in values_seen.items()}
    net = DenseNet(nodes=list(nodes), parents={k: list(v) for k, v in parents.items()}, domains=domains)
    for node, series in P.items():
        scope = net.scope(node)
        assert list(series.index.names) == list(scope), (series.index.names, scope)
        arr = np.zeros([len(domains[v]) for v in scope], dtype=np.float64)
        pos = [{val: i for i, val in enumerate(domains[v])} for v in scope]
        for key, p in series.items():
            if not isinstance(key, tuple):
                key = (key,)
            arr[tuple(pos[i][k] for i, k in enumerate(key))] = p
        net.cpt[node] = arr
    return net


def full_joint(net: DenseNet) -> Factor:
    """Brute-force joint over all variables (independent check of the elimination;
    only for tiny networks).  Mirrors full_joint_dist (bayes_net.py:398-465)."""
    fs = [Factor(net.scope(n), net.cpt[n]) for n in net.nodes]
    j = pointwise_mul(fs)
    order = tuple(sorted(j.vars))
    perm = [j.vars.index(v) for v in order]
    vals = np.transpose(j.values, perm)
    return Factor(order, vals / vals.sum())


def brute_force_query(net: DenseNet, query_vars, event: dict):
    """Posterior from the full joint (tiny networks only)."""
    j = full_joint(net)
    index = []
    keep = []
    for v in j.vars:
        if v in event:
            index.append(net.domains[v].index(event[v]))
        else:
            index.append(slice(None))
            keep.append(v)
    vals = j.values[tuple(index)]
    drop = tuple(i for i, v in enumerate(keep) if v not in query_vars)
    vals = vals.sum(axis=drop)
    return tuple(v for v in keep if v in query_vars), vals / vals.sum()



def impute(net: DenseNet, sample: dict) -> dict:
    """`BayesNet.impute` (bayes_net.py:877-908): the `None` entries of `sample` are replaced by
    the most probable joint state of the missing variables given the others (`idxmax` of the
    exact posterior: the first maximum in sorted-index order)."""
    missing = [k for k, v in sample.items() if v is None]
    event = {k: v for k, v in sample.items() if v is not None}
    names, values, _ = query(net, *missing, event=event)
    best = np.unravel_index(int(np.argmax(values)), values.shape)  # C order == sorted MultiIndex order
    filled = dict(event)
    for name, idx in zip(names, best):
        filled[name] = net.domains[name][idx]
    return filled


def gibbs_conditional(net: DenseNet, node):
    """P(node | Markov boundary), the table `_gibbs_sampling` precomputes for every non-event
    variable (bayes_net.py:699-712): the product of the node's CPT and its children's CPTs,
    normalised over the node for every configuration of the boundary.

    Returns (boundary, table): boundary = parents, children and the children's other parents,
    sorted (bayes_net.py:1002-1039); table has axes [*boundary, node].  Configurations whose
    product is zero for every state (which the reference's zero-dropping join leaves out) are NaN."""
    children = [c for c in net.nodes if node in net.parents.get(c, ())]
    prod = pointwise_mul([Factor(net.scope(n), net.cpt[n]) for n in [node, *children]])
    boundary = sorted(v for v in prod.vars if v != node)
    perm = [prod.vars.index(v) for v in [*boundary, node]]
    vals = np.transpose(prod.values, perm)
    with np.errstate(invalid="ignore", divide="ignore"):
        table = vals / vals.sum(axis=-1, keepdims=True)
    return boundary, table


def gibbs_conditional_at(net: DenseNet, node, state: dict):
    """One row of `gibbs_conditional`: P(node | Markov boundary) for the boundary values in
    `state` (node -> state value; other entries are ignored), without building the table over the
    whole boundary, which a variable with many children cannot afford.  NaN when every state of
    `node` has probability zero."""
    children = [c for c in net.nodes if node in net.parents.get(c, ())]
    dom = net.domains[node]
    w = np.ones(len(dom))
    for n in [node, *children]:
        index = tuple(slice(None) if v == node else net.domains[v].index(state[v]) for v in net.scope(n))
        w = w * net.cpt[n][index]
    with np.errstate(invalid="ignore", divide="ignore"):
        return w / w.sum()
