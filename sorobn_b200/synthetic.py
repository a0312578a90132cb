"""Synthetic Bayesian networks of the shapes BASELINE.json names.

`grid(10, 10, 5)` is the "synthetic 10x10 grid, 5 states/node" network and
`random_dag(50, 4, 8)` the "50-node random DAG, max 4 parents, 8 states/node"
one.  A spec is plain data (edges + one pandas Series per node), so the same spec
can be loaded into this package's `BayesNet` or, in the build container, into the
reference's `sorobn.BayesNet` (that is how `oracle/gen_golden.py` pins parity).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import pandas as pd

__all__ = ["NetSpec", "grid", "random_dag", "chain", "load"]


@dataclass
class NetSpec:
    name: str
    nodes: list  # every node, in generation order
    parents: dict  # node -> sorted list of parents (roots absent)
    n_states: dict  # node -> number of states
    cpt: dict  # node -> ndarray, axes [*parents, node], float64, rows sum to 1

    @property
    def edges(self):
        return [(p, c) for c, ps in self.parents.items() for p in ps]

    def series(self, node) -> pd.Series:
        """The CPT as the pandas Series `BayesNet.P[node]` expects."""
        scope = [*self.parents.get(node, []), node]
        arr = self.cpt[node]
        if len(scope) == 1:
            s = pd.Series(arr, index=pd.Index(range(self.n_states[node]), name=node))
        else:
            idx = pd.MultiIndex.from_product([range(self.n_states[v]) for v in scope], names=scope)
            s = pd.Series(arr.reshape(-1), index=idx)
        return s


def _random_cpt(rng, parent_cards, card, alpha=1.0):
    shape = (*parent_cards, card)
    arr = rng.gamma(alpha, 1.0, size=shape)
    arr /= arr.sum(axis=-1, keepdims=True)
    return arr


def grid(rows: int, cols: int, n_states, seed: int = 0, alpha: float = 1.0) -> NetSpec:
    """rows x cols lattice; node (i, j) has parents (i-1, j) and (i, j-1).

    Node names are strings "gRRCC" so that lexicographic order == row-major order.
    `n_states` is one cardinality for every node or a sequence cycled over the nodes in
    row-major order.
    """
    rng = np.random.default_rng(seed)
    name = lambda i, j: f"g{i:02d}{j:02d}"
    nodes, parents, cards, cpt = [], {}, {}, {}
    for i in range(rows):
        for j in range(cols):
            n = name(i, j)
            ps = []
            if i > 0:
                ps.append(name(i - 1, j))
            if j > 0:
                ps.append(name(i, j - 1))
            ps.sort()
            if ps:
                parents[n] = ps
            k = len(nodes)
            cards[n] = int(n_states) if np.isscalar(n_states) else int(n_states[k % len(n_states)])
            nodes.append(n)
    for n in nodes:
        cpt[n] = _random_cpt(rng, [cards[p] for p in parents.get(n, [])], cards[n], alpha)
    tag = n_states if np.isscalar(n_states) else "x".join(map(str, n_states))
    return NetSpec(f"grid{rows}x{cols}s{tag}", nodes, parents, cards, cpt)


def random_dag(n_nodes: int, max_parents: int, n_states, seed: int = 0, alpha: float = 1.0,
               window: int | None = None) -> NetSpec:
    """Random DAG: node k draws 0..max_parents parents among the `window` nodes
    before it (all earlier nodes when window is None).  A finite window keeps the
    induced width bounded, like the banded structure of real diagnostic networks.
    `n_states` is one cardinality for every node or a sequence cycled over the nodes."""
    rng = np.random.default_rng(seed)
    width = len(str(n_nodes - 1))
    nodes = [f"v{k:0{width}d}" for k in range(n_nodes)]
    states = [n_states] * n_nodes if isinstance(n_states, int) else [n_states[k % len(n_states)] for k in range(n_nodes)]
    parents, cards, cpt = {}, {n: int(c) for n, c in zip(nodes, states)}, {}
    for k, n in enumerate(nodes):
        lo = 0 if window is None else max(0, k - window)
        pool = nodes[lo:k]
        n_par = int(rng.integers(0, max_parents + 1))
        n_par = min(n_par, len(pool))
        if n_par:
            ps = sorted(rng.choice(pool, size=n_par, replace=False).tolist())
            parents[n] = ps
    for n in nodes:
        cpt[n] = _random_cpt(rng, [cards[p] for p in parents.get(n, [])], cards[n], alpha)
    tag = n_states if isinstance(n_states, int) else "x".join(map(str, n_states))
    return NetSpec(f"dag{n_nodes}p{max_parents}s{tag}", nodes, parents, cards, cpt)


def chain(n_nodes: int, n_states: int, seed: int = 0) -> NetSpec:
    rng = np.random.default_rng(seed)
    width = len(str(n_nodes - 1))
    nodes = [f"c{k:0{width}d}" for k in range(n_nodes)]
    parents = {nodes[k]: [nodes[k - 1]] for k in range(1, n_nodes)}
    cards = {n: n_states for n in nodes}
    cpt = {n: _random_cpt(rng, [cards[p] for p in parents.get(n, [])], cards[n]) for n in nodes}
    return NetSpec(f"chain{n_nodes}s{n_states}", nodes, parents, cards, cpt)


def load(spec: NetSpec, cls, **kwargs):
    """Instantiate `cls` (this package's BayesNet or the reference's) from a spec."""
    structure = list(spec.edges) + [n for n in spec.nodes if n not in spec.parents
                                    and not any(n in ps for ps in spec.parents.values())]
    bn = cls(*structure, **kwargs)
    for n in spec.nodes:
        bn.P[n] = spec.series(n)
    bn.prepare()
    return bn


def random_events(spec: NetSpec, evidence_vars, n_rows: int, seed: int = 0) -> pd.DataFrame:
    """Evidence rows drawn by forward-sampling the network (so every row has
    positive probability), restricted to `evidence_vars`."""
    rng = np.random.default_rng(seed)
    state = {}
    # nodes are generated parents-first, so generation order is topological
    for n in spec.nodes:
        ps = spec.parents.get(n, [])
        table = spec.cpt[n]
        if ps:
            probs = table[tuple(state[p] for p in ps)]
        else:
            probs = np.broadcast_to(table, (n_rows, table.shape[-1]))
        cdf = np.cumsum(probs, axis=-1)
        u = rng.random((n_rows, 1))
        state[n] = np.minimum((u > cdf).sum(axis=-1), table.shape[-1] - 1)
    return pd.DataFrame({v: state[v] for v in evidence_vars})

