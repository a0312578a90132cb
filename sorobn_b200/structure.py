"""Structure learning from complete discrete data.

* `family_scores` / `hill_climb`: score-based learning.  Every family's contingency table is counted, and
  reduced to its BIC or BDeu score, on the GPU over codes uploaded once (engine.Tally, csrc/sbn_tally.cu);
  the greedy search over DAGs runs here, on the host.
* `chow_liu`: the Chow-Liu tree (reference: /root/reference/sorobn/structure.py), host-side (pandas / numpy)
  like the reference: mutual information of every pair of columns, maximum spanning tree over those
  weights, edges oriented away from a root.  One deviation from the reference: its Kruskal loop stops as
  soon as every vertex has a neighbour (structure.py:33-41), so on some data it returns a FOREST; this one
  always completes the spanning tree.  On the reference's own example (tests/golden/chow_liu.json) the edge
  lists coincide; where they would not, this function has one extra edge per remaining component.

Every learner returns items of the `BayesNet` constructor grammar, so `BayesNet(*edges).fit(X)` follows.
"""
from __future__ import annotations

import itertools
import math

import numpy as np
import pandas as pd

from . import engine

__all__ = ["chow_liu", "climb", "family_scores", "hill_climb", "mutual_info"]

SCORES = ("bic", "bdeu")
MAX_STATES = 255
MAX_TABLE = engine.TALLY_MAX_TABLE
_BATCH_ENTRIES = 1 << 26  # table entries counted per device call (8 bytes each in the arena)


def mutual_info(puv: pd.Series, pu: pd.Series, pv: pd.Series) -> float:
    """I(u; v) from the joint `puv` (MultiIndex [u, v]) and the marginals (structure.py:59-67)."""
    u_name, v_name = puv.index.names
    mu = pu.reindex(puv.index.get_level_values(u_name)).to_numpy()
    mv = pv.reindex(puv.index.get_level_values(v_name)).to_numpy()
    joint = puv.to_numpy()
    return float((joint * np.log(joint / (mu * mv))).sum())


class _Forest:
    """Union-find with path halving and union by size (structure.py:70-98)."""

    def __init__(self, items):
        self.parent = {x: x for x in items}
        self.size = {x: 1 for x in items}

    def find(self, x):
        while self.parent[x] != x:
            self.parent[x] = self.parent[self.parent[x]]
            x = self.parent[x]
        return x

    def union(self, a, b):
        a, b = self.find(a), self.find(b)
        if a == b:
            return False
        if self.size[a] < self.size[b]:
            a, b = b, a
        self.parent[b] = a
        self.size[a] += self.size[b]
        return True


def chow_liu(X: pd.DataFrame, root=None):
    """Edges (parent, child) of the Chow-Liu tree of `X` (structure.py:9-56): the maximum
    spanning tree of the pairwise mutual informations (Kruskal), oriented away from `root`
    (default: the first column)."""
    marginals = {c: X[c].value_counts(normalize=True) for c in X.columns}
    n = len(X)
    scored = []
    for u, v in itertools.combinations(sorted(X.columns), 2):
        joint = X.groupby([u, v]).size() / n
        scored.append((mutual_info(joint, marginals[u], marginals[v]), u, v))
    # stable sort by decreasing mutual information: ties keep the (u, v) enumeration order, as
    # the reference's `sorted(..., reverse=True)` on the same keys does
    scored.sort(key=lambda t: t[0], reverse=True)

    forest = _Forest(X.columns)
    neighbours = {c: set() for c in X.columns}
    taken = 0
    for _, u, v in scored:
        if forest.union(u, v):
            neighbours[u].add(v)
            neighbours[v].add(u)
            taken += 1
            if taken == len(X.columns) - 1:
                break

    root = X.columns[0] if root is None else root
    edges, seen, stack = [], {root}, [root]
    while stack:
        node = stack.pop()
        for nb in sorted(neighbours[node] - seen, reverse=True):
            seen.add(nb)
            edges.append((node, nb))
            stack.append(nb)
    return edges


# ------------------------------------------------------------------------- score-based learning
def _check_score(score, ess):
    if score not in SCORES:
        raise ValueError(f"score must be one of {SCORES}, not {score!r}")
    if not ess > 0:
        raise ValueError(f"ess must be positive, not {ess!r}")


def _encode(X: pd.DataFrame):
    """(column names, uint8 state codes [n_vars, n_rows], states per column) of a complete discrete frame."""
    if not isinstance(X, pd.DataFrame) or X.shape[0] == 0 or X.shape[1] == 0:
        raise ValueError("X must be a DataFrame with at least one row and one column")
    if not X.columns.is_unique:
        raise ValueError("X has duplicate column names")
    columns = list(X.columns)
    codes = np.empty((len(columns), len(X)), dtype=np.uint8)
    cards = []
    for v, name in enumerate(columns):
        col, states = pd.factorize(X[name], sort=True)
        if (col < 0).any():
            raise ValueError(f"column {name!r} has missing cells (None or NaN); structure learning needs complete data")
        if len(states) > MAX_STATES:
            raise ValueError(f"column {name!r} has {len(states)} states; at most {MAX_STATES} are supported")
        codes[v] = col
        cards.append(len(states))
    return columns, codes, cards


def _family_ids(families, columns, cards):
    """[child id, *parent ids] of every (child, parents) pair of column names, checked."""
    index = {c: i for i, c in enumerate(columns)}
    out = []
    for child, parents in families:
        parents = tuple(parents)
        for name in (child, *parents):
            if name not in index:
                raise ValueError(f"unknown column {name!r} in family ({child!r}, {parents!r})")
        if child in parents:
            raise ValueError(f"{child!r} is listed among its own parents")
        if len(set(parents)) != len(parents):
            raise ValueError(f"duplicate parent in family ({child!r}, {parents!r})")
        ids = [index[child], *(index[p] for p in parents)]
        if math.prod(cards[i] for i in ids) > MAX_TABLE:
            raise ValueError(f"the table of family ({child!r}, {parents!r}) has more than {MAX_TABLE} entries")
        out.append(ids)
    return out


def _device_scores(tally, ids, score, ess):
    """Scores of the families `ids` on `tally`, in device calls of at most _BATCH_ENTRIES table entries."""
    out, batch, entries = [], [], 0
    for fam in ids:
        size = math.prod(int(tally.cards[i]) for i in fam)
        if batch and entries + size > _BATCH_ENTRIES:
            out.append(tally.scores(batch, score, ess))
            batch, entries = [], 0
        batch.append(fam)
        entries += size
    if batch:
        out.append(tally.scores(batch, score, ess))
    return np.concatenate(out) if out else np.empty(0)


def family_scores(X: pd.DataFrame, families, score: str = "bic", ess: float = 1.0, device: int | None = None) -> np.ndarray:
    """The decomposable score of every family, computed on the GPU: float64 [len(families)].

    `families` is a list of (child, parents) pairs of column names of `X`; `parents` is a tuple, which may be
    empty.  `X` is uploaded to `device` once, and each family's table is counted and scored there.

    Data: `X` must be complete, discrete data.  A column's states are its sorted distinct values, and r is
    their number; q is the product of the parents' r and counts every parent configuration, seen or not.
    With N the number of rows, N_jk the rows with parent configuration j and child state k, N_j = sum_k N_jk:

    * BIC:  sum_j sum_k N_jk ln(N_jk / N_j) - 1/2 ln(N) q (r - 1), with 0 ln 0 = 0;
    * BDeu, with equivalent sample size a = `ess`:
      sum_j [lnG(a/q) - lnG(N_j + a/q) + sum_k (lnG(N_jk + a/(q r)) - lnG(a/(q r)))].

    ValueError for a missing cell (None or NaN: structure from incomplete data is not supported), a column
    with more than 255 states, an empty frame, an unknown or duplicate column in a family or a child among its
    own parents, `score` other than "bic" / "bdeu", `ess` <= 0, and a family whose table has more than 2^22
    entries.
    """
    _check_score(score, ess)
    columns, codes, cards = _encode(X)
    ids = _family_ids(families, columns, cards)
    if not ids:
        return np.empty(0)
    tally = engine.Tally(codes, cards, device)
    try:
        return _device_scores(tally, ids, score, ess)
    finally:
        tally.close()



def _start_parents(columns, cards, start, max_parents):
    """Parent sets (column positions) of the edge list `start`, checked: known columns, acyclic, at most
    `max_parents` parents and tables of at most MAX_TABLE entries."""
    index = {c: i for i, c in enumerate(columns)}
    parents = [set() for _ in columns]
    for edge in start or ():
        u, v = edge
        for name in (u, v):
            if name not in index:
                raise ValueError(f"start edge {edge!r} names the unknown column {name!r}")
        if u == v:
            raise ValueError(f"start edge {edge!r} is a self-loop")
        parents[index[v]].add(index[u])
    for v, ps in enumerate(parents):
        if len(ps) > max_parents:
            raise ValueError(f"start gives {columns[v]!r} {len(ps)} parents; max_parents is {max_parents}")
        if cards[v] * math.prod(cards[p] for p in ps) > MAX_TABLE:
            raise ValueError(f"start gives {columns[v]!r} a table of more than {MAX_TABLE} entries")
    state = [0] * len(columns)  # 0 unseen, 1 on the DFS stack, 2 done

    def visit(v):
        state[v] = 1
        for p in parents[v]:
            if state[p] == 1 or (state[p] == 0 and visit(p)):
                return True
        state[v] = 2
        return False

    if any(state[v] == 0 and visit(v) for v in range(len(columns))):
        raise ValueError("start is cyclic")
    return parents


def climb(columns, cards, n_rows, scorer, max_parents=3, start=None, tol=1e-9):
    """Greedy hill-climbing over DAGs on `columns` (with `cards` states each, `n_rows` rows of data): checks
    `start` and `max_parents`, then returns a generator of the graphs it passes through, the start first and
    then the graph after every move, each as (parent, child) edges sorted by (child position, parent position).

    `scorer(families)` returns the scores of a list of (child, parents tuple) families, parents in column
    order; it is called once per step, with every family the step needs that no earlier call scored.

    Legal moves: add u->v when there is no edge between u and v, v has fewer than `max_parents` parents and v
    is not an ancestor of u; remove u->v; reverse u->v when u has fewer than `max_parents` parents and no path
    u ~> v exists but the edge.  A move whose new family's table would pass 2^22 entries is illegal.  A move's
    change in score is the change of the families it touches (both, for a reversal).  Each step takes the best
    change, stops when it is <= tol * n_rows, and otherwise applies the first move, in the order add < remove <
    reverse and then (u, v) by column position, whose change is within 1e-9 * max(1, |best|) of the best: BIC
    and BDeu are score-equivalent, so adding u->v or v->u changes the score by the same amount up to rounding.
    """
    if max_parents < 0:
        raise ValueError(f"max_parents must be >= 0, not {max_parents}")
    parents = _start_parents(columns, cards, start, max_parents)
    return _climb_steps(list(columns), list(cards), n_rows, scorer, max_parents, parents, tol)


def _climb_steps(columns, cards, n_rows, scorer, max_parents, parents, tol):
    n = len(columns)
    cache = {}

    def graph():
        return [(columns[p], columns[v]) for v in range(n) for p in sorted(parents[v])]

    def fits(v, ps):
        return cards[v] * math.prod(cards[p] for p in ps) <= MAX_TABLE

    yield graph()
    while True:
        ancestors = [set() for _ in range(n)]
        for v in range(n):
            stack = list(parents[v])
            while stack:
                p = stack.pop()
                if p not in ancestors[v]:
                    ancestors[v].add(p)
                    stack.extend(parents[p])
        moves = []  # (kind, u, v, ((child, old parents, new parents), ...)); kind 0 add, 1 remove, 2 reverse
        for u in range(n):
            for v in range(n):
                if u == v:
                    continue
                if u in parents[v]:
                    moves.append((1, u, v, ((v, parents[v], parents[v] - {u}),)))
                    others = any(u in ancestors[p] for p in parents[v] if p != u)
                    if len(parents[u]) < max_parents and not others and fits(u, parents[u] | {v}):
                        moves.append((2, u, v, ((v, parents[v], parents[v] - {u}), (u, parents[u], parents[u] | {v}))))
                elif v not in parents[u] and len(parents[v]) < max_parents and v not in ancestors[u] \
                        and fits(v, parents[v] | {u}):
                    moves.append((0, u, v, ((v, parents[v], parents[v] | {u}),)))
        if not moves:
            return
        keys = {(c, tuple(sorted(ps))) for _, _, _, touched in moves for c, old, new in touched for ps in (old, new)}
        missing = sorted(k for k in keys if k not in cache)
        if missing:
            got = scorer([(columns[c], tuple(columns[p] for p in ps)) for c, ps in missing])
            cache.update(zip(missing, (float(x) for x in got)))

        def delta(touched):
            return sum(cache[(c, tuple(sorted(new)))] - cache[(c, tuple(sorted(old)))] for c, old, new in touched)

        scored = sorted((kind, u, v, delta(touched), touched) for kind, u, v, touched in moves)
        best = max(d for _, _, _, d, _ in scored)
        if best <= tol * n_rows:
            return
        floor = best - 1e-9 * max(1.0, abs(best))
        kind, u, v, _, touched = next(m for m in scored if m[3] >= floor)
        for c, _, new in touched:
            parents[c] = set(new)
        yield graph()


def hill_climb(X: pd.DataFrame, score: str = "bic", max_parents: int = 3, ess: float = 1.0, start=None,
               tol: float = 1e-9, device: int | None = None) -> list:
    """Learn a DAG on the columns of `X` by greedy hill-climbing (see `climb` for the moves and the tie rule),
    every family score counted on the GPU over codes uploaded once.

    `start` is a list of (parent, child) edges to start from (default: the empty graph).  Returns structure
    items of the `BayesNet` constructor: the (parent, child) edges sorted by (child column position, parent
    column position), then the bare name of every column without an edge, so that `BayesNet(*hill_climb(X))
    .fit(X)` builds a network over every column.

    Data: `X` must be complete, discrete data.  A column's states are its sorted distinct values, and r is
    their number; q is the product of the parents' r and counts every parent configuration, seen or not.
    With N the number of rows, N_jk the rows with parent configuration j and child state k, N_j = sum_k N_jk:

    * BIC:  sum_j sum_k N_jk ln(N_jk / N_j) - 1/2 ln(N) q (r - 1), with 0 ln 0 = 0;
    * BDeu, with equivalent sample size a = `ess`:
      sum_j [lnG(a/q) - lnG(N_j + a/q) + sum_k (lnG(N_jk + a/(q r)) - lnG(a/(q r)))].

    ValueError for a missing cell (None or NaN: structure from incomplete data is not supported), a column
    with more than 255 states, an empty frame, `score` other than "bic" / "bdeu", `ess` <= 0, `max_parents` < 0,
    and a `start` that is cyclic, names unknown columns or exceeds `max_parents`.  A move that would create a
    family of more than 2^22 table entries is illegal rather than an error.
    """
    _check_score(score, ess)
    columns, codes, cards = _encode(X)
    tally = None

    def scorer(families):
        return _device_scores(tally, _family_ids(families, columns, cards), score, ess)

    steps = climb(columns, cards, len(X), scorer, max_parents, start, tol)
    tally = engine.Tally(codes, cards, device)
    try:
        for edges in steps:
            pass
    finally:
        tally.close()
    linked = {name for edge in edges for name in edge}
    return edges + [c for c in columns if c not in linked]

