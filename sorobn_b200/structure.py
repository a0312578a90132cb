"""Structure learning from complete discrete data.

* `family_scores` / `hill_climb`: score-based learning.  Every family's contingency table is counted, and
  reduced to its BIC or BDeu score, on the GPU over codes uploaded once (engine.Tally, csrc/sbn_tally.cu);
  the greedy search over DAGs runs here, on the host.
* `ci_tests` / `pc_cpdag` / `pc`: constraint-based learning by the PC algorithm (PC-stable skeleton, separating
  sets, v-structures, Meek's rules R1-R3).  Every conditional-independence test of one level of the search is
  counted and reduced to its G^2 or X^2 statistic, degrees of freedom and p-value on the GPU in one batch over the
  same resident codes; `pc_search` (the search, driven by any tester) runs here, on the host.
* `chow_liu`: the Chow-Liu tree (reference: /root/reference/sorobn/structure.py), host-side (pandas / numpy)
  like the reference: mutual information of every pair of columns, maximum spanning tree over those
  weights, edges oriented away from a root.  One deviation from the reference: its Kruskal loop stops as
  soon as every vertex has a neighbour (structure.py:33-41), so on some data it returns a FOREST; this one
  always completes the spanning tree.  On the reference's own example (tests/golden/chow_liu.json) the edge
  lists coincide; where they would not, this function has one extra edge per remaining component.

Every learner returns items of the `BayesNet` constructor grammar, so `BayesNet(*edges).fit(X)` follows.
"""
from __future__ import annotations

import collections
import itertools
import math

import numpy as np
import pandas as pd

from . import engine

__all__ = ["CPDAG", "chow_liu", "ci_tests", "climb", "family_scores", "hill_climb", "mutual_info", "pc", "pc_cpdag",
           "pc_search"]

SCORES = ("bic", "bdeu")
TESTS = ("g2", "chi2")
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



# ------------------------------------------------------------------------- constraint-based learning
CPDAG = collections.namedtuple("CPDAG", ["directed", "undirected", "sepsets"])
CPDAG.__doc__ = """The result of `pc_search`: `directed` (parent, child) edges and `undirected` (a, b) edges, a before b
in column order, each list sorted by column position; `sepsets` maps every non-adjacent pair (u, v), u before v,
to the tuple of columns whose test separated them."""


def _test_ids(tests, columns, cards):
    """[x id, y id, *given ids] of every (x, y, given) triple of column names, checked."""
    index = {c: i for i, c in enumerate(columns)}
    out = []
    for x, y, given in tests:
        given = tuple(given)
        for name in (x, y, *given):
            if name not in index:
                raise ValueError(f"unknown column {name!r} in test ({x!r}, {y!r}, {given!r})")
        if x == y:
            raise ValueError(f"test ({x!r}, {y!r}, {given!r}) tests a column against itself")
        if x in given or y in given:
            raise ValueError(f"test ({x!r}, {y!r}, {given!r}) conditions on one of its own pair")
        if len(set(given)) != len(given):
            raise ValueError(f"duplicate column in the conditioning set of test ({x!r}, {y!r}, {given!r})")
        ids = [index[x], index[y], *(index[g] for g in given)]
        if math.prod(cards[i] for i in ids) > MAX_TABLE:
            raise ValueError(f"the table of test ({x!r}, {y!r}, {given!r}) has more than {MAX_TABLE} entries")
        out.append(ids)
    return out


def _device_tests(tally, ids, test):
    """(statistic, dof, p-value) of the tests `ids` on `tally`, in device calls of at most _BATCH_ENTRIES table
    entries: float64 [len(ids), 3]."""
    out, batch, entries = [], [], 0
    for t in ids:
        size = math.prod(int(tally.cards[i]) for i in t)
        if batch and entries + size > _BATCH_ENTRIES:
            out.append(tally.tests(batch, test))
            batch, entries = [], 0
        batch.append(t)
        entries += size
    if batch:
        out.append(tally.tests(batch, test))
    return np.concatenate(out) if out else np.empty((0, 3))


def _check_test(test):
    if test not in TESTS:
        raise ValueError(f"test must be one of {TESTS}, not {test!r}")


def ci_tests(X: pd.DataFrame, tests, test: str = "g2", device: int | None = None) -> np.ndarray:
    """Conditional-independence tests x _|_ y | given on the data `X`, each table counted and reduced on the GPU:
    float64 [len(tests), 3] of (statistic, degrees of freedom, p-value).

    `tests` is a list of (x, y, given) column names of `X`, `given` a tuple that may be empty.  Data as in
    `family_scores`: complete, discrete, a column's states its sorted distinct values.  Per configuration z of
    `given` (a stratum), N_z is its rows, N_xz = sum_y N_xyz and N_yz = sum_x N_xyz:

    * "g2": G^2 = 2 sum N_xyz ln(N_xyz N_z / (N_xz N_yz)) over the non-zero cells;
    * "chi2": Pearson X^2 = sum (N_xyz - E)^2 / E with E = N_xz N_yz / N_z, over the cells with E > 0.

    dof = sum_z (a_z - 1)(b_z - 1), with a_z (b_z) the states of x (y) seen in stratum z; an empty stratum adds 0
    (scipy's `chi2_contingency` on each stratum's observed rows and columns, summed).  p = Q(dof / 2, stat / 2),
    the chi-square survival function, and 1 when dof = 0.

    ValueError for a missing cell, a column with more than 255 states or an empty frame, an unknown column, x == y,
    x or y among `given`, a duplicate in `given`, a table of more than 2^22 entries, and `test` other than "g2" /
    "chi2".
    """
    _check_test(test)
    columns, codes, cards = _encode(X)
    ids = _test_ids(tests, columns, cards)
    if not ids:
        return np.empty((0, 3))
    tally = engine.Tally(codes, cards, device)
    try:
        return _device_tests(tally, ids, test)
    finally:
        tally.close()


def _check_pc(alpha, max_cond):
    if not 0.0 < alpha < 1.0:
        raise ValueError(f"alpha must lie in (0, 1), not {alpha!r}")
    if max_cond is not None and max_cond < 0:
        raise ValueError(f"max_cond must be None or >= 0, not {max_cond!r}")


def _reaches(directed, src, dst):
    """True when a directed path src ~> dst exists along the (a, b) edges of `directed`."""
    out = collections.defaultdict(list)
    for a, b in directed:
        out[a].append(b)
    seen, stack = {src}, [src]
    while stack:
        a = stack.pop()
        if a == dst:
            return True
        for b in out[a]:
            if b not in seen:
                seen.add(b)
                stack.append(b)
    return False


def _orient(directed, a, b):
    """Orient the undirected edge a - b as a -> b unless that would close a directed cycle; True if it did."""
    if _reaches(directed, b, a):
        return False
    directed.add((a, b))
    return True


def _undirected(adj, directed):
    return [(a, b) for a in range(len(adj)) for b in sorted(adj[a])
            if a < b and (a, b) not in directed and (b, a) not in directed]


def _colliders(adj, directed, sepsets):
    """Orient the v-structures u -> z <- v of the unshielded triples, in (u, v, z) position order."""
    n = len(adj)
    for u in range(n):
        for v in range(u + 1, n):
            if v in adj[u]:
                continue
            for z in sorted(adj[u] & adj[v]):
                if z in sepsets[(u, v)]:
                    continue
                for a in (u, v):
                    if (a, z) not in directed and (z, a) not in directed:
                        _orient(directed, a, z)


def _meek(adj, directed):
    """Apply Meek's rules R1-R3 to a fixpoint: each round orients the first (edge, rule, direction) that fires,
    scanning undirected edges a - b (a < b) in position order, then R1, R2, R3, then a -> b before b -> a."""

    def fires(rule, i, j):
        if rule == 1:  # k -> i - j, k and j non-adjacent
            return any((k, i) in directed and k not in adj[j] for k in adj[i])
        if rule == 2:  # i -> k -> j
            return any((i, k) in directed and (k, j) in directed for k in adj[i])
        und = [k for k in adj[i] if k != j and (k, i) not in directed and (i, k) not in directed and (k, j) in directed]
        return any(l not in adj[k] for k, l in itertools.combinations(und, 2))  # i - k -> j, i - l -> j

    while True:
        for a, b in _undirected(adj, directed):
            if any(fires(rule, i, j) and _orient(directed, i, j) for rule in (1, 2, 3) for i, j in ((a, b), (b, a))):
                break
        else:
            return


def pc_search(columns, cards, tester, alpha: float = 0.05, max_cond: int | None = None) -> CPDAG:
    """The PC algorithm over `columns` (with `cards` states each), driven by `tester`; returns a `CPDAG`.

    `tester(tests)` gets every distinct test of one level as (x, y, given) column names, x before y in column
    order and `given` in column order, and returns their p-values; a NaN p-value means "not tested" and counts as
    dependent.  A test whose table would pass 2^22 entries is not sent: its p-value is NaN.

    * Skeleton (PC-stable).  Start from the complete graph.  At level l = 0, 1, 2, .. freeze every adjacency set
      adj(.) at the start of the level.  For each adjacent pair u < v (by column position) the candidate sets are
      the l-subsets of adj(u) \\ {v}, in lexicographic position order, then those of adj(v) \\ {u}; the edge is
      removed (after the level) when some candidate has p >= alpha, and sepset(u, v) is the first such candidate
      in that order.  The search stops after a level at which no pair has l + 1 candidates, or after level
      `max_cond`.  Every test of a level is known from the frozen adjacencies, so one tester call per level gives
      exactly what sequential PC-stable with early exit gives.
    * V-structures.  Visit the unshielded triples u - z - v, u < v non-adjacent, in (u, v, z) position order;
      when z is not in sepset(u, v), orient u -> z and then v -> z.  An edge already oriented keeps its first
      orientation, and an orientation that would close a directed cycle is skipped.
    * Meek's rules R1-R3, to a fixpoint: scan the undirected edges a - b (a < b) in position order and apply the
      first rule that fires (R1, R2, R3, each tried as a -> b and then b -> a); an orientation that would close a
      directed cycle is skipped.  R1: k -> i - j, k and j non-adjacent gives i -> j.  R2: i -> k -> j gives i -> j.
      R3: i - k -> j and i - l -> j with k and l non-adjacent, i - j, gives i -> j.

    ValueError for `alpha` outside (0, 1) and `max_cond` < 0.
    """
    _check_pc(alpha, max_cond)
    columns, cards = list(columns), [int(r) for r in cards]
    n = len(columns)
    adj = [set(range(n)) - {v} for v in range(n)]
    sepsets = {}
    level = 0
    while max_cond is None or level <= max_cond:
        frozen = [sorted(a) for a in adj]
        cands = {}
        for u in range(n):
            for v in frozen[u]:
                if v > u:
                    cands[(u, v)] = [*itertools.combinations([w for w in frozen[u] if w != v], level),
                                     *itertools.combinations([w for w in frozen[v] if w != u], level)]
        if not any(cands.values()):
            break
        keys = list(dict.fromkeys(((u, v, s) for (u, v), sets in cands.items() for s in sets)))
        sent = [k for k in keys if math.prod(cards[i] for i in (k[0], k[1], *k[2])) <= MAX_TABLE]
        pvals = dict.fromkeys(keys, math.nan)
        if sent:
            got = tester([(columns[u], columns[v], tuple(columns[i] for i in s)) for u, v, s in sent])
            pvals.update(zip(sent, (float(p) for p in got)))
        for (u, v), sets in cands.items():
            for s in sets:
                if pvals[(u, v, s)] >= alpha:
                    adj[u].discard(v)
                    adj[v].discard(u)
                    sepsets[(u, v)] = s
                    break
        level += 1
    directed = set()
    _colliders(adj, directed, sepsets)
    _meek(adj, directed)
    return CPDAG(directed=[(columns[a], columns[b]) for a, b in sorted(directed)],
                 undirected=[(columns[a], columns[b]) for a, b in _undirected(adj, directed)],
                 sepsets={(columns[u], columns[v]): tuple(columns[i] for i in s) for (u, v), s in sorted(sepsets.items())})


def _dag_edges(columns, cpdag):
    """The (parent, child) edges of one DAG in the class of `cpdag`, by Dor and Tarsi's extension: repeatedly take
    the lowest-position node with no outgoing directed edge whose undirected neighbours are adjacent to all of its
    other neighbours (or, if none qualifies, the lowest-position node with no outgoing directed edge), direct its
    undirected edges into it and remove it.  Sorted by (child position, parent position)."""
    index = {c: i for i, c in enumerate(columns)}
    n = len(columns)
    directed = {(index[a], index[b]) for a, b in cpdag.directed}
    undirected = {frozenset((index[a], index[b])) for a, b in cpdag.undirected}
    edges = set(directed)
    alive = set(range(n))

    def nbrs(x):
        return {b for a, b in directed if a == x and b in alive} | {a for a, b in directed if b == x and a in alive} | \
               {y for e in undirected if x in e for y in e if y != x and y in alive}

    def adjacent(a, b):
        return (a, b) in directed or (b, a) in directed or frozenset((a, b)) in undirected

    while alive:
        sinks = [x for x in sorted(alive) if not any(a == x and b in alive for a, b in directed)]
        pick = sinks[0]
        for x in sinks:
            around = nbrs(x)
            und = [y for y in around if frozenset((x, y)) in undirected]
            if all(adjacent(y, w) for y in und for w in around if w != y):
                pick = x
                break
        for e in [e for e in undirected if pick in e]:
            (y,) = e - {pick}
            if y in alive:
                edges.add((y, pick))
                undirected.discard(e)
        alive.discard(pick)
    return [(columns[a], columns[b]) for a, b in sorted(edges, key=lambda e: (e[1], e[0]))]


def pc_cpdag(X: pd.DataFrame, alpha: float = 0.05, test: str = "g2", max_cond: int | None = None,
             device: int | None = None) -> CPDAG:
    """The Markov equivalence class of `X`'s network by the PC algorithm (`pc_search`), each level's tests counted
    and reduced to p-values on the GPU (`ci_tests`) over codes uploaded once.

    Data as in `ci_tests`: complete and discrete; incomplete data is refused, as `hill_climb` refuses it.
    ValueError for a missing cell, a column with more than 255 states, an empty frame, `test` other than "g2" /
    "chi2", `alpha` outside (0, 1) and `max_cond` < 0.
    """
    _check_test(test)
    _check_pc(alpha, max_cond)
    columns, codes, cards = _encode(X)
    tally = engine.Tally(codes, cards, device)
    try:
        return pc_search(columns, cards, lambda tests: _device_tests(tally, _test_ids(tests, columns, cards), test)[:, 2],
                         alpha, max_cond)
    finally:
        tally.close()


def pc(X: pd.DataFrame, alpha: float = 0.05, test: str = "g2", max_cond: int | None = None,
       device: int | None = None) -> list:
    """Learn a DAG on the columns of `X` by the PC algorithm (`pc_cpdag`, same arguments and errors), then pick
    one DAG of the class by Dor and Tarsi's extension: repeatedly take the lowest-position node with no outgoing
    directed edge whose undirected neighbours are adjacent to all of its other neighbours, direct its undirected
    edges into it and remove it; if no node qualifies (only with conflicting finite-sample orientations), take the
    lowest-position node with no outgoing directed edge.

    Returns structure items of the `BayesNet` constructor, as `hill_climb` does: the (parent, child) edges sorted
    by (child column position, parent column position), then the bare name of every column without an edge, so
    that `BayesNet(*pc(X)).fit(X)` builds a network over every column.
    """
    cpdag = pc_cpdag(X, alpha, test, max_cond, device)
    columns = list(X.columns)
    edges = _dag_edges(columns, cpdag)
    linked = {name for edge in edges for name in edge}
    return edges + [c for c in columns if c not in linked]
