"""Float64 oracle of score-based structure learning (test infrastructure; shares no code with
sorobn_b200/structure.py): contingency tables by np.bincount on flat family indices, BIC and BDeu with
math.lgamma, and a plain-Python greedy hill-climb following the documented move and tie rules."""
import math

import numpy as np


def encode(X):
    """{column: (int64 codes, number of states)}, states = the sorted distinct values."""
    out = {}
    for name in X.columns:
        values = X[name].tolist()
        states = sorted(set(values))
        pos = {s: i for i, s in enumerate(states)}
        out[name] = (np.array([pos[x] for x in values], dtype=np.int64), len(states))
    return out


def counts(data, child, parents):
    """The family's table, flat, child fastest, then the first parent, and so on."""
    flat = np.zeros(len(data[child][0]), dtype=np.int64)
    size = 1
    for m in (child, *parents):
        codes, r = data[m]
        flat += codes * size
        size *= r
    return np.bincount(flat, minlength=size)


def bic(table, r, n):
    rows = table.reshape(-1, r)
    total = 0.0
    for row in rows:
        nj = int(row.sum())
        for nk in row:
            if nk:
                total += int(nk) * math.log(int(nk) / nj)
    return total - 0.5 * math.log(n) * rows.shape[0] * (r - 1)


def bdeu(table, r, ess):
    rows = table.reshape(-1, r)
    q = rows.shape[0]
    a_j, a_jk = ess / q, ess / (q * r)
    total = 0.0
    for row in rows:
        total += math.lgamma(a_j) - math.lgamma(int(row.sum()) + a_j)
        for nk in row:
            total += math.lgamma(int(nk) + a_jk) - math.lgamma(a_jk)
    return total


def bdeu_gammaln(table, r, ess):
    """BDeu through scipy's gammaln, vectorised: the cross-check of `bdeu`."""
    from scipy.special import gammaln

    rows = table.reshape(-1, r).astype(np.float64)
    q = rows.shape[0]
    a_j, a_jk = ess / q, ess / (q * r)
    return float(np.sum(gammaln(a_j) - gammaln(rows.sum(axis=1) + a_j))
                 + np.sum(gammaln(rows + a_jk) - gammaln(a_jk)))


def bdeu_sequential(child_codes, parent_codes, r, q, ess):
    """Brute-force BDeu of a 2-variable family: the log marginal likelihood as the product over the rows, in
    order, of the Dirichlet-multinomial predictive probability of the row given the rows before it."""
    a_j, a_jk = ess / q, ess / (q * r)
    seen = np.zeros((q, r))
    total = 0.0
    for k, j in zip(child_codes, parent_codes):
        total += math.log((seen[j, k] + a_jk) / (seen[j].sum() + a_j))
        seen[j, k] += 1
    return total


def family_score(data, child, parents, score, ess=1.0):
    table = counts(data, child, parents)
    r = data[child][1]
    if score == "bic":
        return bic(table, r, len(data[child][0]))
    return bdeu(table, r, ess)


def scorer(X, score, ess=1.0):
    """families -> scores, the callable the search takes."""
    data = encode(X)
    return lambda families: [family_score(data, c, ps, score, ess) for c, ps in families]


def _reaches(children, a, b):
    """Whether a directed path a ~> b exists."""
    todo, seen = [a], {a}
    while todo:
        x = todo.pop()
        if x == b:
            return True
        for y in children[x]:
            if y not in seen:
                seen.add(y)
                todo.append(y)
    return False


def hill_climb(columns, cards, n_rows, score_fn, max_parents, start=(), tol=1e-9, margin=None):
    """Every graph the greedy search passes through (start first), each as sorted (parent, child) edges.
    `score_fn(child, parents_tuple)` scores one family.  With `margin`, asserts at every step that each move
    outside the tie band is at least margin * max(1, |best|) below the best change."""
    pos = {c: i for i, c in enumerate(columns)}
    edges = set(start)
    memo = {}

    def score(child, parents):
        key = (child, tuple(sorted(parents, key=pos.get)))
        if key not in memo:
            memo[key] = score_fn(*key)
        return memo[key]

    def table_ok(child, parents):
        size = cards[child]
        for p in parents:
            size *= cards[p]
        return size <= 1 << 22

    def snapshot():
        return sorted(edges, key=lambda e: (pos[e[1]], pos[e[0]]))

    history = [snapshot()]
    while True:
        par = {c: {u for u, v in edges if v == c} for c in columns}
        kids = {c: {v for u, v in edges if u == c} for c in columns}
        cands = []
        for u in columns:
            for v in columns:
                if u == v:
                    continue
                if (u, v) in edges:
                    d_v = score(v, par[v] - {u}) - score(v, par[v])
                    cands.append(((1, pos[u], pos[v]), d_v, (u, v), None))
                    if len(par[u]) < max_parents and table_ok(u, par[u] | {v}):
                        kids[u].discard(v)
                        other_path = _reaches(kids, u, v)
                        kids[u].add(v)
                        if not other_path:
                            d_u = score(u, par[u] | {v}) - score(u, par[u])
                            cands.append(((2, pos[u], pos[v]), d_v + d_u, (u, v), (v, u)))
                elif (v, u) not in edges and len(par[v]) < max_parents and not _reaches(kids, v, u) \
                        and table_ok(v, par[v] | {u}):
                    d = score(v, par[v] | {u}) - score(v, par[v])
                    cands.append(((0, pos[u], pos[v]), d, None, (u, v)))
        if not cands:
            return history
        best = max(c[1] for c in cands)
        if best <= tol * n_rows:
            return history
        band = 1e-9 * max(1.0, abs(best))
        if margin is not None:
            for c in cands:
                assert c[1] >= best - band or c[1] <= best - margin * max(1.0, abs(best)), \
                    f"move {c[0]} is {best - c[1]:.3e} below the best {best:.6f}: too close to the tie band"
        chosen = min(c for c in cands if c[1] >= best - band)
        _, _, drop, add = chosen
        if drop:
            edges.discard(drop)
        if add:
            edges.add(add)
        history.append(snapshot())


def total_score(data, edges, score, ess=1.0):
    par = {c: [] for c in data}
    for u, v in edges:
        par[v].append(u)
    return sum(family_score(data, c, tuple(ps), score, ess) for c, ps in par.items())
