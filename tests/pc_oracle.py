"""Oracles of the PC algorithm (test infrastructure; shares no code with sorobn_b200/structure.py):

* `d_separated`: d-separation in a DAG, by reachability in the moralised graph of the ancestral set;
* `cpdag`: the CPDAG of a DAG by brute force, every orientation of its skeleton with the same v-structures;
* `sequential_pc`: plain PC-stable, one test at a time with early exit, and its own orientation code on an
  adjacency matrix, following the rules written in the docstring of structure.pc_search."""
import itertools
import math

import numpy as np

MAX_TABLE = 1 << 22


# ------------------------------------------------------------------------------------ d-separation
def d_separated(parents, x, y, given):
    """True when x and y are d-separated by `given` in the DAG {node: parents}."""
    given = set(given)
    anc, stack = set(), [x, y, *given]
    while stack:
        v = stack.pop()
        if v not in anc:
            anc.add(v)
            stack.extend(parents.get(v, ()))
    moral = {v: set() for v in anc}
    for v in anc:
        ps = list(parents.get(v, ()))
        for p in ps:
            moral[v].add(p)
            moral[p].add(v)
        for p, q in itertools.combinations(ps, 2):
            moral[p].add(q)
            moral[q].add(p)
    seen, stack = {x}, [x]
    while stack:
        v = stack.pop()
        if v == y:
            return False
        for w in moral[v]:
            if w not in seen and w not in given:
                seen.add(w)
                stack.append(w)
    return True


def d_sep_tester(parents):
    """A pc_search tester that knows the truth: p = 1 when d-separated, else 0."""
    return lambda tests: [1.0 if d_separated(parents, x, y, given) else 0.0 for x, y, given in tests]


# ------------------------------------------------------------------------------------ brute-force CPDAG
def _acyclic(nodes, edges):
    indeg = {v: 0 for v in nodes}
    out = {v: [] for v in nodes}
    for a, b in edges:
        indeg[b] += 1
        out[a].append(b)
    ready = [v for v in nodes if indeg[v] == 0]
    done = 0
    while ready:
        v = ready.pop()
        done += 1
        for w in out[v]:
            indeg[w] -= 1
            if indeg[w] == 0:
                ready.append(w)
    return done == len(nodes)


def v_structures(edges):
    pa = {}
    for a, b in edges:
        pa.setdefault(b, set()).add(a)
    adj = {frozenset(e) for e in edges}
    return {(min(a, c), max(a, c), b) for b, ps in pa.items() for a, c in itertools.combinations(sorted(ps), 2)
            if frozenset((a, c)) not in adj}


def cpdag(nodes, edges):
    """(directed set, undirected set of frozensets, every DAG of the class as a set of edges)."""
    skel = sorted({tuple(sorted(e)) for e in edges})
    want = v_structures(edges)
    kept = []
    for bits in itertools.product((0, 1), repeat=len(skel)):
        dag = [(a, b) if bit == 0 else (b, a) for (a, b), bit in zip(skel, bits)]
        if _acyclic(nodes, dag) and v_structures(dag) == want:
            kept.append(set(dag))
    directed = set.intersection(*kept) if kept else set()
    undirected = {frozenset(e) for e in skel} - {frozenset(e) for e in directed}
    return directed, undirected, kept


# ------------------------------------------------------------------------------------ sequential PC-stable
def sequential_pc(columns, cards, p_value, alpha, max_cond=None):
    """(directed set, undirected set of frozensets, {(u, v): sepset}) in column names.  `p_value(x, y, given)`
    answers one test; a table over 2^22 entries is never asked and counts as dependent, as is a NaN."""
    n = len(columns)
    pos = {c: i for i, c in enumerate(columns)}
    adj = np.ones((n, n), dtype=bool)
    np.fill_diagonal(adj, False)
    sep = {}
    level = 0
    while max_cond is None or level <= max_cond:
        frozen = adj.copy()
        for u in range(n):
            for v in range(u + 1, n):
                if not frozen[u, v]:
                    continue
                nu = [w for w in range(n) if frozen[u, w] and w != v]
                nv = [w for w in range(n) if frozen[v, w] and w != u]
                for s in itertools.chain(itertools.combinations(nu, level), itertools.combinations(nv, level)):
                    if math.prod(cards[pos[columns[i]]] for i in (u, v, *s)) > MAX_TABLE:
                        continue
                    p = p_value(columns[u], columns[v], tuple(columns[i] for i in s))
                    if p >= alpha:
                        adj[u, v] = adj[v, u] = False
                        sep[(u, v)] = s
                        break
        # go on while some adjacent pair has level + 1 other neighbours on either side
        if not any(adj[u, v] and (adj[u].sum() - 1 >= level + 1 or adj[v].sum() - 1 >= level + 1)
                   for u in range(n) for v in range(n) if u < v):
            break
        level += 1

    # G[a, b] and G[b, a] both set: a - b; only G[a, b]: a -> b
    G = adj.astype(np.int8)

    def undirected(a, b):
        return G[a, b] == 1 and G[b, a] == 1

    def arrow(a, b):
        return G[a, b] == 1 and G[b, a] == 0

    def adjacent(a, b):
        return G[a, b] == 1 or G[b, a] == 1

    def path(a, b):  # directed path a ~> b
        seen, stack = {a}, [a]
        while stack:
            v = stack.pop()
            if v == b:
                return True
            for w in range(n):
                if arrow(v, w) and w not in seen:
                    seen.add(w)
                    stack.append(w)
        return False

    def orient(a, b):
        if path(b, a):
            return False
        G[b, a] = 0
        return True

    for u in range(n):
        for v in range(u + 1, n):
            if adjacent(u, v):
                continue
            for z in range(n):
                if adjacent(u, z) and adjacent(v, z) and z not in sep[(u, v)]:
                    if undirected(u, z):
                        orient(u, z)
                    if undirected(v, z):
                        orient(v, z)

    def rule(k, i, j):
        others = [w for w in range(n) if w not in (i, j)]
        if k == 1:
            return any(arrow(w, i) and not adjacent(w, j) for w in others)
        if k == 2:
            return any(arrow(i, w) and arrow(w, j) for w in others)
        return any(undirected(i, w1) and undirected(i, w2) and arrow(w1, j) and arrow(w2, j) and not adjacent(w1, w2)
                   for w1, w2 in itertools.combinations(others, 2))

    changed = True
    while changed:
        changed = False
        for a in range(n):
            for b in range(a + 1, n):
                if not undirected(a, b):
                    continue
                for k in (1, 2, 3):
                    for i, j in ((a, b), (b, a)):
                        if rule(k, i, j) and orient(i, j):
                            changed = True
                            break
                    if changed:
                        break
                if changed:
                    break
            if changed:
                break

    directed = {(columns[a], columns[b]) for a in range(n) for b in range(n) if arrow(a, b)}
    und = {frozenset((columns[a], columns[b])) for a in range(n) for b in range(a + 1, n) if undirected(a, b)}
    seps = {(columns[u], columns[v]): tuple(columns[i] for i in s) for (u, v), s in sep.items()}
    return directed, und, seps


def extends(dag_edges, directed, undirected, nodes):
    """True when `dag_edges` is an acyclic orientation of the PDAG keeping its directed edges."""
    dag = set(dag_edges)
    if not directed <= dag or not _acyclic(nodes, dag):
        return False
    return {frozenset(e) for e in dag} == {frozenset(e) for e in directed} | set(undirected)
