"""Host-side mirror of `sorobn.BayesNet` for the exact-inference path.

Same surface as the reference (/root/reference/sorobn/bayes_net.py:259-1075) for
everything on the hot path: the constructor's structure grammar, the `P` dict of
pandas Series, `prepare()`, `query(..., algorithm="exact")` and `impute()`, plus the
cheap structural helpers.  What differs is where the arithmetic runs: `prepare()`
additionally compiles the CPTs into dense fp32 tables, and `query()` hands a flat
variable-elimination program to the CUDA engine (`sorobn_b200.engine`, a ctypes
shim over `libsorobn_b200.so`).  There is no CPU fallback: without the CUDA library
or a GPU `query()` raises.

`query_many()` is the batched form of `query()` (one posterior per evidence row of a
DataFrame); it is what the multi-GPU sharding and the benchmark drive.

`predict_proba` / `predict_log_proba` / `full_joint_dist` (bayes_net.py:398-465, :934-973) run
on the same kernels: the probability of a row is the normaliser of an elimination with the
row as evidence.

The approximate algorithms run on the device too (csrc/sbn_gibbs.cuh): `algorithm="gibbs"`
(bayes_net.py:665-737) one chain per evidence row, `"likelihood"` (:621-663) and `"rejection"`
(:577-619) n_iterations forward samples per row.  `fit` / `partial_fit` / `sample`
(:467-575) stay on the host (pandas / numpy), as in the reference.

`expected_counts` / `fit_em` learn from incomplete data (missing cells, latent nodes) by
expectation-maximisation; the E-step runs on the device as one counts program per missingness
pattern (planner.build_counts_plan, csrc/sbn_count.cuh).  `sample_many` draws exact posterior
samples of the missing cells and latent nodes, one sample program per pattern
(planner.build_sample_plan, csrc/sbn_sample.cuh).  `mpe_many` / `mpe` find their most probable
explanation, one log-domain max-sum program per pattern (planner.build_mpe_plan, csrc/sbn_mpe.cuh).
`map_many` / `map` find the marginal MAP state of chosen variables (by default the missing cells), the
other unobserved variables summed out: one log-sum-exp, then max-sum program per pattern
(planner.build_map_plan).
"""
from __future__ import annotations

import graphlib
import random
import threading
import typing
from collections import OrderedDict, defaultdict

import numpy as np
import pandas as pd

from . import planner as _planner

__all__ = ["BayesNet"]


def _as_list(obj):
    return obj if isinstance(obj, list) else [obj]


class _PatternRunner:
    """The device programs of one missingness pattern (a counts, sample, MPE or MAP plan): the float32 program,
    and the float64 one for the rows it flags (created when first needed; never for an MPE or MAP plan, whose
    logs do not underflow).  `set_cpts` gives both new tables in place (counts programs)."""

    def __init__(self, plan, device):
        from . import engine  # raises if libsorobn_b200.so cannot be loaded

        self.plan, self.device = plan, device
        self.f32 = engine.Program(plan, device=device)
        self._f64 = None
        self._blob64 = None

    def set_cpts(self, cpts):
        blob32, self._blob64 = _planner.refresh_tables(self.plan, cpts)
        self.f32.set_tables(blob32)
        if self._f64 is not None:
            self._f64.set_tables(self._blob64)

    def f64(self):
        if self._f64 is None:
            from . import engine

            self._f64 = engine.Program(self.plan, device=self.device, f64=True)
            if self._blob64 is not None:
                self._f64.set_tables(self._blob64)
        return self._f64

    def close(self):
        self.f32.close()
        if self._f64 is not None:
            self._f64.close()


class BayesNet:
    """Bayesian network with CUDA exact inference.

    Parameters mirror bayes_net.py:286: `structure` items are either bare nodes or
    (parent(s), child(ren)) tuples whose members may be lists.
    """

    def __init__(self, *structure, prior_count: int = None, seed: int = None, device: int | None = None):
        self.prior_count = prior_count
        self.seed = seed
        self._rng = random.Random(seed)  # seeds the device samplers (bayes_net.py:289)
        self.device = device

        parents = defaultdict(set)
        children = defaultdict(set)
        lone = set()
        for item in structure:
            if isinstance(item, tuple):
                srcs, dsts = item
                for s in _as_list(srcs):
                    for d in _as_list(dsts):
                        parents[d].add(s)
                        children[s].add(d)
            else:
                lone.add(item)

        # bayes_net.py:312-315: plain dicts of sorted lists
        self.parents = {n: sorted(ps) for n, ps in parents.items()}
        self.children = {n: sorted(cs) for n, cs in children.items()}

        # bayes_net.py:317-322: topological order, lexicographic within a level.
        # graphlib raises CycleError for a cyclic structure, as the reference does.
        sorter = graphlib.TopologicalSorter()
        for n in sorted({*self.parents, *self.children, *lone}):
            sorter.add(n, *self.parents.get(n, []))
        self.nodes = list(sorter.static_order())

        self.P = {}
        self._P_sizes = {}
        self._compiled = None
        # compiled device programs, one per (query vars, evidence vars, mode); least recently
        # used ones are dropped (their streams, graph and scratch are freed with them)
        self._engine_cache = OrderedDict()
        self._cache_lock = threading.RLock()  # query_many(devices=...) looks programs up from worker threads
        self.max_cached_programs = 128

    def __getstate__(self):
        """Copies and pickles carry the network, not the device objects (programs hold CUDA
        handles that must have exactly one owner); they are rebuilt on first use."""
        state = self.__dict__.copy()
        state["_engine_cache"] = OrderedDict()
        state.pop("_cache_lock", None)
        return state

    def __setstate__(self, state):
        self.__dict__.update(state)
        self._cache_lock = threading.RLock()

    # ------------------------------------------------------------------ structure
    def ancestors(self, node):
        """bayes_net.py:373-378."""
        found = set()
        frontier = list(self.parents.get(node, ()))
        while frontier:
            p = frontier.pop()
            if p not in found:
                found.add(p)
                frontier.extend(self.parents.get(p, ()))
        return found

    @property
    def roots(self):
        return [n for n in self.nodes if n not in self.parents]

    @property
    def leaves(self):
        return [n for n in self.nodes if n not in self.children]

    @property
    def is_tree(self):
        return all(len(ps) <= 1 for ps in self.parents.values())

    def markov_boundary(self, node):
        """Parents, children and the children's other parents (bayes_net.py:1002-1039)."""
        kids = self.children.get(node, [])
        blanket = set(self.parents.get(node, [])) | set(kids)
        for k in kids:
            blanket |= set(self.parents[k])
        blanket.discard(node)
        return sorted(blanket)

    def impute_many(self, samples: pd.DataFrame, **query_params) -> pd.DataFrame:
        """Batched `impute` (bayes_net.py:877-908): every missing cell (None / NaN) of `samples`
        is replaced by the most probable joint value of that row's missing variables given its
        observed ones.  Rows are grouped by which columns they lack; each group is one
        `query_many` call, i.e. one device program run over all its rows."""
        out = samples.copy()
        missing = samples.isna()
        patterns = missing.apply(lambda r: tuple(c for c in samples.columns if r[c]), axis=1)
        for pattern, rows in samples.groupby(patterns, sort=False).groups.items():
            if not pattern:
                continue
            observed = [c for c in samples.columns if c not in pattern]
            if not observed:
                raise ValueError("a row with every variable missing cannot be imputed")
            post = self.query_many(*pattern, events=samples.loc[rows, observed], **query_params)
            values = post.to_numpy()
            impossible = np.isnan(values).all(axis=1)
            if impossible.any():
                # `impute` raises here too (idxmax of the reference's empty posterior, bayes_net.py:902)
                raise ValueError(f"{int(impossible.sum())} row(s) have evidence of probability zero "
                                 f"(first: {post.index[impossible][0]!r}); they cannot be imputed")
            best = values.argmax(axis=1)
            labels = post.columns  # joint states, variables sorted by name
            names = list(labels.names)
            for k, name in enumerate(names):
                values = labels.get_level_values(k) if len(names) > 1 else labels
                out.loc[rows, name] = np.asarray(values, dtype=object)[best]
        return out.infer_objects()

    def graphviz(self):
        """The structure as a `graphviz.Digraph` (bayes_net.py:910-929); the module is imported
        here, so it is only needed when this is called."""
        import graphviz

        g = graphviz.Digraph()
        for node in self.nodes:
            g.node(str(node))
        for parent, kids in self.children.items():
            for kid in kids:
                g.edge(str(parent), str(kid))
        return g

    def _repr_svg_(self):
        return self.graphviz()

    def iter_dfs(self):
        """Depth-first walk from each root (bayes_net.py:1041-1075)."""
        seen = set()

        def walk(n):
            yield n
            seen.add(n)
            for c in self.children.get(n, []):
                if c not in seen:
                    yield from walk(c)

        for r in self.roots:
            yield from walk(r)

    # -------------------------------------------------------------------- prepare
    def prepare(self) -> "BayesNet":
        """House-keeping (bayes_net.py:327-371) + compile the tables for the device.

        The pandas side ends in the same state as the reference's: each `P[node]` is
        a Series named "P(node | parents)" whose index levels are
        [*parents, node], sorted.  Then every CPT is densified into an fp32 table
        (domain order == the sorted level values) ready to be shipped.
        """
        for node in list(self.P):
            table = self.P[node]
            node_parents = self.parents.get(node, [])

            if isinstance(table, pd.DataFrame):
                # bayes_net.py:339-358
                if "p" not in table.columns:
                    raise ValueError(
                        f"DataFrame for '{node}' must have a 'p' column containing probabilities"
                    )
                given = [c for c in table.columns if c != "p"]
                wanted = set(node_parents) | {node}
                if set(given) != wanted:
                    raise ValueError(
                        f"DataFrame for '{node}' has columns {given}, but expected {sorted(wanted)} (plus 'p')"
                    )
                table = table.set_index([*node_parents, node])["p"]
                self.P[node] = table

            if node not in self.parents:
                table.index.name = node
            elif set(table.index.names) == {*node_parents, node}:
                table = table.reorder_levels([*node_parents, node])
            else:
                table.index.names = [*node_parents, node]
            # reorder_levels returns a new object: sort it and store it back so that
            # P[node] always carries [*parents, node] levels, sorted
            table = table.sort_index()
            table.name = (
                f"P({node} | {', '.join(map(str, node_parents))})" if node in self.parents else f"P({node})"
            )
            self.P[node] = table

        self._compile()
        return self

    def _compile(self):
        missing = [n for n in self.nodes if n not in self.P]
        if missing:
            # The reference tolerates a partially specified network until a query
            # touches the hole; keep that: compile lazily once everything is there.
            self._compiled = None
            self._engine_cache = OrderedDict()
            return
        seen = {n: set() for n in self.nodes}
        for node, series in self.P.items():
            idx = series.index
            if isinstance(idx, pd.MultiIndex):
                for lvl, name in enumerate(idx.names):
                    seen[name].update(idx.get_level_values(lvl).unique().tolist())
            else:
                seen[node].update(idx.unique().tolist())
        domains = {n: sorted(v) for n, v in seen.items()}
        vid = {n: i for i, n in enumerate(self.nodes)}
        cpts = []
        for node in self.nodes:
            scope = [*self.parents.get(node, []), node]
            series = self.P[node]
            shape = [len(domains[v]) for v in scope]
            dense = np.zeros(shape, dtype=np.float64)
            idx = series.index
            if isinstance(idx, pd.MultiIndex):
                codes = [pd.Index(domains[v]).get_indexer(idx.get_level_values(l)) for l, v in enumerate(scope)]
            else:
                codes = [pd.Index(domains[node]).get_indexer(idx)]
            dense[tuple(codes)] = series.to_numpy(dtype=np.float64)
            cpts.append(dense)
        self._compiled = _planner.CompiledNet(
            names=list(self.nodes),
            domains=[domains[n] for n in self.nodes],
            parents=[[vid[p] for p in self.parents.get(n, [])] for n in self.nodes],
            cpt=cpts,
        )
        self._engine_cache = OrderedDict()

    # ------------------------------------------------------------- learning / sampling
    def partial_fit(self, X: pd.DataFrame) -> "BayesNet":
        """Update every CPT from a batch of rows (host side, pandas; bayes_net.py:467-510).

        Counts are kept per node (`_P_sizes` holds the number of rows behind every parent
        configuration), so feeding the data in chunks gives the same tables as one `fit`.
        With `prior_count`, every combination of the values seen in the first batch gets one
        pseudo-observation, as in the reference."""
        for child, parents in self.parents.items():
            scope = [*parents, child]
            seen = X.groupby(scope).size()
            if child in self.P:
                counts = (self.P[child] * self._P_sizes[child]).add(seen, fill_value=0)
            else:
                counts = seen
                if self.prior_count:
                    grid = pd.MultiIndex.from_product([X[v].unique() for v in scope], names=scope)
                    counts = counts.add(pd.Series(1, index=grid), fill_value=0)
            totals = counts.groupby(parents).sum()
            self._P_sizes[child] = totals
            self.P[child] = counts / totals
        for root in self.roots:
            if root in self.P:
                counts = (self.P[root] * self._P_sizes[root]).add(X[root].value_counts(), fill_value=0)
                self._P_sizes[root] += len(X)
                self.P[root] = counts / self._P_sizes[root]
            else:
                self._P_sizes[root] = len(X)
                self.P[root] = X[root].value_counts(normalize=True)
        self.prepare()
        return self

    def fit(self, X: pd.DataFrame) -> "BayesNet":
        """Estimate every CPT from `X` (bayes_net.py:512-516)."""
        self.P = {}
        self._P_sizes = {}
        return self.partial_fit(X)

    # ------------------------------------------------------- expected counts / EM
    def expected_counts(self, X: pd.DataFrame) -> dict:
        """The E-step of expectation-maximisation: for every node v, the sum over the rows of `X` of
        P(v, parents(v) | the row's observed cells), computed on the GPU.

        A missing cell is None or NaN; a node without a column in `X` is latent (unobserved in every
        row).  Returns {node: float64 Series} indexed like the densified CPT -- levels [*parents, v],
        every combination of the compiled domains, zeros kept.  Raises ValueError for a value outside
        its variable's domain and for rows whose observed cells have probability zero.

        Rows are grouped by missingness pattern (the set of observed columns); each pattern is one
        counts program (planner.build_counts_plan), so the cost grows with the number of distinct
        patterns as well as with the rows."""
        groups = self._count_patterns(X)
        net = self._compiled
        offsets, n_counts = _planner.count_layout(net)
        # each pattern's programs are fetched right before they run: with more patterns than the cache holds,
        # fetching one may close the least recently used ones, which have run by then
        counts, _ = self._e_step(X, groups, lambda k, ev: self._counts_runner(ev), n_counts)
        out = {}
        for v, name in enumerate(net.names):
            size = int(np.prod(net.cpt[v].shape))
            out[name] = pd.Series(counts[offsets[v]:offsets[v] + size], index=self._family_index(v), name=name)
        return out

    def fit_em(self, X: pd.DataFrame, max_iter: int = 100, tol: float = 1e-6) -> "BayesNet":
        """Fit the CPTs to `X` by expectation-maximisation, when cells are missing (None / NaN) or nodes
        are latent (no column in `X`).

        Start: the current CPTs if every node has one; otherwise, if every node is a column of `X`, the
        available-case `fit(X)`; otherwise ValueError (a latent variable's domain, and a start that
        breaks its symmetry, must come from the user).  Each iteration runs `expected_counts` (the
        programs are planned once per call; only their tables change) and normalises the counts per
        parent configuration, after one pseudo-observation per entry with `prior_count`.  Entries of
        zero expected count are left out of the Series, as `fit` leaves out unseen combinations.
        Iteration stops when the observed-data log-likelihood sum_b log P(observed cells of b) rises by
        less than `tol` per row, or after `max_iter` iterations.  The log-likelihood of every iteration
        is kept in `em_log_likelihood_`; `_P_sizes` holds the final expected counts, so a later
        `partial_fit` continues from them."""
        if int(max_iter) < 1:
            raise ValueError(f"max_iter must be at least 1, not {max_iter}")
        if all(n in self.P for n in self.nodes):
            if self._compiled is None:
                self.prepare()
        elif all(n in X.columns for n in self.nodes):
            self.fit(X)
        else:
            latent = [n for n in self.nodes if n not in X.columns]
            raise ValueError(f"fit_em needs initial CPTs in P when nodes have no column in X ({latent[:5]}): a latent "
                             "variable's states and a start that breaks its symmetry must come from the user")
        groups = self._count_patterns(X)
        net = self._compiled
        offsets, n_counts = _planner.count_layout(net)
        n_rows = len(X.index)
        runners = [_PatternRunner(_planner.build_counts_plan(net, ev), self.device) for ev, _, _ in groups]
        cpts = [np.array(c, dtype=np.float64) for c in net.cpt]
        lls = []
        try:
            for it in range(int(max_iter)):
                if it:
                    for r in runners:
                        r.set_cpts(cpts)
                counts, ll = self._e_step(X, groups, lambda k, ev: runners[k], n_counts)
                lls.append(ll)
                fam = [counts[offsets[v]:offsets[v] + c.size].reshape(c.shape) for v, c in enumerate(cpts)]
                if self.prior_count:
                    fam = [f + 1.0 for f in fam]
                totals = [f.sum(axis=-1) for f in fam]
                with np.errstate(invalid="ignore", divide="ignore"):
                    cpts = [np.where(t[..., None] > 0, f / t[..., None], 0.0) for f, t in zip(fam, totals)]
                if it and ll - lls[-2] < tol * n_rows:
                    break
        finally:
            for r in runners:
                r.close()
        self.em_log_likelihood_ = lls
        for v, node in enumerate(net.names):
            table = pd.Series(cpts[v].reshape(-1), index=self._family_index(v))
            self.P[node] = table[fam[v].reshape(-1) > 0]
            parents = self.parents.get(node)
            if parents:
                tot = totals[v].reshape(-1)
                index = self._family_index(v, parents_only=True)
                self._P_sizes[node] = pd.Series(tot, index=index)[tot > 0]
            else:
                self._P_sizes[node] = float(totals[v])
        self.prepare()
        return self

    def _family_index(self, v, parents_only=False):
        """Index of every combination of the compiled domains of [*parents, v] (or of the parents alone)."""
        net = self._compiled
        scope = list(net.scope(v))[:-1] if parents_only else list(net.scope(v))
        names = [net.names[u] for u in scope]
        if len(scope) == 1:
            return pd.Index(net.domains[scope[0]], name=names[0])
        return pd.MultiIndex.from_product([net.domains[u] for u in scope], names=names)

    def _count_patterns(self, X):
        """[(observed var ids, sorted; positions of the rows; uint8 codes [n_observed, n_rows])] per
        missingness pattern of `X`."""
        if self._compiled is None:
            self._compile()
            if self._compiled is None:
                raise ValueError("every node needs a CPT in P before computing expected counts; call prepare()")
        net = self._compiled
        cols = list(X.columns)
        for c in cols:
            if c not in net.index:
                raise KeyError(c)
        n = len(X.index)
        missing = X.isna().to_numpy().reshape(n, len(cols))
        codes = np.zeros((len(cols), n), dtype=np.uint8)
        for i, c in enumerate(cols):
            v = net.index[c]
            idx = pd.Index(net.domains[v]).get_indexer(pd.Index(X[c].to_numpy()))
            bad = (idx < 0) & ~missing[:, i]
            if bad.any():
                b = int(np.flatnonzero(bad)[0])
                raise ValueError(f"column {c!r}: {X[c].iloc[b]!r} (row {X.index[b]!r}) is not a state of the variable")
            codes[i] = np.where(idx < 0, 0, idx).astype(np.uint8)
        if n == 0:
            return []
        # group the rows by their observed-column bitmask, packed into 64-bit words (np.unique(axis=0) on the
        # boolean matrix sorts structured rows: seconds for a million rows)
        bits = np.packbits(~missing, axis=1)
        width = max(8, -(-bits.shape[1] // 8) * 8)  # bytes per row: whole 64-bit words, at least one
        bits = np.pad(bits, ((0, 0), (0, width - bits.shape[1])))
        words = np.ascontiguousarray(bits).view(np.uint64)
        order = np.lexsort(words.T[::-1]) if words.shape[1] > 1 else np.argsort(words[:, 0], kind="stable")
        ordered = words[order]
        starts = np.flatnonzero(np.r_[True, (ordered[1:] != ordered[:-1]).any(axis=1)])
        groups = []
        for s, e in zip(starts, np.r_[starts[1:], n]):
            rows = np.sort(order[s:e])
            observed = ~missing[rows[0]]
            col_of = {net.index[cols[i]]: i for i in range(len(cols)) if observed[i]}
            ev = tuple(sorted(col_of))
            groups.append((ev, rows, np.ascontiguousarray(codes[[col_of[v] for v in ev]][:, rows])))
        return groups

    def _counts_runner(self, ev):
        """The cached counts programs of one missingness pattern."""
        return self._pattern_runner("counts", ev)

    def _sample_runner(self, ev):
        """The cached sample programs of one missingness pattern."""
        return self._pattern_runner("sample", ev)

    def _mpe_runner(self, ev):
        """The cached MPE program of one missingness pattern."""
        return self._pattern_runner("mpe", ev)

    def _map_runner(self, ev, map_vars):
        """The cached marginal MAP program of one missingness pattern and MAP set (sorted var ids)."""
        return self._pattern_runner("map", ev, map_vars)

    def _pattern_runner(self, kind, ev, map_vars=None):
        """The cached programs of one missingness pattern, `kind` "counts", "sample", "mpe" or "map" (a "map"
        program is keyed by its MAP variables too; dropped by `prepare()`, as every program)."""
        with self._cache_lock:
            key = (kind, ev, self.device) if kind != "map" else (kind, ev, map_vars, self.device)
            hit = self._engine_cache.get(key)
            if hit is None:
                if kind == "map":
                    plan = _planner.build_map_plan(self._compiled, ev, map_vars)
                else:
                    plan = {"counts": _planner.build_counts_plan, "sample": _planner.build_sample_plan,
                            "mpe": _planner.build_mpe_plan}[kind](self._compiled, ev)
                hit = self._engine_cache[key] = _PatternRunner(plan, self.device)
                self._evict()
            else:
                self._engine_cache.move_to_end(key)
            return hit

    def _e_step(self, X, groups, runner_of, n_counts):
        """(expected counts [n_counts], observed-data log-likelihood) of every pattern's rows;
        `runner_of(k, observed var ids)` gives the programs of pattern k.  Rows the float32 program flags
        are settled by the float64 one; rows still without a probability raise."""
        counts = np.zeros(n_counts, dtype=np.float64)
        ll = 0.0
        for k, (ev, rows, codes) in enumerate(groups):
            runner = runner_of(k, ev)
            c, prob = runner.f32.counts(codes, len(rows))
            counts += c
            prob = prob.astype(np.float64)
            flagged = np.flatnonzero(np.isnan(prob))
            if len(flagged):
                c, prob[flagged] = runner.f64().counts(np.ascontiguousarray(codes[:, flagged]), len(flagged))
                counts += c
            impossible = np.isnan(prob)
            if impossible.any():
                raise ValueError(f"{int(impossible.sum())} row(s) have observed cells of probability zero "
                                 f"(first: {X.index[rows[impossible][0]]!r}); their expected counts are undefined")
            ll += float(np.log(prob).sum())
        return counts, ll

    def sample_many(self, events: pd.DataFrame, n: int = 1, seed: int | None = None) -> pd.DataFrame:
        """`n` exact draws of every unobserved variable from P(unobserved | the row's observed cells), for
        every row of `events`, computed on the GPU.

        A missing cell is None or NaN; a node without a column is latent.  Both are sampled; observed
        cells are copied through.  Returns `len(events) * n` rows indexed by (the events label, `draw`
        0 .. n - 1), the draws of a row adjacent and the rows in `events` order, with one column per node
        (sorted, dtypes inferred, as `sample`).  `seed=None` takes 64 bits from the network's stream.  The
        draws of a row depend only on the seed, its position in `events`, the draw index and its
        missingness pattern.  Raises ValueError for a value outside its variable's domain, for rows whose
        observed cells have probability zero and for `n < 1`.

        Rows are grouped by missingness pattern; each pattern is one sample program
        (planner.build_sample_plan): the upward pass of variable elimination, then one draw per bucket
        of the elimination, top-down (csrc/sbn_sample.cuh)."""
        if int(n) < 1:
            raise ValueError(f"n must be at least 1, not {n}")
        n = int(n)
        groups = self._count_patterns(events)
        net = self._compiled
        seed = self._rng.getrandbits(64) if seed is None else int(seed) & (2**64 - 1)
        n_rows = len(events.index)
        codes = np.zeros((len(net.names), n_rows, n), dtype=np.uint8)
        for ev, rows, ev_codes in groups:
            # fetched right before it runs: with more patterns than the cache holds, fetching one may close
            # the least recently used programs, which have run by then
            runner = self._sample_runner(ev)
            drawn, prob = self._draw(runner.f32, ev_codes, rows, n, seed)
            flagged = np.flatnonzero(np.isnan(prob))
            if len(flagged):
                drawn[:, :, flagged], prob[flagged] = self._draw(runner.f64(), np.ascontiguousarray(ev_codes[:, flagged]),
                                                                 rows[flagged], n, seed)
            impossible = np.isnan(prob)
            if impossible.any():
                raise ValueError(f"{int(impossible.sum())} row(s) have observed cells of probability zero "
                                 f"(first: {events.index[rows[impossible][0]]!r}); they have no posterior to sample from")
            for i, v in enumerate(ev):
                codes[v][rows] = ev_codes[i][:, None]
            for j, v in enumerate(runner.plan.sampled):
                codes[v][rows] = drawn[j].T
        index = pd.MultiIndex.from_arrays([np.repeat(events.index.to_numpy(), n), np.tile(np.arange(n), n_rows)],
                                          names=[events.index.name, "draw"])
        frame = pd.DataFrame({name: np.asarray(net.domains[v], dtype=object)[codes[v].reshape(-1)]
                              for v, name in enumerate(net.names)}, index=index)
        return frame.infer_objects().sort_index(axis="columns")

    def mpe_many(self, events: pd.DataFrame, return_log_proba: bool = False):
        """The most probable explanation of every row of `events`, computed on the GPU: the joint state of
        every unobserved variable that maximises P(unobserved, the row's observed cells).

        A missing cell is None or NaN; a node without a column is latent.  Both are decoded; observed
        cells are copied through.  Returns one row per row of `events` (same index) with one column per
        node (sorted, dtypes inferred, as `sample_many`).  With `return_log_proba=True` returns (frame,
        Series of log P(explanation, observed cells) in float64, same index); a row with every cell
        observed decodes nothing and gets log P(row).  Ties go to the first joint state of a bucket of
        the elimination (first variable fastest).  Raises ValueError for a value outside its variable's
        domain and for rows whose observed cells have probability zero.

        Unlike `impute_many`, which takes the mode of the dense posterior over the joint of the missing
        columns, the cost grows with the number of variables, not with their joint.  Rows are grouped by
        missingness pattern; each pattern is one MPE program (planner.build_mpe_plan): the upward pass of
        variable elimination in the log domain with max in place of sum, then one argmax per bucket,
        top-down (csrc/sbn_mpe.cuh)."""
        groups = self._count_patterns(events)
        net = self._compiled
        n_rows = len(events.index)
        codes = np.zeros((len(net.names), n_rows), dtype=np.uint8)
        log_p = np.zeros(n_rows, dtype=np.float64)
        for ev, rows, ev_codes in groups:
            # fetched right before it runs, as in `sample_many`
            runner = self._mpe_runner(ev)
            decoded, lp = runner.f32.mpe(ev_codes, len(rows))
            impossible = ~(lp > -np.inf)
            if impossible.any():
                raise ValueError(f"{int(impossible.sum())} row(s) have observed cells of probability zero "
                                 f"(first: {events.index[rows[impossible][0]]!r}); they have nothing to explain")
            for i, v in enumerate(ev):
                codes[v][rows] = ev_codes[i]
            for j, v in enumerate(runner.plan.sampled):
                codes[v][rows] = decoded[j]
            log_p[rows] = lp
        frame = pd.DataFrame({name: np.asarray(net.domains[v], dtype=object)[codes[v]]
                              for v, name in enumerate(net.names)}, index=events.index)
        frame = frame.infer_objects().sort_index(axis="columns")
        if return_log_proba:
            return frame, pd.Series(log_p, index=events.index)
        return frame

    def mpe(self, event: dict) -> pd.Series:
        """The most probable explanation of one event: `mpe_many(pd.DataFrame([event])).iloc[0]`, a Series
        indexed by node name."""
        return self.mpe_many(pd.DataFrame([event])).iloc[0]

    def map_many(self, events: pd.DataFrame, variables=None, return_log_proba: bool = False):
        """The marginal MAP state of every row of `events`, computed on the GPU: the joint state of the MAP
        variables that maximises P(MAP variables, the row's observed cells), every other unobserved variable
        summed out.

        A missing cell is None or NaN; a node without a column is unobserved.  With `variables=None` the MAP
        variables of a row are its missing cells and every node without a column is summed out: the answer
        `impute_many` gives, for any number of missing cells.  With `variables=[...]` the listed nodes are
        decoded, latent ones included; a listed node the row observes is copied through, and every other
        unobserved node is summed out (its missing cells stay missing).  Returns one row per row of `events`
        (same index) whose columns are those of `events` and `variables`, sorted, with dtypes inferred as in
        `mpe_many`.  With `return_log_proba=True` returns (frame, Series of log P(MAP state, observed cells)
        in float64, same index).  Ties go to the first joint state of a bucket of the elimination (first
        variable fastest).  Raises ValueError for a value outside its variable's domain and for rows whose
        observed cells have probability zero.

        Unlike `impute_many`, which builds the dense posterior over the joint of the missing columns, the
        cost grows with the number of variables, not with their joint.  Unlike `mpe_many`, the unobserved
        variables outside the MAP set are summed out, not maximised.  Rows are grouped by missingness pattern;
        each pattern is one marginal MAP program (planner.build_map_plan): the upward pass of variable
        elimination in the log domain, log-sum-exp over the summed variables, then max over the MAP ones,
        then one argmax per MAP bucket, top-down."""
        groups = self._count_patterns(events)
        net = self._compiled
        listed = None
        if variables is not None:
            unknown = [v for v in variables if v not in net.index]
            if unknown:
                raise ValueError(f"{unknown[:5]} are not nodes of the network")
            listed = sorted({net.index[v] for v in variables})
        columns = [net.index[c] for c in events.columns]
        out_vars = sorted(set(columns) | set(listed or ()), key=lambda v: net.names[v])
        n_rows = len(events.index)
        codes = np.zeros((len(net.names), n_rows), dtype=np.uint8)
        known = np.zeros((len(net.names), n_rows), dtype=bool)  # observed or decoded
        log_p = np.zeros(n_rows, dtype=np.float64)
        for ev, rows, ev_codes in groups:
            observed = set(ev)
            if listed is None:
                map_vars = tuple(v for v in sorted(columns) if v not in observed)
            else:
                map_vars = tuple(v for v in listed if v not in observed)
            for i, v in enumerate(ev):
                codes[v][rows] = ev_codes[i]
                known[v][rows] = True
            if not map_vars and not ev:
                continue  # nothing observed, nothing to decode: log P = log 1
            # fetched right before it runs, as in `sample_many`
            runner = self._map_runner(ev, map_vars)
            decoded, lp = runner.f32.map(ev_codes, len(rows))
            impossible = ~(lp > -np.inf)
            if impossible.any():
                raise ValueError(f"{int(impossible.sum())} row(s) have observed cells of probability zero "
                                 f"(first: {events.index[rows[impossible][0]]!r}); they have no MAP state")
            for j, v in enumerate(runner.plan.sampled):
                codes[v][rows] = decoded[j]
                known[v][rows] = True
            log_p[rows] = lp
        frame = pd.DataFrame({net.names[v]: np.where(known[v], np.asarray(net.domains[v], dtype=object)[codes[v]], None)
                              for v in out_vars}, index=events.index)
        frame = frame.infer_objects().sort_index(axis="columns")
        if return_log_proba:
            return frame, pd.Series(log_p, index=events.index)
        return frame

    def map(self, event: dict, variables=None) -> pd.Series:
        """The marginal MAP state of one event: `map_many(pd.DataFrame([event]), variables).iloc[0]`, a Series
        indexed by node name."""
        return self.map_many(pd.DataFrame([event]), variables).iloc[0]

    @staticmethod
    def _draw(program, ev_codes, rows, n, seed):
        """(drawn codes [n_sampled, n, len(rows)], P(observed) float64) of the rows at positions `rows`
        (sorted): one call per run of consecutive positions, whose first position is the call's row_base,
        so that a row's random stream is its position whatever the grouping."""
        starts = np.flatnonzero(np.r_[True, np.diff(rows) != 1])
        parts = [program.sample(np.ascontiguousarray(ev_codes[:, a:b]), b - a, n, seed, row_base=int(rows[a]))
                 for a, b in zip(starts, np.r_[starts[1:], len(rows)])]
        return np.concatenate([d for d, _ in parts], axis=2), np.concatenate([p for _, p in parts]).astype(np.float64)

    def sample(self, n=1, init: dict | None = None, method="forward"):
        """Forward (ancestral) samples (bayes_net.py:550-575): a Series for n == 1, otherwise a
        DataFrame with the columns sorted.  Variables named in `init` keep the given value.
        Vectorised over the n samples on the host; the stream comes from `seed`."""
        if method != "forward":
            raise ValueError("Unknown method, must be one of: forward")
        if self._compiled is None:
            self._compile()
            if self._compiled is None:
                raise ValueError("every node needs a CPT in P before sampling; call prepare()")
        net = self._compiled
        init = init or {}
        rng = np.random.default_rng(self._rng.getrandbits(63))
        n = int(n)
        codes = np.zeros((len(net.names), n), dtype=np.int64)
        for v, name in enumerate(net.names):
            if name in init:
                codes[v] = net.domains[v].index(init[name])
                continue
            table = net.cpt[v]
            probs = table[tuple(codes[p] for p in net.parents[v])] if net.parents[v] else np.broadcast_to(table, (n, table.shape[-1]))
            cdf = np.cumsum(probs, axis=-1)
            u = rng.random((n, 1)) * cdf[:, -1:]
            codes[v] = np.minimum((u > cdf).sum(axis=-1), table.shape[-1] - 1)
        frame = pd.DataFrame({name: np.asarray(net.domains[v], dtype=object)[codes[v]] for v, name in enumerate(net.names)})
        frame = frame.infer_objects().sort_index(axis="columns")
        return frame if n > 1 else frame.iloc[0]

    # ---------------------------------------------------------------------- query
    def _plan(self, query, evidence_vars, mode, robust=False, device=None, marginals=False, replica=0):
        """(plan, program) of P(query | evidence vars), cached.  marginals=True: `query` are the targets of
        a marginals program (planner.build_marginals_plan), cached under its own mode key.  replica=k > 0:
        a separate program on the same device, for the k-th other thread that runs this query there at the
        same time (a program's scratch, staging buffers and graph capture serve one caller at a time)."""
        with self._cache_lock:
            return self._plan_locked(query, evidence_vars, mode, robust, device, marginals, replica)

    def _plan_locked(self, query, evidence_vars, mode, robust, device, marginals=False, replica=0):
        if self._compiled is None:
            self._compile()
            if self._compiled is None:
                raise ValueError("every node needs a CPT in P before querying; call prepare()")
        net = self._compiled
        device = self.device if device is None else device
        key = (tuple(query), tuple(evidence_vars), ("marginals", mode) if marginals else mode, robust,
               (device, replica) if replica else device)
        hit = self._engine_cache.get(key)
        if hit is None:
            for name in (*query, *evidence_vars):
                if name not in net.index:
                    raise KeyError(name)
            twin = next((v for k, v in self._engine_cache.items() if isinstance(v, tuple) and k[:4] == key[:4]), None)
            if twin:
                plan = twin[0]  # the same plan serves every device
            elif marginals:
                plan = _planner.build_marginals_plan(net, [net.index[e] for e in evidence_vars],
                                                     targets=[net.index[q] for q in query], mode=mode)
            else:
                plan = _planner.build_plan(net, [net.index[q] for q in query], [net.index[e] for e in evidence_vars],
                                           mode=mode, allow_empty_query=True)
            from . import engine  # raises if libsorobn_b200.so cannot be loaded

            # single-event programs run in float64 (latency-bound anyway); batches in float32,
            # except the robust re-run of flagged rows (mode key "batched64")
            hit = (plan, engine.Program(plan, device=device, f64=(mode == _planner.MODE_FLAT or robust)))
            self._engine_cache[key] = hit
            self._evict()
        else:
            self._engine_cache.move_to_end(key)
        return hit

    def _evict(self):
        """Drop the least recently used device objects (programs and samplers) beyond the cap."""
        while len(self._engine_cache) > self.max_cached_programs:
            _, old = self._engine_cache.popitem(last=False)
            (old[1] if isinstance(old, tuple) else old).close()

    def _encode_events(self, evidence_vars, columns):
        """State values -> uint8 codes [n_ev, B].  Unknown values get code 255 and the
        row is reported as impossible evidence (the reference's boolean filter at
        bayes_net.py:772-774 leaves an empty factor, hence an empty answer)."""
        net = self._compiled
        n = len(columns[0]) if columns else 0
        codes = np.empty((len(evidence_vars), n), dtype=np.uint8)
        bad = np.zeros(n, dtype=bool)
        for i, (name, col) in enumerate(zip(evidence_vars, columns)):
            dom = pd.Index(net.domains[net.index[name]])
            c = dom.get_indexer(pd.Index(col))
            bad |= c < 0
            codes[i] = np.where(c < 0, 0, c).astype(np.uint8)
        return codes, bad

    def _answer_index(self, plan):
        net = self._compiled
        names = [net.names[v] for v in plan.query]
        doms = [net.domains[v] for v in plan.query]
        if len(names) == 1:
            return pd.Index(doms[0], name=names[0])
        return pd.MultiIndex.from_product(doms, names=names)

    def query(self, *query, event: dict, algorithm="exact", n_iterations=100) -> pd.Series:
        """Answer P(query | event) (bayes_net.py:796-875), exact inference on the GPU.

        The answer is a Series named "P(q1, q2)" indexed by the query variables
        (levels sorted by name, rows sorted by state); states with zero posterior
        are left out, as the reference's zero-filtering join does
        (bayes_net.py:253-256).
        """
        if not query:
            raise ValueError("At least one query variable has to be specified")
        for q in query:
            if q in event:
                raise ValueError("A query variable cannot be part of the event")
        if algorithm in ("gibbs", "likelihood", "rejection"):
            freq = self._sample_query(algorithm, query, tuple(event), [[event[v]] for v in event], 1, n_iterations)
            values = freq[0][:, 0].astype(np.float64)
            name = f"P({', '.join(map(str, query))})"
            if np.isnan(values).any():  # rejection sampling kept no sample: the reference's answer is empty
                return pd.Series([], index=freq[1][:0], name=name, dtype=np.float64)
            answer = pd.Series(values, index=freq[1], name=name)
            return answer[answer > 0]  # the reference only lists the states that were sampled
        if algorithm != "exact":
            raise ValueError("Unknown algorithm, must be one of: exact, gibbs, likelihood, rejection")

        ev_vars = tuple(event)
        plan, program = self._plan(query, ev_vars, _planner.MODE_FLAT)
        # One event is launch-latency bound on the device (~20 us): the host side must not cost ten
        # times that.  State codes come from per-variable dicts, the answer's index is cached on the plan.
        net = self._compiled
        codes = np.empty((len(ev_vars), 1), dtype=np.uint8)
        bad = False
        for i, v in enumerate(ev_vars):
            code = self._code_of(net.index[v]).get(event[v], -1)
            bad |= code < 0
            codes[i, 0] = max(code, 0)
        index = getattr(plan, "_answer_index_cache", None)
        if index is None:
            index = plan._answer_index_cache = self._answer_index(plan)
        name = f"P({', '.join(map(str, query))})"
        if bad:  # a value outside the variable's domain: the reference's filter leaves nothing
            return pd.Series([], index=index[:0], name=name, dtype=np.float64)
        post = program.run(codes, 1)[:, 0].astype(np.float64)
        if np.isnan(post).any():  # impossible evidence: P(event) == 0
            return pd.Series([], index=index[:0], name=name, dtype=np.float64)
        keep = post > 0
        if keep.all():
            return pd.Series(post, index=index, name=name)
        return pd.Series(post[keep], index=index[keep], name=name)

    def _code_of(self, v):
        """state value -> uint8 code of variable id `v` (position in its sorted domain)."""
        cache = self.__dict__.setdefault("_code_cache", {})
        table = cache.get(v)
        if table is None or cache.get("net") is not self._compiled:
            if cache.get("net") is not self._compiled:
                cache.clear()
                cache["net"] = self._compiled
            table = cache[v] = {value: k for k, value in enumerate(self._compiled.domains[v])}
        return table

    def _sample_query(self, algorithm, query, ev_vars, columns, n_rows, n_iterations):
        """The approximate algorithms on the device, per evidence row: one Gibbs chain
        (bayes_net.py:665-737), or n_iterations forward samples for likelihood weighting
        (:621-663) / rejection sampling (:577-619).  Returns (estimates [Q, n_rows], index)."""
        if self._compiled is None:
            self._compile()
            if self._compiled is None:
                raise ValueError("every node needs a CPT in P before querying; call prepare()")
        net = self._compiled
        for name in (*query, *ev_vars):
            if name not in net.index:
                raise KeyError(name)
        key = ("sampler", tuple(query), tuple(ev_vars))
        sampler = self._engine_cache.get(key)
        q_sorted = sorted(query)  # same key as the exact path (planner: sorted by name) and bayes_net.py:873
        if sampler is None:
            from . import engine

            nonevents = sorted(set(self.nodes) - set(ev_vars))  # bayes_net.py:697, the Gibbs cycle order
            sampler = engine.GibbsSampler(net, [net.index[q] for q in q_sorted], [net.index[e] for e in ev_vars],
                                          [net.index[v] for v in nonevents], device=self.device)
            self._engine_cache[key] = sampler
            self._evict()
        codes, bad = self._encode_events(ev_vars, columns)
        if bad.any():
            raise ValueError("an event value is not a state of its variable")
        freq = sampler.run(codes, n_rows, n_iterations, self._rng.getrandbits(63), algorithm=algorithm)
        doms = [net.domains[net.index[q]] for q in q_sorted]
        index = pd.Index(doms[0], name=q_sorted[0]) if len(q_sorted) == 1 else pd.MultiIndex.from_product(doms, names=q_sorted)
        return freq, index

    def query_many(self, *query, events: pd.DataFrame, algorithm="exact", n_iterations=100,
                   devices: typing.Sequence[int] | None = None) -> pd.DataFrame:
        """Batched `query`: one posterior per row of `events` (columns = evidence
        variables).  Returns a DataFrame with one row per evidence row and one column
        per joint state of the query variables (same order as `query`'s index);
        impossible rows are NaN.  Zero-probability states stay (as 0.0).

        devices: CUDA device ids to shard the rows over (exact algorithm).  Rows are independent,
        so each device answers a contiguous slice with its own program (one host thread per
        device; the C ABI call releases the GIL) and the slices land in one host array: there is
        no collective.  One process per GPU under torchrun is `sorobn_b200.sharding.query_many_sharded`."""
        if not query:
            raise ValueError("At least one query variable has to be specified")
        ev_vars = tuple(events.columns)
        for q in query:
            if q in ev_vars:
                raise ValueError("A query variable cannot be part of the event")
        if algorithm in ("gibbs", "likelihood", "rejection"):
            freq, index = self._sample_query(algorithm, query, ev_vars, [events[v].to_numpy() for v in ev_vars],
                                             len(events.index), n_iterations)
            return pd.DataFrame(freq.T.astype(np.float64), index=events.index, columns=index)
        if algorithm != "exact":
            raise ValueError("Unknown algorithm, must be one of: exact, gibbs, likelihood, rejection")
        plan, _ = self._plan(query, ev_vars, _planner.MODE_BATCHED, device=None if devices is None else devices[0])
        n = len(events.index)
        if n == 0:
            return pd.DataFrame(np.zeros((0, plan.Q)), index=events.index, columns=self._answer_index(plan))
        codes, bad = self._encode_events(ev_vars, [events[v].to_numpy() for v in ev_vars])
        if not ev_vars:
            bad = np.zeros(n, dtype=bool)
        if devices is None or len(devices) <= 1:
            post = self._posterior_codes(query, ev_vars, codes, bad, device=None if devices is None else devices[0])
        else:
            post = self._posterior_codes_multi(query, ev_vars, codes, bad, list(devices))
        out = pd.DataFrame(post.T, index=events.index, columns=self._answer_index(plan))
        if bad.any():
            out.loc[events.index[bad]] = np.nan
        return out

    def _posterior_codes(self, query, ev_vars, codes, bad, device=None, marginals=False, replica=0):
        """Posterior float64 [Q, n] for uint8 evidence codes [n_ev, n] on one device.  Rows the
        float32 program flags (NaN: impossible evidence, or an entry below the float32 range)
        are settled in float64 -- a few one by one with the single-event program, many as one
        batch with the batched float64 program; a row that is still NaN there is impossible.
        marginals=True: `query` are the targets of a marginals program (every segment normalised)."""
        n = codes.shape[1] if len(ev_vars) else len(bad)
        _, program = self._plan(query, ev_vars, _planner.MODE_BATCHED, device=device, marginals=marginals, replica=replica)
        post = self._run_evicting(program, codes, n).astype(np.float64)  # [Q, n]
        suspect = np.isnan(post).any(axis=0) & ~bad
        rows = np.nonzero(suspect)[0]
        if len(rows) > 8:
            _, robust = self._plan(query, ev_vars, _planner.MODE_BATCHED, robust=True, device=device, marginals=marginals,
                                   replica=replica)
            post[:, rows] = robust.run(np.ascontiguousarray(codes[:, rows]), len(rows))
        elif len(rows):
            _, flat = self._plan(query, ev_vars, _planner.MODE_FLAT, device=device, marginals=marginals, replica=replica)
            for b in rows:
                post[:, b] = flat.run(np.ascontiguousarray(codes[:, b:b + 1]), 1)[:, 0]
        return post

    def _targets(self, variables, ev_vars):
        """Target names of a marginals query, sorted: `variables`, or every variable that is not evidence."""
        if self._compiled is None:
            self._compile()
            if self._compiled is None:
                raise ValueError("every node needs a CPT in P before querying; call prepare()")
        if variables is None:
            variables = [n for n in self.nodes if n not in set(ev_vars)]
        variables = list(variables)
        for v in variables:
            if v in ev_vars:
                raise ValueError("A query variable cannot be part of the event")
            if v not in self._compiled.index:
                raise KeyError(v)
        if not variables:
            raise ValueError("At least one query variable has to be specified")
        return tuple(sorted(set(variables)))

    def marginals_many(self, events: pd.DataFrame, variables=None) -> pd.DataFrame:
        """The posterior marginal of every variable in `variables` (default: every variable that is not
        a column of `events`), for every row of `events`, from ONE device program: an upward and a
        downward pass over the bucket tree of the elimination, then one readout per variable
        (planner.build_marginals_plan).  Equals `query_many(v, events=events)` for each v.

        Returns one row per evidence row; the columns are a MultiIndex of (variable, state), variables
        sorted by name, states sorted.  Zero-probability states stay (as 0.0); impossible rows and rows
        with a value outside its variable's domain are NaN."""
        ev_vars = tuple(events.columns)
        targets = self._targets(variables, ev_vars)
        net = self._compiled
        columns = pd.MultiIndex.from_tuples([(t, s) for t in targets for s in net.domains[net.index[t]]],
                                            names=["variable", "state"])
        n = len(events.index)
        if n == 0:
            return pd.DataFrame(np.zeros((0, len(columns))), index=events.index, columns=columns)
        codes, bad = self._encode_events(ev_vars, [events[v].to_numpy() for v in ev_vars])
        if not ev_vars:
            bad = np.zeros(n, dtype=bool)
        post = self._posterior_codes(targets, ev_vars, codes, bad, marginals=True)
        out = pd.DataFrame(post.T, index=events.index, columns=columns)
        if bad.any():
            out.loc[events.index[bad]] = np.nan
        return out

    def marginals(self, event: dict, variables=None) -> dict:
        """`marginals_many` for one event, in float64 (as `query`): {variable: Series}, each Series equal to
        `query(variable, event=event)` -- named "P(variable)", zero states left out, empty for evidence of
        probability zero."""
        ev_vars = tuple(event)
        targets = self._targets(variables, ev_vars)
        net = self._compiled
        plan, program = self._plan(targets, ev_vars, _planner.MODE_FLAT, marginals=True)
        codes = np.empty((len(ev_vars), 1), dtype=np.uint8)
        bad = False
        for i, v in enumerate(ev_vars):
            code = self._code_of(net.index[v]).get(event[v], -1)
            bad |= code < 0
            codes[i, 0] = max(code, 0)
        post = None if bad else program.run(codes, 1)[:, 0].astype(np.float64)
        out, q = {}, 0
        for t in targets:
            index = pd.Index(net.domains[net.index[t]], name=t)
            seg = None if post is None else post[q:q + len(index)]
            q += len(index)
            if seg is None or np.isnan(seg).any():
                out[t] = pd.Series([], index=index[:0], name=f"P({t})", dtype=np.float64)
            else:
                keep = seg > 0
                out[t] = pd.Series(seg[keep], index=index[keep], name=f"P({t})")
        return out

    def _run_evicting(self, program, codes, n):
        """`program.run`, retried once after closing every OTHER cached device object when the device
        is out of memory: each program owns a scratch arena sized for its largest batch (3.9 GB for
        100k rows of the benchmark grid), and a BayesNet caches up to `max_cached_programs` of them --
        many evidence patterns at large batches would otherwise exhaust the GPU long before the LRU
        cap evicts anything (VERDICT r1)."""
        from . import engine

        try:
            return program.run(codes, n)
        except engine.EngineError as exc:
            if exc.code != engine.SBN_E_NOMEM:
                raise
        with self._cache_lock:
            for key in [k for k, v in self._engine_cache.items() if (v[1] if isinstance(v, tuple) else v) is not program]:
                old = self._engine_cache.pop(key)
                (old[1] if isinstance(old, tuple) else old).close()
        return program.run(codes, n)

    def _posterior_codes_multi(self, query, ev_vars, codes, bad, devices):
        """Row-shard `_posterior_codes` over several GPUs of this process: contiguous balanced
        slices (sharding.row_shard), one thread per listed device.  A device listed several times
        gets one set of programs per listing: no program is run by two threads at once."""
        import threading

        from .sharding import row_shard

        n = len(bad)
        world = len(devices)
        # programs are created up front, on this thread (the cache is not thread-safe)
        replicas = [devices[:r].count(d) for r, d in enumerate(devices)]
        for d, k in zip(devices, replicas):
            self._plan(query, ev_vars, _planner.MODE_BATCHED, device=d, replica=k)
        plan, _ = self._plan(query, ev_vars, _planner.MODE_BATCHED, device=devices[0])
        post = np.empty((plan.Q, n), dtype=np.float64)
        errors = []

        def work(r):
            sl = row_shard(n, r, world)
            if sl.stop == sl.start:
                return
            try:
                post[:, sl] = self._posterior_codes(query, ev_vars, np.ascontiguousarray(codes[:, sl]), bad[sl],
                                                    device=devices[r], replica=replicas[r])
            except Exception as exc:  # surfaced on the calling thread
                errors.append(exc)

        threads = [threading.Thread(target=work, args=(r,)) for r in range(world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            raise errors[0]
        return post

    # ------------------------------------------------------- joint / likelihood of rows
    def full_joint_dist(self, event: dict = None, keep_zeros=False) -> pd.Series:
        """The normalised product of every CPT (bayes_net.py:398-465), computed on the GPU
        as one exact query over all the variables with no evidence.  Like the reference the
        levels are sorted by name and combinations of probability zero are left out unless
        `keep_zeros`.  Practical for small networks only (the joint has prod(card) rows)."""
        names = sorted(self.nodes)
        plan, program = self._plan(tuple(names), (), _planner.MODE_FLAT)
        post = program.run(np.zeros((0, 1), dtype=np.uint8), 1)[:, 0].astype(np.float64)
        fjd = pd.Series(post, index=self._answer_index(plan), name=f"P({', '.join(map(str, names))})")
        return fjd if keep_zeros else fjd[post > 0]

    def predict_proba(self, X: typing.Union[dict, pd.DataFrame]):
        """Probability of each row of `X` (bayes_net.py:934-962).

        The reference builds the full joint, sums out the columns `X` lacks and looks the
        rows up.  Here P(row) is the normaliser of a variable elimination with the row as
        evidence and no query variable: same number, no joint, any network size.  Rows of
        probability zero give 0.0 (the reference's joint has no such row and raises
        KeyError).  With a single column the reference returns the whole marginal instead
        of per-row values; this returns per-row values in every case."""
        if isinstance(X, dict):
            return self.predict_proba(pd.DataFrame([X])).iloc[0]
        ev_vars = tuple(sorted(X.columns))
        n = len(X.index)
        name = f"P({', '.join(map(str, ev_vars))})"
        if len(ev_vars) == 1:
            index = pd.Index(X[ev_vars[0]], name=ev_vars[0])
        else:
            index = pd.MultiIndex.from_frame(X[list(ev_vars)])
        if n == 0:
            return pd.Series([], index=index, name=name, dtype=np.float64)
        plan, program = self._plan((), ev_vars, _planner.MODE_BATCHED)
        codes, bad = self._encode_events(ev_vars, [X[v].to_numpy() for v in ev_vars])
        prob = program.evidence(codes, n).astype(np.float64)
        rows = np.nonzero(np.isnan(prob) & ~bad)[0]
        if len(rows) > 8:  # below the float32 range (or exactly zero): settle in float64
            _, robust = self._plan((), ev_vars, _planner.MODE_BATCHED, robust=True)
            prob[rows] = robust.evidence(np.ascontiguousarray(codes[:, rows]), len(rows))
        elif len(rows):
            _, flat = self._plan((), ev_vars, _planner.MODE_FLAT)
            for b in rows:
                prob[b] = flat.evidence(np.ascontiguousarray(codes[:, b:b + 1]), 1)[0]
        prob[np.isnan(prob) | bad] = 0.0
        return pd.Series(prob, index=index, name=name)

    def predict_log_proba(self, X: typing.Union[dict, pd.DataFrame]):
        """Log-likelihood of each row (bayes_net.py:964-973)."""
        with np.errstate(divide="ignore"):
            return np.log(self.predict_proba(X))

    def impute(self, sample: dict, **query_params) -> pd.Series:
        """Fill the `None` entries of `sample` with their most probable joint value
        (bayes_net.py:877-908)."""
        known = {k: v for k, v in sample.items() if v is not None}
        unknown = [k for k, v in sample.items() if v is None]
        posterior = self.query(*unknown, event=known, **query_params)
        best = posterior.idxmax()
        if not isinstance(best, tuple):
            best = (best,)
        for k, v in zip(posterior.index.names, best):
            known[k] = v
        return pd.Series(known)
