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
(planner.build_map_plan).  `joint_marginals_many` returns, for every row, the joint posterior of every CPT
family or of chosen groups of variables, one joint program per pattern (planner.build_joint_plan).
`marginals_many(..., algorithm="bp")` approximates every marginal by loopy belief propagation on the device, one
row per thread (sorobn_b200/bp.py, csrc/sbn_bp.cu), for networks too wide to eliminate exactly, and
`mpe_many(..., algorithm="bp")` decodes every row by max-product belief propagation there, and
`expected_counts(..., algorithm="bp")` / `fit_em(..., algorithm="bp")` take their E-step from the family beliefs of
sum-product belief propagation (bp.compile_counts_graph), reduced on the device.
"""
from __future__ import annotations

import graphlib
import random
import threading
import typing
import warnings
from collections import OrderedDict, defaultdict

import numpy as np
import pandas as pd

from . import bp as _bp
from . import planner as _planner

__all__ = ["BayesNet"]


def _as_list(obj):
    return obj if isinstance(obj, list) else [obj]


class _Programs:
    """The float32 and float64 device programs of one plan on one device, each created when first needed; every
    exact-inference entry of the program cache is one.  `set_cpts` gives both new tables in place."""

    def __init__(self, plan, device):
        self.plan, self.device = plan, device
        self._programs = {}  # f64 -> engine.Program
        self._blobs = None  # (float32, float64) tables of the last set_cpts

    def program(self, f64):
        prog = self._programs.get(f64)
        if prog is None:
            from . import engine  # raises if libsorobn_b200.so cannot be loaded

            prog = self._programs[f64] = engine.Program(self.plan, device=self.device, f64=f64)
            if self._blobs is not None:
                prog.set_tables(self._blobs[f64])
        return prog

    def f32(self):
        return self.program(False)

    def f64(self):
        return self.program(True)

    def set_cpts(self, cpts):
        self._blobs = _planner.refresh_tables(self.plan, cpts)
        for f64, prog in self._programs.items():
            prog.set_tables(self._blobs[f64])

    def close(self):
        for prog in self._programs.values():
            prog.close()


def _posterior_series(post, index, name):
    """One event's posterior (float64, or None for a value outside its variable's domain) as the reference gives
    it: states of probability zero left out, empty for evidence of probability zero (NaN)."""
    if post is None or np.isnan(post).any():
        return pd.Series([], index=index[:0], name=name, dtype=np.float64)
    keep = post > 0
    if keep.all():
        return pd.Series(post, index=index, name=name)
    return pd.Series(post[keep], index=index[keep], name=name)


def _lik_rows(lik, rows):
    """The likelihood rows at positions `rows` of a `BayesNet._soft_matrix` matrix: a numpy fancy index, or a torch
    index on the tensor's device."""
    if isinstance(lik, np.ndarray):
        return lik[rows]
    import torch

    return lik[torch.as_tensor(np.asarray(rows), device=lik.device)]


def _check_possible(index, rows, impossible, consequence):
    """ValueError for the rows at positions `rows[impossible]` of a frame with `index`, whose observed cells have
    probability zero; `consequence` ends the message."""
    if impossible.any():
        raise ValueError(f"{int(impossible.sum())} row(s) have observed cells of probability zero "
                         f"(first: {index[rows[impossible][0]]!r}); {consequence}")


class _BpCounts:
    """The expected-counts graph of one missingness pattern on the device: the engine handle and `perm`, which maps
    the device's blob-order counts back to the dense CPTs and the dense CPTs to the blob."""

    def __init__(self, net, ev, device):
        from . import engine

        g = _bp.compile_counts_graph(net, ev)
        self.perm = g.perm
        self.runner = engine.BeliefPropagation(g.words, g.tables, device=device)

    def close(self):
        self.runner.close()


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
        # device objects: the `_Programs` of one plan on one device, keyed (*plan key, device), and Gibbs
        # samplers; least recently used ones are closed (their streams, graph and scratch are freed with them)
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
    def expected_counts(self, X: pd.DataFrame, likelihoods: dict | None = None, algorithm="exact", n_iterations=100,
                        damping=0.5, tol=1e-5) -> dict:
        """The E-step of expectation-maximisation: for every node v, the sum over the rows of `X` of
        P(v, parents(v) | the row's observed cells), computed on the GPU.

        A missing cell is None or NaN; a node without a column in `X` is latent (unobserved in every
        row).  Returns {node: float64 Series} indexed like the densified CPT -- levels [*parents, v],
        every combination of the compiled domains, zeros kept.  Raises ValueError for a value outside
        its variable's domain and for rows whose observed cells have probability zero.

        Rows are grouped by missingness pattern (the set of observed columns); each pattern is one
        counts program (planner.build_counts_plan), so the cost grows with the number of distinct
        patterns as well as with the rows.

        likelihoods: soft (virtual) evidence, {node: values} with one likelihood row per row of `X`, as in
        `query_many`: the counts are then those of P(v, parents(v) | observed cells, likelihoods).  A soft
        node may not be a column of `X`; a row whose cells and likelihoods have probability zero (an
        all-zero likelihood row makes one) raises ValueError.

        algorithm="bp": each row's family posteriors are the family beliefs of sum-product loopy belief propagation
        instead (sorobn_b200/bp.py, "Expected counts", defines them), for networks whose induced width the exact
        planner refuses.  Every CPT is a factor and every unobserved node a variable; messages are swept and damped
        as in `marginals_many(algorithm="bp")` (n_iterations, damping, tol as there), then the device forms every
        family belief of the row and sums them over the rows.  One compiled graph per missingness pattern; the same
        {node: Series} as the exact path, equal to it on polytrees.  A row whose messages or beliefs sum to zero, or
        whose observed cells alone hit a CPT entry of zero, raises the exact path's ValueError; on loopy networks BP
        may miss impossible evidence, whose rows then add counts silently.  Rows that did not converge add the
        beliefs of their last sweep and raise one RuntimeWarning with their count.  No soft evidence."""
        if algorithm not in ("exact", "bp"):
            raise ValueError("Unknown algorithm, must be one of: exact, bp")
        if algorithm == "bp":
            if likelihoods is not None:
                self._check_soft_call(algorithm, None)
            _bp.check_arguments(n_iterations, damping, tol)
            groups = self._count_patterns(X)
            net = self._compiled
            offsets, n_counts = _planner.count_layout(net)
            # each pattern's graph is fetched right before it runs, as in `sample_many`
            counts, _, stuck = self._bp_e_step(
                X, groups, lambda k, ev: self._cached(("bp_counts", ev), lambda: _BpCounts(net, ev, self.device)),
                n_counts, n_iterations, damping, tol)
            if stuck:
                self._warn_bp_stuck(f"{stuck} of {len(X.index)} rows", n_iterations, tol)
            return {name: pd.Series(counts[offsets[v]:offsets[v] + int(np.prod(net.cpt[v].shape))],
                                    index=self._family_index(v), name=name) for v, name in enumerate(net.names)}
        groups = self._count_patterns(X)
        soft = self._pattern_soft(likelihoods, X)
        net = self._compiled
        offsets, n_counts = _planner.count_layout(net)
        # each pattern's programs are fetched right before they run: with more patterns than the cache holds,
        # fetching one may close the least recently used ones, which have run by then
        counts, _ = self._e_step(X, groups, lambda k, ev: self._pattern_runner("counts", ev, soft=soft[0]), n_counts,
                                 soft[1])
        out = {}
        for v, name in enumerate(net.names):
            size = int(np.prod(net.cpt[v].shape))
            out[name] = pd.Series(counts[offsets[v]:offsets[v] + size], index=self._family_index(v), name=name)
        return out

    def joint_marginals_many(self, X: pd.DataFrame, groups=None, likelihoods: dict | None = None) -> dict:
        """For every row of `X`, the joint posterior of every CPT family, or of chosen groups of variables, given
        the row's observed cells (and likelihoods), computed on the GPU.

        Missing data follows `expected_counts`: the columns of `X` are observed cells, None or NaN is a missing
        cell, a node without a column is latent, and `likelihoods` is soft evidence.  `groups` lists the entries
        to return: a node name gives that node's family with axes [*parents, node] (the dense CPT order of
        `cpt_tensors`); a tuple of node names gives that group, in the given order.  Default: every node's family.
        A single name or tuple is one entry.

        Returns {entry: DataFrame} indexed like `X`, with one column per joint state of the group (a MultiIndex
        with one level per member, states sorted); each row sums to 1.  An observed member is a one-hot on the
        row's observed state, so the frame's shape does not depend on the row's missingness.  A row whose observed
        cells and likelihoods have probability zero is NaN in every frame.  Raises ValueError for a value outside
        its variable's domain, an unknown node and a duplicate member.

        Summed over the rows, the family frames are `expected_counts(X)`.  Rows are grouped by missingness pattern;
        each pattern is one joint program (planner.build_joint_plan): the counts program's upward and downward
        passes with a per-row readout of every group in place of the count steps (csrc/sbn_count.cuh
        `sbn_joint_step`).  Rows the float32 program cannot hold re-run in float64."""
        net = self._net("computing joint posteriors")
        if groups is None:
            groups = list(net.names)
        elif isinstance(groups, (str, tuple)):
            groups = [groups]
        entries, gids = [], []
        for g in groups:
            members = (g,) if isinstance(g, str) else tuple(g)
            unknown = [m for m in members if m not in net.index]
            if unknown:
                raise ValueError(f"group {g!r}: {unknown[:5]} are not nodes of the network")
            if isinstance(g, str):
                ids = tuple(net.scope(net.index[g]))
            else:
                ids = tuple(net.index[m] for m in members)
                if not ids or len(set(ids)) != len(ids):
                    raise ValueError(f"group {g!r} is empty or has a duplicate member")
            if g not in entries:
                entries.append(g)
                gids.append(ids)
        gids = tuple(gids)
        pattern_groups = self._count_patterns(X)
        soft, lik = self._pattern_soft(likelihoods, X)
        n = len(X.index)
        dense = [np.zeros((n, int(np.prod([int(net.card[u]) for u in ids])))) for ids in gids]
        for ev, rows, codes in pattern_groups:
            col = {v: i for i, v in enumerate(ev)}
            if all(u in col for ids in gids for u in ids):
                # nothing to read out: P(observed) alone decides the rows, from the pattern's counts program
                runner = self._pattern_runner("counts", ev, soft=soft)
                run = (lambda p, c, r: (None, p.counts(c, len(r))[1])) if lik is None else \
                    (lambda p, c, r: (None, p.counts(c, len(r), lik=_lik_rows(lik, r))[1]))
            else:
                # fetched right before it runs, as in `sample_many`
                runner = self._programs(("joint", ev, gids, soft), lambda: _planner.build_pattern_plan(
                    net, "joint", ev, soft=soft, groups=gids))
                run = lambda p, c, r: p.joint(c, len(r), lik=None if lik is None else _lik_rows(lik, r))  # noqa: E731
            out, prob, flagged, again = self._run_pattern(runner, run, codes, rows)
            bad = np.isnan(prob)
            for k, ids in enumerate(gids):
                cards = [int(net.card[u]) for u in ids]
                strides = [int(np.prod(cards[j + 1:], dtype=np.int64)) for j in range(len(ids))]
                base = np.zeros(len(rows), dtype=np.int64)
                for u, s in zip(ids, strides):
                    if u in col:
                        base += codes[col[u]].astype(np.int64) * s
                M = [(int(net.card[u]), s) for u, s in zip(ids, strides) if u not in col]
                if not M:
                    dense[k][rows, base] = 1.0
                else:
                    uoff = np.zeros(1, dtype=np.int64)
                    for c, s in M:  # each later member slower: the first one fastest
                        uoff = (uoff[None, :] + np.arange(c, dtype=np.int64)[:, None] * s).reshape(-1)
                    q0 = runner.plan.group_rows[k]
                    block = out[q0:q0 + len(uoff)].astype(np.float64)
                    if again is not None:
                        block[:, flagged] = again[q0:q0 + len(uoff)]
                    dense[k][rows[:, None], base[:, None] + uoff[None, :]] = block.T
                dense[k][rows[bad]] = np.nan
        return {g: pd.DataFrame(d, index=X.index, columns=pd.MultiIndex.from_product(
            [net.domains[u] for u in ids], names=[net.names[u] for u in ids])) for g, ids, d in zip(entries, gids, dense)}

    def fit_em(self, X: pd.DataFrame, max_iter: int = 100, tol: float = 1e-6,
               likelihoods: dict | None = None, algorithm="exact", n_iterations=100, damping=0.5,
               bp_tol=1e-5) -> "BayesNet":
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
        `partial_fit` continues from them.

        likelihoods: soft evidence (e.g. probabilistic labels of a latent node), as in `expected_counts`.  They
        stay fixed across the iterations, and `em_log_likelihood_` holds sum_b log P(observed cells of b,
        likelihoods of b), on the scale of the given likelihoods.

        algorithm="bp": Bethe-EM, for networks whose induced width the exact planner refuses.  Each E-step is
        `expected_counts(algorithm="bp")` with n_iterations, damping and `bp_tol` (its tol; `tol` stays EM's), one
        graph compiled per missingness pattern and only its tables replaced per iteration.  Every other rule is the
        exact one (start, prior_count, write-back, `_P_sizes`, the stopping rule), with the log-likelihood replaced by
        the sum of the rows' Bethe log-likelihoods (bp.py, "Expected counts"), which `em_log_likelihood_` then
        holds: exact on polytrees, an approximation of log P on loopy networks.  Bethe-EM is not monotone; a
        decrease also stops the loop.  On loopy networks BP can miss impossible evidence, whose rows then add counts
        silently.  Rows that did not converge in some E-step raise one RuntimeWarning per call.  No soft evidence."""
        if algorithm not in ("exact", "bp"):
            raise ValueError("Unknown algorithm, must be one of: exact, bp")
        if algorithm == "bp":
            if likelihoods is not None:
                self._check_soft_call(algorithm, None)
            _bp.check_arguments(n_iterations, damping, bp_tol)
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
        soft, lik = self._pattern_soft(likelihoods, X)
        net = self._compiled
        offsets, n_counts = _planner.count_layout(net)
        n_rows = len(X.index)
        if algorithm == "bp":
            runners = [_BpCounts(net, ev, self.device) for ev, _, _ in groups]
        else:
            runners = [_Programs(_planner.build_pattern_plan(net, "counts", ev, soft=soft), self.device)
                       for ev, _, _ in groups]
        cpts = [np.array(c, dtype=np.float64) for c in net.cpt]
        lls = []
        stuck = 0
        try:
            for it in range(int(max_iter)):
                if algorithm == "bp":
                    if it:
                        flat = np.concatenate([c.reshape(-1) for c in cpts])
                        for r in runners:
                            r.runner.set_tables(flat[r.perm])
                    counts, ll, s = self._bp_e_step(X, groups, lambda k, ev: runners[k], n_counts, n_iterations,
                                                    damping, bp_tol)
                    stuck = max(stuck, s)
                else:
                    if it:
                        for r in runners:
                            r.set_cpts(cpts)
                    counts, ll = self._e_step(X, groups, lambda k, ev: runners[k], n_counts, lik)
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
        if stuck:
            self._warn_bp_stuck(f"up to {stuck} of {n_rows} rows per E-step", n_iterations, bp_tol)
        self.em_log_likelihood_ = lls
        self._write_cpts(cpts, keep=[f.reshape(-1) > 0 for f in fam])
        for v, node in enumerate(net.names):
            parents = self.parents.get(node)
            if parents:
                tot = totals[v].reshape(-1)
                index = self._family_index(v, parents_only=True)
                self._P_sizes[node] = pd.Series(tot, index=index)[tot > 0]
            else:
                self._P_sizes[node] = float(totals[v])
        self.prepare()
        return self

    def _write_cpts(self, cpts, keep=None):
        """Store dense CPTs (var id -> ndarray [*parents, v] over the compiled domains) in `P`, every entry or those
        where keep[v] (flat) is set; the caller calls prepare()."""
        for v, node in enumerate(self._compiled.names):
            if cpts[v] is None:
                continue
            table = pd.Series(np.asarray(cpts[v], dtype=np.float64).reshape(-1), index=self._family_index(v))
            self.P[node] = table if keep is None else table[keep[v]]

    # ------------------------------------------------------------ gradients
    def encode_rows(self, X: pd.DataFrame):
        """The rows of `X` grouped by missingness pattern and encoded, once: `log_likelihood` takes the result in
        place of `X`, which saves the encoding in a training loop that passes the same rows every step."""
        from .autograd import EncodedRows

        return EncodedRows(self._count_patterns(X), X.index, X.columns)

    def log_likelihood(self, X, cpts: dict | None = None, likelihoods: dict | None = None):
        """log P(observed cells of b, likelihoods of b) of every row of `X` (a frame as in `expected_counts`, or
        `encode_rows(X)`), as a float64 torch tensor [n] on the network's device, computed on the GPU and
        differentiable (DESIGN.md "Gradients of the log-likelihood").

        cpts: {node: tensor [*parents, node]} over the compiled domains (`cpt_tensors()` gives the current ones
        in that layout), used in place of the node's CPT; gradients flow into these tensors, e.g. the softmax of a
        logits Parameter.  Every row must sum to 1 (within 1e-6), and a tensor that requires grad may have no zero
        entry (parameterise through softmax).  likelihoods: soft evidence as in `expected_counts`; gradients flow
        into its torch tensors.  Rows are grouped by missingness pattern, one gradient program per pattern; rows
        the float32 program cannot hold re-run in float64.  A row of probability zero raises ValueError.  One
        device only; second derivatives are not supported."""
        from . import autograd

        return autograd.log_likelihood(self, X, cpts, likelihoods)

    def cpt_tensors(self) -> dict:
        """{node: float64 torch tensor [*parents, node]}: the current dense CPTs over the compiled (sorted)
        domains, in the layout `log_likelihood(cpts=...)` and `assign_cpts` take."""
        import torch

        net = self._net("reading the CPTs")
        return {name: torch.tensor(net.cpt[v], dtype=torch.float64) for v, name in enumerate(net.names)}

    def assign_cpts(self, cpts: dict) -> "BayesNet":
        """Write dense CPTs {node: array or tensor [*parents, node]} (the layout of `cpt_tensors`) into `P`, every
        entry kept, and prepare() the network."""
        net = self._net("assigning CPTs")
        dense = [None] * len(net.names)
        for node, values in cpts.items():
            if node not in net.index:
                raise ValueError(f"a CPT for {node!r}, which is not a node of the network")
            v = net.index[node]
            arr = values.detach().cpu().numpy() if hasattr(values, "detach") else values
            arr = np.asarray(arr, dtype=np.float64)
            if arr.shape != net.cpt[v].shape:
                raise ValueError(f"the CPT of {node!r} has shape {arr.shape}, expected {net.cpt[v].shape}")
            dense[v] = arr
        self._write_cpts(dense)
        return self.prepare()

    def _family_index(self, v, parents_only=False):
        """Index of every combination of the compiled domains of [*parents, v] (or of the parents alone)."""
        scope = list(self._compiled.scope(v))
        return self._states_index(scope[:-1] if parents_only else scope)

    def _states_index(self, var_ids):
        """Index of every joint state of the compiled domains of `var_ids`, one level per variable."""
        net = self._compiled
        names = [net.names[v] for v in var_ids]
        if len(var_ids) == 1:
            return pd.Index(net.domains[var_ids[0]], name=names[0])
        return pd.MultiIndex.from_product([net.domains[v] for v in var_ids], names=names)

    def _count_patterns(self, X):
        """[(observed var ids, sorted; positions of the rows; uint8 codes [n_observed, n_rows])] per
        missingness pattern of `X`."""
        net = self._net("computing expected counts")
        cols = list(X.columns)
        for c in cols:
            if c not in net.index:
                raise KeyError(c)
        n = len(X.index)
        missing = X.isna().to_numpy().reshape(n, len(cols))
        codes = np.zeros((len(cols), n), dtype=np.uint8)
        for i, c in enumerate(cols):
            codes[i], unknown = self._encode_column(net.index[c], X[c].to_numpy())
            bad = unknown & ~missing[:, i]
            if bad.any():
                b = int(np.flatnonzero(bad)[0])
                raise ValueError(f"column {c!r}: {X[c].iloc[b]!r} (row {X.index[b]!r}) is not a state of the variable")
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

    def _pattern_runner(self, kind, ev, map_vars=None, soft=()):
        """The cached programs of one missingness pattern, `kind` "counts", "sample", "mpe" or "map" (a "map"
        plan is keyed by its MAP variables, sorted var ids, too), with the soft-evidence var ids `soft` (sorted
        by name; part of the key only when there are any)."""
        extra = (map_vars,) if kind == "map" else ()
        if not soft and kind != "grad":  # there is no build_grad_plan
            build = getattr(_planner, f"build_{kind}_plan")
            return self._programs((kind, ev, *extra), lambda: build(self._compiled, ev, *extra))
        return self._programs((kind, ev, *extra, soft),
                              lambda: _planner.build_pattern_plan(self._compiled, kind, ev, soft=soft, map_vars=map_vars))

    def _pattern_soft(self, likelihoods, events, single=False):
        """(soft-evidence var ids sorted by name, likelihoods [n, sum of cards]) of `likelihoods` for the rows of
        the frame `events`, whose columns may not be soft nodes (`_soft_matrix`); ((), None) without them."""
        if likelihoods is None:
            return (), None
        names, lik = self._soft_matrix(likelihoods, len(events.index), tuple(events.columns), single=single)
        return tuple(self._compiled.index[n] for n in names), lik

    @staticmethod
    def _run_pattern(runner, run, codes, rows):
        """run(program, codes, rows) -> (result, P(observed)) on a pattern's float32 program, then on its float64
        program for the rows the float32 one flags (P(observed) NaN).  Returns (float32 result, P(observed)
        float64, positions of the flagged rows, their float64 result or None); a row still NaN is impossible."""
        out, prob = run(runner.f32(), codes, rows)
        prob = prob.astype(np.float64)
        flagged = np.flatnonzero(np.isnan(prob))
        again = None
        if len(flagged):
            again, prob[flagged] = run(runner.f64(), np.ascontiguousarray(codes[:, flagged]), rows[flagged])
        return out, prob, flagged, again

    def _e_step(self, X, groups, runner_of, n_counts, lik=None):
        """(expected counts [n_counts], observed-data log-likelihood) of every pattern's rows;
        `runner_of(k, observed var ids)` gives the programs of pattern k, and `lik` the likelihoods of every row
        of `X` for programs with soft evidence (the log-likelihood is then sum log P(observed, lik)).  Rows the
        float32 program flags are settled by the float64 one; rows still without a probability raise."""
        counts = np.zeros(n_counts, dtype=np.float64)
        ll = 0.0

        def run(p, c, r):
            if lik is None:
                return p.counts(c, len(r))
            cnt, prob, log_ev = p.counts(c, len(r), lik=_lik_rows(lik, r), log_evidence=True)
            return (cnt, log_ev), prob

        for k, (ev, rows, codes) in enumerate(groups):
            c, prob, flagged, again = self._run_pattern(runner_of(k, ev), run, codes, rows)
            if lik is not None:
                c, log_ev = c
                if again is not None:
                    again, log_ev[flagged] = again
            counts += c
            if again is not None:
                counts += again
            _check_possible(X.index, rows, np.isnan(prob), "their expected counts are undefined")
            ll += float(np.log(prob).sum()) if lik is None else float(log_ev.sum())
        return counts, ll

    def _bp_e_step(self, X, groups, runner_of, n_counts, n_iterations, damping, tol):
        """(expected counts [n_counts] in count_layout order, sum of the rows' Bethe log-likelihoods, rows that did
        not converge) of belief propagation over every pattern; `runner_of(k, observed var ids)` gives pattern k's
        `_BpCounts`.  Dead rows raise the exact path's ValueError."""
        counts = np.zeros(n_counts, dtype=np.float64)
        ll, stuck = 0.0, 0
        for k, (ev, rows, codes) in enumerate(groups):
            r = runner_of(k, ev)
            c, log_z, iters = r.runner.counts(codes, len(rows), n_iterations, damping, tol)
            _check_possible(X.index, rows, np.isnan(log_z), "their expected counts are undefined")
            counts[r.perm] += c
            ll += float(log_z.sum())
            stuck += int(np.count_nonzero(iters > n_iterations))
        return counts, ll, stuck

    @staticmethod
    def _warn_bp_stuck(which, n_iterations, tol):
        warnings.warn(f"belief propagation: {which} did not converge to tol={tol:g} in {n_iterations} sweeps; they "
                      "add the beliefs of their last sweep", RuntimeWarning, stacklevel=3)

    def sample_many(self, events: pd.DataFrame, n: int = 1, seed: int | None = None,
                    likelihoods: dict | None = None) -> pd.DataFrame:
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
        of the elimination, top-down (csrc/sbn_sample.cuh).

        likelihoods: soft evidence, as in `expected_counts`: the draws come from P(unobserved | observed
        cells, likelihoods), and the soft nodes are drawn too."""
        if int(n) < 1:
            raise ValueError(f"n must be at least 1, not {n}")
        n = int(n)
        groups = self._count_patterns(events)
        soft, lik = self._pattern_soft(likelihoods, events)
        net = self._compiled
        seed = self._rng.getrandbits(64) if seed is None else int(seed) & (2**64 - 1)
        n_rows = len(events.index)
        codes = np.zeros((len(net.names), n_rows, n), dtype=np.uint8)
        for ev, rows, ev_codes in groups:
            # fetched right before it runs: with more patterns than the cache holds, fetching one may close
            # the least recently used programs, which have run by then
            runner = self._pattern_runner("sample", ev, soft=soft)
            drawn, prob, flagged, again = self._run_pattern(runner, lambda p, c, r: self._draw(p, c, r, n, seed, lik),
                                                            ev_codes, rows)
            if again is not None:
                drawn[:, :, flagged] = again
            _check_possible(events.index, rows, np.isnan(prob), "they have no posterior to sample from")
            for i, v in enumerate(ev):
                codes[v][rows] = ev_codes[i][:, None]
            for j, v in enumerate(runner.plan.sampled):
                codes[v][rows] = drawn[j].T
        index = pd.MultiIndex.from_arrays([np.repeat(events.index.to_numpy(), n), np.tile(np.arange(n), n_rows)],
                                          names=[events.index.name, "draw"])
        return self._codes_frame(codes.reshape(len(net.names), -1), index)

    def mpe_many(self, events: pd.DataFrame, return_log_proba: bool = False, likelihoods: dict | None = None,
                 algorithm="exact", n_iterations=100, damping=0.5, tol=1e-5):
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
        top-down (csrc/sbn_mpe.cuh).

        likelihoods: soft evidence, as in `expected_counts` (noisy observations: Viterbi-style decoding).  The
        soft nodes are decoded too, and the log probability is log P(explanation, observed cells, likelihoods)
        on the scale of the given likelihoods.

        algorithm="bp": max-product loopy belief propagation on the device instead of elimination, for networks
        whose induced width the exact planner refuses (sorobn_b200/bp.py, "Max-product", defines it).  Every CPT is
        a factor and every unobserved node a variable; max-product messages are swept synchronously, each
        factor-to-variable message damped as (1 - damping) * new + damping * old, until the largest change of any
        message of the row falls below `tol` or `n_iterations` sweeps have run.  Each variable then takes the first
        state of its largest belief, and the row's log P(explanation, observed cells) is summed over the CPTs in
        float64.  Exact on polytrees whose MPE is unique; on loopy networks an approximation whose log P is that
        of the assignment returned, never above the exact MPE's, and on grids often far below it (DESIGN.md,
        "Max-product belief propagation", gives measured gaps).  Rows are grouped by missingness pattern, one
        compiled graph per pattern; the frame and the log P Series are those of the exact path.  A row whose
        messages or beliefs sum to zero, or whose observed cells alone hit a CPT entry of zero, raises the exact
        path's ValueError: any assignment of positive probability keeps every message non-zero, so its observed
        cells are impossible.  A row whose decode has probability zero (the per-variable decode can combine tied
        states of different maximisers, and loopy messages are approximate) is returned with log P = -inf, and one
        RuntimeWarning gives their count; rows that did not converge keep the decode of their last sweep and raise one
        RuntimeWarning with their count.  ValueError for `likelihoods` (no soft evidence) and unless 0 <= damping < 1, n_iterations >= 1 and
        tol >= 0."""
        return self._mpe_frame(events, return_log_proba, likelihoods, algorithm=algorithm, n_iterations=n_iterations,
                               damping=damping, tol=tol)

    def mpe(self, event: dict, likelihoods: dict | None = None, algorithm="exact", n_iterations=100, damping=0.5,
            tol=1e-5) -> pd.Series:
        """The most probable explanation of one event: `mpe_many(pd.DataFrame([event])).iloc[0]`, a Series
        indexed by node name.  likelihoods: soft evidence of the event, {node: a vector over the node's sorted
        domain, or a {state: weight} dict}, as in `query`.  algorithm, n_iterations, damping, tol: as in
        `mpe_many`."""
        return self._mpe_frame(pd.DataFrame([event]), False, likelihoods, single=True, algorithm=algorithm,
                               n_iterations=n_iterations, damping=damping, tol=tol).iloc[0]

    def _mpe_frame(self, events, return_log_proba, likelihoods, single=False, algorithm="exact", n_iterations=100,
                   damping=0.5, tol=1e-5):
        if algorithm not in ("exact", "bp"):
            raise ValueError("Unknown algorithm, must be one of: exact, bp")
        if algorithm == "bp":
            if likelihoods is not None:
                self._check_soft_call(algorithm, None)
            _bp.check_arguments(n_iterations, damping, tol)
        groups = self._count_patterns(events)
        if algorithm == "bp":
            codes, log_p = self._bp_decode(events, groups, n_iterations, damping, tol)
        else:
            soft = self._pattern_soft(likelihoods, events, single)
            codes, _, log_p = self._decode(events, groups, "mpe", "they have nothing to explain", soft=soft)
        frame = self._codes_frame(codes, events.index)
        return (frame, pd.Series(log_p, index=events.index)) if return_log_proba else frame

    def _bp_decode(self, events, groups, n_iterations, damping, tol):
        """(codes [n_nodes, n], log P [n]) of max-product belief propagation (bp.compile_mpe_graph) over the pattern
        groups of `events`, one cached graph per pattern: the observed codes copied through, the decoded ones in
        var id order.  Dead rows raise; one RuntimeWarning each counts the rows whose decode has probability zero
        and the rows that did not converge."""
        from . import engine

        net = self._compiled
        n_rows = len(events.index)
        codes = np.zeros((len(net.names), n_rows), dtype=np.uint8)
        log_p = np.zeros(n_rows, dtype=np.float64)
        zero = stuck = 0
        for ev, rows, ev_codes in groups:
            for i, v in enumerate(ev):
                codes[v][rows] = ev_codes[i]

            def build(ev=ev):
                g = _bp.compile_mpe_graph(net, ev)
                return engine.BeliefPropagation(g.words, g.tables, device=self.device)

            # fetched right before it runs, as in `sample_many`
            runner = self._cached(("bp_mpe", ev), build)
            decoded, lp, iters = runner.mpe(ev_codes, len(rows), n_iterations, damping, tol)
            _check_possible(events.index, rows, np.isnan(lp), "they have nothing to explain")
            observed = set(ev)
            hidden = [v for v in range(len(net.names)) if v not in observed]
            for j, v in enumerate(hidden):
                codes[v][rows] = decoded[j]
            log_p[rows] = lp
            zero += int(np.count_nonzero(lp == -np.inf))
            stuck += int(np.count_nonzero(iters > n_iterations))
        if zero:
            warnings.warn(f"belief propagation: {zero} of {n_rows} rows decoded an explanation of probability zero "
                          "(log P = -inf)", RuntimeWarning, stacklevel=4)
        if stuck:
            warnings.warn(f"belief propagation: {stuck} of {n_rows} rows did not converge to tol={tol:g} in "
                          f"{n_iterations} sweeps; they keep the decode of their last sweep", RuntimeWarning,
                          stacklevel=4)
        return codes, log_p

    def map_many(self, events: pd.DataFrame, variables=None, return_log_proba: bool = False,
                 likelihoods: dict | None = None):
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
        then one argmax per MAP bucket, top-down.

        likelihoods: soft evidence, as in `expected_counts`.  With `variables=None` the soft nodes are summed
        out; list one to decode it.  The log probability is then log P(MAP state, observed cells,
        likelihoods) on the scale of the given likelihoods."""
        return self._map_frame(events, variables, return_log_proba, likelihoods)

    def _map_frame(self, events, variables, return_log_proba, likelihoods, single=False):
        groups = self._count_patterns(events)
        soft = self._pattern_soft(likelihoods, events, single)
        net = self._compiled
        listed = None
        if variables is not None:
            unknown = [v for v in variables if v not in net.index]
            if unknown:
                raise ValueError(f"{unknown[:5]} are not nodes of the network")
            listed = sorted({net.index[v] for v in variables})
        columns = [net.index[c] for c in events.columns]
        chosen = sorted(columns) if listed is None else listed
        codes, known, log_p = self._decode(events, groups, "map", "they have no MAP state",
                                           lambda ev: tuple(v for v in chosen if v not in ev), soft)
        out_vars = sorted(set(columns) | set(listed or ()), key=lambda v: net.names[v])
        frame = self._codes_frame(codes, events.index, out_vars, known)
        return (frame, pd.Series(log_p, index=events.index)) if return_log_proba else frame

    def map(self, event: dict, variables=None, likelihoods: dict | None = None) -> pd.Series:
        """The marginal MAP state of one event: `map_many(pd.DataFrame([event]), variables).iloc[0]`, a Series
        indexed by node name.  likelihoods: soft evidence of the event, as in `mpe`."""
        return self._map_frame(pd.DataFrame([event]), variables, False, likelihoods, single=True).iloc[0]

    def _decode(self, events, groups, kind, consequence, map_vars_of=None, soft=((), None)):
        """(codes [n_nodes, n], known [n_nodes, n] (observed or decoded), log P [n]) of the MPE (`kind` "mpe")
        or marginal MAP ("map") programs of the pattern groups of `events`: the observed codes copied through,
        the decoded ones in `plan.sampled` order.  MAP takes the MAP variables of a pattern from
        `map_vars_of(observed var ids)` and skips a pattern that observes and decodes nothing (log P = log 1)
        unless there is soft evidence.  `soft` is `_pattern_soft`'s (var ids, likelihoods of every row)."""
        soft, lik = soft
        net = self._compiled
        n_rows = len(events.index)
        codes = np.zeros((len(net.names), n_rows), dtype=np.uint8)
        known = np.zeros((len(net.names), n_rows), dtype=bool)
        log_p = np.zeros(n_rows, dtype=np.float64)
        for ev, rows, ev_codes in groups:
            map_vars = None if map_vars_of is None else map_vars_of(ev)
            for i, v in enumerate(ev):
                codes[v][rows] = ev_codes[i]
                known[v][rows] = True
            if map_vars == () and not ev and not soft:
                continue
            # fetched right before it runs, as in `sample_many`
            runner = self._pattern_runner(kind, ev, map_vars, soft)
            if lik is None:
                decoded, lp = getattr(runner.f32(), kind)(ev_codes, len(rows))
            else:
                decoded, lp = getattr(runner.f32(), kind)(ev_codes, len(rows), lik=_lik_rows(lik, rows))
            _check_possible(events.index, rows, ~(lp > -np.inf), consequence)
            for j, v in enumerate(runner.plan.sampled):
                codes[v][rows] = decoded[j]
                known[v][rows] = True
            log_p[rows] = lp
        return codes, known, log_p

    def _codes_frame(self, codes, index, variables=None, known=None):
        """The frame of state codes [n_nodes, n]: one column per var id in `variables` (default: every node) of
        its domain values, None where `known` is False, the columns sorted and their dtypes inferred."""
        net = self._compiled
        columns = {}
        for v in range(len(net.names)) if variables is None else variables:
            values = np.asarray(net.domains[v], dtype=object)[codes[v]]
            columns[net.names[v]] = values if known is None else np.where(known[v], values, None)
        return pd.DataFrame(columns, index=index).infer_objects().sort_index(axis="columns")

    @staticmethod
    def _draw(program, ev_codes, rows, n, seed, lik=None):
        """(drawn codes [n_sampled, n, len(rows)], P(observed) float64) of the rows at positions `rows`
        (sorted): one call per run of consecutive positions, whose first position is the call's row_base,
        so that a row's random stream is its position whatever the grouping.  `lik` (the likelihoods of every
        position, for a program with soft evidence) is sliced along with each run."""
        starts = np.flatnonzero(np.r_[True, np.diff(rows) != 1])
        parts = []
        for a, b in zip(starts, np.r_[starts[1:], len(rows)]):
            soft = {} if lik is None else {"lik": lik[int(rows[a]):int(rows[a]) + b - a]}
            parts.append(program.sample(np.ascontiguousarray(ev_codes[:, a:b]), b - a, n, seed, row_base=int(rows[a]),
                                        **soft))
        return np.concatenate([d for d, _ in parts], axis=2), np.concatenate([p for _, p in parts]).astype(np.float64)

    def sample(self, n=1, init: dict | None = None, method="forward"):
        """Forward (ancestral) samples (bayes_net.py:550-575): a Series for n == 1, otherwise a
        DataFrame with the columns sorted.  Variables named in `init` keep the given value.
        Vectorised over the n samples on the host; the stream comes from `seed`."""
        if method != "forward":
            raise ValueError("Unknown method, must be one of: forward")
        net = self._net("sampling")
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
        frame = self._codes_frame(codes, None)
        return frame if n > 1 else frame.iloc[0]

    # ---------------------------------------------------------------------- query
    def _net(self, purpose):
        """The compiled network, compiled now if `P` has been completed since; ValueError while a node has no CPT."""
        if self._compiled is None:
            self._compile()
            if self._compiled is None:
                raise ValueError(f"every node needs a CPT in P before {purpose}; call prepare()")
        return self._compiled

    def _cached(self, key, build):
        """The cache entry under `key`, built by `build()` on a miss.  A hit becomes the most recently used entry;
        a miss closes the least recently used entries beyond `max_cached_programs`."""
        with self._cache_lock:
            hit = self._engine_cache.get(key)
            if hit is None:
                hit = self._engine_cache[key] = build()
                self._evict()
            else:
                self._engine_cache.move_to_end(key)
            return hit

    def _programs(self, plan_key, build_plan, device=None, replica=0):
        """The cached `_Programs` of the plan `plan_key` names, on `device` (default: the network's).  replica=k > 0:
        separate programs on the same device, for the k-th other thread that runs this plan there at the same
        time (a program's scratch, staging buffers and graph capture serve one caller at a time).  The plan is
        shared by every device and replica: a miss takes it from another entry of the same plan before calling
        `build_plan()`."""
        device = self.device if device is None else device

        def build():
            twin = next((v for k, v in self._engine_cache.items() if k[:-1] == plan_key), None)
            return _Programs(twin.plan if twin is not None else build_plan(), device)

        return self._cached((*plan_key, (device, replica) if replica else device), build)

    def _query_programs(self, query, evidence_vars, mode, device=None, marginals=False, replica=0):
        """The cached `_Programs` of P(query | evidence vars), plan key (query, evidence vars, mode, marginals);
        marginals=True: `query` are the targets of a marginals program (planner.build_marginals_plan)."""
        net = self._net("querying")

        def build_plan():
            for name in (*query, *evidence_vars):
                if name not in net.index:
                    raise KeyError(name)
            ev = [net.index[e] for e in evidence_vars]
            if marginals:
                return _planner.build_marginals_plan(net, ev, targets=[net.index[q] for q in query], mode=mode)
            return _planner.build_plan(net, [net.index[q] for q in query], ev, mode=mode, allow_empty_query=True)

        return self._programs((tuple(query), tuple(evidence_vars), mode, marginals), build_plan, device, replica)

    def _plan(self, query, evidence_vars, mode, robust=False, device=None, marginals=False, replica=0):
        """(plan, program) of P(query | evidence vars), cached: the float64 program of a single-event
        (MODE_FLAT) plan, which is latency-bound anyway; of a batched plan the float32 program, or with `robust`
        the float64 one that settles the rows the float32 program flags.  The other arguments are
        `_query_programs`'."""
        with self._cache_lock:
            entry = self._query_programs(query, evidence_vars, mode, device, marginals, replica)
            return entry.plan, entry.program(mode == _planner.MODE_FLAT or robust)

    def _evict(self):
        """Drop the least recently used device objects (programs and samplers) beyond the cap."""
        while len(self._engine_cache) > self.max_cached_programs:
            _, old = self._engine_cache.popitem(last=False)
            old.close()

    def _encode_column(self, v, values):
        """(uint8 codes of `values` in the sorted domain of var id `v`, 0 where a value is not a state of it; the
        mask of those values, missing ones included)."""
        idx = pd.Index(self._compiled.domains[v]).get_indexer(pd.Index(values))
        unknown = idx < 0
        return np.where(unknown, 0, idx).astype(np.uint8), unknown

    def _encode_events(self, events, evidence_vars):
        """The columns `evidence_vars` of the frame `events` -> (uint8 codes [n_ev, n], bad [n]).  A row with a
        value outside its variable's domain is bad: the reference's boolean filter at bayes_net.py:772-774 leaves
        an empty factor, hence an empty answer."""
        n = len(events.index)
        codes = np.empty((len(evidence_vars), n), dtype=np.uint8)
        bad = np.zeros(n, dtype=bool)
        for i, name in enumerate(evidence_vars):
            codes[i], unknown = self._encode_column(self._compiled.index[name], events[name].to_numpy())
            bad |= unknown
        return codes, bad

    def _event_posterior(self, program, evidence_vars, event):
        """The float64 posterior of one event on a single-event program, or None when a value is outside its
        variable's domain (the reference's filter leaves nothing).  One event is launch-latency bound on the
        device (~20 us): the host side must not cost ten times that, so state codes come from per-variable
        dicts."""
        net = self._compiled
        codes = np.empty((len(evidence_vars), 1), dtype=np.uint8)
        for i, v in enumerate(evidence_vars):
            code = self._code_of(net.index[v]).get(event[v], -1)
            if code < 0:
                return None
            codes[i, 0] = code
        return program.run(codes, 1)[:, 0].astype(np.float64)

    def _answer_index(self, plan):
        return self._states_index(plan.query)

    def query(self, *query, event: dict, algorithm="exact", n_iterations=100, likelihoods: dict | None = None) -> pd.Series:
        """Answer P(query | event) (bayes_net.py:796-875), exact inference on the GPU.

        The answer is a Series named "P(q1, q2)" indexed by the query variables
        (levels sorted by name, rows sorted by state); states with zero posterior
        are left out, as the reference's zero-filtering join does
        (bayes_net.py:253-256).

        likelihoods: soft evidence, {node: a vector over the node's sorted domain, or a {state: weight}
        dict}, as in `query_many`; computed in float64.
        """
        if not query:
            raise ValueError("At least one query variable has to be specified")
        for q in query:
            if q in event:
                raise ValueError("A query variable cannot be part of the event")
        name = f"P({', '.join(map(str, query))})"
        if likelihoods is not None:
            self._check_soft_call(algorithm, None)
            ev_vars = tuple(event)
            soft, lik = self._soft_matrix(likelihoods, 1, ev_vars, single=True)
            entry = self._soft_programs(query, ev_vars, soft, marginals=False)
            index = self._answer_index(entry.plan)
            codes, bad = self._encode_events(pd.DataFrame({v: [event[v]] for v in ev_vars}, index=[0]), ev_vars)
            post = None if bad[0] else entry.f64().run_soft(codes, lik, 1)[:, 0]
            return _posterior_series(post, index, name)
        if algorithm == "bp":
            post = self._bp_query(query, pd.DataFrame({v: [event[v]] for v in event}, index=[0]), n_iterations)
            return _posterior_series(post[:, 0], self._states_index([self._compiled.index[query[0]]]), name)
        if algorithm in ("gibbs", "likelihood", "rejection"):
            events = pd.DataFrame({v: [event[v]] for v in event}, index=[0])
            freq, index = self._sample_query(algorithm, query, events, n_iterations)
            values = freq[:, 0].astype(np.float64)
            if np.isnan(values).any():  # rejection sampling kept no sample: the reference's answer is empty
                return pd.Series([], index=index[:0], name=name, dtype=np.float64)
            answer = pd.Series(values, index=index, name=name)
            return answer[answer > 0]  # the reference only lists the states that were sampled
        if algorithm != "exact":
            raise ValueError("Unknown algorithm, must be one of: exact, gibbs, likelihood, rejection, bp")

        ev_vars = tuple(event)
        plan, program = self._plan(query, ev_vars, _planner.MODE_FLAT)
        index = getattr(plan, "_answer_index_cache", None)  # cached on the plan: the warm path stays lean
        if index is None:
            index = plan._answer_index_cache = self._answer_index(plan)
        return _posterior_series(self._event_posterior(program, ev_vars, event), index, name)

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

    def _sample_query(self, algorithm, query, events, n_iterations):
        """The approximate algorithms on the device, per row of `events` (columns = evidence variables): one
        Gibbs chain (bayes_net.py:665-737), or n_iterations forward samples for likelihood weighting
        (:621-663) / rejection sampling (:577-619).  Returns (estimates [Q, n_rows], index)."""
        net = self._net("querying")
        ev_vars = tuple(events.columns)
        for name in (*query, *ev_vars):
            if name not in net.index:
                raise KeyError(name)
        q_sorted = sorted(query)  # same key as the exact path (planner: sorted by name) and bayes_net.py:873

        def build():
            from . import engine

            nonevents = sorted(set(self.nodes) - set(ev_vars))  # bayes_net.py:697, the Gibbs cycle order
            return engine.GibbsSampler(net, [net.index[q] for q in q_sorted], [net.index[e] for e in ev_vars],
                                       [net.index[v] for v in nonevents], device=self.device)

        sampler = self._cached(("sampler", tuple(query), ev_vars), build)
        codes, bad = self._encode_events(events, ev_vars)
        if bad.any():
            raise ValueError("an event value is not a state of its variable")
        freq = sampler.run(codes, len(events.index), n_iterations, self._rng.getrandbits(63), algorithm=algorithm)
        return freq, self._states_index([net.index[q] for q in q_sorted])

    def query_many(self, *query, events: pd.DataFrame, algorithm="exact", n_iterations=100,
                   devices: typing.Sequence[int] | None = None, likelihoods: dict | None = None) -> pd.DataFrame:
        """Batched `query`: one posterior per row of `events` (columns = evidence
        variables).  Returns a DataFrame with one row per evidence row and one column
        per joint state of the query variables (same order as `query`'s index);
        impossible rows are NaN.  Zero-probability states stay (as 0.0).

        devices: CUDA device ids to shard the rows over (exact algorithm).  Rows are independent,
        so each device answers a contiguous slice with its own program (one host thread per
        device; the C ABI call releases the GIL) and the slices land in one host array: there is
        no collective.  One process per GPU under torchrun is `sorobn_b200.sharding.query_many_sharded`.

        likelihoods: soft (virtual) evidence, {node: values}, one likelihood over the node's states
        per row: P(query | row) is then proportional to sum P(x, row) * prod_node values[node](x_node).
        `values` is a [len(events), card] numpy array or torch tensor (columns in the node's sorted
        domain order; a CUDA tensor is read on the device) or a DataFrame whose columns are the node's
        states.  Entries must be finite and non-negative; a row of zeros makes the row impossible (NaN),
        and scaling a row changes nothing.  A soft node may be queried, but may not be a column of
        `events`.  Exact algorithm only, on one device."""
        if not query:
            raise ValueError("At least one query variable has to be specified")
        ev_vars = tuple(events.columns)
        for q in query:
            if q in ev_vars:
                raise ValueError("A query variable cannot be part of the event")
        if likelihoods is not None:
            self._check_soft_call(algorithm, devices)
            soft, lik = self._soft_matrix(likelihoods, len(events.index), ev_vars)
            plan = self._soft_programs(query, ev_vars, soft, marginals=False).plan
            return self._soft_frame(query, events, soft, lik, self._answer_index(plan), marginals=False)
        if algorithm == "bp":
            if devices is not None:
                raise ValueError("algorithm='bp' runs on one device: devices=[...] is not supported")
            post = self._bp_query(query, events, n_iterations)
            return pd.DataFrame(post.T, index=events.index, columns=self._states_index([self._compiled.index[query[0]]]))
        if algorithm in ("gibbs", "likelihood", "rejection"):
            freq, index = self._sample_query(algorithm, query, events, n_iterations)
            return pd.DataFrame(freq.T.astype(np.float64), index=events.index, columns=index)
        if algorithm != "exact":
            raise ValueError("Unknown algorithm, must be one of: exact, gibbs, likelihood, rejection, bp")
        plan, _ = self._plan(query, ev_vars, _planner.MODE_BATCHED, device=None if devices is None else devices[0])
        return self._posterior_frame(query, events, self._answer_index(plan), devices=devices)

    def _posterior_frame(self, query, events, columns, marginals=False, devices=None):
        """The posterior of every row of `events` as a frame with `columns`: encoded, run on the device(s) with
        the float64 rescue, and NaN for the rows with a value outside its variable's domain."""
        if len(events.index) == 0:
            return pd.DataFrame(np.zeros((0, len(columns))), index=events.index, columns=columns)
        ev_vars = tuple(events.columns)
        codes, bad = self._encode_events(events, ev_vars)
        if devices is None or len(devices) <= 1:
            post = self._posterior_codes(query, ev_vars, codes, bad, device=None if devices is None else devices[0],
                                         marginals=marginals)
        else:
            post = self._posterior_codes_multi(query, ev_vars, codes, bad, list(devices))
        return self._answer_frame(post, events.index, columns, bad)

    @staticmethod
    def _answer_frame(post, index, columns, bad):
        """The posteriors [Q, n] as a frame, the bad rows NaN."""
        out = pd.DataFrame(post.T, index=index, columns=columns)
        if bad.any():
            out.loc[index[bad]] = np.nan
        return out

    def _posterior_codes(self, query, ev_vars, codes, bad, device=None, marginals=False, replica=0):
        """Posterior float64 [Q, n] for uint8 evidence codes [n_ev, n] on one device, the rows the float32
        program flags settled by `_rescue`.  marginals=True: `query` are the targets of a marginals program
        (every segment normalised)."""
        entry = self._query_programs(query, ev_vars, _planner.MODE_BATCHED, device, marginals, replica)
        post = self._run_evicting(entry, codes, len(bad)).astype(np.float64)  # [Q, n]
        return self._rescue(post, np.isnan(post).any(axis=0) & ~bad, codes, "run", query, ev_vars, device, marginals,
                            replica)

    def _rescue(self, out, flagged, codes, method, query, ev_vars, device=None, marginals=False, replica=0):
        """Settle in float64 the `flagged` rows (last axis of `out`) of a batched float32 program's `method`
        ("run": posteriors, or "evidence": P(event)): flagged rows are NaN, for impossible evidence or an entry
        below the float32 range.  More than 8 run as one batch on the batched plan's float64 program, fewer one
        by one on the single-event program; a row still NaN there is impossible."""
        rows = np.flatnonzero(flagged)
        if len(rows) > 8:
            _, robust = self._plan(query, ev_vars, _planner.MODE_BATCHED, robust=True, device=device,
                                   marginals=marginals, replica=replica)
            out[..., rows] = getattr(robust, method)(np.ascontiguousarray(codes[:, rows]), len(rows))
        elif len(rows):
            _, flat = self._plan(query, ev_vars, _planner.MODE_FLAT, device=device, marginals=marginals,
                                 replica=replica)
            for b in rows:
                out[..., b] = getattr(flat, method)(np.ascontiguousarray(codes[:, b:b + 1]), 1)[..., 0]
        return out

    # ---------------------------------------------------------------- soft evidence
    @staticmethod
    def _check_soft_call(algorithm, devices):
        if algorithm != "exact":
            raise ValueError("soft evidence (likelihoods) needs algorithm='exact'")
        if devices is not None:
            raise ValueError("soft evidence (likelihoods) runs on one device: devices=[...] is not supported")

    def _soft_matrix(self, likelihoods, n, ev_vars, single=False):
        """(soft node names sorted, likelihoods [n, sum of cards]: a numpy float64 array, or a torch tensor on the
        device when any value is a CUDA tensor) of `likelihoods` {node: values}; ValueError for a node that is not
        in the network or is a hard-evidence column, for a wrong shape, a state outside the node's domain, or an
        entry that is NaN, infinite or negative.  `single` (one event): a value may also be a 1-D vector or a
        {state: weight} dict."""
        net = self._net("querying")
        if not isinstance(likelihoods, dict) or not likelihoods:
            raise ValueError("likelihoods must be a non-empty {node: values} dict")
        names = sorted(likelihoods)
        blocks = []
        for name in names:
            if name not in net.index:
                raise ValueError(f"likelihoods for {name!r}, which is not a node of the network")
            if name in ev_vars:
                raise ValueError(f"{name!r} has both hard evidence and likelihoods")
            domain = net.domains[net.index[name]]
            values = likelihoods[name]
            if single and isinstance(values, dict):
                values = pd.DataFrame([values])
            if isinstance(values, (pd.DataFrame, pd.Series)):
                frame = values.to_frame().T if isinstance(values, pd.Series) else values
                unknown = [c for c in frame.columns if c not in set(domain)]
                if unknown:
                    raise ValueError(f"likelihoods for {name!r}: {unknown[:5]} are not states of the node")
                values = frame.reindex(columns=domain).to_numpy(dtype=np.float64)
            elif not type(values).__module__.startswith("torch"):
                values = np.asarray(values, dtype=np.float64)
            if single and values.ndim == 1:
                values = values.reshape(1, -1)
            if tuple(values.shape) != (n, len(domain)):
                raise ValueError(f"likelihoods for {name!r} have shape {tuple(values.shape)}, expected {(n, len(domain))}")
            blocks.append(values)
        torch_blocks = [b for b in blocks if not isinstance(b, np.ndarray)]
        cuda = next((b.device for b in torch_blocks if b.is_cuda), None)
        if cuda is None:
            lik = np.concatenate([b if isinstance(b, np.ndarray) else b.detach().cpu().numpy().astype(np.float64)
                                  for b in blocks], axis=1)
            finite, negative = np.isfinite(lik).all(), (lik < 0).any()
        else:
            import torch

            lik = torch.cat([torch.as_tensor(b).to(device=cuda, dtype=torch.float64) for b in blocks], dim=1)
            finite, negative = bool(torch.isfinite(lik).all()), bool((lik < 0).any())
        if not finite:
            raise ValueError("likelihoods must be finite (no NaN or inf)")
        if negative:
            raise ValueError("likelihoods must be non-negative")
        return tuple(names), lik

    def _soft_programs(self, query, ev_vars, soft, marginals):
        """The cached `_Programs` of P(query | hard columns `ev_vars`, likelihoods of `soft`), plan key (query,
        evidence vars, mode, marginals, soft nodes): batched only, the float64 twin settles flagged rows."""
        net = self._net("querying")

        def build_plan():
            for name in (*query, *ev_vars):
                if name not in net.index:
                    raise KeyError(name)
            ev, sv = [net.index[e] for e in ev_vars], [net.index[s] for s in soft]
            if marginals:
                return _planner.build_marginals_plan(net, ev, targets=[net.index[q] for q in query], soft=sv)
            return _planner.build_plan(net, [net.index[q] for q in query], ev, allow_empty_query=True, soft=sv)

        return self._programs((tuple(query), tuple(ev_vars), _planner.MODE_BATCHED, marginals, tuple(soft)), build_plan)

    def _soft_codes(self, query, ev_vars, soft, codes, bad, lik, marginals, log_evidence=False):
        """(posterior float64 [Q, n], log P(e, lik) [n] or None) of a soft-evidence program; the rows the float32
        program flags (NaN) re-run on the float64 program with their likelihoods; rows with a value outside its
        variable's domain (`bad`) are left to the caller."""
        entry = self._soft_programs(query, ev_vars, soft, marginals)
        n = len(bad)
        res = entry.f32().run_soft(codes, lik, n, log_evidence=log_evidence)
        post, log_ev = res if log_evidence else (res, None)
        post = post.astype(np.float64)
        flagged = np.isnan(post).any(axis=0) & ~bad
        if log_evidence:
            flagged |= np.isnan(log_ev) & ~bad
        rows = np.flatnonzero(flagged)
        if len(rows):
            again = entry.f64().run_soft(np.ascontiguousarray(codes[:, rows]), _lik_rows(lik, rows), len(rows),
                                         log_evidence=log_evidence)
            if log_evidence:
                post[:, rows], log_ev[rows] = again
            else:
                post[:, rows] = again
        return post, log_ev

    def _soft_frame(self, query, events, soft, lik, columns, marginals):
        """`_posterior_frame` with likelihoods: the posterior of every row of `events`."""
        ev_vars = tuple(events.columns)
        if len(events.index) == 0:
            return pd.DataFrame(np.zeros((0, len(columns))), index=events.index, columns=columns)
        codes, bad = self._encode_events(events, ev_vars)
        post, _ = self._soft_codes(query, ev_vars, soft, codes, bad, lik, marginals)
        return self._answer_frame(post, events.index, columns, bad)

    def _targets(self, variables, ev_vars):
        """Target names of a marginals query, sorted: `variables`, or every variable that is not evidence."""
        net = self._net("querying")
        if variables is None:
            variables = [n for n in self.nodes if n not in set(ev_vars)]
        variables = list(variables)
        for v in variables:
            if v in ev_vars:
                raise ValueError("A query variable cannot be part of the event")
            if v not in net.index:
                raise KeyError(v)
        if not variables:
            raise ValueError("At least one query variable has to be specified")
        return tuple(sorted(set(variables)))

    def marginals_many(self, events: pd.DataFrame, variables=None, likelihoods: dict | None = None, algorithm="exact",
                       n_iterations=100, damping=0.5, tol=1e-5) -> pd.DataFrame:
        """The posterior marginal of every variable in `variables` (default: every variable that is not
        a column of `events`), for every row of `events`, from ONE device program: an upward and a
        downward pass over the bucket tree of the elimination, then one readout per variable
        (planner.build_marginals_plan).  Equals `query_many(v, events=events)` for each v.

        Returns one row per evidence row; the columns are a MultiIndex of (variable, state), variables
        sorted by name, states sorted.  Zero-probability states stay (as 0.0); impossible rows and rows
        with a value outside its variable's domain are NaN.  `likelihoods`: soft evidence, as in
        `query_many`; a soft node may be a target.

        algorithm="bp": loopy belief propagation on the device instead of elimination, for networks whose induced
        width the exact planner refuses (sorobn_b200/bp.py defines it).  Sum-product messages on the factor graph of
        the CPT families are swept synchronously, each factor-to-variable message damped as (1 - damping) * new +
        damping * old, until the largest change of any message of the row falls below `tol` or `n_iterations`
        sweeps have run (tol=0 runs exactly n_iterations).  Deterministic, exact on polytrees, approximate on loopy
        networks, where it may also miss impossible evidence.  Same frame as the exact path; rows that did not
        converge keep their last beliefs and raise one RuntimeWarning with their count.  ValueError unless
        0 <= damping < 1, n_iterations >= 1 and tol >= 0.  No soft evidence."""
        if algorithm not in ("exact", "bp"):
            raise ValueError("Unknown algorithm, must be one of: exact, bp")
        if likelihoods is not None:
            self._check_soft_call(algorithm, None)
        if algorithm == "bp":
            _bp.check_arguments(n_iterations, damping, tol)
        ev_vars = tuple(events.columns)
        targets = self._targets(variables, ev_vars)
        net = self._compiled
        columns = pd.MultiIndex.from_tuples([(t, s) for t in targets for s in net.domains[net.index[t]]],
                                            names=["variable", "state"])
        if algorithm == "bp":
            return pd.DataFrame(self._bp_run(targets, events, n_iterations, damping, tol).T, index=events.index,
                                columns=columns)
        if likelihoods is not None:
            soft, lik = self._soft_matrix(likelihoods, len(events.index), ev_vars)
            return self._soft_frame(targets, events, soft, lik, columns, marginals=True)
        return self._posterior_frame(targets, events, columns, marginals=True)

    def _bp_run(self, targets, events, n_iterations, damping, tol):
        """Loopy belief propagation (bp.py) of the sorted `targets` for every row of `events`: beliefs float64
        [Q, n] in the targets' column order, NaN for a row that met a zero sum or has a value outside its
        variable's domain.  One RuntimeWarning counts the rows that did not converge."""
        from . import engine

        net = self._net("querying")
        ev_vars = tuple(events.columns)
        for name in (*targets, *ev_vars):
            if name not in net.index:
                raise KeyError(name)

        def build():
            g = _bp.compile_graph(net, [net.index[e] for e in ev_vars], [net.index[t] for t in targets])
            return engine.BeliefPropagation(g.words, g.tables, device=self.device)

        runner = self._cached(("bp", tuple(targets), ev_vars), build)
        n = len(events.index)
        if n == 0:
            return np.zeros((runner.Q, 0))
        codes, bad = self._encode_events(events, ev_vars)
        out, iters = runner.run(codes, n, n_iterations, damping, tol)
        out = out.astype(np.float64)
        out[:, bad] = np.nan
        stuck = int(np.count_nonzero((iters > n_iterations) & ~bad))
        if stuck:
            warnings.warn(f"belief propagation: {stuck} of {n} rows did not converge to tol={tol:g} in {n_iterations} "
                          "sweeps; they keep the beliefs of their last sweep", RuntimeWarning, stacklevel=3)
        return out

    def _bp_query(self, query, events, n_iterations):
        """`query` / `query_many` with algorithm="bp": one query variable, the default damping and tol."""
        if len(query) != 1:
            raise ValueError("algorithm='bp' answers one query variable at a time: belief propagation gives no joint "
                             "over variables of different families")
        _bp.check_arguments(n_iterations, 0.5, 1e-5)
        ev_vars = tuple(events.columns)
        if query[0] not in self._net("querying").index:
            raise KeyError(query[0])
        return self._bp_run(self._targets(query, ev_vars), events, n_iterations, 0.5, 1e-5)

    def marginals(self, event: dict, variables=None) -> dict:
        """`marginals_many` for one event, in float64 (as `query`): {variable: Series}, each Series equal to
        `query(variable, event=event)` -- named "P(variable)", zero states left out, empty for evidence of
        probability zero."""
        ev_vars = tuple(event)
        targets = self._targets(variables, ev_vars)
        net = self._compiled
        _, program = self._plan(targets, ev_vars, _planner.MODE_FLAT, marginals=True)
        post = self._event_posterior(program, ev_vars, event)
        out, q = {}, 0
        for t in targets:
            index = self._states_index([net.index[t]])
            out[t] = _posterior_series(None if post is None else post[q:q + len(index)], index, f"P({t})")
            q += len(index)
        return out

    def _run_evicting(self, entry, codes, n):
        """`entry.f32().run`, retried once after closing every OTHER cached device object when the device
        is out of memory: each program owns a scratch arena sized for its largest batch (3.9 GB for
        100k rows of the benchmark grid), and a BayesNet caches up to `max_cached_programs` of them --
        many evidence patterns at large batches would otherwise exhaust the GPU long before the LRU
        cap evicts anything (VERDICT r1)."""
        from . import engine

        try:
            return entry.f32().run(codes, n)
        except engine.EngineError as exc:
            if exc.code != engine.SBN_E_NOMEM:
                raise
        with self._cache_lock:
            for key in [k for k, v in self._engine_cache.items() if v is not entry]:
                self._engine_cache.pop(key).close()
        return entry.f32().run(codes, n)

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

    def predict_proba(self, X: typing.Union[dict, pd.DataFrame], likelihoods: dict | None = None):
        """Probability of each row of `X` (bayes_net.py:934-962).

        The reference builds the full joint, sums out the columns `X` lacks and looks the
        rows up.  Here P(row) is the normaliser of a variable elimination with the row as
        evidence and no query variable: same number, no joint, any network size.  Rows of
        probability zero give 0.0 (the reference's joint has no such row and raises
        KeyError).  With a single column the reference returns the whole marginal instead
        of per-row values; this returns per-row values in every case.

        likelihoods: soft evidence, as in `query_many`: each row then gives
        P(row, likelihoods) = sum_x P(x, row) * prod_node values[node](x_node)."""
        if likelihoods is not None:
            with np.errstate(under="ignore"):
                return np.exp(self.predict_log_proba(X, likelihoods=likelihoods))
        if isinstance(X, dict):
            return self.predict_proba(pd.DataFrame([X])).iloc[0]
        ev_vars, name, index = self._proba_index(X)
        n = len(X.index)
        if n == 0:
            return pd.Series([], index=index, name=name, dtype=np.float64)
        _, program = self._plan((), ev_vars, _planner.MODE_BATCHED)
        codes, bad = self._encode_events(X, ev_vars)
        prob = program.evidence(codes, n).astype(np.float64)
        prob = self._rescue(prob, np.isnan(prob) & ~bad, codes, "evidence", (), ev_vars)
        prob[np.isnan(prob) | bad] = 0.0
        return pd.Series(prob, index=index, name=name)

    def _proba_index(self, X):
        """(evidence columns sorted, Series name, index) of `predict_proba`'s answer for the frame `X`."""
        ev_vars = tuple(sorted(X.columns))
        name = f"P({', '.join(map(str, ev_vars))})"
        if len(ev_vars) == 1:
            return ev_vars, name, pd.Index(X[ev_vars[0]], name=ev_vars[0])
        return ev_vars, name, pd.MultiIndex.from_frame(X[list(ev_vars)])

    def predict_log_proba(self, X: typing.Union[dict, pd.DataFrame], likelihoods: dict | None = None):
        """Log-likelihood of each row (bayes_net.py:964-973).  With `likelihoods` (soft evidence, as in
        `query_many`), log P(row, likelihoods) straight from the device's log-normaliser, -inf for a row of
        probability zero."""
        if likelihoods is None:
            with np.errstate(divide="ignore"):
                return np.log(self.predict_proba(X))
        single = isinstance(X, dict)  # one event: a likelihood may be a vector or a {state: weight} dict
        frame = pd.DataFrame([X]) if single else X
        ev_vars, name, index = self._proba_index(frame)
        n = len(frame.index)
        soft, lik = self._soft_matrix(likelihoods, n, ev_vars, single=single)
        if n == 0:
            return pd.Series([], index=index, name=name, dtype=np.float64)
        codes, bad = self._encode_events(frame, ev_vars)
        _, log_ev = self._soft_codes((), ev_vars, soft, codes, bad, lik, marginals=False, log_evidence=True)
        log_ev[np.isnan(log_ev) | bad] = -np.inf
        out = pd.Series(log_ev, index=index, name=name)
        return out.iloc[0] if single else out

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
