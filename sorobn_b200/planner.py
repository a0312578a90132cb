"""Variable-elimination planner: (network, query vars, evidence vars) -> device program.

The reference interleaves planning and arithmetic inside
`BayesNet._variable_elimination` (/root/reference/sorobn/bayes_net.py:739-794):
it works out the relevant and hidden nodes, slices every CPT by the event, then for
each hidden node multiplies the factors that mention it (`pointwise_mul`,
bayes_net.py:253) and sums it out (`CDTAccessor.sum_out`, bayes_net.py:54).

Here the same decisions are taken once per (query vars, evidence vars) pair and
frozen into a flat int32 program; the arithmetic then runs on the device for any
number of evidence rows.  Each program step is one fused
"product of k factors -> sum out one axis" kernel launch:

    out[o, b] = sum_x  prod_i  in_i[ off_i(o) + x * sx_i + evoff_i(b) ]   (, b)

* `o` runs over the output scope (mixed radix, axis 0 fastest), `b` over evidence
  rows.  A factor that depends on the evidence is *batched*: stored `[scope..., B]`
  with the row axis innermost so that a warp reads 32 x 4 consecutive rows of one
  scope entry with 128-bit loads.
* Evidence never materialises sliced tables: a CPT axis that belongs to an
  evidence variable is indexed per row with that row's state code
  (`evoff_i(b) = sum_k ev[col_k, b] * stride_k`).
* Factors that do not depend on evidence stay unbatched and are computed once per
  call by the flat kernel.

Program layout (int32 words) -- parsed by csrc/sbn_api.cu and by
oracle/program_interp.py (the CPU checker used in tests):

    header : MAGIC VERSION mode n_ev n_tables n_slots n_steps Q post_slot post_batched n_soft 0
    tables : (offset_floats, size) * n_tables         -- into the float table blob
    slots  : (batched, size_per_row) * n_slots        -- scratch buffers
    soft   : (slot, card) * n_soft                    -- likelihood slots (header word 10 or 11, see below)
    steps  : kind n_in out_slot n_axes n_elim | cards[n_axes] | ecards[n_elim] |
             per input: is_slot id batched n_ev (col stride card)*n_ev estrides[n_elim] strides[n_axes]

A step sums out `n_elim` variables at once (0 = product only): the reference's
`sum_out(*variables)` (bayes_net.py:54) also takes several.  With `merge_sum_outs=True` the
planner folds a pure sum-out (an elimination whose only factor is the previous product) into
its producer, which saves writing and re-reading the intermediate (-11.7 % HBM bytes on the
benchmark grid).  It is OFF by default: such launches run on the plain kernel today, whose
50 L1 loads per output cost more than the HBM bytes saved (measured 1.59 ms against 0.78 ms
for the two tiled launches replaced); it becomes the default once the tiled kernel takes an
input that spans both tile axes.

`mode` 0 = flat (one evidence row, nothing batched: evidence offsets are uniform),
1 = batched.  The posterior is produced by the last step into `post_slot`
(`[Q]` or `[Q, B]`, unnormalised) and normalised per row by the engine.

Soft evidence (`soft=` of `build_plan`, `build_marginals_plan` and `build_pattern_plan`; batched plans
only): every soft variable v carries a per-row likelihood lambda_v over its states, one batched leaf factor
over (v) in a slot no step writes.  The engine fills those slots before step 0 of every run
(csrc/sbn_soft.cuh), each row divided by its maximum, from the caller's `[n_rows][ld_lik]` likelihood
matrix whose columns are the soft variables sorted by name, states in domain order.  The soft section lists
`(slot, card)` per soft variable in that column order.  `n_soft` is header word 10 of versions 4 and 5 and
word 11 of versions 6 to 9 (their word 10 holds `n_counts` / `n_sampled`).  The log-domain versions 8 and 9
hold log(lambda_v / max lambda_v) in the slot, -inf for a zero entry.  A soft variable is unobserved: a
counts plan gives its family's counts, sample and MPE plans draw or decode it, and a MAP plan sums it out
unless it is a MAP variable.  With `n_soft = 0` the words are those of a plan without soft evidence.

Marginals programs (`build_marginals_plan`, VERSION 5) answer P(t | e) for many targets t at
once.  They use the same words, with two differences:

    header : MAGIC 5 mode n_ev n_tables n_slots n_steps Q -1 0 0 0     -- no posterior slot
    kind 2 : 2 n_in -1 1 n_elim q_offset | card_t | ecards[n_elim] | inputs as above

A kind-2 step (KIND_MARGINAL, the readout of target t from its bucket) has one output axis, the
target, and sums out the `n_elim` other variables of the bucket, with no MAX_ELIM / MAX_Z limit.
It writes the target's `card_t` posterior entries, already normalised per row, at rows
`q_offset ..` of the run's output.  Targets are sorted by name and Q = sum of their cards.
Intermediates of a version-5 program may have several consumers; `build_plan`'s version-4
programs are unchanged.

Counts programs (`build_counts_plan`, VERSION 6) compute the E-step of expectation-maximisation:
for every CPT family (v, parents(v)), sum over the rows of P(family | the row's observed cells).
They reuse the version-5 upward and downward passes and add a count step (kind 3):

    header : MAGIC 6 mode n_ev n_tables n_slots n_steps 1 p_slot p_batched n_counts 0
    kind 3 : 3 n_in -1 n_axes n_elim c_offset n_key (col stride card)*n_key cstrides[n_axes] |
             cards[n_axes] | ecards[n_elim] | inputs as above

`p_slot` holds P(observed cells) of every row (`[1]` or `[1, B]`): the product of the upward
pass's leftover scalars, computed once per run.  The run's per-row output is that probability, NaN
where it is below the float range rule (1e-30 in float32, 1e-290 in float64, or zero / NaN); such
a row adds nothing to the counts.  The count table (`n_counts` float64 entries) is every CPT's
dense `[*parents, v]` array in CompiledNet order, concatenated.  A kind-3 step for node v has the
unobserved members M_v of v's family as output axes.  It reads the smallest bucket whose scope
holds M_v and, per row, adds

    sum_{elims} prod_i in_i[...] / P(observed)     (n_in = 0, M_v empty: 1)

at `c_offset + key(row) + sum_m state_m * cstrides[m]`, with key(row) = sum_k ev[col_k] * stride_k
over the observed family members.  No step writes a slot that a later one still needs: a kind-3
step writes only the count table.

Sample programs (`build_sample_plan`, VERSION 7) draw exact posterior samples of every unobserved
variable: the version-5 upward pass (no downward pass), then one sample step (kind 4) per bucket in
reverse elimination order (forward filtering, backward sampling):

    header : MAGIC 7 1 n_ev n_tables n_slots n_steps 1 p_slot p_batched n_sampled 0
    kind 4 : 4 n_in -1 0 n_x d_first | cards[n_x] |
             per input: is_slot id batched n_terms (col stride card)*n_terms strides[n_x]

`p_slot` holds P(observed cells) of every row, as in version 6.  The drawn codes are extra code
rows: row `n_ev + j` is the j-th sampled variable, `[n_sampled][n_draws][ld]` uint8.  A kind-4 step
draws the joint state X of its bucket's eliminated variables (`n_x` of them, first one fastest,
at most MAX_Z joint states) with probability proportional to

    w(X) = prod_i in_i[ sum_x X_x * strides_i[x] + sum_t code_t(row, draw) * stride_t ]

where the terms `(col stride card)` gather observed columns (col < n_ev) or variables drawn by an
earlier step (col >= n_ev): the bucket's separator, which lies above it in the bucket tree.  A
batched input's gathered offset is multiplied by the row pitch.  The step writes the codes of its
variables to drawn rows `d_first .. d_first + n_x - 1`; steps write consecutive rows, so the
sampled variables are numbered in drawing order.  A sample step writes no slot.

MPE programs (`build_mpe_plan`, VERSION 8) find the most probable explanation of every row: the joint
state x* of every unobserved variable that maximises P(x, e).  They are sample programs in the log
domain, with an argmax step (kind 5) in place of every sample step:

    header : MAGIC 8 1 n_ev n_tables n_slots n_steps 1 p_slot p_batched n_decoded 0
    kind 5 : the words of kind 4

The table blob holds log(table) (the float64 logs cast to float32; a zero entry is -inf), and every
kind-0 / kind-1 step means max-sum: `out = max_x sum_i in_i[...]`, or `sum_i in_i[...]` for a
product-only step.  `p_slot` holds max log P(x, e) of every row, the sum of the upward pass's leftover
scalars (-inf: the observed cells are impossible).  A kind-5 step decodes its bucket's variables given
the decoded separator: the first joint state z (first variable fastest) with the largest

    w(z) = sum_i in_i[ sum_x X_x * strides_i[x] + sum_t code_t(row) * stride_t ].

Logs, because the maximum is a product of one entry of every CPT: it shrinks with the network and with
every observed cell, past the float32 range of the sum-product programs, where its log cannot underflow.

Marginal MAP programs (`build_map_plan`, VERSION 9) find, for every row, the joint state of chosen MAP
variables that maximises P(x_MAP, e), every other unobserved variable summed out.  They are MPE programs
whose elimination order puts every summed variable before any MAP variable, and whose kind-0 / kind-1
steps carry one more word, the reduction of their eliminated variables:

    kind 0/1 : kind n_in out_slot n_axes n_elim reduce | cards | ecards | inputs as above

`reduce` 1 = log-sum-exp, `out = log sum_x exp(sum_i in_i[...])` (a bucket of summed variables); 0 = max,
as in version 8 (a bucket of MAP variables, and every product-only step).  No launch mixes the two.
Argmax steps (kind 5, the words of version 8) decode the MAP buckets only: their separators hold MAP and
observed variables alone, because every summed variable is gone by then.  `p_slot` holds
max_{x_MAP} log P(x_MAP, e).

Gradient programs (`build_pattern_plan(net, "grad", ...)`, VERSION 10) give the derivatives of
log P(observed cells, lik) of every row (DESIGN.md "Gradients of the log-likelihood").  They are counts
programs plus one derivative readout (kind 6) per soft variable s:

    header : MAGIC 10 1 n_ev n_tables n_slots n_steps Q p_slot p_batched n_counts n_soft
    kind 6 : 6 n_in -1 1 n_elim q_offset | card_s | ecards[n_elim] | inputs as above

Q = 1 + the likelihood columns.  The count steps add each row's family posterior times a per-row weight
w_b given at run time (a fully observed family adds w_b), which is sum_b w_b * theta * d log P_b / d theta.
A kind-6 step reads the bucket k that lambda_s entered, with every input of that bucket except lambda_s:

    D_s(x, b) = sum_{U_k - s} pi_k * prod_{f in F_k, f != lambda_s} f  /  P(observed)

written at rows `q_offset ..` (1 + the soft variable's first likelihood column) of the run's output; row 0 is
P(observed).  D_s is d log P / d lambda_s, exact where lambda_s(x) = 0.  `Plan.forward_steps` lists the steps
P(observed) depends on (the upward pass): a forward run issues only those.

Joint programs (`build_joint_plan`, `build_pattern_plan(net, "joint", ...)`, VERSION 11) give, for every row,
the joint posterior of chosen groups of variables (by default every CPT family) given the row's observed cells
and likelihoods.  They are counts programs whose count steps are per-row readouts (kind 7):

    header : MAGIC 11 1 n_ev n_tables n_slots n_steps Q p_slot p_batched 0 n_soft
    kind 7 : 7 n_in -1 n_axes n_elim q_offset | cards[n_axes] | ecards[n_elim] | inputs as above

`p_slot` holds P(observed, lik / max) of every row, as in version 6.  A kind-7 step reads the unobserved
members M_g of group g (its output axes, in the group's order, the first one fastest) from the smallest bucket
that holds them, and writes

    sum_{U_k - M_g} pi_k * prod_{f in F_k} f / P(observed)

at rows `q_offset .. q_offset + |M_g| - 1` of the run's `[Q][ld]` output; Q is the sum of those sizes over the
groups.  A group the pattern observes completely has no step (its posterior is a one-hot on the observed
codes).  A family lies in the bucket its CPT entered; a group that lies in no CPT's scope gets a constant table
of ones over M_g, entered with the CPTs, so that elimination builds a bucket holding it (`Plan.ones`).  Those
tables follow the CPTs' in the table section.
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field

import numpy as np

MAGIC = 0x53424E31  # "SBN1"
VERSION = 4
MAX_IN = 8  # factors fused per launch (csrc/sbn_kernels.cuh: SBN_MAX_IN)
MAX_AXES = 20  # output axes per step (SBN_MAX_AXES)
MAX_EV = 8  # evidence axes per input (SBN_MAX_EV)
TILE_EDGE = 5  # largest register-tile edge of sbn_step_tiled
MAX_ELIM = 3  # variables summed out by one launch (SBN_MAX_ELIM)
MAX_Z = 256  # joint states of the variables summed out by one launch
# Largest table (entries) that may keep evidence axes.  Much larger tables make a consumer gather
# from a big table (62 KB at 16384 entries on the grid) for every output.
LIFT_MAX = int(os.environ.get("SOROBN_B200_LIFT_MAX", "4096"))
TILED_MAX_IN = 4  # inputs of one launch of the tiled kernel (csrc: kTiledMaxIn)
SLICE_MIN_BYTES = 64 * 1024  # tables of one launch beyond this are laid out for sliced staging (csrc: SBN_SMEM_BUDGET)
PRELOAD_MAX_IN = 3  # the tiled kernel's preload schedule (all operands of a block in registers)
MODE_FLAT, MODE_BATCHED = 0, 1
KIND_FLAT, KIND_BATCHED = 0, 1
KIND_MARGINAL = 2  # readout of one target's marginal from a bucket (marginals programs only)
# Joint states one readout sums out: its offset table, [SBN_MAX_IN][cz] int32 words, is capped at 2^24
# words (csrc/sbn_api.cu: kMarginalZoffMax / SBN_MAX_IN)
MARGINAL_MAX_Z = 2**21
VERSION_MARGINALS = 5
KIND_COUNT = 3  # expected counts of one CPT family, summed over the rows (counts programs only)
VERSION_COUNTS = 6
KIND_SAMPLE = 4  # draw one bucket's eliminated variables given the drawn separator (sample programs only)
VERSION_SAMPLE = 7
SAMPLE_MAX_CARD = 255  # a sampled variable's states (its codes are uint8)
SAMPLE_MAX_TERMS = 16  # gathered (col stride card) terms per input of a sample step (csrc: SBN_SAMPLE_MAX_TERMS)
KIND_ARGMAX = 5  # decode one bucket's eliminated variables given the decoded separator (MPE programs only)
VERSION_MPE = 8
VERSION_MAP = 9  # marginal MAP: the MPE words plus a reduction word on kind-0 / kind-1 steps
KIND_DERIV = 6  # derivative of P(observed) by one soft variable's likelihood, over P(observed) (gradient programs only)
VERSION_GRAD = 10
KIND_JOINT = 7  # per-row joint posterior of one group of variables (joint programs only)
VERSION_JOINT = 11
REDUCE_MAX, REDUCE_LOGSUMEXP = 0, 1
HEADER_WORDS = 12


@dataclass
class CompiledNet:
    """Dense, integer-indexed form of a prepared BayesNet (built by
    `BayesNet.prepare()`; the analogue of the pandas housekeeping at
    bayes_net.py:327-371 plus "ship the tables to the device")."""

    names: list  # var id -> node name, topological order (== BayesNet.nodes)
    domains: list  # var id -> sorted list of state values
    parents: list  # var id -> list of parent ids (sorted by name, like the reference)
    cpt: list  # var id -> float64 ndarray, axes [*parents, var]
    card: np.ndarray = None
    index: dict = field(default_factory=dict)  # name -> var id

    def __post_init__(self):
        self.card = np.array([len(d) for d in self.domains], dtype=np.int64)
        self.index = {n: i for i, n in enumerate(self.names)}

    def scope(self, v):
        return (*self.parents[v], v)

    def ancestors(self, v):
        seen = set()
        stack = list(self.parents[v])
        while stack:
            p = stack.pop()
            if p not in seen:
                seen.add(p)
                stack.extend(self.parents[p])
        return seen


@dataclass
class _Factor:
    is_slot: bool
    buf: int  # table index or slot index
    vars: tuple  # free variable ids
    strides: tuple  # element stride per free variable
    ev: tuple  # ((ev_col, stride, card), ...) -- CPTs and tables that kept evidence axes (never batched)
    batched: bool

    @property
    def depends_on_evidence(self):
        return self.batched or bool(self.ev)


@dataclass
class Step:
    kind: int
    inputs: list  # of (factor, strides-per-eliminated-axis, strides-per-out-axis)
    out_id: int  # logical id of the factor produced (slots are assigned afterwards)
    out_vars: tuple  # axis 0 (fastest) first
    cards: tuple
    elims: tuple  # variables summed out by this launch
    ecards: tuple
    out_slot: int = -1
    q_offset: int = -1  # KIND_MARGINAL: first posterior entry of the target's segment; KIND_COUNT: c_offset;
    # KIND_SAMPLE / KIND_ARGMAX: first drawn-code row it writes
    key: tuple = ()  # KIND_COUNT: ((ev_col, stride, card), ...) of the observed family members
    cstrides: tuple = ()  # KIND_COUNT: count-table stride of every output axis
    norm: object = None  # KIND_COUNT / KIND_SAMPLE / KIND_ARGMAX: the factor in the header's p_slot
    reduce: int = REDUCE_MAX  # kind 0 / 1 of a marginal MAP plan: REDUCE_LOGSUMEXP sums its elims out

    @property
    def cx(self):
        return int(np.prod(self.ecards, dtype=np.int64)) if self.ecards else 1


@dataclass
class Plan:
    mode: int
    query: tuple  # query var ids, in output (sorted-name) order, slowest axis first
    evidence: tuple  # evidence var ids == evidence columns
    order: list  # elimination order (var ids)
    tables: list  # var ids whose CPTs are shipped, in table order
    slots: list  # (batched, size)
    steps: list
    post_slot: int
    Q: int
    words: np.ndarray = None
    table_blob: np.ndarray = None
    table_blob64: np.ndarray = None
    table_offsets: list = None
    version: int = VERSION
    targets: tuple = ()  # marginals plans: target var ids, sorted by name (== posterior segment order)
    n_counts: int = 0  # counts plans: entries of the count table
    count_offsets: list = None  # counts plans: first count-table entry of every var id's family
    table_axes: list = None  # var ids of every shipped table's axes, outermost first (refresh_tables)
    table_scopes: list = None  # the CPT scope [*parents, v] every table was transposed from
    sampled: tuple = ()  # sample / MPE plans: the var id of every drawn (decoded) code row, in drawing order
    soft: tuple = ()  # soft-evidence var ids, sorted by name (== likelihood column order)
    soft_slots: tuple = ()  # the slot of every soft variable's likelihood, in `soft` order
    # gradient plans: indices of the steps P(observed) depends on, in program order.  The engine derives the same set
    # from the slot words (csrc/sbn_api.cu parse); the CPU replay reads this one, and a GPU test checks the two agree
    forward_steps: tuple = ()
    groups: tuple = ()  # joint plans: the var ids of every group, in call order
    group_rows: tuple = ()  # joint plans: each group's first output row, -1 for a group the pattern observes completely
    ones: tuple = ()  # joint plans: the unobserved members of every group given a table of ones, in table order

    # ---- cost model (DESIGN.md "algorithmic bytes") -------------------------------
    def bytes_per_row(self, n_draws=1):
        """Algorithmic HBM bytes per evidence row: every batched step reads each
        batched input once and writes its output once (fp32), plus the evidence
        codes in and the posterior out.  A sample step reads, per draw, the part of each
        batched input its drawn separator selects and writes its codes (`n_draws` draws); an
        argmax step counts as a sample step with one draw."""
        total = 0
        for st in self.steps:
            if st.kind in (KIND_SAMPLE, KIND_ARGMAX):
                nd = n_draws if st.kind == KIND_SAMPLE else 1
                for f, es, _ in st.inputs:
                    if f.batched:
                        total += 4 * nd * int(np.prod([c for c, s in zip(st.ecards, es) if s], dtype=np.int64))
                total += nd * len(st.elims)
                continue
            if st.kind not in (KIND_BATCHED, KIND_MARGINAL, KIND_COUNT, KIND_JOINT):
                continue
            for f, _, _ in st.inputs:
                if f.batched:
                    total += 4 * int(np.prod([self._card[v] for v in f.vars], dtype=np.int64))
            if st.kind == KIND_COUNT:
                total += 4  # P(observed); the count table is per program, not per row
                continue
            total += 4 * int(np.prod(st.cards, dtype=np.int64))
        if self.version == VERSION:
            # normalise: read unnormalised posterior, write posterior (a marginals program's
            # readouts write their segments normalised, counted above)
            total += 8 * self.Q
        elif self.version in (VERSION_COUNTS, VERSION_SAMPLE, VERSION_MPE, VERSION_MAP, VERSION_JOINT):
            total += 4  # P(observed) (max log P(x, e)) out
        total += len(self.evidence)  # uint8 codes
        if self.soft:
            # the pack reads the caller's likelihoods, writes them to their slots and writes sum log(max)
            total += 8 * sum(int(self._card[v]) for v in self.soft) + 8
        return total

    def step_bytes_per_row(self):
        out = []
        for st in self.steps:
            if st.kind not in (KIND_BATCHED, KIND_MARGINAL):
                out.append(0)
                continue
            t = 4 * int(np.prod(st.cards, dtype=np.int64))
            for f, _, _ in st.inputs:
                if f.batched:
                    t += 4 * int(np.prod([self._card[v] for v in f.vars], dtype=np.int64))
            out.append(t)
        return out

    def flops_per_row(self):
        total = 0
        for st in self.steps:
            if st.kind != KIND_BATCHED:
                continue
            total += int(np.prod(st.cards, dtype=np.int64)) * st.cx * len(st.inputs)
        return total

    def scratch_floats_per_row(self):
        return sum(size for batched, size in self.slots if batched)

    def max_factor_per_row(self):
        return max([size for batched, size in self.slots if batched] or [0])


def _min_fill_order(scopes, hidden, card, first=None):
    """Greedy min-fill (ties: smaller clique, then lower var id).  The reference
    eliminates in set-iteration order (bayes_net.py:779), which is arbitrary and
    does not change the answer; BASELINE.json asks for min-fill.  With `first`, every
    variable of `first` is eliminated before any other (min-fill within each group)."""
    adj = {}
    for sc in scopes:
        for a in sc:
            adj.setdefault(a, set()).update(b for b in sc if b != a)
    for h in hidden:
        adj.setdefault(h, set())
    remaining = sorted(hidden)
    order = []
    while remaining:
        best_key, best_v = None, None
        pool = remaining if first is None else ([v for v in remaining if v in first] or remaining)
        for v in pool:
            nb = list(adj[v])
            fill = 0
            for i in range(len(nb)):
                ai = adj[nb[i]]
                for j in range(i + 1, len(nb)):
                    if nb[j] not in ai:
                        fill += 1
            size = 1
            for u in nb:
                size *= int(card[u])
            key = (fill, size, v)
            if best_key is None or key < best_key:
                best_key, best_v = key, v
        v = best_v
        nb = adj.pop(v)
        for a in nb:
            adj[a].discard(v)
            adj[a].update(b for b in nb if b != a)
        remaining.remove(v)
        order.append(v)
    return order


def _check_soft(net, evidence, soft, mode):
    """`soft` as var ids sorted by name (the likelihood column order); ValueError for a bad set."""
    soft = tuple(soft)
    if not soft:
        return ()
    if len(set(soft)) != len(soft):
        raise ValueError("duplicate soft-evidence variable")
    if set(soft) & set(evidence):
        raise ValueError("a soft-evidence variable cannot also be a hard-evidence column")
    if mode != MODE_BATCHED:
        raise ValueError("soft evidence needs a batched plan")
    return tuple(sorted(soft, key=lambda v: net.names[v]))


def build_plan(net: CompiledNet, query, evidence, mode=MODE_BATCHED, order=None, max_in=MAX_IN,
               merge_sum_outs=None, lift_evidence=True, allow_empty_query=False, fuse_elims=None, soft=()) -> Plan:
    """Plan P(query | evidence) for `net`.

    query / evidence are sequences of var ids.  `evidence` fixes the evidence
    *columns*; their values arrive at run time.  `soft` are the var ids whose per-row
    likelihoods arrive at run time (soft evidence, see the module docstring); a soft
    variable may be queried.
    """
    query, evidence = tuple(query), tuple(evidence)
    soft = _check_soft(net, evidence, soft, mode)
    if not query and not allow_empty_query:
        # bayes_net.py:840-841
        raise ValueError("At least one query variable has to be specified")
    if not query and not evidence and not soft:
        raise ValueError("nothing to compute: no query variable and no evidence")
    if set(query) & set(evidence):
        # bayes_net.py:843-845
        raise ValueError("A query variable cannot be part of the event")
    if len(set(query)) != len(query):
        raise ValueError("duplicate variable in query or event")
    return _build(net, VERSION, evidence, query=query, mode=mode, order=order, max_in=max_in,
                  lift_evidence=lift_evidence, fuse_elims=fuse_elims, merge_sum_outs=merge_sum_outs, soft=soft)


def build_marginals_plan(net: CompiledNet, evidence, targets=None, mode=MODE_BATCHED, order=None, max_in=MAX_IN,
                         lift_evidence=True, fuse_elims=None, soft=()) -> Plan:
    """Plan P(t | evidence) for every target t at once (a version-5 program, see the module docstring).

    `targets` defaults to every variable that is not evidence.  The posterior is the
    concatenation of the targets' marginals, targets sorted by name, states in domain order.
    `soft` are the var ids with per-row likelihoods, as for `build_plan`; they may be targets."""
    evidence = tuple(evidence)
    soft = _check_soft(net, evidence, soft, mode)
    if targets is None:
        targets = [v for v in range(len(net.names)) if v not in set(evidence)]
    targets = tuple(targets)
    if not targets:
        raise ValueError("no target variable: every variable is evidence")
    if set(targets) & set(evidence):
        raise ValueError("A query variable cannot be part of the event")
    if len(set(targets)) != len(targets):
        raise ValueError("duplicate target variable")
    return _build(net, VERSION_MARGINALS, evidence, targets=targets, mode=mode, order=order, max_in=max_in,
                  lift_evidence=lift_evidence, fuse_elims=fuse_elims, soft=soft)


def build_counts_plan(net: CompiledNet, evidence, mode=MODE_BATCHED, order=None, max_in=MAX_IN, lift_evidence=True,
                      fuse_elims=None) -> Plan:
    """Plan the expected counts of every CPT family given the observed columns `evidence` (a version-6
    program, see the module docstring): one program serves every row of one missingness pattern.
    Its count table is laid out by `count_layout`."""
    evidence = tuple(evidence)
    hidden = tuple(v for v in range(len(net.names)) if v not in set(evidence))
    return _build(net, VERSION_COUNTS, evidence, targets=hidden, mode=mode, order=order, max_in=max_in,
                  lift_evidence=lift_evidence, fuse_elims=fuse_elims)


def build_sample_plan(net: CompiledNet, evidence, order=None, max_in=MAX_IN, lift_evidence=True, fuse_elims=None) -> Plan:
    """Plan exact posterior draws of every variable that is not in `evidence` (a version-7 program, see
    the module docstring): the upward pass of variable elimination, then one sample step per bucket,
    top-down.  `Plan.sampled` names the variable of every drawn-code row."""
    evidence = tuple(evidence)
    hidden = tuple(v for v in range(len(net.names)) if v not in set(evidence))
    return _build(net, VERSION_SAMPLE, evidence, targets=hidden, order=order, max_in=max_in,
                  lift_evidence=lift_evidence, fuse_elims=fuse_elims)


def build_mpe_plan(net: CompiledNet, evidence, order=None, max_in=MAX_IN, lift_evidence=True, fuse_elims=None) -> Plan:
    """Plan the most probable explanation of every row (a version-8 program, see the module docstring):
    the sample plan's steps in the log domain, the upward pass max-sum, then one argmax step per bucket,
    top-down.  Every variable that is not in `evidence` is decoded -- barren nodes too: their CPT rows
    do not max to 1 -- and `Plan.sampled` names the variable of every decoded-code row."""
    evidence = tuple(evidence)
    hidden = tuple(v for v in range(len(net.names)) if v not in set(evidence))
    return _build(net, VERSION_MPE, evidence, targets=hidden, order=order, max_in=max_in,
                  lift_evidence=lift_evidence, fuse_elims=fuse_elims)


def build_map_plan(net: CompiledNet, evidence, map_vars, order=None, max_in=MAX_IN, lift_evidence=True,
                   fuse_elims=None) -> Plan:
    """Plan the marginal MAP state of `map_vars` for every row (a version-9 program, see the module
    docstring): the joint state of the MAP variables that maximises P(x_MAP, e), every other unobserved
    variable summed out.  Only the MAP variables, the evidence and their ancestors are relevant: a barren
    summed variable sums to one and drops out.  The upward pass eliminates the summed variables first
    (log-sum-exp), then the MAP variables (max-sum); one argmax step per MAP bucket follows, top-down.
    `order`, if given, must list every summed variable before any MAP variable.  `Plan.sampled` names the
    variable of every decoded-code row."""
    evidence, map_vars = tuple(evidence), tuple(map_vars)
    if len(set(map_vars)) != len(map_vars):
        raise ValueError("duplicate MAP variable")
    if set(map_vars) & set(evidence):
        raise ValueError("A MAP variable cannot be part of the event")
    if not map_vars and not evidence:
        raise ValueError("nothing to compute: no MAP variable and no evidence")
    return _build(net, VERSION_MAP, evidence, targets=map_vars, order=order, max_in=max_in,
                  lift_evidence=lift_evidence, fuse_elims=fuse_elims)


def build_joint_plan(net: CompiledNet, evidence, groups=None, soft=(), order=None, max_in=MAX_IN, lift_evidence=True,
                     fuse_elims=None) -> Plan:
    """Plan the joint posterior of every group of `groups` for each row of one missingness pattern (a version-11
    program, see the module docstring): `groups` are tuples of var ids (default: every CPT family, in
    [*parents, v] order), `evidence` the observed columns and `soft` the var ids with per-row likelihoods.
    `Plan.group_rows` gives each group's first output row (-1: observed completely).  ValueError for a
    duplicate member, and when no group has an unobserved member (the program would output nothing)."""
    evidence = tuple(evidence)
    soft = _check_soft(net, evidence, soft, MODE_BATCHED)
    if groups is None:
        groups = [net.scope(v) for v in range(len(net.names))]
    groups = tuple(tuple(int(u) for u in g) for g in groups)
    for g in groups:
        if not g or len(set(g)) != len(g):
            raise ValueError(f"group {[net.names[u] for u in g]} is empty or has a duplicate member")
        if any(u < 0 or u >= len(net.names) for u in g):
            raise ValueError(f"group {g} names a variable the network does not have")
    if not any(u not in set(evidence) for g in groups for u in g):
        raise ValueError("every group is observed completely: a joint program would output nothing")
    hidden = tuple(v for v in range(len(net.names)) if v not in set(evidence))
    return _build(net, VERSION_JOINT, evidence, targets=hidden, order=order, max_in=max_in, lift_evidence=lift_evidence,
                  fuse_elims=fuse_elims, soft=soft, groups=groups)


def build_pattern_plan(net: CompiledNet, kind, evidence, soft=(), map_vars=None, groups=None, **kw) -> Plan:
    """The plan of one missingness pattern with soft evidence: `kind` "counts", "sample", "mpe" or "map" (then
    `map_vars` are the MAP variables), the observed columns `evidence` and the var ids `soft` whose per-row
    likelihoods arrive at run time (see the module docstring).  A soft variable may not be evidence; it may be
    a MAP variable.  With `soft=()` the plan is the one of the kind's own builder (`build_counts_plan`, ...),
    word for word; `kw` are that builder's options.

    `kind` "grad" plans the gradient program of the pattern (version 10, soft evidence or not): the counts
    program's steps with weighted counts, plus one derivative readout per soft variable.  `kind` "joint" plans
    the joint posteriors of `groups` (version 11, soft evidence or not; `build_joint_plan`)."""
    builders = {"counts": build_counts_plan, "sample": build_sample_plan, "mpe": build_mpe_plan, "map": build_map_plan}
    if kind not in builders and kind not in ("grad", "joint"):
        raise ValueError(f"kind must be one of {sorted([*builders, 'grad', 'joint'])}, not {kind!r}")
    if (map_vars is not None) != (kind == "map"):
        raise ValueError("map_vars go with kind 'map' only, and kind 'map' needs them")
    if groups is not None and kind != "joint":
        raise ValueError("groups go with kind 'joint' only")
    if kind == "joint":
        if kw.get("mode", MODE_BATCHED) != MODE_BATCHED:
            raise ValueError("a joint program is batched")
        kw.pop("mode", None)
        return build_joint_plan(net, evidence, groups, soft=soft, **kw)
    evidence = tuple(evidence)
    soft = _check_soft(net, evidence, soft, kw.get("mode", MODE_BATCHED))
    if kind == "grad":
        if kw.get("mode", MODE_BATCHED) != MODE_BATCHED:
            raise ValueError("a gradient program is batched")
        hidden = tuple(v for v in range(len(net.names)) if v not in set(evidence))
        return _build(net, VERSION_GRAD, evidence, targets=hidden, soft=soft, **kw)
    if not soft:
        return builders[kind](net, evidence, *(() if map_vars is None else (map_vars,)), **kw)
    hidden = tuple(v for v in range(len(net.names)) if v not in set(evidence))
    if kind == "counts":
        return _build(net, VERSION_COUNTS, evidence, targets=hidden, soft=soft, **kw)
    if kind in ("sample", "mpe"):
        return _build(net, VERSION_SAMPLE if kind == "sample" else VERSION_MPE, evidence, targets=hidden, soft=soft, **kw)
    map_vars = tuple(map_vars)
    if len(set(map_vars)) != len(map_vars):
        raise ValueError("duplicate MAP variable")
    if set(map_vars) & set(evidence):
        raise ValueError("A MAP variable cannot be part of the event")
    # with soft evidence a plan that decodes nothing still has its log P(e, lik) to compute
    return _build(net, VERSION_MAP, evidence, targets=map_vars, soft=soft, **kw)


def count_layout(net: CompiledNet):
    """(first count-table entry of every var id's family, total entries): the dense `[*parents, v]`
    arrays of the CPTs in CompiledNet order, concatenated."""
    offsets, off = [], 0
    for v in range(len(net.names)):
        offsets.append(off)
        off += int(np.prod([int(net.card[u]) for u in net.scope(v)], dtype=np.int64))
    return offsets, off


def refresh_tables(plan: Plan, cpts):
    """The (float32, float64) table blobs of `plan` for new CPT values `cpts` (var id -> ndarray
    [*parents, v], the same domains): the layout of the planned tables (axis permutations, relayouts,
    offsets) is kept, so a program can take them in place of its own (engine.Program.set_tables)."""
    arrays = []
    for t, v in enumerate(plan.tables):
        scope = list(plan.table_scopes[t])
        arr = np.asarray(cpts[v], dtype=np.float64)
        if arr.shape != tuple(int(plan._card[u]) for u in scope):
            raise ValueError(f"the CPT of var {v} has shape {arr.shape}; the plan has {[int(plan._card[u]) for u in scope]}")
        arrays.append(np.ascontiguousarray(np.transpose(arr, [scope.index(u) for u in plan.table_axes[t]])))
    blob64, _ = _blobs(arrays)
    return blob64.astype(np.float32), blob64


class _Builder:
    """The planning state every program kind shares: the shipped tables, the steps emitted so far and
    the next logical id, with the launch-building rules over them (`emit` and the products built on
    it).  `_build` makes one per plan and runs the upward pass through it; the kind's tail adds its
    own steps and ends with `finish`."""

    def __init__(self, net, evidence, mode, max_in, lift_evidence, tables):
        self.net, self.card = net, net.card
        self.evidence = evidence
        self.ev_col = {v: i for i, v in enumerate(evidence)}
        self.mode, self.max_in, self.lift_evidence = mode, max_in, lift_evidence
        self.order = None  # elimination order (var ids), set by `_build`
        self.steps = []
        self.tables = tables  # var ids whose CPTs are shipped, in table order
        self.table_arrays = []
        self.table_axes = []  # variable of every axis of table_arrays[t], outermost first
        self.next_id = 0
        self.summed = frozenset()  # marginal MAP plans: the variables a launch sums out by log-sum-exp
        self.soft = ()  # (var id, logical id of its likelihood) per soft-evidence variable, sorted by name

    def size(self, vs):
        """Joint states of the variables `vs`."""
        return int(np.prod([self.card[v] for v in vs], dtype=np.int64)) if vs else 1

    def largest(self, inputs):
        """The largest batched operand (the largest table when none is batched)."""
        return max(inputs, key=lambda f: (f.batched, self.size(f.vars)))

    def emit(self, inputs, elims, out_vars, may_lift=True):
        """One fused launch: multiply `inputs`, sum out `elims` (empty: product only).
        out_vars is given fastest axis first.  The output gets a logical id; physical
        slots are assigned after the merge pass.

        Deferred evidence instantiation: when every input is a table (CPTs, or tables built
        this way), the product depends on the evidence row only through the few evidence
        columns those tables are indexed by.  It is then computed ONCE, as a table that keeps
        those evidence variables as ordinary (innermost) axes, by an evidence-independent flat
        launch; consumers gather from it like from a CPT.  The reference filters every CPT by
        the event first (bayes_net.py:772-774); filtering after multiplying gives the same
        numbers and turns per-row work into per-call work."""
        card, evidence = self.card, self.evidence
        elims = tuple(elims)
        ecards = tuple(int(card[e]) for e in elims)
        n_summed = sum(e in self.summed for e in elims)
        assert n_summed in (0, len(elims)), "a launch may not both sum out and maximise"
        reduce = REDUCE_LOGSUMEXP if n_summed else REDUCE_MAX
        dep = any(f.depends_on_evidence for f in inputs)
        batched = dep and self.mode == MODE_BATCHED
        if len(out_vars) > MAX_AXES:
            raise ValueError(f"a factor over {len(out_vars)} variables exceeds the kernel's {MAX_AXES} axes")
        cards = tuple(int(card[u]) for u in out_vars)
        size = self.size(out_vars)
        if size >= 2**31:
            raise ValueError("a factor with >= 2^31 entries per row does not fit the 32-bit scope index")

        lifted_cols = None
        if batched and self.lift_evidence and may_lift and not any(f.batched for f in inputs):
            cols = []
            for f in inputs:
                for col, _, c in f.ev:
                    if (col, c) not in cols:
                        cols.append((col, c))
            lifted = size * int(np.prod([c for _, c in cols], dtype=np.int64))
            if len(cols) <= MAX_EV and lifted <= LIFT_MAX and len(out_vars) + len(cols) <= MAX_AXES:
                lifted_cols = cols

        ins = []
        out_id = self.next_id
        self.next_id += 1
        if lifted_cols is not None:
            ev_vars = [evidence[col] for col, _ in lifted_cols]
            axes = tuple(ev_vars) + tuple(out_vars)  # evidence axes innermost
            axis_cards = tuple(c for _, c in lifted_cols) + cards
            for f in inputs:
                pos = {u: sd for u, sd in zip(f.vars, f.strides)}
                pos.update({evidence[col]: sd for col, sd, _ in f.ev})
                es = tuple(pos.get(e, 0) for e in elims)
                plain = _Factor(f.is_slot, f.buf, f.vars, f.strides, (), False)  # evidence axes are output axes here
                ins.append((plain, es, tuple(pos.get(u, 0) for u in axes)))
            self.steps.append(Step(KIND_FLAT, ins, out_id, axes, axis_cards, elims, ecards, reduce=reduce))
            strides = _dense_strides(axis_cards)
            n_ev = len(lifted_cols)
            ev = tuple((col, strides[k], c) for k, (col, c) in enumerate(lifted_cols))
            return _Factor(True, out_id, tuple(out_vars), strides[n_ev:], ev, False)

        for f in inputs:
            pos = {u: s for u, s in zip(f.vars, f.strides)}
            es = tuple(pos.get(e, 0) for e in elims)
            ins.append((f, es, tuple(pos.get(u, 0) for u in out_vars)))
        self.steps.append(Step(KIND_BATCHED if batched else KIND_FLAT, ins, out_id, tuple(out_vars), cards, elims,
                               ecards, reduce=reduce))
        return _Factor(True, out_id, tuple(out_vars), _dense_strides(cards), (), batched)

    def axis_order(self, inputs, out_set):
        """Fastest-first order of the output axes (`_tile_axes` in the kernel docs).

        Axes 0 and 1 span the register tile of csrc/sbn_step_tiled: an input that lacks
        axis 0 is loaded once per tile column, one that lacks both once per tile.  Every
        ordered pair of output axes is scored by the loads per output it implies
        (batched inputs weigh double: they come from L1/L2/HBM, tables from shared
        memory) and the cheapest pair wins; the remaining axes follow the largest
        batched input's own order so that its reads stay sequential."""
        card = self.card
        out = sorted(out_set)
        big = self.largest(inputs)
        tail = [u for _, u in sorted(zip(big.strides, big.vars)) if u in out_set]
        tail += [u for u in out if u not in big.vars]
        if len(out) < 2:
            return out
        best_key, best = None, None
        for a0 in out:
            t0 = min(int(card[a0]), TILE_EDGE)
            for a1 in out:
                if a1 == a0:
                    continue
                t1 = min(int(card[a1]), TILE_EDGE)
                loads = 0.0
                for f in inputs:
                    n = (t0 if a0 in f.vars else 1) * (t1 if a1 in f.vars else 1)
                    loads += n * (2.0 if f.batched else 1.0)
                key = (loads / (t0 * t1), -(t0 * t1), a0, a1)
                if best_key is None or key < best_key:
                    best_key, best = key, (a0, a1)
        return [best[0], best[1]] + [u for u in tail if u not in best]

    def combine_tables(self, inputs, limit=TILED_MAX_IN):
        """A launch with more than TILED_MAX_IN factors falls off the tiled kernel.  When the
        surplus is small tables, multiply those together first: a table-only product is an
        evidence-independent flat launch (see `emit`), and the big launch then gathers one
        value where it gathered several."""
        inputs = list(inputs)
        if self.mode != MODE_BATCHED or not self.lift_evidence:
            return inputs
        while len(inputs) > limit:
            tabs = [f for f in inputs if not f.batched]
            best = None
            for i in range(len(tabs)):
                for j in range(i + 1, len(tabs)):
                    fa, fb = tabs[i], tabs[j]
                    cols = {(col, c) for f in (fa, fb) for col, _, c in f.ev}
                    sz = self.size(set(fa.vars) | set(fb.vars)) * int(np.prod([c for _, c in cols], dtype=np.int64))
                    n_cols = len({col for col, _ in cols})
                    if sz <= LIFT_MAX and n_cols <= MAX_EV and (best is None or sz < best[0]):
                        best = (sz, fa, fb)
            if best is None:
                break
            _, fa, fb = best
            inputs = [f for f in inputs if f is not fa and f is not fb]
            inputs.append(self.emit([fa, fb], (), sorted(set(fa.vars) | set(fb.vars))))
        return inputs

    def fold(self, inputs):
        """At most max_in factors per launch: bayes_net.py:256 reduces pairwise; multiply the
        smallest max_in together first while there are more."""
        inputs = list(inputs)
        while len(inputs) > self.max_in:
            inputs.sort(key=lambda f: self.size(f.vars))
            head, inputs = inputs[:self.max_in], inputs[self.max_in:]
            inputs.append(self.emit(head, (), self.axis_order(head, set().union(*[f.vars for f in head]))))
        return inputs

    def product_chain(self, inputs, elims, final_vars=None):
        """Multiply `inputs` and sum out `elims` in one launch, after combining and folding the
        surplus factors.  With `final_vars`, a product-only launch over exactly those axes."""
        # a launch that sums out several variables keeps to the preload schedule's 3 inputs
        inputs = self.fold(self.combine_tables(inputs, PRELOAD_MAX_IN if len(elims) > 1 else TILED_MAX_IN))
        union = set().union(*[f.vars for f in inputs])
        if final_vars is not None:
            assert union == set(final_vars), (union, final_vars)
            return self.emit(inputs, (), list(final_vars), may_lift=False)
        return self.emit(inputs, elims, self.axis_order(inputs, union - set(elims)))

    def message(self, inputs, out_vars, elims):
        """sum_{elims} prod(inputs) over out_vars, at most MAX_ELIM variables / MAX_Z joint states per launch:
        the first launch multiplies and sums out the first group, each later one sums out the next group."""
        card = self.card
        groups, cur, z = [], [], 1
        for v in sorted(elims, key=lambda v: (-int(card[v]), v)):
            if cur and (len(cur) >= MAX_ELIM or z * int(card[v]) > MAX_Z):
                groups.append(cur)
                cur, z = [], 1
            cur.append(v)
            z *= int(card[v])
        if cur:
            groups.append(cur)
        inputs = self.fold(self.combine_tables(inputs, PRELOAD_MAX_IN if groups and len(groups[0]) > 1
                                               else TILED_MAX_IN))
        if not groups:
            return self.emit(inputs, (), self.axis_order(inputs, set(out_vars)))
        rest = [v for g in groups for v in g]
        f = None
        for g in groups:
            rest = [v for v in rest if v not in g]
            keep = set(out_vars) | set(rest)
            src = inputs if f is None else [f]
            f = self.emit(src, tuple(g), self.axis_order(src, keep))
        return f

    def finish(self, version, post, Q, query=(), **fields):
        """Assign the slots, build the Plan and serialise it.  `post` is the factor the header's slot
        holds (None for a marginals plan: its readouts write the posterior)."""
        slots, where = _assign_slots(self.steps, keep_unbatched=(self.mode == MODE_BATCHED),
                                     park_batched=(version == VERSION),
                                     preset=[(lid, int(self.card[v])) for v, lid in self.soft])
        plan = Plan(mode=self.mode, query=query, evidence=self.evidence, order=list(self.order), tables=self.tables,
                    slots=slots, steps=self.steps, post_slot=-1 if post is None else where[post.buf], Q=Q,
                    version=version, table_axes=[list(a) for a in self.table_axes],
                    table_scopes=[self.net.scope(v) for v in self.tables], soft=tuple(v for v, _ in self.soft),
                    soft_slots=tuple(where[lid] for _, lid in self.soft), **fields)
        plan._card = self.card
        _serialise(plan, self.table_arrays)
        return plan


def _dense_strides(cards):
    """Element strides of a dense array over `cards`, axis 0 fastest."""
    strides, acc = [], 1
    for c in cards:
        strides.append(acc)
        acc *= c
    return tuple(strides)


def _build(net, version, evidence, query=(), targets=(), mode=MODE_BATCHED, order=None, max_in=MAX_IN,
           lift_evidence=True, fuse_elims=None, merge_sum_outs=None, soft=(), groups=None):
    """A plan of program `version` (VERSION, VERSION_MARGINALS, ...): the upward pass of variable
    elimination, then the kind's tail.  `targets` are kept relevant besides the query and the evidence:
    a marginals plan reads them out, and counts, sample and MPE plans pass every unobserved variable.
    `soft` (sorted by name) adds one batched likelihood factor per variable, read from a slot no step
    writes; it enters the variable's bucket, or the final product of a queried variable.  `groups` (joint plans)
    are the var-id tuples whose joint posteriors the plan reads out."""
    if fuse_elims is None:
        fuse_elims = os.environ.get("SOROBN_B200_FUSE", "1") == "1"
    if len(set(evidence)) != len(evidence):
        raise ValueError("duplicate variable in query or event")
    card = net.card
    for v in evidence:
        if card[v] > 255:
            raise ValueError(f"evidence variable {net.names[v]!r} has {card[v]} states; state codes are uint8")

    # bayes_net.py:763-766
    relevant = {*query, *evidence, *targets, *soft}
    for v in list(relevant):
        relevant |= net.ancestors(v)
    hidden = relevant - set(query) - set(evidence)
    b = _Builder(net, evidence, mode, max_in, lift_evidence, sorted(relevant))
    ev_col = b.ev_col
    if version == VERSION_MAP:
        b.summed = frozenset(hidden - set(targets))  # every relevant unobserved variable that is not MAP

    # bayes_net.py:768-776 -- one factor per relevant CPT; evidence axes become
    # per-row gathers instead of boolean filters
    factors = []
    for t, v in enumerate(b.tables):
        scope = net.scope(v)
        # Shipped layout: free axes first (reference order), evidence axes innermost.  Rows of
        # a warp differ only in their evidence codes, so their gathers of one entry then fall
        # into one 32-byte sector / distinct shared-memory banks instead of `stride` apart.
        perm = [i for i, u in enumerate(scope) if u not in ev_col] + [i for i, u in enumerate(scope) if u in ev_col]
        b.table_arrays.append(np.ascontiguousarray(np.transpose(net.cpt[v], perm)))
        pscope = [scope[i] for i in perm]
        b.table_axes.append(list(pscope))
        shape = [int(card[u]) for u in pscope]
        strides = [int(np.prod(shape[i + 1:], dtype=np.int64)) for i in range(len(shape))]
        free = [(u, s) for u, s in zip(pscope, strides) if u not in ev_col]
        ev = tuple((ev_col[u], s, int(card[u])) for u, s in zip(pscope, strides) if u in ev_col)
        if len(ev) > MAX_EV:
            raise ValueError(f"CPT of {net.names[v]!r} has {len(ev)} evidence axes; the kernel supports {MAX_EV}")
        factors.append(_Factor(False, t, tuple(u for u, _ in free), tuple(s for _, s in free), ev, False))
    ones = []
    if version == VERSION_JOINT:
        # a group whose unobserved members lie in no CPT's scope gets a table of ones over them: elimination then
        # builds a bucket that holds the group, and no value changes
        for g in groups:
            M = tuple(u for u in g if u not in ev_col)
            if len(M) < 2 or M in ones or any(set(M) <= set(net.scope(v)) for v in range(len(net.names))):
                continue
            shape = [int(card[u]) for u in M]
            b.table_arrays.append(np.ones(shape, dtype=np.float64))
            b.table_axes.append(list(M))
            factors.append(_Factor(False, len(b.table_arrays) - 1, M, _dense_strides(shape[::-1])[::-1], (), False))
            ones.append(M)
    # the likelihoods: batched leaf factors over one variable each, under logical ids no step produces
    b.soft = tuple((v, b.next_id + k) for k, v in enumerate(soft))
    b.next_id += len(soft)
    factors += [_Factor(True, lid, (v,), (1,), (), True) for v, lid in b.soft]

    if order is None:
        order = _min_fill_order([f.vars for f in factors], hidden, card, first=b.summed if b.summed else None)
    else:
        order = list(order)
        if set(order) != hidden or len(order) != len(hidden):
            raise ValueError("elimination order must be a permutation of the hidden variables")
        if any(v in b.summed for v in order[len(b.summed):]):
            raise ValueError("a marginal MAP order must eliminate every summed variable before any MAP variable")
    b.order = order

    # bayes_net.py:778-786
    # Fused eliminations.  A later variable w of the order joins x's launch when every factor
    # that mentions w is in x's bucket already, or is a table over variables the bucket covers
    # anyway: sum_w sum_x prod(bucket + those tables).  The joint state space is the one the
    # separate launches walk, but the intermediate over w is never written and read back, and
    # the tile axes are chosen for the launch's real output.
    gone = set()
    buckets = []  # (F_k, eliminated variables, U_k, lambda_k) per launch of the loop below
    for k, x in enumerate(order):
        if x in gone:
            continue
        touching = [f for f in factors if x in f.vars]
        factors = [f for f in factors if x not in f.vars]
        elims = [x]
        if fuse_elims and mode == MODE_BATCHED and any(f.batched for f in touching):
            union = set().union(*[f.vars for f in touching])
            z = int(card[x])
            for w in order[k + 1:]:
                if len(elims) >= MAX_ELIM:
                    break
                if w in gone or w not in union or z * int(card[w]) > MAX_Z or (w in b.summed) != (x in b.summed):
                    continue
                extra = [f for f in factors if w in f.vars]
                if any(f.batched or not set(f.vars) <= union for f in extra):
                    continue
                if extra and len(touching) + len(extra) > TILED_MAX_IN:
                    continue
                touching += extra
                factors = [f for f in factors if w not in f.vars]
                elims.append(w)
                z *= int(card[w])
        gone.update(elims)
        try:
            factors.append(b.product_chain(touching, tuple(elims)))
        except ValueError as e:
            if version != VERSION_MAP:
                raise
            # the constrained order can build factors min-fill alone would not: say where
            raise ValueError(f"the bucket of {[net.names[v] for v in elims]}: {e}") from e
        buckets.append((touching, tuple(elims), set().union(*[f.vars for f in touching]), factors[-1]))

    if version == VERSION_MARGINALS:
        return _marginals_passes(b, buckets, factors, targets)
    if version in (VERSION_COUNTS, VERSION_GRAD):
        return _counts_passes(b, buckets, factors, grad=version == VERSION_GRAD)
    if version == VERSION_JOINT:
        return _counts_passes(b, buckets, factors, groups=groups, ones=tuple(ones))
    if version in (VERSION_SAMPLE, VERSION_MPE, VERSION_MAP):
        return _sample_passes(b, buckets, factors, version)

    # bayes_net.py:788-794: product of what is left; the answer's levels are sorted
    # by name (bayes_net.py:872-873) and rows by state (sort_index, :875)
    q_sorted = tuple(sorted(query, key=lambda v: net.names[v]))
    post = b.product_chain(factors, (), final_vars=tuple(reversed(q_sorted)))
    if merge_sum_outs is None:
        merge_sum_outs = os.environ.get("SOROBN_B200_MERGE", "0") == "1"
    b.steps = _merge_sum_outs(b.steps, merge_sum_outs)
    if mode == MODE_BATCHED:
        if os.environ.get("SOROBN_B200_DFS", "1") == "1":
            b.steps = _depth_first_order(b.steps)
        _relayout_big_tables(b.steps, b.table_arrays, b.table_axes, evidence, card)
    return b.finish(VERSION, post, b.size(post.vars), query=q_sorted)


def _marginals_passes(b, buckets, leftovers, targets):
    """Downward pass and readouts of a marginals plan (DESIGN.md "Marginals of every variable").

    `buckets` are the launches of the upward pass: (F_k, eliminated variables, U_k, lambda_k).
    Bucket j's parent is the bucket whose F contains lambda_j.  The message to a child is
        pi_j(S_j) = sum_{U_p - S_j} pi_p * prod_{f in F_p, f != lambda_j} f,
    and a target t is read from the smallest bucket k with t in U_k:
        M_t(t) = sum_{U_k - {t}} pi_k * prod_{f in F_k} f.
    What is left after the upward pass are per-row scalars (the root buckets' messages and the
    tables of evidence-only variables); a root bucket's pi is the product of the others, so that
    every bucket belief is P(U_k, e) and a row of probability zero stays NaN as in `build_plan`."""
    card, names = b.card, b.net.names
    t_sorted = tuple(sorted(targets, key=lambda v: names[v]))
    read = {t: _smallest_bucket(b, buckets, {t}) for t in t_sorted}
    pi = _downward(b, buckets, leftovers, read.values())
    q = 0
    for t in t_sorted:
        ins, elims, ecards = _bucket_read(b, buckets[read[t]], pi[read[t]], (t,))
        cz = b.size(elims)
        if cz > MARGINAL_MAX_Z or cz * int(card[t]) >= 2**31:
            raise ValueError(f"the bucket read for {names[t]!r} is too large for a readout: {cz} joint "
                             f"states summed out (at most {MARGINAL_MAX_Z}) x {int(card[t])} target states (below 2^31)")
        b.steps.append(Step(KIND_MARGINAL, ins, -1, (t,), (int(card[t]),), elims, ecards, q_offset=q))
        q += int(card[t])
    b.steps = _prune_dead(b.steps)
    return b.finish(VERSION_MARGINALS, None, q, targets=t_sorted)


def _counts_passes(b, buckets, leftovers, grad=False, groups=None, ones=()):
    """Downward pass and count steps of a counts plan (DESIGN.md "Expected counts and EM").

    The unobserved members M_v of v's family are read from the smallest bucket k with M_v in U_k (the
    bucket the CPT of v entered has them all):
        counts_v(M_v; key(row)) += sum_{U_k - M_v} pi_k * prod_{f in F_k} f / P(observed),
    where P(observed) is the product of every leftover scalar of the upward pass, computed once.

    grad=True: a gradient plan (version 10), whose derivative readouts (`_deriv_steps`) follow the count
    steps on the same downward messages.

    groups: a joint plan (version 11): the members M_g of every group g (unobserved, in the group's order) are
    read the same way, each into rows of the output (`_joint_steps`), in place of the count steps."""
    card, names, ev_col = b.card, b.net.names, b.ev_col
    if groups is None:
        members = {v: [u for u in b.net.scope(v) if u not in ev_col] for v in range(len(names))}
    else:
        members = {k: [u for u in g if u not in ev_col] for k, g in enumerate(groups)}
    read = {v: _smallest_bucket(b, buckets, set(M)) for v, M in members.items() if M}
    deriv = _deriv_buckets(b, buckets) if grad else {}
    pi = _downward(b, buckets, leftovers, [*read.values(), *deriv.values()])
    prob = b.emit(b.fold(leftovers), (), [], may_lift=False)
    if groups is not None:
        return _joint_steps(b, buckets, pi, read, members, groups, ones, prob)

    c_offsets, n_counts = count_layout(b.net)
    for v, M in members.items():
        scope = b.net.scope(v)
        shape = [int(card[u]) for u in scope]
        stride = {u: int(np.prod(shape[i + 1:], dtype=np.int64)) for i, u in enumerate(scope)}
        key = tuple((ev_col[u], stride[u], int(card[u])) for u in scope if u in ev_col)
        if len(key) > MAX_EV:
            raise ValueError(f"the family of {names[v]!r} has {len(key)} observed members; the kernel gathers {MAX_EV}")
        if not M:  # fully observed family: a histogram of the rows' keys
            b.steps.append(Step(KIND_COUNT, [], -1, (), (), (), (), q_offset=c_offsets[v], key=key, norm=prob))
            continue
        out_vars = tuple(reversed(M))  # v (count-table stride 1) is the fastest output axis
        ins, elims, ecards = _bucket_read(b, buckets[read[v]], pi[read[v]], out_vars)
        cz, cs = b.size(elims), b.size(out_vars)
        if cz > MARGINAL_MAX_Z or cs > MARGINAL_MAX_Z or cz * cs >= 2**31:
            raise ValueError(f"the bucket read for the family of {names[v]!r} is too large for a count step: "
                             f"{cz} joint states summed out and {cs} family states (each at most "
                             f"{MARGINAL_MAX_Z}, their product below 2^31)")
        b.steps.append(Step(KIND_COUNT, ins, -1, out_vars, tuple(int(card[u]) for u in out_vars), elims, ecards,
                            q_offset=c_offsets[v], key=key, cstrides=tuple(stride[u] for u in out_vars), norm=prob))
    if not grad:
        b.steps = _prune_dead(b.steps)
        return b.finish(VERSION_COUNTS, prob, 1, n_counts=n_counts, count_offsets=c_offsets)
    q = _deriv_steps(b, buckets, pi, deriv, prob)
    b.steps = _prune_dead(b.steps)
    forward = _closure(b.steps, prob.buf)
    return b.finish(VERSION_GRAD, prob, q, n_counts=n_counts, count_offsets=c_offsets, forward_steps=forward)


def _joint_steps(b, buckets, pi, read, members, groups, ones, prob):
    """The readouts of a joint plan, groups in call order: group k's members M (first one fastest) from bucket
    read[k], summed over the rest of the bucket and divided by P(observed), at the next |M| output rows."""
    card, names = b.card, b.net.names
    q, rows = 0, []
    for k, g in enumerate(groups):
        M = tuple(members[k])
        if not M:
            rows.append(-1)
            continue
        ins, elims, ecards = _bucket_read(b, buckets[read[k]], pi[read[k]], M)
        cz, cs = b.size(elims), b.size(M)
        if cz > MARGINAL_MAX_Z or cs > MARGINAL_MAX_Z or cz * cs >= 2**31:
            raise ValueError(f"the bucket read for the group {[names[u] for u in g]} is too large for a joint readout: "
                             f"{cz} joint states summed out and {cs} group states (each at most {MARGINAL_MAX_Z}, "
                             "their product below 2^31)")
        b.steps.append(Step(KIND_JOINT, ins, -1, M, tuple(int(card[u]) for u in M), elims, ecards, q_offset=q,
                            norm=prob))
        rows.append(q)
        q += cs
    b.steps = _prune_dead(b.steps)
    return b.finish(VERSION_JOINT, prob, q, groups=tuple(groups), group_rows=tuple(rows), ones=ones)


def _deriv_buckets(b, buckets):
    """{soft var id: the bucket its likelihood entered}; ValueError for a likelihood that was folded into another
    factor first, which leaves no bucket holding it as an input of its own."""
    out = {}
    for v, lid in b.soft:
        k = next((k for k, (F, _, _, _) in enumerate(buckets) if any(f.is_slot and f.buf == lid for f in F)), None)
        if k is None:
            raise ValueError(f"the likelihood of {b.net.names[v]!r} was folded into another factor before its bucket: "
                             "no derivative readout can leave it out")
        out[v] = k
    return out


def _deriv_steps(b, buckets, pi, deriv, prob):
    """The derivative readouts of a gradient plan, soft variables in likelihood-column order: s is read from the
    bucket its likelihood entered, every input but the likelihood, summed over the rest of the bucket.  Returns
    the rows of the run's output (1 + the likelihood columns)."""
    card, names = b.card, b.net.names
    q = 1
    for v, lid in b.soft:
        k = deriv[v]
        F_k, X, _, lam = buckets[k]
        F = [f for f in F_k if not (f.is_slot and f.buf == lid)]
        U = set().union(*[f.vars for f in F], *([pi[k].vars] if pi[k] is not None else []))
        ins, elims, ecards = _bucket_read(b, (F, X, U, lam), pi[k], (v,))
        cz = b.size(elims)
        if cz > MARGINAL_MAX_Z or cz * int(card[v]) >= 2**31:
            raise ValueError(f"the bucket read for the likelihood of {names[v]!r} is too large for a readout: {cz} "
                             f"joint states summed out (at most {MARGINAL_MAX_Z}) x {int(card[v])} states (below 2^31)")
        b.steps.append(Step(KIND_DERIV, ins, -1, (v,), (int(card[v]),), elims, ecards, q_offset=q, norm=prob))
        q += int(card[v])
    return q


def _closure(steps, lid):
    """Indices of the steps the factor of logical id `lid` depends on, in program order."""
    by_id = {st.out_id: st for st in steps if st.kind in (KIND_FLAT, KIND_BATCHED)}
    need, stack = set(), [lid]
    while stack:
        i = stack.pop()
        if i in need or i not in by_id:  # a likelihood has no producer
            continue
        need.add(i)
        stack.extend(f.buf for f, _, _ in by_id[i].inputs if f.is_slot)
    return tuple(i for i, st in enumerate(steps) if st.kind in (KIND_FLAT, KIND_BATCHED) and st.out_id in need)


def _sample_passes(b, buckets, leftovers, version):
    """Sample steps of a sample plan (DESIGN.md "Posterior samples"), or argmax steps of an MPE plan
    (`version` VERSION_MPE, DESIGN.md "Most probable explanation").

    Bucket k eliminated X_k and sent lambda_k(S_k) to a later bucket.  Walking the buckets in reverse
    elimination order, every variable of S_k has been drawn when bucket k is reached, and
        P(X_k | S_k = drawn, e) is proportional to prod_{f in F_k} f(X_k, S_k = drawn, e).
    P(observed) is the product of the upward pass's leftover scalars, as in a counts plan.  In the log
    domain of an MPE plan the same steps mean max-sum: lambda_k(S_k) = max_{X_k} sum_{f in F_k} log f,
    the leftovers sum to max log P(x, e), and the argmax of sum_{f in F_k} log f(X_k, S_k = decoded, e)
    is X_k's state in the maximising assignment.

    A marginal MAP plan (`version` VERSION_MAP, DESIGN.md "Marginal MAP") decodes its MAP buckets only.  Its
    summed buckets come first in the order, so a MAP bucket's factors, and its separator, hold MAP and
    observed variables alone: the same decode over lambda_k(S_k) = max_{X_k} sum_{f in F_k} log f, where
    the f are CPTs and the log-sum-exp messages of the summed buckets."""
    kind = KIND_SAMPLE if version == VERSION_SAMPLE else KIND_ARGMAX
    card, names = b.card, b.net.names
    n_ev = len(b.evidence)
    decodes = [k for k, (_, X, _, _) in enumerate(buckets) if not (set(X) & b.summed)]
    # the folds (products of the factors beyond max_in) do not depend on the draws: they all run before
    # the sample steps, which then form one contiguous run at the end of the program
    inputs_of = {k: b.fold(buckets[k][0]) for k in decodes}
    prob = b.emit(b.fold(leftovers), (), [], may_lift=False)

    drawn = {}  # var id -> drawn-code row
    for k in reversed(decodes):
        _, X, _, _ = buckets[k]
        for x in X:
            if int(card[x]) > SAMPLE_MAX_CARD:
                raise ValueError(f"{names[x]!r} has {int(card[x])} states; drawn codes are uint8 (at most "
                                 f"{SAMPLE_MAX_CARD} states)")
        cz = b.size(X)
        if cz > MAX_Z:
            raise ValueError(f"the bucket of {[names[x] for x in X]} has {cz} joint states; a sample step draws "
                             f"from at most {MAX_Z}")
        ins = []
        for f in inputs_of[k]:
            pos = dict(zip(f.vars, f.strides))
            terms = tuple(f.ev) + tuple((n_ev + drawn[u], pos[u], int(card[u])) for u in f.vars if u not in X)
            if len(terms) > SAMPLE_MAX_TERMS:
                raise ValueError(f"a factor of the bucket of {[names[x] for x in X]} gathers {len(terms)} observed "
                                 f"or drawn variables; a sample step gathers at most {SAMPLE_MAX_TERMS}")
            g = _Factor(f.is_slot, f.buf, f.vars, f.strides, terms, f.batched)
            ins.append((g, tuple(pos.get(x, 0) for x in X), ()))
        b.steps.append(Step(kind, ins, -1, (), (), tuple(X), tuple(int(card[x]) for x in X),
                            q_offset=len(drawn), norm=prob))
        for x in X:
            drawn[x] = len(drawn)
    return b.finish(version, prob, 1, sampled=tuple(sorted(drawn, key=drawn.get)))


def _smallest_bucket(b, buckets, M):
    """The bucket a step reads the variables `M` from: the smallest whose scope U_k holds them all."""
    return min((b.size(U), k) for k, (_, _, U, _) in enumerate(buckets) if M <= U)[1]


def _bucket_read(b, bucket, pi_k, out_vars):
    """The operands of a step that reads `out_vars` from `bucket` (F_k, X_k, U_k, lambda_k) with
    downward message `pi_k`, summing out U_k - out_vars: (inputs with their (summed-out strides,
    output strides), the summed-out variables, their cards).  The caller checks the sizes."""
    F_k, _, U_k, _ = bucket
    inputs = b.fold(([pi_k] if pi_k is not None else []) + list(F_k))
    # joint states of the summed-out variables are walked first-variable fastest: the variables the
    # largest batched operand lacks go first, so each of its entries is read in one stretch
    big = b.largest(inputs)
    pos_big = dict(zip(big.vars, big.strides))
    elims = tuple(sorted(U_k - set(out_vars), key=lambda v: (v in pos_big, pos_big.get(v, 0), v)))
    ins = []
    for f in inputs:
        pos = dict(zip(f.vars, f.strides))
        ins.append((f, tuple(pos.get(e, 0) for e in elims), tuple(pos.get(u, 0) for u in out_vars)))
    return ins, elims, tuple(int(b.card[e]) for e in elims)


def _downward(b, buckets, leftovers, reads):
    """Downward messages pi_k of the buckets on the way from a root to every bucket in `reads`
    (`_marginals_passes`, `_counts_passes`)."""
    n = len(buckets)
    owner = {id(lam): k for k, (_, _, _, lam) in enumerate(buckets)}
    parent = [None] * n
    for k, (F, _, _, _) in enumerate(buckets):
        for f in F:
            j = owner.get(id(f))
            if j is not None:
                parent[j] = k

    need = [False] * n
    for k in reads:
        while k is not None and not need[k]:
            need[k] = True
            k = parent[k]

    pi = {}
    for k in reversed(range(n)):  # a parent is eliminated after its children
        if not need[k]:
            continue
        lam_k = buckets[k][3]
        if parent[k] is None:
            others = [f for f in leftovers if f is not lam_k]
            pi[k] = b.emit(b.fold(others), (), [], may_lift=False) if others else None
            continue
        p = parent[k]
        F_p, _, U_p, _ = buckets[p]
        inputs = ([pi[p]] if pi[p] is not None else []) + [f for f in F_p if f is not lam_k]
        S_k = set(lam_k.vars)
        pi[k] = b.message(inputs, S_k, U_p - S_k) if inputs else None
    return pi


def _prune_dead(steps):
    """Drop the launches nothing reads (the root buckets' own messages when no other root needs them)."""
    used, keep = set(), []
    for st in reversed(steps):
        if st.kind in (KIND_MARGINAL, KIND_COUNT, KIND_DERIV, KIND_JOINT) or st.out_id in used:
            keep.append(st)
            used.update(f.buf for f, _, _ in st.inputs if f.is_slot)
            if st.norm is not None:
                used.add(st.norm.buf)
    return keep[::-1]


def _relayout_big_tables(steps, table_arrays, table_axes, evidence, card):
    """Lay a big CPT out for its (single) consumer.

    A launch stages its tables in shared memory; a CPT that does not fit (SLICE_MIN_BYTES: the
    engine's 64 KB budget) can still be staged slice by slice when the tiles one CTA walks touch
    a contiguous part of it.  Tiles enumerate the output axes >= 2 (axis 2 fastest), so the table
    is shipped with those axes outermost in the same significance order, then the eliminated
    variables, then the two tile axes, then its evidence axes (innermost, as for every table).
    Every CPT enters exactly one launch, so nobody else sees the new layout."""
    for st in steps:
        if st.kind != KIND_BATCHED:
            continue
        tabs = [k for k, (f, _, _) in enumerate(st.inputs) if not f.is_slot]
        total = sum(table_arrays[st.inputs[k][0].buf].size for k in tabs)
        for f, _, _ in st.inputs:  # tables built by deferred evidence instantiation are staged too
            if f.is_slot and not f.batched:
                total += int(np.prod([card[u] for u in f.vars] + [c for _, _, c in f.ev], dtype=np.int64))
        if total * 4 <= SLICE_MIN_BYTES:
            continue
        rank = {}  # variable -> significance (higher = outer)
        for j, u in enumerate(st.out_vars):
            rank[u] = (0, j) if j < 2 else (2, j)
        for j, u in enumerate(st.elims):
            rank[u] = (1, j)
        for k in tabs:
            f, _, _ = st.inputs[k]
            t = f.buf
            axes = table_axes[t]
            ev_vars = {evidence[col] for col, _, _ in f.ev}
            free = [u for u in axes if u not in ev_vars]
            assert set(free) == set(f.vars) and all(u in rank for u in free)
            new_axes = sorted(free, key=lambda u: rank[u], reverse=True) + [u for u in axes if u in ev_vars]
            if new_axes == axes:
                continue
            table_arrays[t] = np.ascontiguousarray(np.transpose(table_arrays[t], [axes.index(u) for u in new_axes]))
            table_axes[t] = new_axes
            shape = [int(card[u]) for u in new_axes]
            stride = {u: int(np.prod(shape[i + 1:], dtype=np.int64)) for i, u in enumerate(new_axes)}
            col_of = {evidence[col]: col for col, _, _ in f.ev}
            ev = tuple((col_of[u], stride[u], int(card[u])) for u in new_axes if u in ev_vars)
            g = _Factor(False, t, f.vars, tuple(stride[u] for u in f.vars), ev, False)
            st.inputs[k] = (g, tuple(stride.get(e, 0) for e in st.elims), tuple(stride.get(u, 0) for u in st.out_vars))


def _merge_sum_outs(steps, enabled=True):
    """Fold a step whose ONLY input is the output of an earlier step into that step.

    Such a step is a pure sum-out (or, with nothing to eliminate, a re-layout) of a factor
    that was just produced: `sum_j (sum_x prod_i f_i)`.  Summing both variables in the
    producer costs the same multiplies and saves writing the intermediate and reading it
    back (25 KB of the 223 KB per query on the benchmark grid).  Every intermediate is
    consumed exactly once, so the producer's original output is never needed."""
    if not enabled:
        return steps
    merged = []
    producer = {}  # logical id -> index into merged
    for st in steps:
        f0 = st.inputs[0][0]
        if len(st.inputs) == 1 and f0.is_slot and not f0.ev and f0.buf in producer:
            a = merged[producer[f0.buf]]
            z = a.cx * st.cx
            if a.kind == st.kind and len(a.elims) + len(st.elims) <= MAX_ELIM and z <= MAX_Z:
                new_inputs = []
                for f, es, ss in a.inputs:
                    # the producer's own axis -> stride map: its output axes include the evidence
                    # axes a lifted step keeps (those strides come from f.ev, not f.strides)
                    pos = dict(zip(a.out_vars, ss))
                    new_inputs.append((f, es + tuple(pos.get(y, 0) for y in st.elims),
                                       tuple(pos.get(u, 0) for u in st.out_vars)))
                a.inputs = new_inputs
                a.elims = a.elims + st.elims
                a.ecards = a.ecards + st.ecards
                a.out_vars, a.cards = st.out_vars, st.cards
                producer[st.out_id] = producer.pop(f0.buf)
                a.out_id = st.out_id
                continue
        merged.append(st)
        producer[st.out_id] = len(merged) - 1
    return merged


def _depth_first_order(steps):
    """Re-order the launches depth first.

    The steps form a tree (every intermediate has exactly one consumer, the last step produces
    the posterior); the elimination order interleaves its branches.  Executing one branch to the
    end before starting the next keeps the fewest intermediates alive -- the children of a step
    are visited in decreasing (peak - result) order, which is optimal for trees (Sethi-Ullman) --
    so the engine's on-chip segments (csrc/sbn_chain.h) can hold them in shared memory, and a run
    of `frontier <- sum table x frontier` steps becomes contiguous.  Any topological order gives
    the same numbers; slots are assigned afterwards, for THIS order."""
    by_id = {st.out_id: i for i, st in enumerate(steps)}
    children = []
    for st in steps:
        # a likelihood slot (soft evidence) is filled before the steps: no step produces it
        children.append([by_id[f.buf] for f, _, _ in st.inputs if f.is_slot and f.buf in by_id])
    size = [int(np.prod(st.cards, dtype=np.int64)) if st.kind == KIND_BATCHED else 0 for st in steps]
    peak = [0] * len(steps)
    order_of = [None] * len(steps)
    # children always precede their consumer in the incoming list: one forward pass suffices
    for i, st in enumerate(steps):
        kids = sorted(children[i], key=lambda c: (-(peak[c] - size[c]), c))
        # An expanding product (an output several times the size of its siblings' outputs) goes last, so that its
        # consumer follows it immediately: the engine can then run the two as one launch (csrc/sbn_pair.h), and the
        # big intermediate is not held while the other sub-trees are computed.
        if len(kids) > 1 and os.environ.get("SOROBN_B200_BIG_LAST", "1") == "1":
            big = max(kids, key=lambda c: size[c])
            if all(size[big] >= 2 * size[c] for c in kids if c != big):
                kids = [c for c in kids if c != big] + [big]
        held, worst = 0, 0
        for c in kids:
            worst = max(worst, held + peak[c])
            held += size[c]
        peak[i] = max(worst, held + size[i])
        order_of[i] = kids
    out, stack = [], [(len(steps) - 1, 0)]
    seen = set()
    while stack:  # iterative post-order
        node, k = stack.pop()
        if k < len(order_of[node]):
            stack.append((node, k + 1))
            stack.append((order_of[node][k], 0))
        elif node not in seen:
            seen.add(node)
            out.append(steps[node])
    assert len(out) == len(steps), "a step does not feed the posterior"
    return out


def _assign_slots(steps, keep_unbatched, park_batched, preset=()):
    """Physical scratch slots by liveness: an output slot is taken before the step's inputs
    are released (a launch never writes a buffer it reads), best fit among the free slots
    of the same kind, and an intermediate is released after its last consumer.  An
    intermediate of a posterior plan has a single consumer; one of the other kinds may have
    several (the factors of a bucket feed its upward message, its downward messages and its
    readouts).  `Step.norm`, the P(observed) a count, sample or argmax step reads, counts as a
    read.  Steps of kinds 2 to 5 write the posterior, the count table or drawn codes, not a
    slot.  Returns (slots, logical id -> slot).

    keep_unbatched: the evidence-independent tables of a batched program are computed ONCE, when
    the program is created (csrc/sbn_api.cu `run_table_steps`), and then read by every run; their
    slots are never recycled (they are a few KB each).

    park_batched (posterior plans): the batched inputs of a batched step are released one batched
    step LATE.  The engine may run a step and its consumer as ONE launch that reads the first step's
    operand and writes the second step's output (csrc/sbn_pair.h), so those two must never share a
    buffer; it plans such launches for posterior programs only.

    preset: (logical id, size per row) of the batched operands written before step 0 (the likelihoods of soft
    evidence): each takes its own slot first, live until its last reader."""
    remaining = {}  # logical id -> reads still to come
    for st in steps:
        for buf in [f.buf for f, _, _ in st.inputs if f.is_slot] + ([st.norm.buf] if st.norm is not None else []):
            remaining[buf] = remaining.get(buf, 0) + 1
    slots = []  # [batched, size, free]
    where = {}  # logical id -> physical slot
    parked = []

    def alloc(batched, size):
        best = None
        for i, (b, sz, free) in enumerate(slots):
            if free and b == batched and sz >= size and (best is None or sz < slots[best][1]):
                best = i
        if best is None:
            slots.append([batched, size, False])
            return len(slots) - 1
        slots[best][2] = False
        return best

    def release(buf, late):
        remaining[buf] -= 1
        if remaining[buf] == 0:
            phys = where[buf]
            if late and slots[phys][0]:
                parked.append(phys)
            else:
                slots[phys][2] = not (keep_unbatched and not slots[phys][0])

    for lid, size in preset:
        where[lid] = alloc(True, size)
    for st in steps:
        writes_slot = st.kind in (KIND_FLAT, KIND_BATCHED)
        if writes_slot:
            st.out_slot = alloc(st.kind == KIND_BATCHED, int(np.prod(st.cards, dtype=np.int64)) if st.cards else 1)
        late = park_batched and st.kind == KIND_BATCHED
        if late:
            for phys in parked:
                slots[phys][2] = True
            parked.clear()
        new_inputs = []
        for f, es, ss in st.inputs:
            if f.is_slot:
                phys = where[f.buf]
                release(f.buf, late)
                f = _Factor(True, phys, f.vars, f.strides, f.ev, f.batched)
            new_inputs.append((f, es, ss))
        st.inputs = new_inputs
        if st.norm is not None:
            release(st.norm.buf, late)
        if writes_slot:
            where[st.out_id] = st.out_slot
    if not slots:  # every operand is a CPT: the engine still expects one scratch slot
        slots.append([False, 1, True])
    return [(bool(b), int(sz)) for b, sz, _ in slots], where


def _blobs(table_arrays):
    """(float64 table blob, [(offset, size)] per table)."""
    blob = []
    offsets = []
    off = 0
    for arr in table_arrays:
        # plain probabilities: every intermediate entry is then <= 1 and fp32 cannot overflow
        # (DESIGN.md "Precision and fp32 range")
        t = arr.astype(np.float64).reshape(-1)
        pad = (-t.size) % 4  # keep every table 16-byte aligned and sized (bulk-TMA copies)
        offsets.append((off, t.size))
        blob.append(t)
        if pad:
            blob.append(np.zeros(pad, dtype=np.float64))
        off += t.size + pad
    return (np.concatenate(blob) if blob else np.zeros(0, dtype=np.float64)), offsets


def _serialise(plan: Plan, table_arrays):
    # float64 copy: only the CPU checker (oracle/program_interp.py) reads it, to
    # separate planner errors from fp32 rounding; the device gets the fp32 blob
    plan.table_blob64, offsets = _blobs(table_arrays)
    if plan.version in (VERSION_MPE, VERSION_MAP):
        # max-sum and log-sum-exp programs work on logs; a zero entry (and the padding) is -inf
        with np.errstate(divide="ignore"):
            plan.table_blob64 = np.log(plan.table_blob64)
    plan.table_blob = plan.table_blob64.astype(np.float32)
    plan.table_offsets = offsets

    extra = [0, 0]
    if plan.version in (VERSION, VERSION_COUNTS, VERSION_SAMPLE, VERSION_MPE, VERSION_MAP, VERSION_GRAD, VERSION_JOINT):
        post = [plan.post_slot, int(plan.slots[plan.post_slot][0])]
        if plan.version in (VERSION_COUNTS, VERSION_GRAD):
            extra = [plan.n_counts, 0]
        elif plan.version in (VERSION_SAMPLE, VERSION_MPE, VERSION_MAP):
            extra = [len(plan.sampled), 0]
    else:
        post = [-1, 0]  # the readouts write the posterior themselves
    if plan.version in (VERSION, VERSION_MARGINALS):
        extra = [len(plan.soft), 0]
    else:
        extra[1] = len(plan.soft)
    w = [MAGIC, plan.version, plan.mode, len(plan.evidence), len(offsets), len(plan.slots), len(plan.steps),
         plan.Q, *post, *extra]
    assert len(w) == HEADER_WORDS
    for o, s in offsets:
        w += [o, s]
    for b, s in plan.slots:
        w += [int(b), s]
    for v, s in zip(plan.soft, plan.soft_slots):
        w += [s, int(plan._card[v])]
    for st in plan.steps:
        w += [st.kind, len(st.inputs), st.out_slot, len(st.cards), len(st.ecards)]
        if st.kind in (KIND_MARGINAL, KIND_DERIV, KIND_JOINT):
            w.append(st.q_offset)
        elif st.kind == KIND_COUNT:
            w += [st.q_offset, len(st.key)]
            for col, s, c in st.key:
                w += [col, s, c]
            w += list(st.cstrides)
        elif st.kind in (KIND_SAMPLE, KIND_ARGMAX):
            w.append(st.q_offset)
        elif plan.version == VERSION_MAP:
            w.append(st.reduce)
        w += list(st.cards)
        w += list(st.ecards)
        for f, estrides, strides in st.inputs:
            w += [int(f.is_slot), f.buf, int(f.batched), len(f.ev)]
            for col, s, c in f.ev:
                w += [col, s, c]
            w += list(estrides)
            w += list(strides)
    arr = np.asarray(w, dtype=np.int64)
    if arr.max(initial=0) >= 2**31:
        raise ValueError("program word overflows int32")
    plan.words = arr.astype(np.int32)
