"""Loopy belief propagation: (network, evidence variables, targets) -> a compiled factor graph.

Every exact program kind eliminates variables, so its cost grows with the induced width of the network; past
a width of about 20 the planner refuses the network.  Loopy belief propagation (sum-product message passing on
the factor graph of the CPT families) costs what the families cost, is deterministic, gives every marginal at
once, and is exact on polytrees.  The device runs one evidence row per thread through every sweep in one launch
(csrc/sbn_bp.cu); `tests/bp_interp.py` replays the same words on the CPU, and `tests/bp_oracle.py` restates the
algorithm below in float64 from the dense network, without these words.

Semantics (every implementation follows them exactly)
-----------------------------------------------------
Factor graph.  The relevant subnetwork is the targets, the evidence variables and all their ancestors (the set
the exact planner keeps).  There is one factor per relevant CPT, its hard-evidence axes indexed by the row's
codes; a factor whose members are all observed is dropped.  The variable nodes are the unobserved relevant
variables.  (A barren node would send exactly uniform messages, so pruning it changes no message.)

Messages.  Every message is normalised to sum 1.  Variable-to-factor messages nu start uniform; factor-to-variable
messages mu start uniform too, and are the "old" messages of the first damping step.

One sweep (synchronous flooding), with damping lambda in [0, 1):
  1. for every factor f and unobserved member v:
         mu'_{f->v}(x) = sum_{x_f \\ v} f(x_f, e) prod_{u != v} nu_{u->f}(x_u), normalised,
         mu_{f->v} = (1 - lambda) mu' + lambda mu_old;
  2. for every variable v and factor f containing v: nu_{v->f} = prod_{g ∋ v, g != f} mu_{g->v}, normalised
     (no damping; a variable with one factor sends the uniform message);
  3. the residual r is the largest |mu_{f->v}(x) - mu_old(x)| over every message and state of the row.  The row
     has converged at sweep t when r < tol: it stops, its beliefs b_v = prod_{f ∋ v} mu_{f->v} (normalised) are
     taken from that sweep's messages, and it records t;
  4. after `n_iterations` sweeps a row that has not converged returns the beliefs of its last sweep and records
     n_iterations + 1.  tol = 0 therefore runs exactly n_iterations sweeps.

Zeros.  A mu' (before damping), nu or belief whose sum is 0 makes the row NaN: the row stops at that sweep and
records it (a belief is formed after the last sweep).  On polytrees this is exactly impossible evidence, as in the
exact path.  On loopy graphs BP need not detect impossible evidence: a row of probability zero may converge to
finite beliefs.

Underflow.  A product of many messages (a variable with 50 children) can underflow.  The running product of nu
and of a belief is formed in double and rescaled as `sbn_gibbs.cuh` rescales the Gibbs weights: after each factor,
a product whose largest entry fell below 2^-32 is multiplied by 2^64.  A power of two changes no ratio, so this is
invisible after normalisation wherever nothing underflowed.  Double keeps the smaller states too: with many
disagreeing neighbours a state can fall more than 2^126 below the largest on the way, past float32's range.  Every
normalisation divides by the sum (a subnormal sum still gives finite ratios).

Max-product (the most probable explanation; `compile_mpe_graph`, `BayesNet.mpe_many(algorithm="bp")`)
--------------------------------------------------------------------------------------------------
Factor graph.  Every unobserved node is a variable and nothing is pruned: in max-product a barren leaf sends
max_x P(x | pa), which depends on its parents (P(A=0) = 0.6, B | A=0 = (0.5, 0.5), B | A=1 = (0.9, 0.1): the MPE
is A=1, B=0 at 0.36 > 0.30, and without B the decode would give A=0).  There is one factor per CPT of the
network, its evidence axes indexed by the row's codes; a factor whose members are all observed is kept with 0
members: the sweep skips it and the score reads it.  Before the first sweep, a 0-member factor whose entry at the
row's codes is 0 makes the row dead (its observed cells are impossible, and no message would show it): it runs no
sweep and records 0.

Sweep.  The sweep above, except that step 1 maximises:
    mu'_{f->v}(x) = max_{x_f \\ v} f(x_f, e) prod_{u != v} nu_{u->f}(x_u)   (the max starting at 0),
then normalised to sum 1 and damped as in sum-product.  Step 2, the residual, tol, the n_iterations + 1 record, the
zero rule and the double products with their rescale are unchanged.

Decode.  After the row's last sweep, each variable's belief product prod_{f ∋ v} mu_{f->v} is formed in double (as
the beliefs above, before normalisation); its code is the first state with the largest product (x walked upwards,
strict >).  A belief that sums to 0 makes the row dead.

Score.  log P(x̂, e) = sum over every factor, 0-member ones included, of log(double(table entry at x̂ and the row's
codes)), in double.  It may be -inf for a live row: the per-variable decode can combine tied states of different
maximisers (even on a polytree: A uniform and B = not A decode A=0, B=0), and loopy messages are approximate.  A
dead row reports NaN and codes 0.  A pattern that observes every node has 0 variables and 0 edges: it runs no sweep,
records 0 and returns only its score.

Expected counts (the E-step of EM; `compile_counts_graph`, `BayesNet.expected_counts(algorithm="bp")`)
-------------------------------------------------------------------------------------------------------
Factor graph.  The max-product graph: every CPT is a factor, with nothing pruned, because every family needs counts;
every unobserved node is a variable; a family whose members are all observed is kept with 0 members.  (In
sum-product a barren unobserved node sends uniform messages, so keeping it changes no other belief; its family gets
P(v | pa) b(pa).)

Sweep.  The sum-product sweep above, unchanged: damping, residual, tol, the n_iterations + 1 record, the zero rule and
the double products with their 2^64 rescale.  As in max-product, a row whose codes hit a 0 entry of a 0-member factor
is dead before the first sweep: it runs no sweep and records 0, and so does a pattern that observes every node.

Family beliefs.  After the row's last sweep, for every factor f with at least one member,
    b_f(x_f) ∝ f(x_f, e) prod_{v ∈ f} nu_{v->f}(x_v),
formed in double from the last sweep's nu and normalised over the configurations of the unobserved members.  A
0-member factor has belief 1 at the row's codes.  A belief that sums to 0 makes the row dead.

Variable beliefs.  b_v is the normalised product of v's mu (the sum-product belief), formed in double.

Bethe log-likelihood of a row, in double with 0 log 0 = 0:
    log Z_B = sum_f sum_{x_f} b_f (log f - log b_f) + sum_v (d_v - 1) sum_x b_v log b_v,
d_v being the number of factors v is an unobserved member of; each 0-member factor adds log f(e).  On a polytree at
BP's fixed point it equals log P(e) exactly; on a pattern that observes every node it is log P(row).  (The device
and the replay sum each factor's terms as H / S + log S, with p = f prod nu, S = sum p and H = sum p (log f - log p),
which is the same number up to rounding.)

Expected counts.  Each live row adds its b_f into the count entry of (x_f, the row's evidence codes).  A dead row adds
nothing, and its log Z_B is NaN.  The device adds the rows without floating-point atomics, so two runs are bitwise
equal.

Words (int32; `sbn_bp_create` bounds-checks every one)
------------------------------------------------------
    header : MAGIC 1 n_ev n_factors n_vars E n_targets Q n_table_floats fac_pos var_pos tgt_pos
    factor : family var | table offset | n_mem | n_evax | n_mem x (card, stride, edge) | n_evax x (col, stride, card)
    var    : var id | card | degree | degree x edge
    target : position of its var record | q_offset

An *edge* (f, v) owns `card(v)` consecutive entries of each direction of the per-row message state: mu_{f->v}
at entries [edge, edge + card) and nu_{v->f} at [E + edge, E + edge + card); 2 E floats per row in all.  A factor's
table in the blob has its unobserved members innermost, dense, member 0 fastest (member i at `stride`), and its
evidence axes outside them: the entry of a row is table offset + sum_k min(code_k, card_k - 1) * stride_k +
sum_i x_i * stride_i.  Factors follow the variable order (topological), members the CPT's axis order [*parents, v],
variables their ids; targets are sorted by name, each at rows q_offset .. q_offset + card of the output.

Version 2 (max-product) has the same layout, with three differences: a factor record may have n_mem = 0; n_vars
and E may be 0; the target section lists every variable record in variable order, with q_offset = its position,
its row of the codes output (Q = n_vars).  Version 3 (expected counts) has the version-2 layout and rules.  Every
factor's blob is its full CPT transposed, evidence axes included, so the blob is a permutation of the dense CPTs
concatenated in `planner.count_layout` order: `Graph.perm` gives it (tables64 == concat(cpt).reshape(-1)[perm]).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

MAGIC = 0x53424250  # "SBBP"
VERSION = 1  # sum-product (compile_graph)
VERSION_MPE = 2  # max-product (compile_mpe_graph)
VERSION_COUNTS = 3  # expected counts (compile_counts_graph)
HEADER_WORDS = 12
MAX_CARD = 256  # states of an unobserved variable (the kernel's widest message)


@dataclass
class Graph:
    words: np.ndarray  # int32
    tables: np.ndarray  # float32 blob (tables64: the same in float64)
    tables64: np.ndarray
    families: tuple  # var id of each factor's CPT, factor order
    variables: tuple  # unobserved relevant var ids, variable order
    targets: tuple  # var ids, output order
    q_offsets: tuple
    Q: int
    n_edges: int  # E: entries of one direction of the message state per row
    perm: np.ndarray | None = None  # version 3: int64, tables64 == concat of the dense CPTs, flattened, [perm]

    def message_bytes_per_sweep(self) -> int:
        """Bytes of message state one sweep of one row accesses in the device scratch, as csrc/sbn_bp.cu walks
        it: step 1 reads, for each member of a factor and each configuration of the other members, their nu, then
        reads and writes the member's mu; step 2 reads degree - 1 mu per nu it writes.  Tables and words come
        from shared memory and are not counted; repeated reads of one entry may hit the caches."""
        w = self.words
        fac_pos, var_pos = int(w[9]), int(w[10])
        n_fac, n_var = int(w[3]), int(w[4])
        floats = 0
        p = fac_pos
        for _ in range(n_fac):
            n_mem, n_evax = int(w[p + 2]), int(w[p + 3])
            cards = [int(w[p + 4 + 3 * i]) for i in range(n_mem)]
            T = int(np.prod(cards))
            for c in cards:
                # T / c configurations of the other members, each reading their nu; then mu read and written
                floats += (T // c) * (n_mem - 1) + 2 * c
            p += 4 + 3 * n_mem + 3 * n_evax
        p = var_pos
        for _ in range(n_var):
            c, deg = int(w[p + 1]), int(w[p + 2])
            floats += deg * (max(deg - 1, 0) * c + c)
            p += 3 + deg
        return 4 * floats


def relevant_set(net, evidence, targets):
    """Targets, evidence and all their ancestors (planner._build's relevant set)."""
    relevant = {*targets, *evidence}
    for v in list(relevant):
        relevant |= net.ancestors(v)
    return relevant


def compile_graph(net, evidence, targets) -> Graph:
    """The factor graph of `net` (planner.CompiledNet) given the evidence var ids (the columns of the codes, in
    order) and the target var ids, as words and a table blob (module docstring)."""
    evidence, targets = [int(e) for e in evidence], [int(t) for t in targets]
    if not targets:
        raise ValueError("at least one target is needed")
    if set(targets) & set(evidence):
        raise ValueError("a target cannot be an evidence variable")
    return _compile(net, evidence, relevant_set(net, evidence, targets), targets, VERSION)


def compile_mpe_graph(net, evidence) -> Graph:
    """The max-product factor graph of `net` given the evidence var ids (module docstring, "Max-product"): every
    CPT a factor, every unobserved node a variable and a target, as version-2 words and a table blob."""
    evidence = [int(e) for e in evidence]
    observed = set(evidence)
    variables = [v for v in range(len(net.names)) if v not in observed]
    return _compile(net, evidence, set(range(len(net.names))), variables, VERSION_MPE)


def compile_counts_graph(net, evidence) -> Graph:
    """The expected-counts factor graph of `net` given the evidence var ids (module docstring, "Expected counts"):
    the graph of `compile_mpe_graph` as version-3 words, with `perm` set."""
    evidence = [int(e) for e in evidence]
    observed = set(evidence)
    variables = [v for v in range(len(net.names)) if v not in observed]
    return _compile(net, evidence, set(range(len(net.names))), variables, VERSION_COUNTS)


def _compile(net, evidence, relevant, targets, version) -> Graph:
    """Words and blob of the factors of the `relevant` CPTs (version 1 drops those with every member observed);
    version 1 targets are sorted by name and span their cards, version 2 targets are every variable in order."""
    if len(set(evidence)) != len(evidence):
        raise ValueError("duplicate evidence variable")
    card = [int(c) for c in net.card]
    for v in evidence:
        if card[v] > 255:
            raise ValueError(f"evidence variable {net.names[v]!r} has {card[v]} states; state codes are uint8")
    ev_col = {v: k for k, v in enumerate(evidence)}
    variables = [v for v in sorted(relevant) if v not in ev_col]
    for v in variables:
        if card[v] > MAX_CARD:
            raise ValueError(f"{net.names[v]!r} has {card[v]} states; belief propagation takes at most {MAX_CARD}")

    fac_words, blobs, families, perms = [], [], [], []
    if version == VERSION_COUNTS:
        from .planner import count_layout

        first = count_layout(net)[0]
    edges_of = {v: [] for v in variables}
    E = 0
    off = 0
    for v in sorted(relevant):
        scope = list(net.scope(v))
        members = [u for u in scope if u not in ev_col]
        if not members and version == VERSION:
            continue
        evax = [u for u in scope if u in ev_col]
        T = int(np.prod([card[u] for u in members]))
        # blob axes, slowest first: evidence axes (last first), then members (last first): member 0 fastest
        order = list(reversed(evax)) + list(reversed(members))
        arr = np.transpose(np.asarray(net.cpt[v], dtype=np.float64), [scope.index(u) for u in order])
        blobs.append(np.ascontiguousarray(arr).reshape(-1))
        if version == VERSION_COUNTS:
            flat = first[v] + np.arange(arr.size, dtype=np.int64).reshape(np.shape(net.cpt[v]))
            perms.append(np.transpose(flat, [scope.index(u) for u in order]).reshape(-1))
        rec = [v, off, len(members), len(evax)]
        stride = 1
        for u in members:
            rec += [card[u], stride, E]
            edges_of[u].append(E)
            stride *= card[u]
            E += card[u]
        for u in evax:
            rec += [ev_col[u], stride, card[u]]
            stride *= card[u]
        fac_words.append(rec)
        families.append(v)
        off += stride
    var_words, var_rel = [], {}
    pos = 0
    for v in variables:
        var_rel[v] = pos
        rec = [v, card[v], len(edges_of[v]), *edges_of[v]]
        var_words.append(rec)
        pos += len(rec)
    if version == VERSION:
        names = {t: net.names[t] for t in targets}
        targets = sorted(set(targets), key=lambda t: names[t])
    q_offsets, Q = [], 0
    for t in targets:
        q_offsets.append(Q)
        Q += card[t] if version == VERSION else 1

    fac_flat = [w for rec in fac_words for w in rec]
    var_flat = [w for rec in var_words for w in rec]
    fac_pos = HEADER_WORDS
    var_pos = fac_pos + len(fac_flat)
    tgt_pos = var_pos + len(var_flat)
    tgt_flat = []
    for t, q in zip(targets, q_offsets):
        tgt_flat += [var_pos + var_rel[t], q]
    tables64 = np.concatenate(blobs) if blobs else np.zeros(0)
    header = [MAGIC, version, len(evidence), len(fac_words), len(variables), E, len(targets), Q, tables64.size,
              fac_pos, var_pos, tgt_pos]
    words = np.asarray(header + fac_flat + var_flat + tgt_flat, dtype=np.int64)
    if words.max(initial=0) >= 2**31 or tables64.size >= 2**31:
        raise ValueError("the factor graph does not fit 32-bit words")
    perm = (np.concatenate(perms) if perms else np.zeros(0, dtype=np.int64)) if version == VERSION_COUNTS else None
    return Graph(words.astype(np.int32), tables64.astype(np.float32), tables64, tuple(families), tuple(variables),
                 tuple(targets), tuple(q_offsets), Q, E, perm)


def check_arguments(n_iterations, damping, tol):
    """ValueError unless n_iterations >= 1, 0 <= damping < 1 and tol >= 0 (all finite)."""
    if isinstance(n_iterations, bool) or int(n_iterations) != n_iterations or n_iterations < 1 or n_iterations >= 2**31 - 1:
        raise ValueError(f"n_iterations must be a positive integer, not {n_iterations!r}")
    if not (np.isfinite(damping) and 0.0 <= damping < 1.0):
        raise ValueError(f"damping must be in [0, 1), not {damping!r}")
    if not (np.isfinite(tol) and tol >= 0.0):
        raise ValueError(f"tol must be finite and >= 0, not {tol!r}")
