"""CPU replay of the device samplers (TEST INFRASTRUCTURE, not product).

The sampler kernels of `sorobn_b200/csrc/sbn_gibbs.cuh` draw every random number from
Philox-4x32-10, which is counter-based, and compare plain IEEE float32 values (the build has no
fast-math and no multiply-add that could contract into an FMA).  So the same stream and the same
float32 operations in numpy give the same output bit for bit:

* `gibbs`: `sbn_gibbs_flat_kernel` and `sbn_gibbs_kernel` (`GibbsSampler.run(..., "gibbs")`);
* `forward(..., "rejection")`: `sbn_forward_kernel`, algo 2;
* `forward(..., "likelihood")`: `sbn_forward_kernel`, algo 1, up to the order in which the
  kernel's atomics add the float64 per-sample likelihoods.

Inputs are a `planner.CompiledNet` and uint8 evidence codes [n_ev, n_rows], as
`engine.GibbsSampler` takes them; the tables are `net.cpt[v]` cast to float32, axes
[*parents, v], as the sampler ships them.  Everything is vectorised over chains (or samples).

`lw_expectation` is the exact expectation of the reference's likelihood-weighting estimator,
which the device estimator converges to.
"""
from __future__ import annotations

import itertools

import numpy as np

__all__ = ["philox4x32", "Stream", "gibbs_weights", "gibbs", "forward", "lw_expectation", "RESCALE_BELOW", "RESCALE_BY"]

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)

# sbn_gibbs_weights: weights whose largest entry falls below 2^-32 after a child's factor are
# multiplied by 2^64 (SBN_GIBBS_TINY, SBN_GIBBS_RESCALE)
RESCALE_BELOW = np.float32(2.0 ** -32)
RESCALE_BY = np.float32(2.0 ** 64)


def philox4x32(ctr, key):
    """Philox-4x32-10 of counter blocks `ctr` (4 uint32 arrays) under `key` (2 uint32), as
    `sbn_philox` computes it.  Returns the four output words."""
    c = [np.asarray(x, dtype=np.uint32).copy() for x in ctr]
    k0, k1 = np.uint32(key[0]), np.uint32(key[1])
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = _M0 * c[0].astype(np.uint64)
            p1 = _M1 * c[2].astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & _LO).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & _LO).astype(np.uint32)
            c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
            k0 = np.uint32(k0 + _W0)
            k1 = np.uint32(k1 + _W1)
    return c


class Stream:
    """`SbnRng` for many chains at once: key = (seed low, seed high), counter block
    [counter, 0, chain low, chain high]; each block's words are used as 3, 2, 1, 0.  Every chain
    draws in lockstep, so the counter is shared."""

    def __init__(self, seed, chains):
        seed = int(seed) & (2**64 - 1)
        chains = np.asarray(chains, dtype=np.uint64)
        self.key = (seed & 0xFFFFFFFF, seed >> 32)
        self.lo = (chains & _LO).astype(np.uint32)
        self.hi = (chains >> np.uint64(32)).astype(np.uint32)
        self.counter = 0
        self.buf = None
        self.have = 0

    def uniform(self):
        """float32 in (0, 1]: ((word >> 8) + 1) * 2^-24, exact."""
        if self.have == 0:
            n = self.lo.shape
            self.buf = philox4x32([np.full(n, self.counter, np.uint32), np.zeros(n, np.uint32), self.lo, self.hi],
                                  self.key)
            self.counter += 1
            self.have = 4
        self.have -= 1
        w = self.buf[self.have]
        return ((w >> np.uint32(8)).astype(np.float32) + np.float32(1.0)) * np.float32(2.0 ** -24)


class _Tables:
    """float32 CPTs of a CompiledNet, flattened, with the stride of each parent in its child's flat table,
    and each variable's children in ascending id order (the order of sbn_gibbs_create's child lists)."""

    def __init__(self, net):
        self.card = [int(c) for c in net.card]
        self.parents = [list(p) for p in net.parents]
        self.flat = [np.ascontiguousarray(np.asarray(t, dtype=np.float32).reshape(-1)) for t in net.cpt]
        self.stride = []
        for v, ps in enumerate(self.parents):
            s, out = self.card[v], []
            for p in reversed(ps):
                out.append(s)
                s *= self.card[p]
            self.stride.append(dict(zip(reversed(ps), out)))
        self.children = [[c for c in range(len(self.card)) if v in self.parents[c]] for v in range(len(self.card))]

    def base(self, v, state, skip=None):
        """Flat offset of v's CPT row for the current parent states (`skip`: a parent left at 0)."""
        b = np.zeros(state.shape[1], dtype=np.int64)
        for p in self.parents[v]:
            if p != skip:
                b += state[p] * self.stride[v][p]
        return b


def _draw(tab, base, u, card):
    """First x with u <= (float32 running sum of the row up to x); card - 1 when there is none."""
    acc = np.zeros(u.shape, dtype=np.float32)
    pick = np.full(u.shape, card - 1, dtype=np.int64)
    open_ = np.ones(u.shape, dtype=bool)
    for x in range(card):
        acc = acc + tab[base + x]
        hit = open_ & (u <= acc)
        pick[hit] = x
        open_ &= ~hit
    return pick


def _clamped(net, evidence, codes):
    return [np.minimum(np.asarray(codes[k], dtype=np.int64), int(net.card[v]) - 1) for k, v in enumerate(evidence)]


def _query_index(tabs, query, state):
    qi = np.zeros(state.shape[1], dtype=np.int64)
    for q in query:
        qi = qi * tabs.card[q] + state[q]
    return qi


def gibbs_weights(tabs, v, state):
    """float32 un-normalised P(v = x | blanket) [card, n], as `sbn_gibbs_weights`: own CPT entry, then
    one factor per child in ascending id order, rescaled by 2^64 whenever the largest weight of a
    chain falls below 2^-32 after a child's factor."""
    c = tabs.card[v]
    base = tabs.base(v, state)
    w = np.stack([tabs.flat[v][base + x] for x in range(c)])
    for ch in tabs.children[v]:
        cb = tabs.base(ch, state, skip=v) + state[ch]
        sv = tabs.stride[ch][v]
        w = w * np.stack([tabs.flat[ch][cb + x * sv] for x in range(c)])
        small = w.max(axis=0) < RESCALE_BELOW
        if small.any():
            w[:, small] *= RESCALE_BY
    return w


def gibbs(net, query, evidence, cycle, codes, n_chains, n_iterations, seed, stats=None):
    """Frequencies [Q, n_chains] float32 of `GibbsSampler.run(codes, n_chains, n_iterations, seed,
    "gibbs")`: chain id = evidence row.  One uniform per non-event variable in id order for the
    initial forward sample (event variables clamped to min(code, card - 1)), then one per update,
    whether the update's conditional is all zero (the chain keeps its value) or not.
    `stats`, a dict, receives "all_zero": the number of such updates over all chains."""
    tabs = _Tables(net)
    n = int(n_chains)
    rng = Stream(seed, np.arange(n, dtype=np.uint64))
    state = np.full((len(tabs.card), n), -1, dtype=np.int64)
    for v, code in zip(evidence, _clamped(net, evidence, codes)):
        state[v] = code
    observed = set(int(v) for v in evidence)
    for v in range(len(tabs.card)):
        if v not in observed:
            state[v] = _draw(tabs.flat[v], tabs.base(v, state), rng.uniform(), tabs.card[v])
    Q = int(np.prod([tabs.card[q] for q in query]))
    counts = np.zeros((Q, n), dtype=np.int64)
    cols = np.arange(n)
    cycle = [int(v) for v in cycle]
    all_zero = 0
    for it in range(int(n_iterations)):
        v = cycle[it % len(cycle)]
        c = tabs.card[v]
        w = gibbs_weights(tabs, v, state)
        cum = np.empty_like(w)
        total = np.zeros(n, dtype=np.float32)
        for x in range(c):
            total = total + w[x]
            cum[x] = total
        u = rng.uniform() * total
        pick = np.minimum((cum < u).sum(axis=0), c - 1)
        state[v] = np.where(total > 0, pick, state[v])
        all_zero += int((total == 0).sum())
        counts[_query_index(tabs, query, state), cols] += 1
    if stats is not None:
        stats["all_zero"] = all_zero
    return counts.astype(np.float32) * (np.float32(1.0) / np.float32(n_iterations))


def forward(net, query, evidence, codes, n_rows, n_iterations, seed, algorithm):
    """Output [Q, n_rows] float32 of `GibbsSampler.run(..., algorithm)` for "likelihood" or
    "rejection".  Sample `it` of row `r` has its own stream, chain id r * n_iterations + it.

    rejection: one uniform per variable; a sample is kept when every event variable drew its code;
    float32 counts over their float32 sum in state order (NaN when nothing is kept).
    likelihood: one uniform per non-event variable, event variables clamped; the sample's weight is
    the float64 product of the float32 CPT entries of every variable in id order; per-state mean
    weight, normalised in float64, rounded to float32 (NaN when every weight is 0)."""
    if algorithm not in ("likelihood", "rejection"):
        raise ValueError(algorithm)
    tabs = _Tables(net)
    n_rows, n_it = int(n_rows), int(n_iterations)
    S = n_rows * n_it
    rng = Stream(seed, np.arange(S, dtype=np.uint64))
    ev = {int(v): np.repeat(code, n_it) for v, code in zip(evidence, _clamped(net, evidence, codes))}
    state = np.zeros((len(tabs.card), S), dtype=np.int64)
    lik = np.ones(S, dtype=np.float64)
    keep = np.ones(S, dtype=bool)
    for v in range(len(tabs.card)):
        base = tabs.base(v, state)
        if algorithm == "likelihood" and v in ev:
            x = ev[v]
        else:
            x = _draw(tabs.flat[v], base, rng.uniform(), tabs.card[v])
            if v in ev:
                keep &= x == ev[v]
        lik *= tabs.flat[v][base + x].astype(np.float64)
        state[v] = x
    Q = int(np.prod([tabs.card[q] for q in query]))
    qi = _query_index(tabs, query, state).reshape(n_rows, n_it)
    out = np.empty((Q, n_rows), dtype=np.float32)
    lik = lik.reshape(n_rows, n_it)
    keep = keep.reshape(n_rows, n_it)
    for r in range(n_rows):
        if algorithm == "rejection":
            cnt = np.bincount(qi[r][keep[r]], minlength=Q).astype(np.float32)
            total = np.float32(0.0)
            for q in range(Q):
                total = np.float32(total + cnt[q])
            out[:, r] = cnt / total if total > 0 else np.nan
        else:
            sums = np.bincount(qi[r], weights=lik[r], minlength=Q)
            cnt = np.bincount(qi[r], minlength=Q)
            mean = np.where(cnt > 0, sums / np.maximum(cnt, 1), 0.0)
            total = 0.0
            for q in range(Q):
                total += mean[q]
            out[:, r] = (mean / total).astype(np.float32) if total > 0 else np.nan
    return out


def lw_expectation(net, query, event):
    """Exact expectation of the reference's likelihood-weighting estimator (bayes_net.py:621-663),
    by enumeration of every joint state (tiny networks only).  Samples are drawn from
    g(s) = prod over non-event variables of P(v | parents) with the event clamped, each is weighted
    by the JOINT probability P(s) (bayes_net.py:546 multiplies over all variables), the per-state
    MEAN weight is taken (:660) and normalised (:661).

    `query`: variable names; `event`: name -> state value.  Returns {tuple of query codes, in
    name order: probability}."""
    names = net.names
    doms = [range(int(c)) for c in net.card]
    qids = sorted((net.index[q] for q in query), key=lambda v: names[v])
    ev = {net.index[k]: net.domains[net.index[k]].index(v) for k, v in event.items()}
    num = {}
    den = {}
    for s in itertools.product(*doms):
        if any(s[v] != x for v, x in ev.items()):
            continue
        joint, g = 1.0, 1.0
        for v in range(len(names)):
            p = net.cpt[v][tuple(s[u] for u in net.parents[v]) + (s[v],)]
            joint *= p
            if v not in ev:
                g *= p
        key = tuple(s[v] for v in qids)
        num[key] = num.get(key, 0.0) + g * joint
        den[key] = den.get(key, 0.0) + g
    means = {k: num[k] / den[k] for k in num if den[k] > 0}
    total = sum(means.values())
    return {k: v / total for k, v in means.items()}
