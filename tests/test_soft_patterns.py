"""Counts, sample, MPE and marginal MAP plans with soft evidence (planner.build_pattern_plan), checked on the CPU.

tests/soft_pattern_interp.py replays the words as the device runs them; the float64 ground truth is the existing
oracles (em_oracle, mpe_oracle, map_oracle) on Pearl's virtual-child network of every row (soft_oracle.virtual),
whose log values gain log_k and whose `__soft__*` families are dropped from the counts."""
import numpy as np
import pytest

import em_oracle
import map_oracle
import mpe_oracle
import soft_oracle
import soft_pattern_interp as spi
from oracle import program_interp
from sorobn_b200 import planner
from test_soft_plan import CORPUS, EXAMPLES, digest, fixed_plans, network, plan_nets

KINDS = ("counts", "sample", "mpe", "map")


def cases(net, seed):
    """(hard evidence, soft, MAP variables) var-id triples: soft only, soft with hard cells, a soft MAP variable."""
    rng = np.random.default_rng(seed)
    n = len(net.names)
    out = []
    for k in range(3):
        perm = [int(v) for v in rng.permutation(n)]
        n_soft = min(1 + k, n - 1)
        soft = tuple(perm[:n_soft])
        rest = perm[n_soft:]
        ev = tuple(rest[1:1 + min(k + 1, max(0, len(rest) - 2))]) if k else ()
        map_vars = (soft[0],) if k == 2 else (rest[0],)
        out.append((ev, soft, map_vars))
    return out


def random_lik(rng, net, soft, n_rows, zeros=True):
    """Likelihoods over 8 orders of magnitude; with `zeros`, some zero entries and row 0 all zeros."""
    n_lik = sum(int(net.card[v]) for v in soft)
    lik = rng.random((n_rows, n_lik)) * 10.0 ** rng.integers(-4, 4, size=(n_rows, 1))
    if zeros:
        lik[rng.random(lik.shape) < 0.1] = 0.0
        lik[0] = 0.0
    return lik


def codes_of(rng, net, evidence, n_rows):
    if not evidence:
        return np.zeros((0, n_rows), dtype=np.uint8)
    return np.stack([rng.integers(0, int(net.card[v]), n_rows) for v in evidence]).astype(np.uint8)


def virtual_rows(net, plan, ev, codes, lik):
    """(virtual network, event with the soft children observed, log_k) of every row; network None: impossible."""
    dn = soft_oracle.dense(net)
    out = []
    for hard, s in soft_oracle.rows(net, ev, codes, plan.soft, lik):
        vnet, event, log_k = soft_oracle.virtual(dn, s)
        out.append((vnet, None if event is None else {**hard, **event}, log_k))
    return out


def oracle_possible(vnet, event):
    from oracle import ve_oracle

    return event is not None and ve_oracle.evidence_probability(vnet, event) > 0


# ----------------------------------------------------------------------------- the words
@pytest.mark.parametrize("kind", KINDS)
def test_soft_section_follows_the_slots_with_its_count_in_word_11(kind):
    net = network("alarm")
    for ev, soft, map_vars in cases(net, 3):
        plan = planner.build_pattern_plan(net, kind, ev, soft=soft, map_vars=map_vars if kind == "map" else None)
        assert plan.soft == tuple(sorted(soft, key=lambda v: net.names[v]))
        assert int(plan.words[11]) == len(soft)
        section, plain = spi.split(plan.words)
        assert section == [(s, int(net.card[v])) for v, s in zip(plan.soft, plan.soft_slots)]
        _, _, slots, steps = program_interp.parse(plain)
        for s, card in section:
            assert slots[s][0] == 1 and slots[s][1] >= card
            reads = [i for i, st in enumerate(steps) if any(inp["is_slot"] and inp["buf"] == s for inp in st["inputs"])]
            writes = [i for i, st in enumerate(steps) if st["kind"] in (0, 1) and st["out_slot"] == s]
            assert reads and (not writes or min(writes) > min(reads))
        if kind in ("sample", "mpe"):
            assert set(plan.soft) <= set(plan.sampled)  # soft variables are drawn / decoded
        if kind == "map":
            assert set(plan.sampled) == set(map_vars)  # and summed out unless MAP variables


def test_without_soft_evidence_the_pattern_plan_is_the_builders_plan():
    """build_pattern_plan(..., soft=()) is byte-equal to the four builders on the plans pinned by
    test_soft_plan.test_plans_without_soft_evidence_keep_their_words."""

    class Pattern:
        def __getattr__(self, name):
            return getattr(planner, name)

        @staticmethod
        def build_counts_plan(net, ev, **kw):
            return planner.build_pattern_plan(net, "counts", ev, **kw)

        @staticmethod
        def build_sample_plan(net, ev):
            return planner.build_pattern_plan(net, "sample", ev)

        @staticmethod
        def build_mpe_plan(net, ev):
            return planner.build_pattern_plan(net, "mpe", ev)

        @staticmethod
        def build_map_plan(net, ev, map_vars):
            return planner.build_pattern_plan(net, "map", ev, map_vars=map_vars)

    nets = plan_nets()
    want = dict((name, (plan.words, digest(plan))) for name, plan in fixed_plans(planner, nets))
    n = 0
    for name, plan in fixed_plans(Pattern(), nets):
        if plan.version in (6, 7, 8, 9):
            assert np.array_equal(plan.words, want[name][0]), name
            assert digest(plan) == want[name][1], name
            n += 1
    assert n > 50


def test_refusals():
    net = network("asia")
    a, b, c = net.index["Smoker"], net.index["Lung cancer"], net.index["Dispnea"]
    with pytest.raises(ValueError, match="hard-evidence"):
        planner.build_pattern_plan(net, "counts", (a,), soft=(a,))
    with pytest.raises(ValueError, match="duplicate"):
        planner.build_pattern_plan(net, "mpe", (), soft=(a, a))
    with pytest.raises(ValueError, match="kind"):
        planner.build_pattern_plan(net, "posterior", (), soft=(a,))
    with pytest.raises(ValueError, match="map_vars"):
        planner.build_pattern_plan(net, "map", (c,), soft=(a,))
    with pytest.raises(ValueError, match="map_vars"):
        planner.build_pattern_plan(net, "mpe", (c,), soft=(a,), map_vars=(b,))
    with pytest.raises(ValueError, match="MAP variable"):
        planner.build_pattern_plan(net, "map", (c,), soft=(a,), map_vars=(c,))
    # without soft evidence a MAP plan that computes nothing is still refused; with it, it has log P(e, lik)
    with pytest.raises(ValueError, match="nothing to compute"):
        planner.build_pattern_plan(net, "map", (), map_vars=())
    plan = planner.build_pattern_plan(net, "map", (), soft=(a,), map_vars=())
    assert plan.sampled == () and plan.soft == (a,)
    # the replay takes likelihoods for a soft program only
    plain = planner.build_mpe_plan(net, (c,))
    with pytest.raises(AssertionError):
        spi.run_mpe(plain.words, plain.table_blob, np.zeros((1, 1), np.uint8), np.ones((1, 2)), n_rows=1)


# ----------------------------------------------------------------------------- against the float64 oracles
@pytest.mark.parametrize("name", EXAMPLES + CORPUS[:3])
def test_counts_match_the_virtual_evidence_oracle(name):
    net = network(name)
    rng = np.random.default_rng(5)
    offsets, _ = planner.count_layout(net)
    for ev, soft, _ in cases(net, 9):
        plan = planner.build_pattern_plan(net, "counts", ev, soft=soft)
        B = 4
        codes, lik = codes_of(rng, net, ev, B), random_lik(rng, net, plan.soft, B)
        for b, (vnet, event, log_k) in enumerate(virtual_rows(net, plan, ev, codes, lik)):
            counts, prob, log_ev = spi.run_counts(plan.words, plan.table_blob64, codes[:, b:b + 1], lik[b:b + 1])
            if not oracle_possible(vnet, event):
                assert np.isnan(prob[0]) and not counts.any(), (name, b)
                continue
            want = em_oracle.expected_counts(vnet, [event])
            for v, node in enumerate(net.names):
                got = counts[offsets[v]:offsets[v] + net.cpt[v].size].reshape(net.cpt[v].shape)
                np.testing.assert_allclose(got, want[node], rtol=1e-9, atol=1e-12)
            le = em_oracle.log_likelihood(vnet, [event]) + log_k
            assert abs(log_ev[0] - le) <= 1e-9 * max(1.0, abs(le)), (name, b, log_ev[0], le)


@pytest.mark.parametrize("name", EXAMPLES + CORPUS[:3])
def test_mpe_matches_the_virtual_evidence_oracle(name):
    net = network(name)
    rng = np.random.default_rng(6)
    for ev, soft, _ in cases(net, 10):
        plan = planner.build_pattern_plan(net, "mpe", ev, soft=soft)
        B = 5
        codes, lik = codes_of(rng, net, ev, B), random_lik(rng, net, plan.soft, B)
        decoded, lp = spi.run_mpe(plan.words, plan.table_blob64, codes, lik, n_rows=B, dtype=np.float64)
        for b, (vnet, event, log_k) in enumerate(virtual_rows(net, plan, ev, codes, lik)):
            if not oracle_possible(vnet, event):
                assert lp[b] == -np.inf, (name, b)
                continue
            try:
                x, L = mpe_oracle.brute_force(vnet, event)
            except ValueError:  # too many joint states to enumerate
                x, L = mpe_oracle.max_sum(vnet, event)
            L += log_k
            assert abs(lp[b] - L) <= 1e-9 * max(1.0, abs(L)), (name, b, lp[b], L)
            got = {net.names[v]: net.domains[v][int(decoded[j, b])] for j, v in enumerate(plan.sampled)}
            # ties aside the codes are the oracle's: the decoded state must reach the maximum
            assert abs(mpe_oracle.log_joint(vnet, {**event, **got}) + log_k - L) <= 1e-9 * max(1.0, abs(L))


@pytest.mark.parametrize("name", EXAMPLES + CORPUS[:3])
def test_map_matches_the_virtual_evidence_oracle(name):
    net = network(name)
    rng = np.random.default_rng(7)
    for ev, soft, map_vars in cases(net, 12):
        plan = planner.build_pattern_plan(net, "map", ev, soft=soft, map_vars=map_vars)
        B = 5
        codes, lik = codes_of(rng, net, ev, B), random_lik(rng, net, plan.soft, B)
        decoded, lp = spi.run_mpe(plan.words, plan.table_blob64, codes, lik, n_rows=B, dtype=np.float64)
        names = [net.names[v] for v in map_vars]
        for b, (vnet, event, log_k) in enumerate(virtual_rows(net, plan, ev, codes, lik)):
            if not oracle_possible(vnet, event):
                assert lp[b] == -np.inf, (name, b)
                continue
            x, L, gap = map_oracle.solve(vnet, event, names)
            L += log_k
            assert abs(lp[b] - L) <= 1e-9 * max(1.0, abs(L)), (name, b, lp[b], L)
            got = {net.names[v]: net.domains[v][int(decoded[j, b])] for j, v in enumerate(plan.sampled)}
            if gap > 1e-9:
                assert got == x, (name, b)
            else:
                assert abs(map_oracle.log_prob(vnet, event, got) + log_k - L) <= 1e-9 * max(1.0, abs(L))


@pytest.mark.parametrize("name", ["asia", "sprinkler", "grades"])
def test_sample_draws_follow_the_exact_posterior(name):
    """The replay's draws of every unobserved variable, soft ones included, against the virtual-evidence
    posterior: within 5 standard errors for 4,000 draws of each of two rows."""
    net = network(name)
    rng = np.random.default_rng(8)
    dn = soft_oracle.dense(net)
    for ev, soft, _ in cases(net, 13)[:2]:
        plan = planner.build_pattern_plan(net, "sample", ev, soft=soft)
        B, D = 2, 4000
        codes, lik = codes_of(rng, net, ev, B), random_lik(rng, net, plan.soft, B, zeros=False)
        drawn, prob, _, log_ev = spi.run_sample(plan.words, plan.table_blob64, codes, lik, n_rows=B, n_draws=D,
                                                seed=11)
        for b, (hard, s) in enumerate(soft_oracle.rows(net, ev, codes, plan.soft, lik)):
            assert abs(log_ev[b] - soft_oracle.log_evidence(dn, hard, s)) <= 1e-9 * max(1.0, abs(log_ev[b]))
            for j, v in enumerate(plan.sampled):
                want = soft_oracle.posterior(dn, [net.names[v]], hard, s)
                freq = np.bincount(drawn[j, :, b], minlength=int(net.card[v])) / D
                se = np.sqrt(want * (1 - want) / D) + 1e-12
                assert (np.abs(freq - want) <= 5 * se + 1e-3).all(), (name, b, net.names[v], freq, want)


# ----------------------------------------------------------------------------- one-hot, all-ones and scale
@pytest.mark.parametrize("kind", KINDS)
def test_one_hot_is_hard_evidence_all_ones_is_nothing_and_scale_shifts_only_the_log(kind):
    net = network("alarm")
    soft_v, other = net.index["Alarm"], net.index["John calls"]
    mv = (net.index["Burglary"],)
    B = 6
    rng = np.random.default_rng(4)
    card = int(net.card[soft_v])
    hot = rng.integers(0, card, B).astype(np.uint8)
    obs = rng.integers(0, int(net.card[other]), B).astype(np.uint8)[None, :]
    extra = dict(map_vars=mv) if kind == "map" else {}
    soft = planner.build_pattern_plan(net, kind, (other,), soft=(soft_v,), **extra)
    ev = tuple(sorted((other, soft_v)))
    hard = planner.build_pattern_plan(net, kind, ev, **extra)
    none = planner.build_pattern_plan(net, kind, (other,), **extra)
    hard_codes = np.stack([obs[0] if v == other else hot for v in ev])
    onehot, ones = np.eye(card)[hot] * 0.25, np.ones((B, card))
    scaled = rng.random((B, card)) + 0.1
    c = 7.5
    if kind == "counts":
        got = spi.run_counts(soft.words, soft.table_blob64, obs, onehot, n_rows=B)
        want = program_interp.run_counts(hard.words, hard.table_blob64, hard_codes, n_rows=B)
        np.testing.assert_allclose(got[0], want[0], rtol=1e-12)
        np.testing.assert_allclose(got[2], np.log(want[1]) + np.log(0.25), rtol=1e-12)
        got = spi.run_counts(soft.words, soft.table_blob64, obs, ones, n_rows=B)
        want = program_interp.run_counts(none.words, none.table_blob64, obs, n_rows=B)
        np.testing.assert_allclose(got[0], want[0], rtol=1e-12)
        a = spi.run_counts(soft.words, soft.table_blob64, obs, scaled, n_rows=B)
        z = spi.run_counts(soft.words, soft.table_blob64, obs, scaled * c, n_rows=B)
        np.testing.assert_allclose(a[0], z[0], rtol=1e-12)
        np.testing.assert_allclose(z[2] - a[2], np.log(c), rtol=1e-9)
    elif kind == "sample":
        # the soft variable is drawn, and one-hot pins it; P(observed) is the hard plan's
        got, prob, _, _ = spi.run_sample(soft.words, soft.table_blob64, obs, onehot, n_rows=B, n_draws=3, seed=5)
        _, want, _ = program_interp.run_sample(hard.words, hard.table_blob64, hard_codes, n_rows=B, n_draws=3, seed=5)
        assert (got[soft.sampled.index(soft_v)] == hot[None, :]).all()
        np.testing.assert_allclose(prob, want, rtol=1e-12)
        conds_soft = spi.run_sample(soft.words, soft.table_blob64, obs, ones, n_rows=B, n_draws=3, seed=5)
        conds_none = program_interp.run_sample(none.words, none.table_blob64, obs, n_rows=B, n_draws=3, seed=5)
        np.testing.assert_allclose(conds_soft[1], conds_none[1], rtol=1e-12)
        a = spi.run_sample(soft.words, soft.table_blob64, obs, scaled, n_rows=B, n_draws=3, seed=5)
        z = spi.run_sample(soft.words, soft.table_blob64, obs, scaled * c, n_rows=B, n_draws=3, seed=5)
        assert (a[0] == z[0]).all()
        np.testing.assert_allclose(z[3] - a[3], np.log(c), rtol=1e-9)
    else:
        got, lp = spi.run_mpe(soft.words, soft.table_blob64, obs, onehot, n_rows=B, dtype=np.float64)
        want, wlp = program_interp.run_mpe(hard.words, hard.table_blob64, hard_codes, n_rows=B, dtype=np.float64)
        hard_row = {v: j for j, v in enumerate(hard.sampled)}
        for j, v in enumerate(soft.sampled):
            assert (got[j] == (hot if v == soft_v else want[hard_row[v]])).all(), net.names[v]
        np.testing.assert_allclose(lp, wlp + np.log(0.25), rtol=1e-12)
        got, lp = spi.run_mpe(soft.words, soft.table_blob64, obs, ones, n_rows=B, dtype=np.float64)
        want, wlp = program_interp.run_mpe(none.words, none.table_blob64, obs, n_rows=B, dtype=np.float64)
        assert (got == want).all()
        np.testing.assert_allclose(lp, wlp, rtol=1e-12)
        a = spi.run_mpe(soft.words, soft.table_blob64, obs, scaled, n_rows=B, dtype=np.float64)
        z = spi.run_mpe(soft.words, soft.table_blob64, obs, scaled * c, n_rows=B, dtype=np.float64)
        assert (a[0] == z[0]).all()
        np.testing.assert_allclose(z[1] - a[1], np.log(c), rtol=1e-9)
