"""Soft-evidence plans (planner `soft=`, likelihood slots of versions 4 and 5), checked on the CPU.

tests/soft_oracle.py answers in float64 without the planner (Pearl's virtual-evidence children on the dense
oracle); tests/soft_interp.py fills the likelihood slots as the device's pack does and oracle/program_interp.py
executes the serialised words
the device's pack fills.  Plans without soft evidence must keep their words: they are hashed against the
words the planner wrote before soft evidence existed (tests/golden/plan_words_parent.json)."""
import hashlib
import json
import os

import numpy as np
import pytest

import kernel_corpus
import soft_interp
import soft_oracle
from oracle import program_interp
from sorobn_b200 import examples, planner, workloads

EXAMPLES = ["alarm", "asia", "sprinkler", "grades"]
CORPUS = ["dag9p2s4x1x4x4_seed54_q1-8_e2", "dag14p4s5x8_seed1_zeros_q10-13_e1", "dag16p4s8_seed0_q15_e2",
          "grid7x7s5_seed39_q48_e18", "dag19p7s3_seed93_q12_e3"]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def network(name):
    if name in EXAMPLES:
        return getattr(examples, name)()._compiled
    case = next(c for c in kernel_corpus.CASES if c["name"] == name)
    return kernel_corpus.compiled_net(kernel_corpus.make_spec(case))


def random_lik(rng, net, soft, n_rows):
    """Likelihoods [n_rows, sum of cards] over 12 orders of magnitude, with zeros; row 0 all zeros (impossible)."""
    n_lik = sum(int(net.card[v]) for v in soft)
    lik = rng.random((n_rows, n_lik)) * 10.0 ** rng.integers(-6, 6, size=(n_rows, 1))
    lik[rng.random(lik.shape) < 0.1] = 0.0
    lik[0] = 0.0
    return lik


def codes_of(rng, net, evidence, n_rows):
    if not evidence:
        return np.zeros((0, n_rows), dtype=np.uint8)
    return np.stack([rng.integers(0, int(net.card[v]), n_rows) for v in evidence]).astype(np.uint8)


def cases(net, seed):
    """(query, hard evidence, soft) var-id triples: soft hidden, soft queried, and mixed hard and soft."""
    rng = np.random.default_rng(seed)
    n = len(net.names)
    out = []
    for k in range(4):
        perm = [int(v) for v in rng.permutation(n)]
        n_soft = min(1 + k % 3, n - 1)
        soft = tuple(perm[:n_soft])
        rest = perm[n_soft:]
        ev = tuple(rest[1:1 + min(k, len(rest) - 1)]) if k % 2 else ()
        query = (soft[0],) if k == 2 else (rest[0],)
        out.append((query, ev, soft))
    return out


def check_posterior(net, plan, ev, codes, lik, post, log_ev=None):
    dn = soft_oracle.dense(net)
    q_names = [net.names[v] for v in plan.query]
    for b, (hard, s) in enumerate(soft_oracle.rows(net, ev, codes, plan.soft, lik)):
        want = soft_oracle.posterior(dn, q_names, hard, s)
        if np.isnan(want).all():
            assert np.isnan(post[:, b]).all(), b
            continue
        np.testing.assert_allclose(post[:, b], want, rtol=1e-12, atol=1e-300)
        if log_ev is not None:
            le = soft_oracle.log_evidence(dn, hard, s)
            assert abs(log_ev[b] - le) <= 1e-12 * max(1.0, abs(le)), (b, log_ev[b], le)


@pytest.mark.parametrize("name", EXAMPLES + CORPUS)
def test_posterior_matches_virtual_evidence_oracle(name):
    net = network(name)
    rng = np.random.default_rng(1)
    for query, ev, soft in cases(net, 7):
        plan = planner.build_plan(net, query, ev, soft=soft)
        B = 6
        codes, lik = codes_of(rng, net, ev, B), random_lik(rng, net, plan.soft, B)
        post, _, log_ev = soft_interp.run(plan.words, plan.table_blob64, codes, lik, n_rows=B)
        check_posterior(net, plan, ev, codes, lik, post, log_ev)


@pytest.mark.parametrize("name", EXAMPLES + CORPUS[:3])
def test_marginals_match_virtual_evidence_oracle(name):
    net = network(name)
    rng = np.random.default_rng(2)
    dn = soft_oracle.dense(net)
    for _, ev, soft in cases(net, 11):
        targets = [v for v in range(len(net.names)) if v not in ev]  # soft variables are targets too
        plan = planner.build_marginals_plan(net, ev, targets=targets, soft=soft)
        B = 5
        codes, lik = codes_of(rng, net, ev, B), random_lik(rng, net, plan.soft, B)
        post = soft_interp.run_marginals(plan.words, plan.table_blob64, codes, lik, n_rows=B)
        starts = program_interp.segment_starts(plan)
        for b, (hard, s) in enumerate(soft_oracle.rows(net, ev, codes, plan.soft, lik)):
            for t, q0 in zip(plan.targets, starts):
                want = soft_oracle.posterior(dn, [net.names[t]], hard, s)
                got = post[q0:q0 + int(net.card[t]), b]
                if np.isnan(want).all():
                    assert np.isnan(got).all()
                else:
                    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-300)


def test_one_hot_is_hard_evidence_and_ones_are_no_evidence():
    net = network("alarm")
    soft_v, q = net.index["Alarm"], (net.index["Burglary"],)
    rng = np.random.default_rng(3)
    B = 4
    card = int(net.card[soft_v])
    codes = rng.integers(0, card, B).astype(np.uint8)
    onehot = np.eye(card)[codes] * 0.3
    soft = planner.build_plan(net, q, (), soft=(soft_v,))
    hard = planner.build_plan(net, q, (soft_v,))
    got = soft_interp.run(soft.words, soft.table_blob64, np.zeros((0, B), np.uint8), onehot, n_rows=B)[0]
    want = program_interp.run(hard.words, hard.table_blob64, codes[None, :])
    np.testing.assert_allclose(got, want, rtol=1e-13)
    none = planner.build_plan(net, q, ())
    got = soft_interp.run(soft.words, soft.table_blob64, np.zeros((0, B), np.uint8), np.ones((B, card)), n_rows=B)[0]
    want = program_interp.run(none.words, none.table_blob64, np.zeros((0, B), np.uint8), n_rows=B)
    np.testing.assert_allclose(got, want, rtol=1e-13)


# ----------------------------------------------------------------------------- plan invariants and refusals
@pytest.mark.parametrize("name", EXAMPLES + CORPUS)
def test_likelihood_slots_are_live_from_the_start_and_listed_in_column_order(name):
    net = network(name)
    for query, ev, soft in cases(net, 5):
        for plan in (planner.build_plan(net, query, ev, soft=soft),
                     planner.build_marginals_plan(net, ev, soft=soft)):
            assert plan.soft == tuple(sorted(soft, key=lambda v: net.names[v]))
            section, plain = soft_interp.split(plan.words)
            _, _, slots, steps = program_interp.parse(plain)
            assert plan.words[10] == len(soft)
            assert section == [(s, int(net.card[v])) for v, s in zip(plan.soft, plan.soft_slots)]
            assert len(set(plan.soft_slots)) == len(soft)
            for s, card in section:
                assert slots[s][0] == 1 and slots[s][1] >= card
                reads = [i for i, st in enumerate(steps) if any(inp["is_slot"] and inp["buf"] == s for inp in st["inputs"])]
                writes = [i for i, st in enumerate(steps) if st["kind"] in (0, 1) and st["out_slot"] == s]
                # filled before step 0: the first access is a read (later steps may reuse the slot)
                assert reads and (not writes or min(writes) > min(reads))


def test_refusals():
    net = network("asia")
    a, b, c = net.index["Smoker"], net.index["Lung cancer"], net.index["Dispnea"]
    with pytest.raises(ValueError, match="hard-evidence"):
        planner.build_plan(net, (b,), (a,), soft=(a,))
    with pytest.raises(ValueError, match="duplicate"):
        planner.build_plan(net, (b,), (), soft=(a, a))
    with pytest.raises(ValueError, match="batched"):
        planner.build_plan(net, (b,), (), soft=(a,), mode=planner.MODE_FLAT)
    with pytest.raises(ValueError, match="hard-evidence"):
        planner.build_marginals_plan(net, (a,), soft=(a,))
    for build in (planner.build_counts_plan, planner.build_sample_plan, planner.build_mpe_plan):
        with pytest.raises(TypeError):
            build(net, (c,), soft=(a,))
    with pytest.raises(TypeError):
        planner.build_map_plan(net, (c,), (b,), soft=(a,))
    # the replay (as the engine) takes likelihoods for a soft program only, one column per soft state
    plain = planner.build_plan(net, (b,), ())
    with pytest.raises(AssertionError):
        soft_interp.run(plain.words, plain.table_blob64, np.zeros((0, 1), np.uint8), np.ones((1, 2)), n_rows=1)
    plan = planner.build_plan(net, (b,), (), soft=(a,))
    with pytest.raises(AssertionError):
        soft_interp.run(plan.words, plan.table_blob64, np.zeros((0, 1), np.uint8), np.ones((1, 3)), n_rows=1)


# ------------------------------------------------------------------------------ plans without soft evidence
def fixed_plans(pl, nets):
    """(name, plan) of plans without soft evidence over the example networks, the corpus and the benchmark grid,
    built by planner module `pl` on the CompiledNets `nets` {name: net}."""
    for name, net in nets.items():
        n = len(net.names)
        rng = np.random.default_rng(len(name))
        for k in range(3):
            perm = [int(v) for v in rng.permutation(n)]
            ev = tuple(perm[1:1 + k * max(1, n // 5)])
            yield f"{name}/post{k}", pl.build_plan(net, (perm[0],), ev)
            yield f"{name}/flat{k}", pl.build_plan(net, (perm[0],), ev, mode=pl.MODE_FLAT)
            if n <= 20:
                yield f"{name}/marg{k}", pl.build_marginals_plan(net, ev)
                yield f"{name}/counts{k}", pl.build_counts_plan(net, ev)
                yield f"{name}/sample{k}", pl.build_sample_plan(net, ev)
                yield f"{name}/mpe{k}", pl.build_mpe_plan(net, ev)
                yield f"{name}/map{k}", pl.build_map_plan(net, ev, (perm[0],))
        if name.startswith("dag") or name in EXAMPLES:
            yield f"{name}/evidence", pl.build_plan(net, (), tuple(range(n // 2)), allow_empty_query=True)
    w = workloads.grid10x10()  # the benchmark's own plan
    net = nets["grid10x10"]
    yield "grid10x10/bench", pl.build_plan(net, [net.index[q] for q in w.query], [net.index[e] for e in w.evidence])


def plan_nets():
    nets = {name: network(name) for name in EXAMPLES + CORPUS}
    nets["grid10x10"] = workloads.grid10x10().build()._compiled
    return nets


def digest(plan):
    return hashlib.sha256(np.asarray(plan.words, dtype=np.int32).tobytes() +
                          np.asarray(plan.table_blob, dtype=np.float32).tobytes()).hexdigest()


def test_plans_without_soft_evidence_keep_their_words():
    with open(os.path.join(GOLDEN, "plan_words_parent.json")) as f:
        want = json.load(f)["digests"]
    got = {name: digest(plan) for name, plan in fixed_plans(planner, plan_nets())}
    assert got.keys() == want.keys()
    assert [k for k in got if got[k] != want[k]] == []
