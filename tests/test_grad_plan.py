"""Gradient programs (planner.build_pattern_plan kind "grad", version 10), checked on the CPU.

tests/grad_interp.py replays the words as the device runs them; tests/grad_oracle.py gives log P(e_b, lambda_b)
and its gradients by torch autograd over the joint, with no planner or engine code.  The weighted counts must be
sum_b w_b * theta * d log P_b / d theta, and each derivative readout over the row's maximum must be
d log P_b / d lambda_b."""
import numpy as np
import pytest

import grad_interp
import grad_oracle
from sorobn_b200 import planner
from test_soft_plan import CORPUS, EXAMPLES, network

NETS = EXAMPLES + CORPUS[:3] + ["wide"]


def wide():
    """A net whose soft variable has 11 states: its readout takes two passes of the kernel's 8 accumulators."""
    rng = np.random.default_rng(0)

    def cpt(*shape):
        t = rng.random(shape) + 0.05
        return t / t.sum(axis=-1, keepdims=True)

    return planner.CompiledNet(names=["a", "b", "c", "d"], domains=[list(range(11)), list(range(3)), list(range(4)),
                                                                   list(range(5))],
                               parents=[[], [0], [0, 1], [2]], cpt=[cpt(11), cpt(11, 3), cpt(11, 3, 4), cpt(4, 5)])


def net_of(name):
    return wide() if name == "wide" else network(name)


def cases(net, seed):
    """(observed var ids, soft var ids) pairs: soft only, hard and soft, hard only (with latent nodes)."""
    rng = np.random.default_rng(seed)
    n = len(net.names)
    out = []
    for k in range(3):
        perm = [int(v) for v in rng.permutation(n)]
        soft = tuple(perm[:min(1 + k, n - 1)]) if k < 2 else ()
        rest = perm[len(soft):]
        ev = tuple(sorted(rest[:min(2 + k, len(rest) - 1)])) if k else ()
        out.append((ev, soft))
    return out


def random_rows(rng, net, ev, soft, n_rows):
    codes = np.stack([rng.integers(0, int(net.card[v]), n_rows) for v in ev]).astype(np.uint8) if ev \
        else np.zeros((0, n_rows), dtype=np.uint8)
    n_lik = sum(int(net.card[v]) for v in soft)
    lik = rng.random((n_rows, n_lik)) * 10.0 ** rng.integers(-3, 3, size=(n_rows, 1))
    lik[rng.random(lik.shape) < 0.25] = 0.0  # exact zeros: the readouts must stay exact there
    c0 = 0
    for v in soft:  # every row keeps one positive entry per soft variable
        c = int(net.card[v])
        lik[:, c0] = np.maximum(lik[:, c0], 0.5)
        c0 += c
    weights = rng.normal(size=n_rows)
    return codes, lik, weights


def oracle(net, plan, ev, codes, lik, weights):
    n_rows = len(weights)
    full = _full(net, ev, codes, n_rows)
    lik_of = _lik_of(net, plan, lik)
    _, g_cpt, _, logp = grad_oracle.gradients(net.parents, net.card, net.cpt, full, weights, lik_of)
    _, _, g_lik, _ = grad_oracle.gradients(net.parents, net.card, net.cpt, full, np.ones(n_rows), lik_of)
    return g_cpt, g_lik, logp


def possible(net, plan, ev, codes, lik, weights):
    """The rows of positive probability (a network with zero CPT entries makes impossible ones)."""
    import torch

    logp = grad_oracle.log_likelihood(net.parents, net.card, [torch.as_tensor(c) for c in net.cpt],
                                      _full(net, ev, codes, len(weights)),
                                      {v: torch.as_tensor(x) for v, x in _lik_of(net, plan, lik).items()})
    keep = np.isfinite(logp.numpy())
    return codes[:, keep], lik[keep], weights[keep]


def check(net, plan, ev, codes, lik, weights, dtype=np.float64, tol=1e-9):
    codes, lik, weights = possible(net, plan, ev, codes, lik, weights)
    n_rows = len(weights)
    lik_in = lik if plan.soft else None
    blob = plan.table_blob64 if dtype == np.float64 else plan.table_blob
    counts, deriv, prob, log_max = grad_interp.run_grad(plan.words, blob, codes, weights, lik_in, n_rows=n_rows,
                                                        dtype=dtype)
    g_cpt, g_lik, logp = oracle(net, plan, ev, codes, lik, weights)
    want = np.concatenate([(net.cpt[v] * g_cpt[v]).reshape(-1) for v in range(len(net.names))])
    # each entry against the same entry's oracle with |w_b|: signed weights may cancel
    _, g_abs, _, _ = grad_oracle.gradients(net.parents, net.card, net.cpt, _full(net, ev, codes, n_rows), np.abs(weights),
                                           _lik_of(net, plan, lik))
    scale = np.concatenate([(net.cpt[v] * g_abs[v]).reshape(-1) for v in range(len(net.names))])
    assert (np.abs(counts - want) <= tol * np.maximum(scale, 1e-300) + 1e-300).all(), np.abs(counts - want).max()
    np.testing.assert_allclose(np.log(prob.astype(np.float64)) + log_max, logp, rtol=tol, atol=tol)
    c0 = 0
    for v in plan.soft:
        c = int(net.card[v])
        m = lik[:, c0:c0 + c].max(axis=1)
        got = deriv[c0:c0 + c].astype(np.float64).T / m[:, None]
        np.testing.assert_allclose(got, g_lik[v], rtol=tol, atol=tol * np.abs(g_lik[v]).max())
        c0 += c
    fwd, fwd_log_max = grad_interp.run_grad(plan.words, blob, codes, lik=lik_in, n_rows=n_rows, dtype=dtype,
                                            forward_steps=plan.forward_steps)
    np.testing.assert_array_equal(fwd, prob)


def _full(net, ev, codes, n_rows):
    full = -np.ones((len(net.names), n_rows), dtype=np.int64)
    for i, v in enumerate(ev):
        full[v] = codes[i]
    return full


def _lik_of(net, plan, lik):
    out, c0 = {}, 0
    for v in plan.soft:
        out[v] = lik[:, c0:c0 + int(net.card[v])]
        c0 += int(net.card[v])
    return out


@pytest.mark.parametrize("name", NETS)
def test_float64_replay_matches_the_autograd_oracle(name):
    net = net_of(name)
    rng = np.random.default_rng(len(name))
    for k, (ev, soft) in enumerate(cases(net, len(name))):
        plan = planner.build_pattern_plan(net, "grad", ev, soft=soft)
        assert plan.version == planner.VERSION_GRAD and plan.Q == 1 + sum(int(net.card[v]) for v in plan.soft)
        codes, lik, weights = random_rows(rng, net, ev, plan.soft, 12)
        check(net, plan, ev, codes, lik, weights)


def test_float32_replay_is_within_the_counts_tolerance():
    net = network("alarm")
    rng = np.random.default_rng(3)
    for ev, soft in cases(net, 3):
        plan = planner.build_pattern_plan(net, "grad", ev, soft=soft)
        codes, lik, weights = random_rows(rng, net, ev, plan.soft, 17)
        check(net, plan, ev, codes, lik, weights, dtype=np.float32, tol=2e-5)


@pytest.mark.parametrize("name", NETS)
def test_forward_closure_holds_no_count_or_readout_step(name):
    net = net_of(name)
    for ev, soft in cases(net, 7):
        plan = planner.build_pattern_plan(net, "grad", ev, soft=soft)
        kinds = [plan.steps[i].kind for i in plan.forward_steps]
        assert set(kinds) <= {planner.KIND_FLAT, planner.KIND_BATCHED}
        assert plan.steps[plan.forward_steps[-1]].out_slot == plan.post_slot
        n_deriv = sum(st.kind == planner.KIND_DERIV for st in plan.steps)
        assert n_deriv == len(plan.soft)


def test_wide_soft_variable_is_read_in_passes():
    net = wide()
    plan = planner.build_pattern_plan(net, "grad", (3,), soft=(0,))
    assert [st.cards for st in plan.steps if st.kind == planner.KIND_DERIV] == [(11,)]
    rng = np.random.default_rng(5)
    check(net, plan, (3,), *random_rows(rng, net, (3,), plan.soft, 10))


def test_refusals():
    net = network("asia")
    with pytest.raises(ValueError, match="batched"):
        planner.build_pattern_plan(net, "grad", (0,), mode=planner.MODE_FLAT)
    with pytest.raises(ValueError, match="kind must be one of"):
        planner.build_pattern_plan(net, "gradient", (0,))
    with pytest.raises(ValueError, match="soft-evidence variable cannot also be"):
        planner.build_pattern_plan(net, "grad", (0,), soft=(0,))
