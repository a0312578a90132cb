"""Gradient programs and `BayesNet.log_likelihood` on the H100, against tests/grad_oracle.py."""
import numpy as np
import pandas as pd
import pytest
import torch

import grad_oracle
from sorobn_b200 import BayesNet, engine, examples, planner
from test_grad_plan import NETS, _full, _lik_of, cases, net_of, possible, random_rows
from test_grad_host import frame, oracle

pytestmark = pytest.mark.gpu


def run_both(plan, codes, lik, weights, f64=False):
    prog = engine.Program(plan, f64=f64)
    try:
        lik_in = lik if plan.soft else None
        fwd = prog.grad_forward(codes, len(weights), lik=lik_in)
        bwd = prog.grad_backward(codes, len(weights), weights, lik=lik_in)
        again = prog.grad_backward(codes, len(weights), weights, lik=lik_in)
        return fwd, bwd, again
    finally:
        prog.close()


ROWS = [1, 127, 129, 4 * 132 * 128 - 1, 4 * 132 * 128 + 1, 3 * 4 * 132 * 128 + 77]  # block and grid edges


def tiled_rows(rng, net, plan, ev, n_rows, n_distinct=64):
    """n_rows rows drawn from at most n_distinct possible ones (the oracle runs on the distinct rows): (codes, lik,
    weights, index of each row's distinct row, the distinct (codes, lik))."""
    codes, lik, _ = possible(net, plan, ev, *random_rows(rng, net, ev, plan.soft, min(n_rows, n_distinct)))
    idx = rng.integers(0, len(lik), n_rows)
    return codes[:, idx], lik[idx], rng.normal(size=n_rows), idx, (codes, lik)


@pytest.mark.parametrize("name", NETS)
@pytest.mark.parametrize("n_rows", ROWS)
def test_forward_and_backward_match_the_oracle(name, n_rows):
    net = net_of(name)
    rng = np.random.default_rng(n_rows)
    for ev, soft in cases(net, n_rows):
        plan = planner.build_pattern_plan(net, "grad", ev, soft=soft)
        codes, lik, weights, idx, (dcodes, dlik) = tiled_rows(rng, net, plan, ev, n_rows)
        (prob, log_p), (counts, deriv, prob_b), (counts2, deriv2, _) = run_both(plan, codes, lik, weights)
        # two backward calls are bitwise equal; forward and backward agree on P(observed)
        assert counts.tobytes() == counts2.tobytes() and deriv.tobytes() == deriv2.tobytes()
        np.testing.assert_array_equal(prob, prob_b)
        # the counts are linear in the weights: the oracle takes each distinct row with the sum of its weights
        n_d = len(dlik)
        w_d = np.bincount(idx, weights, n_d)
        a_d = np.bincount(idx, np.abs(weights), n_d)
        full, lik_of = _full(net, ev, dcodes, n_d), _lik_of(net, plan, dlik)
        _, g_cpt, _, logp = grad_oracle.gradients(net.parents, net.card, net.cpt, full, w_d, lik_of)
        _, g_abs, _, _ = grad_oracle.gradients(net.parents, net.card, net.cpt, full, a_d, lik_of)
        _, _, g_lik, _ = grad_oracle.gradients(net.parents, net.card, net.cpt, full, np.ones(n_d), lik_of)
        ok = ~np.isnan(prob)  # float32 rows below 1e-30 are the float64 program's
        np.testing.assert_allclose(log_p[ok], logp[idx][ok], rtol=2e-6, atol=2e-6)
        if not ok.all():
            continue
        want = np.concatenate([(net.cpt[v] * g_cpt[v]).reshape(-1) for v in range(len(net.names))])
        scale = np.concatenate([(net.cpt[v] * g_abs[v]).reshape(-1) for v in range(len(net.names))])
        assert (np.abs(counts - want) <= 2e-6 * scale + 1e-12).all(), np.abs(counts - want).max()
        c0 = 0
        for v in plan.soft:
            c = int(net.card[v])
            m = lik[:, c0:c0 + c].max(axis=1)
            got = deriv[c0:c0 + c].astype(np.float64).T / m[:, None]
            want_l = g_lik[v][idx]
            # the counts tests' 2e-6 relative, entry by entry (exact zeros stay zero up to 1e-12 of the row's largest)
            bound = 2e-6 * np.abs(want_l) + 1e-12 * np.abs(want_l).max(axis=1, keepdims=True)
            assert (np.abs(got - want_l) <= bound).all(), (v, (np.abs(got - want_l) / np.abs(want_l)).max())
            c0 += c


def test_forward_issues_the_upward_closure_only():
    """The engine derives the forward run's launches from the slot words; they are the planner's forward_steps."""
    for name in ("alarm", "wide"):
        net = net_of(name)
        for ev, soft in cases(net, 4):
            plan = planner.build_pattern_plan(net, "grad", ev, soft=soft)
            rng = np.random.default_rng(1)
            codes, lik, weights = possible(net, plan, ev, *random_rows(rng, net, ev, plan.soft, 300))
            prog = engine.Program(plan)
            try:
                lik_in = lik if plan.soft else None
                before = prog.info()["launches"]
                prog.grad_forward(codes, len(weights), lik=lik_in)
                fwd = prog.info()["launches"] - before
                prog.grad_backward(codes, len(weights), weights, lik=lik_in)
                bwd = prog.info()["launches"] - before - fwd
            finally:
                prog.close()
            per_row = [i for i, st in enumerate(plan.steps) if st.kind == planner.KIND_BATCHED]
            pack = 1 if plan.soft else 0
            assert fwd == pack + len([i for i in plan.forward_steps if i in per_row]) + 1
            n_count = sum(st.kind == planner.KIND_COUNT for st in plan.steps)
            assert bwd == pack + len(per_row) + 2 * n_count + len(plan.soft) + 1


def test_device_weights_are_read_in_place():
    net = net_of("alarm")
    ev, soft = cases(net, 2)[1]
    plan = planner.build_pattern_plan(net, "grad", ev, soft=soft)
    rng = np.random.default_rng(2)
    codes, lik, weights = possible(net, plan, ev, *random_rows(rng, net, ev, plan.soft, 5000))
    dev = torch.device("cuda", engine.default_device())
    prog = engine.Program(plan)
    try:
        host = prog.grad_backward(codes, len(weights), weights, lik=lik)
        on_device = prog.grad_backward(codes, len(weights), torch.as_tensor(weights, device=dev),
                                       lik=torch.as_tensor(lik, device=dev))
    finally:
        prog.close()
    for a, b in zip(host, on_device):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes()


def chain(n=60, p=0.999):
    """A chain whose rows of disagreeing observations fall far below 1e-30."""
    nodes = [f"x{i:02d}" for i in range(n)]
    bn = BayesNet(*[(a, b) for a, b in zip(nodes[:-1], nodes[1:])])
    bn.P[nodes[0]] = pd.Series({0: 0.5, 1: 0.5})
    for a, b in zip(nodes[:-1], nodes[1:]):
        bn.P[b] = pd.Series({(0, 0): p, (0, 1): 1 - p, (1, 0): 1 - p, (1, 1): p})
    return bn.prepare(), nodes


def test_rows_below_float32_range_are_settled_in_float64():
    bn, nodes = chain()
    n = len(nodes)
    # every row disagrees with its neighbours 20 to 59 times: P between 1e-60 and 1e-177, all flagged in float32
    X = pd.DataFrame([[(i // k) % 2 for i in range(n)] for k in (1, 2, 3)] + [[(i + 1) % 2 for i in range(n)]],
                     columns=nodes)
    tabs = {nodes[5]: bn.cpt_tensors()[nodes[5]].clone().requires_grad_(True)}
    lp = bn.log_likelihood(X, cpts=tabs)
    lp.sum().backward()
    want_lp, g_cpt, _ = oracle(bn, X, {}, {}, np.ones(len(X)))
    assert want_lp.max() < np.log(1e-30)
    np.testing.assert_allclose(lp.detach().cpu().numpy(), want_lp, rtol=1e-9)
    np.testing.assert_allclose(tabs[nodes[5]].grad.numpy(), g_cpt[bn._compiled.index[nodes[5]]], rtol=1e-9)


def test_cuda_likelihoods_and_softmax_logits_receive_their_gradients():
    bn = examples.asia()
    X = frame(bn, 300, 7)
    rng = np.random.default_rng(8)
    dev = torch.device("cuda", engine.default_device())
    raw = torch.tensor(rng.normal(size=(300, 2)), device=dev, requires_grad=True)
    lik = torch.softmax(raw, -1)  # produced by a torch op on the device
    lik.retain_grad()
    name = "Lung cancer"
    logits = torch.tensor(rng.normal(size=tuple(bn.cpt_tensors()[name].shape)), requires_grad=True)
    lp = bn.log_likelihood(X, cpts={name: torch.softmax(logits, -1)}, likelihoods={"Dispnea": lik})
    assert lp.device == dev and lp.dtype == torch.float64
    lp.sum().backward()
    assert lik.grad.device == dev and raw.grad.device == dev
    cpt = torch.softmax(logits, -1).detach().numpy()
    want_lp, g_cpt, g_lik = oracle(bn, X, {name: cpt}, {"Dispnea": lik.detach().cpu().numpy()}, np.ones(300))
    np.testing.assert_allclose(lp.detach().cpu().numpy(), want_lp, rtol=2e-6)
    np.testing.assert_allclose(lik.grad.cpu().numpy(), g_lik[bn._compiled.index["Dispnea"]], rtol=2e-5, atol=1e-7)
    c, g = torch.tensor(cpt), torch.tensor(g_cpt[bn._compiled.index[name]])
    np.testing.assert_allclose(logits.grad.numpy(), (c * (g - (g * c).sum(-1, keepdim=True))).numpy(), rtol=2e-5,
                               atol=1e-6)


def test_zero_likelihood_entries_get_exact_readouts():
    bn = examples.asia()
    X = frame(bn, 200, 9)
    rng = np.random.default_rng(10)
    lik = rng.random((200, 2)) + 0.1
    lik[::3, 1] = 0.0
    t = torch.tensor(lik, requires_grad=True)
    bn.log_likelihood(X, likelihoods={"Dispnea": t}).sum().backward()
    _, _, g_lik = oracle(bn, X, {}, {"Dispnea": lik}, np.ones(200))
    want = g_lik[bn._compiled.index["Dispnea"]]
    assert (want[::3, 1] != 0).all()
    np.testing.assert_allclose(t.grad.numpy(), want, rtol=2e-5, atol=1e-7)


def test_em_fixed_point_is_stationary():
    bn = examples.asia()
    X = frame(bn, 2000, 11)
    bn.prior_count = None
    bn.fit_em(X, max_iter=500, tol=1e-12)
    tabs = {k: v.clone().requires_grad_(True) for k, v in bn.cpt_tensors().items() if (v > 0).all()}
    bn.log_likelihood(X, cpts=tabs).sum().backward()
    for name, t in tabs.items():
        g = t.grad.numpy()
        # the Lagrange condition of the sum-to-one constraint: the gradient is constant along every parent row
        spread = g.max(axis=-1) - g.min(axis=-1)
        assert (spread <= 1e-3 * np.abs(g).max(axis=-1) + 1e-2).all(), (name, spread)


def test_refusals_name_the_right_call():
    net = net_of("asia")
    counts = engine.Program(planner.build_pattern_plan(net, "counts", (0,), soft=(1,)))
    grad = engine.Program(planner.build_pattern_plan(net, "grad", (0,), soft=(1,)))
    codes, lik = np.zeros((1, 4), dtype=np.uint8), np.ones((4, 2))
    try:
        with pytest.raises(engine.EngineError, match="with soft evidence runs through sbn_program_counts_soft_host"):
            counts.grad_forward(codes, 4, lik=lik)
        with pytest.raises(engine.EngineError, match="sbn_program_grad_forward_host"):
            grad.counts(codes, 4, lik=lik)
    finally:
        counts.close()
        grad.close()
