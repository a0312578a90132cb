"""The host side of `BayesNet.log_likelihood`, `encode_rows`, `cpt_tensors` and `assign_cpts` on the CPU: the device
programs are replaced by the CPU replay of their words (tests/grad_interp.py), and only public entry points are
driven.  Ground truth is tests/grad_oracle.py."""
import numpy as np
import pandas as pd
import pytest
import torch

import grad_interp
import grad_oracle
from interpreted_program import InterpretedProgram
from sorobn_b200 import engine, examples, workloads


class GradProgram(InterpretedProgram):
    """InterpretedProgram with the gradient calls; `weights` records (f64, weights) of every backward run."""

    weights = []

    def _lik(self, lik):
        return None if lik is None else np.asarray(lik.cpu().numpy() if hasattr(lik, "cpu") else lik, dtype=self.dtype)

    def grad_forward(self, codes, n_rows, lik=None):
        self._start(n_rows)
        prob, log_max = grad_interp.run_grad(self.plan.words, self.blob, codes, lik=self._lik(lik), n_rows=n_rows,
                                             dtype=self.dtype, min_total=self._min_total(),
                                             forward_steps=self.plan.forward_steps)
        with np.errstate(divide="ignore", invalid="ignore"):
            return prob, np.log(prob.astype(np.float64)) + log_max

    def grad_backward(self, codes, n_rows, weights, lik=None):
        self._start(n_rows)
        w = np.asarray(weights.cpu().numpy() if hasattr(weights, "cpu") else weights, dtype=np.float64)
        GradProgram.weights.append((self.f64, w.copy()))
        counts, deriv, prob, _ = grad_interp.run_grad(self.plan.words, self.blob, codes, w, self._lik(lik),
                                                      n_rows=n_rows, dtype=self.dtype, min_total=self._min_total())
        return counts, deriv, prob


@pytest.fixture
def interpreted(monkeypatch):
    monkeypatch.setattr(InterpretedProgram, "live", [])
    monkeypatch.setattr(InterpretedProgram, "calls", [])
    monkeypatch.setattr(InterpretedProgram, "flag_below", None)
    monkeypatch.setattr(GradProgram, "weights", [])
    monkeypatch.setattr(engine, "Program", GradProgram)
    return GradProgram


def frame(bn, n, seed, cols=("Smoker", "Visit to Asia", "Positive X-ray"), frac=0.35):
    net = bn._compiled
    codes = workloads.forward_sample_codes(net, n, seed)
    rng = np.random.default_rng(seed)
    out = {}
    for c in cols:
        vals = np.asarray(net.domains[net.index[c]], dtype=object)[codes[net.index[c]]].copy()
        vals[rng.random(n) < frac] = None
        out[c] = vals
    return pd.DataFrame(out, index=pd.RangeIndex(3, 3 + n, name="row"))


def oracle(bn, X, cpts, lik, weights):
    """(log P [n], d/d CPT per var id, d/d lik {var id: [n, card]}) of the frame's rows."""
    net = bn._compiled
    full = -np.ones((len(net.names), len(X)), dtype=np.int64)
    for c in X.columns:
        v = net.index[c]
        vals = X[c].to_numpy()
        for b, x in enumerate(vals):
            if x is not None and x == x:
                full[v, b] = net.domains[v].index(x)
    tables = [cpts.get(n, net.cpt[v]) for v, n in enumerate(net.names)]
    _, g_cpt, g_lik, logp = grad_oracle.gradients(net.parents, net.card, tables, full, weights,
                                                  {net.index[k]: x for k, x in lik.items()})
    return logp, g_cpt, g_lik


def test_log_likelihood_and_gradients_match_the_oracle(interpreted):
    bn = examples.asia()
    X = frame(bn, 30, 1)
    rng = np.random.default_rng(2)
    tabs = bn.cpt_tensors()
    name = "Lung cancer"
    shape = tuple(tabs[name].shape)
    logits = torch.tensor(rng.normal(size=shape), requires_grad=True)
    lik = torch.tensor(rng.random((30, 2)) + 0.01, requires_grad=True)
    weights = rng.normal(size=30)
    lp = bn.log_likelihood(X, cpts={name: torch.softmax(logits, -1)}, likelihoods={"Dispnea": lik})
    (lp.cpu() * torch.as_tensor(weights)).sum().backward()
    cpt = torch.softmax(logits, -1).detach().numpy()
    want_lp, g_cpt, g_lik = oracle(bn, X, {name: cpt}, {"Dispnea": lik.detach().numpy()}, weights)
    np.testing.assert_allclose(lp.detach().cpu().numpy(), want_lp, rtol=1e-5)
    # the chain rule through softmax, on the oracle's d/d CPT
    c = torch.tensor(cpt)
    g = torch.tensor(g_cpt[bn._compiled.index[name]])
    want_logits = (c * (g - (g * c).sum(-1, keepdim=True))).numpy()
    np.testing.assert_allclose(logits.grad.numpy(), want_logits, rtol=2e-4, atol=1e-6)
    np.testing.assert_allclose(lik.grad.numpy(), g_lik[bn._compiled.index["Dispnea"]], rtol=2e-4,
                               atol=1e-6)


def test_flagged_rows_rerun_in_float64_with_their_weights(interpreted, monkeypatch):
    bn = examples.asia()
    X = frame(bn, 20, 4)
    monkeypatch.setattr(InterpretedProgram, "flag_below", 0.3)  # flags the rarer rows
    tabs = {k: v.clone().requires_grad_(True) for k, v in bn.cpt_tensors().items() if k == "Smoker"}
    lp = bn.log_likelihood(X, cpts=tabs)
    lp.sum().backward()
    f64_runs = [c for c in InterpretedProgram.calls if c[2]]
    assert f64_runs, "no row was re-run in float64"
    assert any(f64 for f64, _ in interpreted.weights)
    want_lp, g_cpt, _ = oracle(bn, X, {}, {}, np.ones(20))
    np.testing.assert_allclose(lp.detach().cpu().numpy(), want_lp, rtol=1e-5)
    np.testing.assert_allclose(tabs["Smoker"].grad.numpy(), g_cpt[bn._compiled.index["Smoker"]], rtol=1e-4)


def test_encode_rows_is_reused(interpreted):
    bn = examples.asia()
    X = frame(bn, 25, 5)
    rows = bn.encode_rows(X)
    a = bn.log_likelihood(rows)
    b = bn.log_likelihood(X)
    np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())


def test_cpt_tensors_and_assign_cpts_round_trip(interpreted):
    bn = examples.asia()
    tabs = bn.cpt_tensors()
    tabs["Smoker"] = torch.tensor([0.25, 0.75], dtype=torch.float64)
    bn.assign_cpts({"Smoker": tabs["Smoker"]})
    np.testing.assert_array_equal(bn.cpt_tensors()["Smoker"].numpy(), [0.25, 0.75])
    for k, t in bn.cpt_tensors().items():
        assert t.dtype == torch.float64 and tuple(t.shape) == bn._compiled.cpt[bn._compiled.index[k]].shape


def test_input_errors(interpreted):
    bn = examples.asia()
    X = frame(bn, 5, 6)
    tab = bn.cpt_tensors()["Smoker"]
    with pytest.raises(ValueError, match="not a node"):
        bn.log_likelihood(X, cpts={"nope": tab})
    with pytest.raises(ValueError, match="shape"):
        bn.log_likelihood(X, cpts={"Smoker": torch.ones(3, dtype=torch.float64) / 3})
    with pytest.raises(ValueError, match="negative"):
        bn.log_likelihood(X, cpts={"Smoker": torch.tensor([1.5, -0.5], dtype=torch.float64)})
    with pytest.raises(ValueError, match="sum to 1"):
        bn.log_likelihood(X, cpts={"Smoker": torch.tensor([0.5, 0.6], dtype=torch.float64)})
    with pytest.raises(ValueError, match="softmax"):
        bn.log_likelihood(X, cpts={"Smoker": torch.tensor([1.0, 0.0], dtype=torch.float64, requires_grad=True)})
    with pytest.raises(ValueError, match="likelihoods must be non-negative"):
        bn.log_likelihood(X, likelihoods={"Dispnea": -np.ones((5, 2))})
    with pytest.raises(ValueError, match="shape"):
        bn.log_likelihood(X, likelihoods={"Dispnea": np.ones((4, 2))})
    with pytest.raises(ValueError, match="probability zero"):
        bn.log_likelihood(X, likelihoods={"Dispnea": np.zeros((5, 2))})
