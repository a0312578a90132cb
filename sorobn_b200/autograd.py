"""Per-row log-likelihoods of a BayesNet as a differentiable torch function (`BayesNet.log_likelihood`).

For row b with observed cells e_b and soft evidence lambda_b, log P(e_b, lambda_b; theta) is the log of the
network polynomial.  Its derivatives are what a counts program reduces (DESIGN.md "Gradients of the
log-likelihood"):

    d log P_b / d theta_v(x, u)   = P(v = x, pa(v) = u | e_b, lambda_b) / theta_v(x, u)
    d log P_b / d lambda_b,s(x)   = [the bucket of lambda_s without lambda_s, summed to s = x] / P(e_b, lambda_b)

The forward pass runs each missingness pattern's gradient program (planner.build_pattern_plan kind "grad") in
forward mode: the upward pass only.  The backward pass runs it again with the upstream gradient g_b as the row
weight of the count steps: sum_b g_b * d log P_b / d theta comes back as weighted counts, divided here by
theta, and the derivative readouts give d log P_b / d lambda_b after the pack's 1 / max is undone.  Rows the
float32 program flags re-run on the float64 twin, in both passes.  Second derivatives are not supported.
"""
from __future__ import annotations

import numpy as np
import torch

from . import planner as _planner
from .bayes_net import _lik_rows


class EncodedRows:
    """The rows of a frame grouped by missingness pattern (`BayesNet.encode_rows`), to pass to
    `BayesNet.log_likelihood` in place of the frame when the same rows are used again."""

    def __init__(self, groups, index, columns):
        self.groups = groups  # [(observed var ids, row positions, uint8 codes [n_observed, n_rows])]
        self.index = index
        self.columns = tuple(columns)

    def __len__(self):
        return len(self.index)


def _dense_cpts(bn, cpts):
    """(float64 ndarray per var id: the given CPTs over the compiled ones, {var id: the given tensor}); ValueError
    for an unknown node, a wrong shape, a negative entry, a row that does not sum to 1 within 1e-6, or a zero entry
    in a tensor that requires grad."""
    net = bn._compiled
    arrays = [np.asarray(c, dtype=np.float64) for c in net.cpt]
    given = {}
    for node, t in (cpts or {}).items():
        if node not in net.index:
            raise ValueError(f"cpts for {node!r}, which is not a node of the network")
        v = net.index[node]
        tensor = t if isinstance(t, torch.Tensor) else torch.as_tensor(np.asarray(t, dtype=np.float64))
        shape = tuple(int(net.card[u]) for u in net.scope(v))
        if tuple(tensor.shape) != shape:
            raise ValueError(f"the CPT of {node!r} has shape {tuple(tensor.shape)}, expected {shape} "
                             f"(axes {[net.names[u] for u in net.scope(v)]})")
        arr = tensor.detach().to("cpu", torch.float64).numpy()
        if not np.isfinite(arr).all() or (arr < 0).any():
            raise ValueError(f"the CPT of {node!r} has a negative or non-finite entry")
        if np.abs(arr.sum(axis=-1) - 1.0).max(initial=0.0) > 1e-6:
            raise ValueError(f"the CPT of {node!r} has rows that do not sum to 1 (within 1e-6)")
        if tensor.requires_grad and (arr == 0).any():
            raise ValueError(f"the CPT of {node!r} requires grad and has a zero entry, whose derivative is not "
                             "count / theta: parameterise through softmax")
        arrays[v] = arr
        given[v] = tensor
    return arrays, given


def _run(bn, rows, soft, lik, arrays, weights=None):
    """Every pattern's gradient program over `rows`: forward (weights None) -> log P [n]; backward -> (counts,
    derivative readouts [n_lik, n] on the likelihoods / max)."""
    n = len(rows)
    n_counts = _planner.count_layout(bn._compiled)[1]
    log_p = np.full(n, np.nan)
    counts = np.zeros(n_counts)
    n_lik = 0 if lik is None else int(lik.shape[1])
    deriv = np.full((n_lik, n), np.nan)
    for ev, r, codes in rows.groups:
        runner = bn._pattern_runner("grad", ev, soft=soft)
        runner.set_cpts(arrays)
        lik_r = None if lik is None else _lik_rows(lik, r)

        def run(program, c, rr, lik_rr, w):
            if w is None:
                prob, lp = program.grad_forward(c, len(rr), lik=lik_rr)
                return lp, prob
            cnt, d, prob = program.grad_backward(c, len(rr), w, lik=lik_rr)
            return (cnt, d), prob

        w = None if weights is None else _lik_rows(weights, r)  # a CUDA tensor stays on the device
        out, prob = run(runner.f32(), codes, r, lik_r, w)
        flagged = np.flatnonzero(np.isnan(np.asarray(prob, dtype=np.float64)))
        again = None
        if len(flagged):
            again, prob2 = run(runner.f64(), np.ascontiguousarray(codes[:, flagged]), r[flagged],
                               None if lik_r is None else _lik_rows(lik_r, flagged), None if w is None else _lik_rows(w, flagged))
            prob = np.asarray(prob, dtype=np.float64)
            prob[flagged] = prob2
        impossible = np.isnan(np.asarray(prob, dtype=np.float64))
        if impossible.any():
            raise ValueError(f"{int(impossible.sum())} row(s) have observed cells of probability zero "
                             f"(first: {rows.index[r[impossible][0]]!r}); their log-likelihood is -inf")
        if weights is None:
            lp = np.asarray(out, dtype=np.float64)
            if again is not None:
                lp[flagged] = again
            log_p[r] = lp
            continue
        cnt, d = out
        counts += cnt
        d = np.asarray(d, dtype=np.float64)
        if again is not None:
            counts += again[0]
            d[:, flagged] = again[1]
        deriv[:, r] = d
    return log_p if weights is None else (counts, deriv)


class _LogLikelihood(torch.autograd.Function):
    @staticmethod
    def forward(ctx, state, *tensors):
        bn, rows, soft, lik, arrays, given, blocks, device = state
        log_p = _run(bn, rows, soft, lik, arrays)
        ctx.state = state
        return torch.as_tensor(log_p, dtype=torch.float64, device=device)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        bn, rows, soft, lik, arrays, given, blocks, device = ctx.state
        g = grad_out.detach().to(torch.float64).contiguous()
        # the engine reads a CUDA upstream gradient in place as the row weights
        counts, deriv = _run(bn, rows, soft, lik, arrays, weights=g if g.is_cuda else g.numpy())
        net = bn._compiled
        offsets, _ = _planner.count_layout(net)
        grads = []
        for v, t in given.items():
            c = counts[offsets[v]:offsets[v] + arrays[v].size].reshape(arrays[v].shape)
            with np.errstate(divide="ignore", invalid="ignore"):
                gv = np.where(arrays[v] > 0, c / arrays[v], 0.0)
            grads.append(torch.as_tensor(gv, dtype=t.dtype, device=t.device) if t.requires_grad else None)
        # the readouts come back through host memory; the likelihood gradient g_b * readout / max is formed on the
        # likelihood tensor's device
        c0 = 0
        for (name, t) in blocks:
            card = int(net.card[net.index[name]])
            if t is not None:
                block = torch.as_tensor(lik[:, c0:c0 + card]).to(t.device, torch.float64)
                d = torch.as_tensor(np.ascontiguousarray(deriv[c0:c0 + card].T)).to(t.device)
                gl = g.to(t.device)[:, None] * d / block.max(dim=1).values[:, None]
                grads.append(gl.to(t.dtype) if t.requires_grad else None)
            c0 += card
        return (None, *grads)


def log_likelihood(bn, X, cpts=None, likelihoods=None):
    """`BayesNet.log_likelihood`: log P(observed cells of b, lambda_b) of every row, float64 [n] on the network's
    device, differentiable in the tensors of `cpts` and `likelihoods`."""
    bn._net("computing log-likelihoods")
    rows = X if isinstance(X, EncodedRows) else bn.encode_rows(X)
    arrays, given = _dense_cpts(bn, cpts)
    soft, lik, blocks = (), None, []
    if likelihoods is not None:
        names, lik = bn._soft_matrix(likelihoods, len(rows), rows.columns)
        if not isinstance(lik, np.ndarray):
            lik = lik.detach()
        soft = tuple(bn._compiled.index[n] for n in names)
        blocks = [(n, likelihoods[n] if isinstance(likelihoods[n], torch.Tensor) else None) for n in names]
    from . import engine

    # the network's device (a host without one can only run interpreted programs, as the tests do)
    device = torch.device("cuda", engine.default_device() if bn.device is None else bn.device) \
        if torch.cuda.is_available() else torch.device("cpu")
    tensors = [t for t in given.values()] + [t for _, t in blocks if t is not None]
    state = (bn, rows, soft, lik, arrays, given, blocks, device)
    return _LogLikelihood.apply(state, *tensors)
