"""Float64 oracle of per-row log-likelihoods and their gradients (TEST INFRASTRUCTURE, not product).

For row b with observed cells e_b and likelihoods lambda_b, log P(e_b, lambda_b) is the log of

    sum_x prod_v CPT_v(x_v | x_pa(v)) * prod_v E_v[b, x_v]

where E_v[b] is the one-hot vector of v's code where the row observes v, lambda_v[b] for a soft node, and all
ones otherwise.  The sum is a float64 torch einsum over the joint, contracted one variable at a time
(min-degree order) with the row axis kept, so that alarm-sized networks fit; `torch.autograd.grad` then gives
d/d CPT and d/d lambda.  It uses no planner or engine code: only the network's parents, cards and CPTs.
"""
from __future__ import annotations

import string

import numpy as np
import torch

_LETTERS = string.ascii_letters


def _contract(factors, n_vars):
    """sum over every variable of prod(factors); factors: [(var ids, tensor [B, *cards])] -> [B]."""
    factors = list(factors)
    remaining = set(range(n_vars))
    while remaining:
        # min-degree: the variable whose elimination touches the fewest other variables
        def degree(v):
            return len(set().union(*[set(vs) for vs, _ in factors if v in vs]) - {v})

        x = min(remaining, key=lambda v: (degree(v), v))
        remaining.discard(x)
        touching = [f for f in factors if x in f[0]]
        factors = [f for f in factors if x not in f[0]]
        if not touching:
            continue
        out_vars = sorted(set().union(*[set(vs) for vs, _ in touching]) - {x})
        letter = {v: _LETTERS[i + 1] for i, v in enumerate(sorted(set().union(*[set(vs) for vs, _ in touching])))}
        spec = ",".join("a" + "".join(letter[v] for v in vs) for vs, _ in touching)
        spec += "->a" + "".join(letter[v] for v in out_vars)
        factors.append((tuple(out_vars), torch.einsum(spec, *[t for _, t in touching])))
    out = None
    for vs, t in factors:
        assert not vs
        out = t if out is None else out * t
    return out


def log_likelihood(parents, cards, cpts, codes, lik=None):
    """log P(e_b, lambda_b) [B] float64.

    parents: var id -> parent ids; cards: var id -> states; cpts: var id -> float64 tensor [*parents, v];
    codes: int array [n_vars, B], -1 where the cell is unobserved (latent nodes are -1 throughout);
    lik: {var id: float64 tensor [B, card]} soft evidence."""
    codes = np.asarray(codes)
    n, B = codes.shape
    lik = lik or {}
    factors = []
    for v in range(n):
        t = cpts[v]
        factors.append(((*parents[v], v), t.unsqueeze(0).expand(B, *t.shape)))
        e = torch.ones(B, int(cards[v]), dtype=torch.float64)
        obs = codes[v] >= 0
        if obs.any():
            e[torch.as_tensor(obs)] = torch.nn.functional.one_hot(
                torch.as_tensor(codes[v][obs], dtype=torch.int64), int(cards[v])).to(torch.float64)
        if v in lik:
            e = e * lik[v]
        factors.append(((v,), e))
    return torch.log(_contract(factors, n))


def gradients(parents, cards, cpts, codes, weights, lik=None):
    """(sum_b w_b log P_b, d/d CPT [per var id, float64 ndarray], d/d lambda {var id: [B, card]}, log P [B])."""
    cpts = [torch.as_tensor(np.asarray(c, dtype=np.float64)).clone().requires_grad_(True) for c in cpts]
    lik = {v: torch.as_tensor(np.asarray(x, dtype=np.float64)).clone().requires_grad_(True)
           for v, x in (lik or {}).items()}
    logp = log_likelihood(parents, cards, cpts, codes, lik)
    w = torch.as_tensor(np.asarray(weights, dtype=np.float64))
    total = (w * logp).sum()
    keys = sorted(lik)
    grads = torch.autograd.grad(total, [*cpts, *[lik[k] for k in keys]], allow_unused=True)
    g_cpt = [g.numpy() if g is not None else np.zeros(c.shape) for g, c in zip(grads[:len(cpts)], cpts)]
    g_lik = {k: g.numpy() for k, g in zip(keys, grads[len(cpts):])}
    return float(total.detach()), g_cpt, g_lik, logp.detach().numpy()
