"""CPU replay of soft-evidence programs (TEST INFRASTRUCTURE): the likelihood slots of a version-4 or version-5
program filled as csrc/sbn_soft.cuh fills them, then the program run by oracle/program_interp.py unchanged.

A soft program's words are those of a program without soft evidence plus the soft section after the slots
(header word 10 = n_soft, then `(slot, card)` per soft variable; planner.py "Soft evidence").  `split` takes that
section out, which leaves words the interpreter parses as they are, with likelihood slots that no step writes.
`run` and `run_marginals` hand those words to `program_interp.run` / `run_marginals` on an execution whose
likelihood slots hold the packed likelihoods before the first step, so every step, readout and normalisation is
the interpreter's own.
"""
from __future__ import annotations

import contextlib

import numpy as np

from oracle import program_interp

HEADER_WORDS = program_interp.HEADER_WORDS


def split(words):
    """(the (slot, card) of every likelihood in likelihood-column order, the words without the soft section)."""
    w = np.asarray(words, dtype=np.int32)
    version, n_soft = int(w[1]), int(w[10])
    if version not in (4, 5) or n_soft == 0:
        return [], w
    p = HEADER_WORDS + 2 * int(w[4]) + 2 * int(w[5])  # after the table and slot sections
    soft = [(int(w[p + 2 * k]), int(w[p + 2 * k + 1])) for k in range(n_soft)]
    plain = np.concatenate([w[:p], w[p + 2 * n_soft:]])
    plain[10] = 0
    return soft, plain


def soft_pack(soft, lik, dtype):
    """The likelihood slots as the pack kernel fills them: `lik` [B, sum of cards] (columns in the order of `soft`)
    cast to `dtype`, every variable's row divided by its maximum in `dtype` (all zeros where the maximum is 0).
    Returns ([card, B] per soft variable, sum over the soft variables of log(maximum) [B] in float64, -inf where a
    maximum is 0)."""
    lik = np.asarray(lik).astype(dtype)
    assert lik.ndim == 2 and lik.shape[1] == sum(c for _, c in soft), "one likelihood column per soft state"
    packed, log_max, c0 = [], np.zeros(lik.shape[0], dtype=np.float64), 0
    for _, card in soft:
        block = lik[:, c0:c0 + card]
        c0 += card
        m = block.max(axis=1)
        with np.errstate(divide="ignore", invalid="ignore"):
            packed.append(np.where(m[:, None] > 0, block / m[:, None], dtype(0)).astype(dtype).T.copy())
            log_max = log_max + np.log(m.astype(np.float64))
    return packed, log_max


@contextlib.contextmanager
def _filled(soft, packed):
    """While active, every interpreter execution starts with the likelihood slots filled.  `program_interp.run` and
    `run_marginals` create their execution through the module's `_Program`, which is swapped for the duration."""
    base = program_interp._Program

    class Filled(base):
        def __init__(self, *args, **kwargs):
            super().__init__(*args, **kwargs)
            for (slot, card), lam in zip(soft, packed):
                assert lam.shape == (card, self.B), "one likelihood row per evidence row"
                self.bufs[slot] = lam

    program_interp._Program = Filled
    try:
        yield
    finally:
        program_interp._Program = base


def run(words, table_blob, ev_codes, lik, n_rows=None, dtype=np.float64):
    """A soft-evidence posterior program (version 4): (normalised posterior [Q, B], its normaliser [B], and
    log P(e, lik) [B] = log(normaliser) + sum log(max), NaN / -inf for an impossible row)."""
    soft, plain = split(words)
    assert soft, "not a soft-evidence program"
    packed, log_max = soft_pack(soft, lik, dtype)
    with _filled(soft, packed):
        post, total = program_interp.run(plain, table_blob, ev_codes, n_rows=n_rows, dtype=dtype, return_totals=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        log_ev = np.log(total.astype(np.float64)) + log_max
    return post, total, log_ev


def run_marginals(words, table_blob, ev_codes, lik, n_rows=None, dtype=np.float64, min_total=None):
    """A soft-evidence marginals program (version 5): the posterior [Q, B] of `program_interp.run_marginals`."""
    soft, plain = split(words)
    assert soft, "not a soft-evidence program"
    packed, _ = soft_pack(soft, lik, dtype)
    with _filled(soft, packed):
        return program_interp.run_marginals(plain, table_blob, ev_codes, n_rows=n_rows, dtype=dtype,
                                            min_total=min_total)
