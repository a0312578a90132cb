"""CPU replay of counts, sample, MPE and marginal MAP programs with soft evidence (versions 6 to 9; TEST
INFRASTRUCTURE): the likelihood slots filled as csrc/sbn_soft.cuh fills them, then the program run by
oracle/program_interp.py unchanged.

The soft section of these versions follows the slots, as in versions 4 and 5, but its count is header word 11
(word 10 holds n_counts / n_sampled).  `split` takes it out, which leaves words the interpreter parses as they
are.  Sum-product kinds (counts, sample) fill the slots with `soft_interp.soft_pack`; the log-domain kinds (MPE,
MAP) with `log_pack`, the numpy form of sbn_soft_pack_log.  `soft_interp`'s version-4/5 replay is untouched.
"""
from __future__ import annotations

import numpy as np

import soft_interp
from oracle import program_interp

HEADER_WORDS = program_interp.HEADER_WORDS


def split(words):
    """(the (slot, card) of every likelihood in likelihood-column order, the words without the soft section) of a
    version 6-9 program."""
    w = np.asarray(words, dtype=np.int32)
    version, n_soft = int(w[1]), int(w[11])
    assert version in (6, 7, 8, 9), f"version {version}: not a counts, sample, MPE or MAP program"
    if n_soft == 0:
        return [], w
    p = HEADER_WORDS + 2 * int(w[4]) + 2 * int(w[5])  # after the table and slot sections
    soft = [(int(w[p + 2 * k]), int(w[p + 2 * k + 1])) for k in range(n_soft)]
    plain = np.concatenate([w[:p], w[p + 2 * n_soft:]])
    plain[11] = 0
    return soft, plain


def log_pack(soft, lik, dtype):
    """The likelihood slots of a log-domain program: log(x / max) per variable's row, computed in float64 from the
    float64 likelihoods (the kernel reads them in double) and rounded once to `dtype` (its __double2float_rn of a
    double log), -inf for a zero entry (an all-zero row is -inf throughout).  Returns ([card, B] per soft variable,
    sum log(max) [B] in float64)."""
    lik = np.asarray(lik, dtype=np.float64)
    assert lik.ndim == 2 and lik.shape[1] == sum(c for _, c in soft), "one likelihood column per soft state"
    packed, log_max, c0 = [], np.zeros(lik.shape[0], dtype=np.float64), 0
    for _, card in soft:
        block = lik[:, c0:c0 + card]
        c0 += card
        m = block.max(axis=1)
        with np.errstate(divide="ignore", invalid="ignore"):
            vals = np.where(block > 0, np.log(block / m[:, None]), -np.inf)
            log_max = log_max + np.log(m)
        packed.append(vals.astype(dtype).T.copy())
    return packed, log_max


def _soft(words, lik, dtype, log):
    soft, plain = split(words)
    assert soft, "not a soft-evidence program"
    packed, log_max = (log_pack if log else soft_interp.soft_pack)(soft, lik, dtype)
    return soft, plain, packed, log_max


def run_counts(words, table_blob, ev_codes, lik, n_rows=None, dtype=np.float64, min_total=None):
    """(counts [n_counts], P(observed, lik / max) [B] in `dtype` (NaN where flagged), log P(observed, lik) [B])."""
    soft, plain, packed, log_max = _soft(words, lik, dtype, log=False)
    with soft_interp._filled(soft, packed):
        counts, prob = program_interp.run_counts(plain, table_blob, ev_codes, n_rows=n_rows, dtype=dtype,
                                                 min_total=min_total)
    with np.errstate(divide="ignore", invalid="ignore"):
        return counts, prob, np.log(prob.astype(np.float64)) + log_max


def run_sample(words, table_blob, ev_codes, lik, n_rows=None, n_draws=1, seed=0, row_base=0, dtype=np.float64,
               min_total=None, given=None):
    """`program_interp.run_sample`'s (drawn, P(observed, lik / max), info), then log P(observed, lik) [B]."""
    soft, plain, packed, log_max = _soft(words, lik, dtype, log=False)
    with soft_interp._filled(soft, packed):
        drawn, prob, info = program_interp.run_sample(plain, table_blob, ev_codes, n_rows=n_rows, n_draws=n_draws,
                                                      seed=seed, row_base=row_base, dtype=dtype, min_total=min_total,
                                                      given=given)
    with np.errstate(divide="ignore", invalid="ignore"):
        return drawn, prob, info, np.log(prob.astype(np.float64)) + log_max


def run_mpe(words, table_blob, ev_codes, lik, n_rows=None, dtype=np.float32):
    """(decoded codes [n_decoded, B], log P(x*, e, lik) [B] in float64: the program's `dtype` maximum plus the
    float64 sum log(max), as the engine adds them) of an MPE or marginal MAP program."""
    soft, plain, packed, log_max = _soft(words, lik, dtype, log=True)
    with soft_interp._filled(soft, packed):
        decoded, lp = program_interp.run_mpe(plain, table_blob, ev_codes, n_rows=n_rows, dtype=dtype)
    return decoded, lp.astype(np.float64) + log_max
