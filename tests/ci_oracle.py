"""Float64 oracle of the conditional-independence tests of constraint-based learning (test infrastructure; shares
no code with sorobn_b200/structure.py): the table of x _|_ y | S by np.bincount, its G^2 or Pearson X^2 statistic
and degrees of freedom in numpy, the p-value by scipy's regularised upper incomplete gamma function, and a tester
for structure.pc_search built from them."""
import math

import numpy as np
from scipy.special import gammaincc


def codes_of(X):
    """({column: int64 codes}, {column: states}), states = the sorted distinct values."""
    codes, cards = {}, {}
    for name in X.columns:
        states = sorted(set(X[name].tolist()))
        pos = {s: i for i, s in enumerate(states)}
        codes[name] = np.array([pos[v] for v in X[name].tolist()], dtype=np.int64)
        cards[name] = len(states)
    return codes, cards


def table(codes, cards, x, y, given=()):
    """Counts [n_strata, r_y, r_x] of the test x _|_ y | given, the first column of `given` fastest among S."""
    flat = np.zeros(len(codes[x]), dtype=np.int64)
    size = 1
    for m in (x, y, *given):
        flat += codes[m] * size
        size *= cards[m]
    return np.bincount(flat, minlength=size).reshape(-1, cards[y], cards[x])


def statistic(tab, kind="g2"):
    """(statistic, dof, p-value) of a stratified table [n_strata, r_y, r_x] of counts."""
    tab = np.asarray(tab, dtype=np.float64)
    nxz = tab.sum(axis=1)[:, None, :]
    nyz = tab.sum(axis=2)[:, :, None]
    nz = tab.sum(axis=(1, 2))[:, None, None]
    if kind == "g2":
        nz_b = np.broadcast_to(nz, tab.shape)
        nx_b, ny_b = np.broadcast_to(nxz, tab.shape), np.broadcast_to(nyz, tab.shape)
        cell = tab > 0
        n = tab[cell]
        stat = 2.0 * float(np.sum(n * np.log(n * nz_b[cell] / (nx_b[cell] * ny_b[cell]))))
    elif kind == "chi2":
        with np.errstate(invalid="ignore", divide="ignore"):
            e = nxz * nyz / nz
        cell = np.isfinite(e) & (e > 0)
        stat = float(np.sum((tab[cell] - e[cell]) ** 2 / e[cell]))
    else:
        raise ValueError(kind)
    a = (tab.sum(axis=1) > 0).sum(axis=1)
    b = (tab.sum(axis=2) > 0).sum(axis=1)
    dof = int(np.sum(np.where(tab.sum(axis=(1, 2)) > 0, (a - 1) * (b - 1), 0)))
    p = float(gammaincc(dof / 2.0, stat / 2.0)) if dof > 0 and stat > 0 else 1.0
    return stat, dof, p


def tester(X, kind="g2"):
    """A structure.pc_search tester on the data X: each test's p-value from `statistic`."""
    codes, cards = codes_of(X)

    def run(tests):
        return [statistic(table(codes, cards, x, y, given), kind)[2] for x, y, given in tests]

    return run


def table_entries(cards, x, y, given=()):
    return math.prod(cards[m] for m in (x, y, *given))
