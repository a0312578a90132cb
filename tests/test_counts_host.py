"""The host side of expected_counts / fit_em, on the CPU: the device programs are replaced by the
version-6 interpreter (oracle/program_interp.py), which refuses to run after close() as a real program
handle does."""
import numpy as np
import pandas as pd
import pytest

import em_oracle
from interpreted_program import InterpretedProgram
from oracle import ve_oracle
from sorobn_b200 import engine, examples, workloads


@pytest.fixture
def interpreted(monkeypatch):
    InterpretedProgram.live = []
    monkeypatch.setattr(engine, "Program", InterpretedProgram)
    return InterpretedProgram


def frame(bn, n, seed, frac):
    """n forward-sampled rows, every column missing independently in a fraction `frac` of them."""
    net = bn._compiled
    codes = workloads.forward_sample_codes(net, n, seed)
    rng = np.random.default_rng(seed + 1)
    cols = {}
    for v, name in enumerate(net.names):
        values = np.asarray(net.domains[v], dtype=object)[codes[v]]
        values[rng.random(n) < frac] = None
        cols[name] = values
    return pd.DataFrame(cols)


def oracle_counts(bn, X):
    rows = [{k: v for k, v in r.items() if v is not None and v == v} for r in X.to_dict("records")]
    return em_oracle.expected_counts(ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes), rows)


def test_more_patterns_than_cached_programs(interpreted):
    bn = examples.asia()
    bn.max_cached_programs = 8
    X = frame(bn, 400, 3, 0.3)
    n_patterns = len(bn._count_patterns(X))
    assert n_patterns > 3 * bn.max_cached_programs
    got = bn.expected_counts(X)
    want = oracle_counts(bn, X)
    for node, s in got.items():
        assert np.allclose(s.to_numpy(), want[node].reshape(-1), rtol=2e-6, atol=1e-9), node
    assert len(bn._engine_cache) <= bn.max_cached_programs
    # a second call reuses the cached programs it can and builds the others again
    again = bn.expected_counts(X)
    for node in got:
        assert np.array_equal(again[node].to_numpy(), got[node].to_numpy())


def test_fit_em_closes_its_programs_and_refuses_no_iterations(interpreted):
    bn = examples.sprinkler()
    X = frame(bn, 300, 4, 0.2)
    with pytest.raises(ValueError, match="max_iter"):
        bn.fit_em(X, max_iter=0)
    bn.fit_em(X, max_iter=5)
    assert 1 <= len(bn.em_log_likelihood_) <= 5
    lls = bn.em_log_likelihood_
    assert all(b >= a - 1e-6 * abs(a) for a, b in zip(lls, lls[1:])), lls
    assert interpreted.live and all(p.closed for p in interpreted.live)
