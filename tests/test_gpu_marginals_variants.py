"""Marginals programs (the readout kernel sbn_marginal_step and the downward-pass messages) on every
network of the variant corpus (tests/kernel_corpus.py: build_marginals), against the float64 oracle.

Per network, the plan targets every variable that is not evidence.  The reference is the float64 CPU
interpreter of the same plan (oracle/program_interp.py), itself held to ve_oracle.query on a sample
of rows.  Every entry of every row is checked, at row counts around the readout's 128-thread CTA and
the step kernels' edges: 1e-6 relative, exact zeros exactly 0, impossible rows NaN, and a NaN segment
on a possible row only where the float32 range rule explains it.  The float64 batch and the float64
single-event program hold 1e-12, on the rows float32 flags as well; the batch run in 128-row pieces
equals the single run bit for bit; the plain kernel and the branched graph agree within 3e-6.

The coverage test takes the kernel census of every network's programs in a fresh interpreter (after
many profiler sessions in one process the profiler stops recording): every `<T, C>` instantiation of
the readout kernel runs, every readout path the plans show is reached, and no marginals run
normalises separately.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import kernel_census
import kernel_corpus
from oracle import program_interp, ve_oracle

pytestmark = pytest.mark.gpu

RTOL = 1e-6
ROW_COUNTS = (1, 2, 127, 128, 129, 255, 257, 513)
N_MAX = max(ROW_COUNTS)
BIG_NAME = "grid10x10s5_seed0_q99_e30"
BIG_ROWS = 8449  # past the join kernel's 2 x SMs x R rows, R = 32, on 132 SMs


class MCase:
    """The programs of one corpus network's marginals plan: default dispatch, plain kernel, branched
    graph, float64 batch and the float64 single-event program; its evidence rows, the float64
    interpreter's answer for them and P(e) of every row."""

    def __init__(self, name, n_rows=N_MAX, reference=True):
        from sorobn_b200 import engine, planner

        self.name = name
        self.spec, self.net, self.dn, self.plan, self.evidence = kernel_corpus.build_marginals(name)
        self.n = n_rows
        self.codes = kernel_corpus.evidence_rows(self.spec, self.evidence, n_rows, seed=1)
        self.starts = program_interp.segment_starts(self.plan)
        if reference:  # the census needs the programs only
            self.want = program_interp.run_marginals(self.plan.words, self.plan.table_blob64, self.codes, n_rows=n_rows)
            self.p_e = np.array([self.evidence_probability(b) for b in range(n_rows)])
        self.default = engine.Program(self.plan)
        self.plain = engine.Program(self.plan)
        self.plain.set_tiled(0)
        self.branched = engine.Program(self.plan)
        self.branched.set_graph(3)
        self.batched64 = engine.Program(self.plan, f64=True)
        flat = planner.build_marginals_plan(self.net, list(self.plan.evidence), mode=planner.MODE_FLAT)
        assert flat.Q == self.plan.Q and list(flat.targets) == list(self.plan.targets)
        self.flat64 = engine.Program(flat, f64=True)

    def event(self, b):
        return dict(zip(self.evidence, (int(x) for x in self.codes[:, b])))

    def evidence_probability(self, b):
        return ve_oracle.evidence_probability(self.dn, self.event(b)) if self.evidence else 1.0

    def census_runs(self):
        """The census switches graph replay off and back on, so the branched program stays out."""
        return [(p, self.codes, self.n) for p in (self.default, self.plain, self.batched64)] + \
            [(self.flat64, np.ascontiguousarray(self.codes[:, :1]), 1)]

    def check_oracle(self, rows):
        """The float64 interpreter against ve_oracle.query, every target, on `rows`."""
        for b in rows:
            if self.p_e[b] == 0:
                assert np.isnan(self.want[:, b]).all(), b
                continue
            ev = self.event(b)
            for t, q0 in zip(self.plan.targets, self.starts):
                ref = ve_oracle.query(self.dn, self.net.names[t], event=ev)[1].reshape(-1)
                got = self.want[q0:q0 + len(ref), b]
                assert np.allclose(got, ref, rtol=1e-12, atol=1e-300), (b, self.net.names[t], got, ref)
                assert (got[ref == 0] == 0).all(), (b, self.net.names[t], got, ref)

    def close(self):
        for p in (self.default, self.plain, self.branched, self.batched64, self.flat64):
            p.close()


def oracle_rows(case, n):
    k = 4 if len(case.plan.targets) > 100 else 8
    return sorted({0, n - 1, *np.linspace(0, n - 1, k).astype(int).tolist()})


@pytest.mark.parametrize("name", kernel_corpus.MARGINALS_CASES)
def test_marginals_case_matches_oracle(name):
    c = MCase(name)
    codes = c.codes
    c.check_oracle(oracle_rows(c, N_MAX))
    full = None
    for n in ROW_COUNTS:
        out = c.default.run(np.ascontiguousarray(codes[:, :n]), n)
        worst, _ = program_interp.check_posterior(out, c.want[:, :n], c.starts, p_event=c.p_e[:n])
        assert worst < RTOL, (n, worst)
        full = out
    flagged = np.flatnonzero(np.isnan(full).any(axis=0) & ~np.isnan(c.want).all(axis=0))
    # the same batch as 128-row pieces, the last one partial, on a fresh program
    chunked = type(c.default)(c.plan)
    pieces = [chunked.run(np.ascontiguousarray(codes[:, lo:lo + 128]), min(128, N_MAX - lo)) for lo in range(0, N_MAX, 128)]
    assert np.array_equal(np.concatenate(pieces, axis=1), full, equal_nan=True)
    chunked.close()
    # the plain kernel and the branched graph
    for other in (c.plain, c.branched):
        assert np.allclose(other.run(codes, N_MAX), full, rtol=3e-6, atol=1e-30, equal_nan=True)
    # float64: the batch on every row, the single-event program on the edge rows and the flagged ones
    worst, _ = program_interp.check_posterior(c.batched64.run(codes, N_MAX), c.want, c.starts)
    assert worst < 1e-12, worst
    for b in sorted({0, N_MAX - 1, *flagged[:4].tolist()}):
        one = np.ascontiguousarray(codes[:, b:b + 1])
        worst, _ = program_interp.check_posterior(c.flat64.run(one, 1), c.want[:, b:b + 1], c.starts)
        assert worst < 1e-12, (b, worst)
    c.close()


def test_large_batch_on_the_benchmark_grid():
    """One batch past the join kernel's row threshold (whether it runs is recorded by the coverage
    test): every entry against the float64 interpreter, a sample of rows against the oracle."""
    c = MCase(BIG_NAME, BIG_ROWS)
    out = c.default.run(c.codes, BIG_ROWS)
    worst, _ = program_interp.check_posterior(out, c.want, c.starts, p_event=c.p_e)
    assert worst < RTOL, worst
    c.check_oracle(oracle_rows(c, BIG_ROWS))
    c.close()


_CENSUS_SCRIPT = """
import json, sys
import kernel_census, kernel_corpus
import test_gpu_marginals_variants as T
cases = [T.MCase(name, reference=False) for name in kernel_corpus.MARGINALS_CASES]
big = T.MCase(T.BIG_NAME, T.BIG_ROWS, reference=False)
runs = [r for c in cases for r in c.census_runs()] + [(big.default, big.codes, T.BIG_ROWS)]
seen = kernel_census.census_many(runs)
k = len(cases[0].census_runs())
out = {c.name: [name for s in seen[i * k:(i + 1) * k] for name, _ in s] for i, c in enumerate(cases)}
out["big"] = [name for name, _ in seen[-1]]
json.dump(out, sys.stdout)
"""


def test_marginals_corpus_covers_the_readout_variants():
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, "-c", _CENSUS_SCRIPT], capture_output=True, text=True, env=env, cwd=here,
                         timeout=1800)
    assert res.returncode == 0, res.stderr[-3000:]
    census = json.loads(res.stdout)
    seen = {}
    for name in kernel_corpus.MARGINALS_CASES:
        names = census[name]
        assert names, f"{name}: the profiler recorded no kernel"
        assert not any("normalise" in n for n in names), (name, names)
        plan = kernel_corpus.build_marginals(name)[3]
        seen[name] = kernel_census.variants([(n, 1) for n in names]) | kernel_corpus.readout_items(plan)
    required = [f"marginal<{t},{c}>" for t in ("float", "double") for c in (2, 4, 8)] + list(kernel_corpus.READOUT_ITEMS)
    lines = []
    for item in required:
        hits = [name for name, s in seen.items() if item in s]
        lines.append(f"  {item:<26} " + (f"hit by {len(hits)}: {hits[0]}" if hits else "NOT HIT"))
    big = kernel_census.variants([(n, 1) for n in census["big"]])
    assert not any("normalise" in n for n in census["big"]), census["big"]
    assert "marginal<float,8>" in big, census["big"]
    joins = sorted(i for i in big if i.startswith("join"))
    lines.append(f"  {BIG_ROWS} rows of {BIG_NAME}: join kernel " + (", ".join(joins) if joins else "not launched"))
    print("\nmarginals coverage\n" + "\n".join(lines))
    union = set().union(*seen.values())
    assert set(required) <= union, sorted(set(required) - union)
