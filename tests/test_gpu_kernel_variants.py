"""Every case of the variant corpus (tests/kernel_corpus.py) on the device, against the float64 oracle.

Per case: evidence rows from every joint code of the evidence columns (probability-zero codes
included) plus forward samples; runs at row counts around the CTA edges of the tiled (256 rows),
slab (128), pair (256) and triple (32 / 128) kernels; the batch run in 128-row pieces, which must
equal the single run bit for bit; the plain kernel and the unpaired program within 3e-6; the float32
and float64 single-event programs and the float64 batch; and the kernel census, which must show the
variants the case claims.  The coverage test checks the census of all cases against the required set.
The census of every case is taken once, in a fresh interpreter: after many profiler sessions in one
process the profiler stops recording some launches.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import kernel_census
import kernel_corpus
from oracle import ve_oracle

pytestmark = pytest.mark.gpu

RTOL = 1e-6
ROW_COUNTS = (1, 2, 3, 127, 129, 255, 256, 257, 513)
N_MAX = max(ROW_COUNTS)


def check_row(got, want, rtol):
    """`want` NaN (impossible evidence) -> `got` all NaN; otherwise relative error per entry, and
    exact zeros stay exactly zero."""
    if np.isnan(want).all():
        assert np.isnan(got).all(), got
        return
    assert np.isfinite(got).all(), (got, want)
    pos = want > 0
    assert (got[~pos] == 0).all(), (got, want)
    assert np.max(np.abs(got[pos] - want[pos]) / want[pos], initial=0.0) < rtol, (got, want)


class Case:
    """The programs of one corpus case: default dispatch, plain kernel, no paired steps, float64
    batch, and the float32 / float64 single-event programs."""

    def __init__(self, case):
        from sorobn_b200 import engine, planner

        self.case = case
        self.spec, self.net, self.dn, self.plan, self.query, self.evidence = kernel_corpus.build(case)
        self.codes = kernel_corpus.evidence_rows(self.spec, self.evidence, N_MAX, seed=case["seed"])
        self.one = np.ascontiguousarray(self.codes[:, :1])
        self.default = engine.Program(self.plan)
        self.plain = engine.Program(self.plan)
        self.plain.set_tiled(False)
        self.unpaired = engine.Program(self.plan)
        self.unpaired.set_tiled(10)
        self.batched64 = engine.Program(self.plan, f64=True)
        flat = planner.build_plan(self.net, list(self.plan.query), list(self.plan.evidence), mode=planner.MODE_FLAT)
        self.flat32 = engine.Program(flat)
        self.flat64 = engine.Program(flat, f64=True)

    def census_runs(self):
        return [(p, self.codes, N_MAX) for p in (self.default, self.plain, self.unpaired, self.batched64)] + \
            [(self.flat32, self.one, 1), (self.flat64, self.one, 1)]


def items_of(cases):
    """Coverage items each case reaches: the census of its programs, plus what its plan shows."""
    runs = [r for c in cases for r in c.census_runs()]
    seen = kernel_census.census_many(runs)
    k = len(cases[0].census_runs())
    return [set().union(*[kernel_census.variants(s) for s in seen[i * k:(i + 1) * k]]) | kernel_corpus.plan_items(c.plan)
            for i, c in enumerate(cases)]


_CENSUS_SCRIPT = """
import json, sys
import kernel_corpus, test_gpu_kernel_variants as T
json.dump([sorted(s) for s in T.items_of([T.Case(case) for case in kernel_corpus.CASES])], sys.stdout)
"""


@pytest.fixture(scope="module")
def corpus_items():
    """Coverage items of every corpus case (`items_of`), taken in a fresh interpreter."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, "-c", _CENSUS_SCRIPT], capture_output=True, text=True, env=env, cwd=here,
                         timeout=1800)
    assert res.returncode == 0, res.stderr[-3000:]
    return {case["name"]: set(items) for case, items in zip(kernel_corpus.CASES, json.loads(res.stdout))}


@pytest.mark.parametrize("case", kernel_corpus.CASES, ids=kernel_corpus.case_id)
def test_variant_case_matches_oracle(case, corpus_items):
    c = Case(case)
    order = [c.net.names[v] for v in c.plan.order]
    codes = c.codes
    cache = {}

    def want(b):
        key = tuple(int(x) for x in codes[:, b])
        if key not in cache:
            ev = dict(zip(c.evidence, key))
            post = ve_oracle.query(c.dn, *c.query, event=ev, order=order)[1].reshape(-1)
            cache[key] = (post, ve_oracle.evidence_probability(c.dn, ev) if ev else 1.0)
        return cache[key]

    full = None
    for n in ROW_COUNTS:
        out = c.default.run(np.ascontiguousarray(codes[:, :n]), n)
        for b in range(n):
            check_row(out[:, b], want(b)[0], RTOL)
        full = out
    # P(event) per row; NaN where the event is impossible
    p = c.default.evidence(codes, N_MAX)
    for b in range(N_MAX):
        w = want(b)[1]
        if w == 0:
            assert np.isnan(p[b]), (b, p[b])
        else:
            assert abs(p[b] - w) <= RTOL * w, (b, p[b], w)
    # the same batch as 128-row pieces, the last one partial, on a fresh program
    chunked = type(c.default)(c.plan)
    pieces = [chunked.run(np.ascontiguousarray(codes[:, lo:lo + 128]), min(128, N_MAX - lo)) for lo in range(0, N_MAX, 128)]
    assert np.array_equal(np.concatenate(pieces, axis=1), full, equal_nan=True)
    # the plain kernel and the program without paired steps
    for other in (c.plain, c.unpaired):
        assert np.allclose(other.run(codes, N_MAX), full, rtol=3e-6, atol=1e-30, equal_nan=True)
    # single-event programs (flat kernel) in float32 and float64, and the batched float64 program
    check_row(c.flat32.run(c.one, 1)[:, 0], want(0)[0], RTOL)
    check_row(c.flat64.run(c.one, 1)[:, 0], want(0)[0], 1e-12)
    out64 = c.batched64.run(codes, N_MAX)
    for b in range(N_MAX):
        check_row(out64[:, b], want(b)[0], 1e-12)

    seen = corpus_items[case["name"]]
    assert set(case["claims"]) <= seen, sorted(set(case["claims"]) - seen)
    assert not seen & set(kernel_corpus.UNREACHABLE), sorted(seen & set(kernel_corpus.UNREACHABLE))


def test_variant_corpus_covers_the_required_items(corpus_items):
    """The census of every corpus case: each required item is reached by some case, or listed in
    UNREACHABLE (a reason from the dispatch code) or OPEN, which no case may reach."""
    seen = corpus_items
    union = set().union(*seen.values())
    lines = []
    for item in sorted(kernel_corpus.required_items()):
        hits = [name for name, s in seen.items() if item in s]
        if hits:
            status = f"hit by {len(hits)}: {hits[0]}"
        elif item in kernel_corpus.UNREACHABLE:
            status = "UNREACHABLE: " + kernel_corpus.UNREACHABLE[item]
        else:
            status = "OPEN: " + kernel_corpus.OPEN.get(item, "(not listed)")
        lines.append(f"  {item:<36} {status}")
    print("\nvariant coverage\n" + "\n".join(lines))
    missing = kernel_corpus.required_items() - union - set(kernel_corpus.UNREACHABLE) - set(kernel_corpus.OPEN)
    assert not missing, sorted(missing)
    assert not union & set(kernel_corpus.UNREACHABLE), sorted(union & set(kernel_corpus.UNREACHABLE))
    assert not union & set(kernel_corpus.OPEN), f"now reached, move into a case's claims: {sorted(union & set(kernel_corpus.OPEN))}"
