"""Every log-domain step instantiation on the device, over the variant corpus (kernel_corpus.LOG_DOMAIN_CASES: every
corpus case, and a naive Bayes network whose marginal MAP log P lies far below float32's range).

The MPE program of a case (planner.build_mpe_plan) and its marginal MAP programs (planner.build_map_plan, the sets
of kernel_corpus.MAP_SETS) run the max-sum and log-sum-exp instantiations of sbn_step_batched (N_IN = 1 .. 8) and
sbn_step_flat, and sbn_argmax_step.  Per program:
  * runs at row counts around the batched kernel's 512-row CTA and the argmax kernel's 128-row CTA, and on two
    cases around kSampleGraphMinRows (4,096: plain launches below, a captured graph from it); every run equals the
    largest one's rows bit for bit, as do its 128-row pieces and its plain launches;
  * MPE: codes and float32 log P bitwise equal to the float32 replay of the words (oracle/program_interp.py) --
    additions and maxima only; marginal MAP: log P within 4e-6 x max(1, |r|) of the replay (expf / logf differ
    from numpy's in the last bits), the same -inf rows, and a decision that differs from the replay's a near-tie
    under the float64 oracle;
  * against the float64 oracles (tests/mpe_oracle.py, tests/map_oracle.py) on the first LOG_DOMAIN_ORACLE_ROWS
    rows: log P within 2e-5 x max(1, |L*|), and a decoded state that is not the oracle's a near-tie;
  * no NaN anywhere.
The census of every program is taken once, in a fresh interpreter, with each program created inside its profiled
run (its evidence-independent kind-0 steps, the only launches of the flat log-domain kernels, run at creation).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import kernel_census
import kernel_corpus
from oracle import program_interp
from sorobn_b200 import engine, planner
from test_log_domain_corpus import LOG_FLT_MIN, Oracle, programs

pytestmark = pytest.mark.gpu

ROW_COUNTS = (1, 2, 3, 5, 127, 128, 129, 511, 512, 513)
GRAPH_ROW_COUNTS = (4095, 4096, 4097)  # around kSampleGraphMinRows (csrc/sbn_api.cu)
GRAPH_CASES = ("grid7x7s5_seed39_q48_e18", "dag300p1s17_seed34_q0_e8")
RTOL = 4e-6  # device against the float32 replay of a marginal MAP program, x max(1, |r|)
TOL = 2e-5  # against the float64 oracle: a near-tie under float32 rounding, x max(1, |L*|)
CENSUS_ROWS = 513
ORACLE_ROWS = kernel_corpus.LOG_DOMAIN_ORACLE_ROWS


def row_counts(name):
    return ROW_COUNTS + (GRAPH_ROW_COUNTS if name in GRAPH_CASES else ())


def bitwise(a, b):
    return a[0].shape == b[0].shape and np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


def run_everywhere(program, codes, counts):
    """The run of every row count and the largest run's 128-row pieces and plain launches, each bitwise equal to
    the largest run's rows.  Returns the largest run (decoded, log P)."""
    decode = program.map if program.plan.version == planner.VERSION_MAP else program.mpe
    n = max(counts)
    whole = decode(codes, n)
    assert whole[1].dtype == np.float32 and not np.isnan(whole[1]).any()
    for k in counts:
        part = decode(np.ascontiguousarray(codes[:, :k]), k)
        assert bitwise(part, (whole[0][:, :k], whole[1][:k])), k
    pieces = [decode(np.ascontiguousarray(codes[:, lo:lo + 128]), min(128, n - lo)) for lo in range(0, n, 128)]
    assert bitwise((np.concatenate([p[0] for p in pieces], axis=1), np.concatenate([p[1] for p in pieces])), whole)
    program.set_graph(False)
    assert bitwise(decode(codes, n), whole)
    program.set_graph(True)
    return whole


@pytest.mark.parametrize("name", kernel_corpus.LOG_DOMAIN_CASES)
def test_mpe_equals_the_float32_replay_bitwise_and_agrees_with_the_oracle(name):
    counts = row_counts(name)
    net, dn, observed, codes, plans = programs(name, max(counts))
    _, plan = plans[0]
    program = engine.Program(plan, device=0)
    got, lp = run_everywhere(program, codes, counts)
    program.close()
    want, wlp = program_interp.run_mpe(plan.words, plan.table_blob, codes, dtype=np.float32)
    assert bitwise((got, lp), (want, wlp))
    oracle = Oracle(net, dn, observed, plan, codes)
    ties = sum(oracle.check(b, got[:, b], lp[b], TOL) for b in range(ORACLE_ROWS))
    print(f"\n{name}: {ties} near-tie(s) of {ORACLE_ROWS} rows")


@pytest.mark.parametrize("name", kernel_corpus.LOG_DOMAIN_CASES)
def test_map_agrees_with_the_float32_replay_and_the_oracle(name):
    counts = row_counts(name)
    net, dn, observed, codes, plans = programs(name, max(counts))
    for label, plan in plans[1:]:
        program = engine.Program(plan, device=0)
        got, lp = run_everywhere(program, codes, counts)
        program.close()
        want, wlp = program_interp.run_mpe(plan.words, plan.table_blob, codes, dtype=np.float32)
        assert got.shape == want.shape
        fin = np.isfinite(wlp)
        assert np.array_equal(np.isfinite(lp), fin) and np.array_equal(lp[~fin], wlp[~fin]), label
        r = wlp[fin].astype(np.float64)
        assert np.all(np.abs(lp[fin] - r) <= RTOL * np.maximum(1.0, np.abs(r))), label
        oracle = Oracle(net, dn, observed, plan, codes)
        differ = np.flatnonzero((got != want).any(axis=0))
        for b in differ:  # a decision the replay makes otherwise: a near-tie under the oracle
            _, L, gap = oracle(b)
            t = TOL * max(1.0, abs(L))
            assert gap <= t and abs(oracle.log_p(b, got[:, b]) - L) <= t, (label, b)
        for b in range(ORACLE_ROWS):
            oracle.check(b, got[:, b], lp[b], TOL)
        if name == kernel_corpus.NAIVE_BAYES_60:
            lo, hi = kernel_corpus.NAIVE_BAYES_60_LOG_P
            L = np.array([oracle(b)[1] for b in range(ORACLE_ROWS)])
            assert lo <= L.min() and L.max() <= hi < LOG_FLT_MIN, (L.min(), L.max())
        print(f"\n{name} {label}: {len(differ)} of {codes.shape[1]} row(s) decode a near-tie differently from the replay")


class _Created:
    """A census run of one plan: the program is created inside the profiled run, decodes the rows with plain
    launches and is closed."""

    def __init__(self, plan):
        self.plan = plan

    def set_graph(self, mode):
        pass

    def run(self, codes, n_rows):
        program = engine.Program(self.plan, device=0)
        program.set_graph(False)
        program.mpe(codes, n_rows)
        program.close()


def census_items():
    """Coverage items of every log-domain case: the census of its programs, plus what its plans show."""
    runs, owners = [], []
    for name in kernel_corpus.LOG_DOMAIN_CASES:
        _, _, _, codes, plans = programs(name, CENSUS_ROWS)
        for _, plan in plans:
            runs.append((_Created(plan), codes, CENSUS_ROWS))
            owners.append((name, plan))
    out = {name: set() for name in kernel_corpus.LOG_DOMAIN_CASES}
    for (name, plan), seen in zip(owners, kernel_census.census_many(runs)):
        out[name] |= kernel_census.variants(seen) | kernel_corpus.log_domain_items(plan)
    return {name: sorted(items) for name, items in out.items()}


_CENSUS_SCRIPT = """
import json, sys
import test_gpu_log_domain_variants as T
json.dump(T.census_items(), sys.stdout)
"""


@pytest.fixture(scope="module")
def log_domain_items():
    """Coverage items of every log-domain case (`census_items`), taken in a fresh interpreter."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, "-c", _CENSUS_SCRIPT], capture_output=True, text=True, env=env, cwd=here,
                         timeout=1800)
    assert res.returncode == 0, res.stderr[-3000:]
    return {name: set(items) for name, items in json.loads(res.stdout).items()}


@pytest.mark.parametrize("name", kernel_corpus.LOG_DOMAIN_CASES)
def test_log_domain_case_reaches_its_claims(name, log_domain_items):
    seen = log_domain_items[name]
    claims = set(kernel_corpus.LOG_DOMAIN_CLAIMS[name])
    assert claims <= seen, sorted(claims - seen)
    assert seen <= kernel_corpus.log_domain_required_items(), sorted(seen - kernel_corpus.log_domain_required_items())


def test_log_domain_corpus_covers_the_required_items(log_domain_items):
    """Each required item is reached by some case, or listed in LOG_DOMAIN_OPEN, which no case may reach."""
    seen = log_domain_items
    union = set().union(*seen.values())
    required = kernel_corpus.log_domain_required_items()
    lines = []
    for item in sorted(required):
        hits = [name for name, s in seen.items() if item in s]
        status = f"hit by {len(hits)}: {hits[0]}" if hits else "OPEN: " + kernel_corpus.LOG_DOMAIN_OPEN.get(item, "(not listed)")
        lines.append(f"  {item:<36} {status}")
    print("\nlog-domain coverage\n" + "\n".join(lines))
    missing = required - union - set(kernel_corpus.LOG_DOMAIN_OPEN)
    assert not missing, sorted(missing)
    assert not union & set(kernel_corpus.LOG_DOMAIN_OPEN), \
        f"now reached, move into a case's claims: {sorted(union & set(kernel_corpus.LOG_DOMAIN_OPEN))}"
