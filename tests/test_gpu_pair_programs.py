"""The paired-step and expanding-product kernels (`csrc/sbn_pair.cu`) on the hand-built programs of
tests/pair_programs.py, against the float64 interpreter of the same words.

Per case, at row counts around the pair kernel's 256-row CTA (and, for the case with 125 tiles, at a
count where one CTA walks several tiles and the last chunk is partial): every entry within 1e-6 of
the interpreter (exact zeros exact, impossible rows all NaN), P(event), the same program without
paired steps, the float64 batch, bitwise repeatability with and without graph replay, bitwise
equality with the batch run in 128-row pieces, the step roles, and the kernel census.  The
coverage test requires all 15 (m1, m2) mode pairs and both triple groups.  The census is taken in a
fresh interpreter: after many profiler sessions in one process the profiler stops recording.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import kernel_census
import pair_programs as pp
from oracle import program_interp
from test_gpu_kernel_variants import check_row

pytestmark = pytest.mark.gpu

RTOL = 1e-6
ROW_COUNTS = (1, 2, 255, 256, 257, 513)
CENSUS_ROWS = 513


def _n_sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def row_counts(case):
    if case["multi_chunk"] is None:
        return ROW_COUNTS
    return ROW_COUNTS + (pp.multi_chunk_rows(case["multi_chunk"], _n_sms()),)


class Case:
    def __init__(self, case):
        from sorobn_b200 import engine

        self.case = case
        self.built = pp.build(case)
        plan = self.built.plan
        self.codes = pp.evidence_rows(self.built, max(row_counts(case)), seed=1)
        uniq, inv = pp.unique_rows(self.codes)
        want, totals = program_interp.run(plan.words, plan.table_blob64, uniq, n_rows=uniq.shape[1], return_totals=True)
        self.want, self.totals = want[:, inv], totals[inv]
        self.default = engine.Program(plan)
        self.pieces = engine.Program(plan)
        self.f64 = engine.Program(plan, f64=True)

    def close(self):
        for p in (self.default, self.pieces, self.f64):
            p.close()


_CENSUS_SCRIPT = f"""
import json, sys
import numpy as np
import kernel_census, pair_programs as pp
from sorobn_b200 import engine
runs = []
for case in pp.CASES:
    built = pp.build(case)
    runs.append((engine.Program(built.plan), pp.evidence_rows(built, {CENSUS_ROWS}, seed=1), {CENSUS_ROWS}))
json.dump([s for s in kernel_census.census_many(runs)], sys.stdout)
"""


@pytest.fixture(scope="module")
def census():
    """kernel_census.variants of each case's default program at CENSUS_ROWS rows."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, "-c", _CENSUS_SCRIPT], capture_output=True, text=True, env=env, cwd=here,
                         timeout=1800)
    assert res.returncode == 0, res.stderr[-3000:]
    seen = json.loads(res.stdout)
    return {c["name"]: kernel_census.variants([tuple(k) for k in s]) for c, s in zip(pp.CASES, seen)}


def _check_rows(got, want, rtol):
    for b in range(got.shape[1]):
        check_row(got[:, b], want[:, b], rtol)


@pytest.mark.parametrize("case", pp.CASES, ids=pp.case_id)
def test_pair_program_matches_the_interpreter(case, census):
    c = Case(case)
    prog = c.default
    if case["roles"] is not None:
        assert prog.step_roles().tolist() == case["roles"], (prog.step_roles(), case["branch"])
    fused = {v for v in census[case["name"]] if v.startswith(("pair", "triple"))}
    assert fused == ({case["census"]} if case["census"] else set()), (fused, case["branch"])

    for n in row_counts(case):
        codes = np.ascontiguousarray(c.codes[:, :n])
        want = c.want[:, :n]
        out = prog.run(codes, n).copy()
        _check_rows(out, want, RTOL)
        # P(event): NaN where the event is impossible
        p = prog.evidence(codes, n)
        tot = c.totals[:n]
        assert np.isnan(p[tot == 0]).all()
        assert np.all(np.abs(p[tot > 0] - tot[tot > 0]) <= RTOL * tot[tot > 0]), n
        # repeatable bit for bit: graph replay, then plain launches
        assert np.array_equal(prog.run(codes, n), out, equal_nan=True)
        prog.set_graph(False)
        assert np.array_equal(prog.run(codes, n), out, equal_nan=True)
        prog.set_graph(True)
        # the per-row arithmetic does not depend on the batch: 128-row pieces give the same bits
        pieces = [c.pieces.run(np.ascontiguousarray(codes[:, lo:lo + 128]), min(128, n - lo)) for lo in range(0, n, 128)]
        assert np.array_equal(np.concatenate(pieces, axis=1), out, equal_nan=True), n
        # one launch per step
        prog.set_tiled(10)
        single = prog.run(codes, n).copy()
        prog.set_tiled(11)
        assert np.allclose(single, out, rtol=3e-6, atol=1e-30, equal_nan=True), n
        _check_rows(single, want, RTOL)
        # the float64 batch (no paired steps)
        _check_rows(c.f64.run(codes, n), want, 1e-12)
    c.close()


def test_pair_programs_cover_every_mode_pair_and_triple_group(census):
    union = set().union(*census.values())
    required = [f"pair ({m1},{m2})" for m1 in range(5) for m2 in range(3)] + ["triple group=1", "triple group=5"]
    lines = []
    for item in required:
        hits = [name for name, s in census.items() if item in s]
        lines.append(f"  {item:<16} " + (f"reached by {len(hits)}: {', '.join(hits)}" if hits else "MISSING"))
    print("\npaired-step coverage\n" + "\n".join(lines))
    assert set(required) <= union, sorted(set(required) - union)
