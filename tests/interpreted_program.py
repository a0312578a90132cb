"""`engine.Program` executed by the CPU interpreter (oracle/program_interp.py), for the host side of every
exact-inference entry point without a GPU.  Like a real program handle, it refuses to run after close()."""
import numpy as np

from oracle import program_interp
from sorobn_b200 import engine, planner


class InterpretedProgram:
    """engine.Program for posterior, marginals, counts, sample, MPE and marginal MAP plans.  `live` lists every
    program created, `calls` every run as (plan version, plan mode, f64, n_rows).  A float32 program flags the
    rows whose total (P(event) or P(observed)) is below `flag_below`: their posterior, P(event) or P(observed)
    comes back NaN, as under the device's range rule (raised so that the float64 path runs)."""

    live = []
    calls = []
    flag_below = None

    def __init__(self, plan, device=None, f64=False):
        assert not (f64 and plan.version in (planner.VERSION_MPE, planner.VERSION_MAP)), \
            "MPE and MAP programs run in float32 only"
        self.plan, self.f64 = plan, f64
        self.Q = plan.Q
        self.dtype = np.float64 if f64 else np.float32
        self.blob = plan.table_blob64 if f64 else plan.table_blob
        self.closed = False
        InterpretedProgram.live.append(self)

    def _start(self, n_rows):
        if self.closed:
            raise engine.EngineError("libsorobn_b200 error -1: null program", code=-1)
        InterpretedProgram.calls.append((self.plan.version, self.plan.mode, self.f64, int(n_rows)))

    def _min_total(self):
        return None if self.f64 or self.flag_below is None else self.flag_below

    def _posterior(self, codes, n_rows):
        """(posterior [Q, n_rows], P(event) [n_rows]) of a posterior or marginals plan (P(event) of posterior plans
        only), NaN where flagged; a flat plan takes one row at a time."""
        codes = np.asarray(codes, dtype=np.uint8)
        if self.plan.mode == planner.MODE_FLAT and n_rows != 1:
            parts = [self._posterior(codes[:, b:b + 1], 1) for b in range(n_rows)]
            return (np.concatenate([p for p, _ in parts], axis=1),
                    None if self.plan.version == planner.VERSION_MARGINALS else np.concatenate([t for _, t in parts]))
        if self.plan.version == planner.VERSION_MARGINALS:
            return program_interp.run_marginals(self.plan.words, self.blob, codes, n_rows=n_rows, dtype=self.dtype,
                                                min_total=self._min_total()), None
        post, total = program_interp.run(self.plan.words, self.blob, codes, n_rows=n_rows, dtype=self.dtype,
                                         return_totals=True)
        if self._min_total() is not None:
            low = ~(total >= self._min_total())
            post[:, low], total[low] = np.nan, np.nan
        return post, total

    def run(self, codes, n_rows):
        self._start(n_rows)
        return self._posterior(codes, n_rows)[0]

    def evidence(self, codes, n_rows):
        self._start(n_rows)
        assert self.plan.version == planner.VERSION, "only posterior programs give P(event)"
        return self._posterior(codes, n_rows)[1]

    def counts(self, codes, n_rows):
        self._start(n_rows)
        return program_interp.run_counts(self.plan.words, self.blob, codes, n_rows=n_rows, dtype=self.dtype,
                                         min_total=self._min_total())

    def sample(self, codes, n_rows, n_draws, seed, row_base=0):
        self._start(n_rows)
        drawn, prob, _ = program_interp.run_sample(self.plan.words, self.plan.table_blob64, codes, n_rows=n_rows,
                                                   n_draws=n_draws, seed=seed, row_base=row_base,
                                                   min_total=self._min_total())
        return drawn, prob.astype(self.dtype)

    def mpe(self, codes, n_rows):
        self._start(n_rows)
        return program_interp.run_mpe(self.plan.words, self.plan.table_blob, codes, n_rows=n_rows, dtype=np.float32)

    def map(self, codes, n_rows):
        assert self.plan.version == planner.VERSION_MAP
        return self.mpe(codes, n_rows)

    def set_tables(self, blob):
        if self.closed:
            raise engine.EngineError("libsorobn_b200 error -1: null program", code=-1)
        self.blob = np.asarray(blob)

    def close(self):
        self.closed = True
