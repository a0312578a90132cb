"""`engine.Program` executed by the CPU interpreter (oracle/program_interp.py), for the host side of
expected_counts / fit_em, sample_many, mpe_many and map_many without a GPU.  Like a real program handle, it
refuses to run after close()."""
import numpy as np

from oracle import program_interp
from sorobn_b200 import engine, planner


class InterpretedProgram:
    """engine.Program for counts, sample, MPE and marginal MAP plans.  `live` lists every program created,
    `calls` every sample call as (f64, n_rows).  The float32 sample program flags the rows whose P(observed)
    is below `flag_below` (the range rule, raised so that the float64 path runs)."""

    live = []
    calls = []
    flag_below = None

    def __init__(self, plan, device=None, f64=False):
        assert not (f64 and plan.version in (planner.VERSION_MPE, planner.VERSION_MAP)), \
            "MPE and MAP programs run in float32 only"
        self.plan, self.f64 = plan, f64
        self.blob = plan.table_blob64 if f64 else plan.table_blob
        self.closed = False
        InterpretedProgram.live.append(self)

    def _check_open(self):
        if self.closed:
            raise engine.EngineError("libsorobn_b200 error -1: null program", code=-1)

    def counts(self, codes, n_rows):
        self._check_open()
        dtype = np.float64 if self.f64 else np.float32
        return program_interp.run_counts(self.plan.words, self.blob, codes, n_rows=n_rows, dtype=dtype)

    def sample(self, codes, n_rows, n_draws, seed, row_base=0):
        self._check_open()
        InterpretedProgram.calls.append((self.f64, int(n_rows)))
        min_total = None if self.f64 or self.flag_below is None else self.flag_below
        drawn, prob, _ = program_interp.run_sample(self.plan.words, self.plan.table_blob64, codes, n_rows=n_rows,
                                                   n_draws=n_draws, seed=seed, row_base=row_base, min_total=min_total)
        return drawn, prob.astype(np.float64 if self.f64 else np.float32)

    def mpe(self, codes, n_rows):
        self._check_open()
        return program_interp.run_mpe(self.plan.words, self.plan.table_blob, codes, n_rows=n_rows, dtype=np.float32)

    def map(self, codes, n_rows):
        assert self.plan.version == planner.VERSION_MAP
        return self.mpe(codes, n_rows)

    def set_tables(self, blob):
        self._check_open()
        self.blob = np.asarray(blob)

    def close(self):
        self.closed = True
