"""ctypes shim over libsorobn_b200.so (the C ABI in include/sorobn_b200.h).

This is the "thin C-ABI/ctypes shim" between the Python host (`BayesNet.query`) and
the CUDA kernels.  There is deliberately no fallback: if the library has not been
built (`python -m sorobn_b200.csrc.build` / `__graft_entry__.build()`), cannot be
loaded, or no sm_90 GPU is visible, construction raises.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libsorobn_b200.so")
_lib = None

SBN_OK = 0
ABI_VERSION = 22


class EngineError(RuntimeError):
    """An error reported by libsorobn_b200; `code` is the SBN_E_* value (-3 = device memory)."""

    def __init__(self, message, code=None):
        super().__init__(message)
        self.code = code


SBN_E_NOMEM = -3


def lib_path() -> str:
    return _LIB_PATH


def load():
    """Load the shared library and declare every entry point of include/sorobn_b200.h."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise EngineError(
            f"{_LIB_PATH} is missing: build the CUDA library first "
            "(python -m sorobn_b200.csrc.build, or __graft_entry__.build()). "
            "sorobn_b200 has no CPU fallback for exact inference."
        )
    lib = ctypes.CDLL(_LIB_PATH)
    c = ctypes
    vp, i64, i32 = c.c_void_p, c.c_int64, c.c_int
    lib.sbn_abi_version.restype = i32
    lib.sbn_abi_version.argtypes = []
    lib.sbn_last_error.restype = c.c_char_p
    lib.sbn_last_error.argtypes = []
    lib.sbn_device_count.restype = i32
    lib.sbn_device_count.argtypes = [c.POINTER(i32)]
    lib.sbn_program_create.restype = i32
    lib.sbn_program_create.argtypes = [i32, vp, i64, vp, i64, c.POINTER(vp)]
    lib.sbn_program_create_f64.restype = i32
    lib.sbn_program_create_f64.argtypes = [i32, vp, i64, vp, i64, c.POINTER(vp)]
    lib.sbn_program_run_host_f64.restype = i32
    lib.sbn_program_run_host_f64.argtypes = [vp, vp, i64, i64, vp, i64]
    lib.sbn_program_evidence_host.restype = i32
    lib.sbn_program_evidence_host.argtypes = [vp, vp, i64, i64, vp]
    lib.sbn_program_evidence_host_f64.restype = i32
    lib.sbn_program_evidence_host_f64.argtypes = [vp, vp, i64, i64, vp]
    for name in ("sbn_program_counts_host", "sbn_program_counts_host_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = [vp, vp, i64, i64, vp, i64, vp]
    for name in ("sbn_program_set_tables", "sbn_program_set_tables_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = [vp, vp, i64]
    for name in ("sbn_program_sample_host", "sbn_program_sample_host_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = [vp, vp, i64, i64, i64, c.c_uint64, i64, vp, vp]
    lib.sbn_program_mpe_host.restype = i32
    for name in ("sbn_program_run_soft_host", "sbn_program_run_soft_host_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = [vp, vp, i64, i64, vp, i64, i32, vp, i64, vp]
    lib.sbn_program_mpe_host.argtypes = [vp, vp, i64, i64, vp, vp]
    for name in ("sbn_program_counts_soft_host", "sbn_program_counts_soft_host_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = [vp, vp, i64, i64, vp, i64, i32, vp, i64, vp, vp]
    for name in ("sbn_program_sample_soft_host", "sbn_program_sample_soft_host_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = [vp, vp, i64, i64, vp, i64, i32, i64, c.c_uint64, i64, vp, vp, vp]
    lib.sbn_program_mpe_soft_host.restype = i32
    lib.sbn_program_mpe_soft_host.argtypes = [vp, vp, i64, i64, vp, i64, i32, vp, vp]
    for name in ("sbn_program_grad_forward_host", "sbn_program_grad_forward_host_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = [vp, vp, i64, i64, vp, i64, i32, vp, vp]
    for name in ("sbn_program_grad_backward_host", "sbn_program_grad_backward_host_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = [vp, vp, i64, i64, vp, i64, i32, vp, i32, vp, i64, vp, i64, vp]
    for name in ("sbn_program_joint_host", "sbn_program_joint_host_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = [vp, vp, i64, i64, vp, i64, i32, vp, i64, vp]
    lib.sbn_program_destroy.restype = None
    lib.sbn_program_destroy.argtypes = [vp]
    lib.sbn_program_reserve.restype = i32
    lib.sbn_program_reserve.argtypes = [vp, i64]
    lib.sbn_program_run_host.restype = i32
    lib.sbn_program_run_host.argtypes = [vp, vp, i64, i64, vp, i64]
    lib.sbn_program_run_device.restype = i32
    lib.sbn_program_run_device.argtypes = [vp, vp, i64, i64, vp, i64, vp]
    lib.sbn_program_step_roles.restype = i32
    lib.sbn_program_step_roles.argtypes = [vp, vp, i64]
    lib.sbn_program_profile.restype = i32
    lib.sbn_program_profile.argtypes = [vp, vp, i64, i64, vp, i64, vp, vp, i64]
    lib.sbn_program_info.restype = i32
    lib.sbn_program_info.argtypes = [vp, vp, i64]
    lib.sbn_program_set_graph.restype = i32
    lib.sbn_program_set_graph.argtypes = [vp, i32]
    lib.sbn_program_set_tiled.restype = i32
    lib.sbn_program_set_tiled.argtypes = [vp, i32]
    lib.sbn_gibbs_create.restype = i32
    lib.sbn_gibbs_create.argtypes = [i32, i32, vp, vp, vp, vp, vp, i64, i32, vp, i32, vp, i32, vp, c.POINTER(vp)]
    lib.sbn_gibbs_run_host.restype = i32
    lib.sbn_gibbs_run_host.argtypes = [vp, vp, i64, i64, i64, c.c_uint64, vp, i64]
    lib.sbn_sampler_run_host.restype = i32
    lib.sbn_sampler_run_host.argtypes = [vp, i32, vp, i64, i64, i64, c.c_uint64, vp, i64]
    lib.sbn_gibbs_conditional.restype = i32
    lib.sbn_gibbs_conditional.argtypes = [vp, i32, vp, vp]
    lib.sbn_gibbs_destroy.restype = None
    lib.sbn_gibbs_destroy.argtypes = [vp]
    lib.sbn_tally_create.restype = i32
    lib.sbn_tally_create.argtypes = [i32, vp, i64, i32, i64, vp, c.POINTER(vp)]
    lib.sbn_tally_counts.restype = i32
    lib.sbn_tally_counts.argtypes = [vp, vp, i64, vp, i64]
    lib.sbn_tally_scores.restype = i32
    lib.sbn_tally_scores.argtypes = [vp, vp, i64, i32, c.c_double, vp, i64]
    lib.sbn_tally_tests.restype = i32
    lib.sbn_tally_tests.argtypes = [vp, vp, i64, i32, vp, i64]
    lib.sbn_tally_destroy.restype = None
    lib.sbn_tally_destroy.argtypes = [vp]
    lib.sbn_bp_create.restype = i32
    lib.sbn_bp_create.argtypes = [i32, vp, i64, vp, i64, c.POINTER(vp)]
    lib.sbn_bp_run_host.restype = i32
    lib.sbn_bp_run_host.argtypes = [vp, vp, i64, i64, i32, c.c_float, c.c_float, vp, i64, vp]
    lib.sbn_bp_mpe_host.restype = i32
    lib.sbn_bp_mpe_host.argtypes = [vp, vp, i64, i64, i32, c.c_float, c.c_float, vp, i64, vp, vp]
    lib.sbn_bp_counts_host.restype = i32
    lib.sbn_bp_counts_host.argtypes = [vp, vp, i64, i64, i32, c.c_float, c.c_float, vp, vp, vp]
    lib.sbn_bp_set_tables.restype = i32
    lib.sbn_bp_set_tables.argtypes = [vp, vp, i64]
    lib.sbn_bp_destroy.restype = None
    lib.sbn_bp_destroy.argtypes = [vp]
    lib.sbn_host_alloc.restype = i32
    lib.sbn_host_alloc.argtypes = [c.POINTER(vp), i64]
    lib.sbn_host_free.restype = i32
    lib.sbn_host_free.argtypes = [vp]
    if lib.sbn_abi_version() != ABI_VERSION:
        raise EngineError(f"libsorobn_b200.so has ABI {lib.sbn_abi_version()}, Python expects {ABI_VERSION}; rebuild")
    _lib = lib
    return lib


EXPORTS = (
    "sbn_abi_version", "sbn_last_error", "sbn_device_count", "sbn_program_create", "sbn_program_create_f64",
    "sbn_program_run_host_f64", "sbn_program_evidence_host", "sbn_program_evidence_host_f64", "sbn_program_destroy",
    "sbn_program_reserve", "sbn_program_run_host", "sbn_program_run_device", "sbn_program_profile",
    "sbn_program_step_roles", "sbn_program_counts_host", "sbn_program_counts_host_f64", "sbn_program_set_tables",
    "sbn_program_set_tables_f64", "sbn_program_sample_host", "sbn_program_sample_host_f64", "sbn_program_mpe_host",
    "sbn_program_run_soft_host", "sbn_program_run_soft_host_f64", "sbn_program_counts_soft_host",
    "sbn_program_counts_soft_host_f64", "sbn_program_sample_soft_host", "sbn_program_sample_soft_host_f64",
    "sbn_program_mpe_soft_host", "sbn_program_grad_forward_host", "sbn_program_grad_forward_host_f64",
    "sbn_program_grad_backward_host", "sbn_program_grad_backward_host_f64", "sbn_program_joint_host",
    "sbn_program_joint_host_f64",
    "sbn_program_info", "sbn_program_set_graph", "sbn_program_set_tiled", "sbn_gibbs_create", "sbn_gibbs_run_host",
    "sbn_sampler_run_host", "sbn_gibbs_conditional", "sbn_gibbs_destroy", "sbn_tally_create", "sbn_tally_counts",
    "sbn_tally_scores", "sbn_tally_tests", "sbn_tally_destroy", "sbn_bp_create", "sbn_bp_run_host", "sbn_bp_mpe_host", "sbn_bp_counts_host",
    "sbn_bp_set_tables", "sbn_bp_destroy",
    "sbn_host_alloc",
    "sbn_host_free",
)


def _check(rc: int):
    if rc != SBN_OK:
        raise EngineError(f"libsorobn_b200 error {rc}: {load().sbn_last_error().decode(errors='replace')}", code=rc)


def device_count() -> int:
    n = ctypes.c_int(0)
    rc = load().sbn_device_count(ctypes.byref(n))
    return n.value if rc == SBN_OK else 0


def default_device() -> int:
    return int(os.environ.get("SOROBN_B200_DEVICE", "0"))


class PinnedArray:
    """A numpy array backed by page-locked host memory (cudaHostAlloc) so that the
    engine's host<->device copies are true asynchronous DMA."""

    def __init__(self, shape, dtype):
        self.shape = tuple(int(s) for s in shape)
        self.dtype = np.dtype(dtype)
        nbytes = max(1, int(np.prod(self.shape)) * self.dtype.itemsize)
        self._ptr = ctypes.c_void_p()
        _check(load().sbn_host_alloc(ctypes.byref(self._ptr), nbytes))
        buf = (ctypes.c_char * nbytes).from_address(self._ptr.value)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(np.prod(self.shape))).reshape(self.shape)

    def free(self):
        if self._ptr is not None and self._ptr.value:
            self.array = None
            load().sbn_host_free(self._ptr)
            self._ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Program:
    """One compiled (query variables, evidence variables) pair on one GPU."""

    def __init__(self, plan, device: int | None = None, f64: bool = False):
        lib = load()
        self.plan = plan
        self.device = default_device() if device is None else int(device)
        self.Q = int(plan.Q)
        self.n_ev = len(plan.evidence)
        self.f64 = bool(f64)
        self.dtype = np.float64 if self.f64 else np.float32
        self._h = ctypes.c_void_p()
        words = np.ascontiguousarray(plan.words, dtype=np.int32)
        if self.f64:
            blob = np.ascontiguousarray(plan.table_blob64, dtype=np.float64)
            _check(lib.sbn_program_create_f64(self.device, words.ctypes.data, words.size, blob.ctypes.data, blob.size,
                                              ctypes.byref(self._h)))
            return
        blob = np.ascontiguousarray(plan.table_blob, dtype=np.float32)
        _check(lib.sbn_program_create(self.device, words.ctypes.data, words.size, blob.ctypes.data, blob.size,
                                      ctypes.byref(self._h)))
        # developer switches (profiling / A-B runs); the defaults are the fast path
        if os.environ.get("SOROBN_B200_TILED"):
            self.set_tiled(int(os.environ["SOROBN_B200_TILED"]))
        if os.environ.get("SOROBN_B200_GRAPH"):
            self.set_graph(int(os.environ["SOROBN_B200_GRAPH"]))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            load().sbn_program_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ control
    def reserve(self, max_rows: int):
        _check(load().sbn_program_reserve(self._h, int(max_rows)))

    def set_graph(self, mode):
        """0 / False: plain launches; 1 / True: CUDA-graph replay (default); 3: graph with the independent
        sub-trees of the elimination as parallel branches."""
        _check(load().sbn_program_set_graph(self._h, int(mode)))

    def set_tiled(self, mode):
        """0: plain kernel; 1: tiled (default); 4: tiled, x-loop schedule only; 5: no slab variant;
        7: on-chip segments on (csrc/sbn_chain.h, opt-in); 6: off again; 9: tensor-map TMA pipeline
        kernel on for the steps it covers (csrc/sbn_tma.h, opt-in); 8: off again; 10: no paired steps; 11: paired
        steps where eligible (default; csrc/sbn_pair.h)."""
        _check(load().sbn_program_set_tiled(self._h, int(mode)))

    def info(self) -> dict:
        buf = (ctypes.c_int64 * 14)()
        _check(load().sbn_program_info(self._h, buf, 14))
        keys = ("Q", "n_ev", "n_steps", "scratch_floats_per_row", "reserved_rows", "launches", "mode",
                "shared_scratch_floats", "segments", "segment_steps", "segment_hbm_bytes_per_row",
                "segment_scratch_floats", "pairs", "pair_bytes_saved_per_row")
        return dict(zip(keys, [int(x) for x in buf]))

    # --------------------------------------------------------------------- runs
    def _evidence(self, codes, n_rows):
        """(uint8 evidence codes [n_ev, n_rows], C-contiguous, and their pointer: None for a program without
        evidence columns); ValueError for another shape.  Keep the array alive until the call returns."""
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        if self.n_ev and codes.shape != (self.n_ev, n_rows):
            raise ValueError(f"evidence codes have shape {codes.shape}, expected {(self.n_ev, n_rows)}")
        return codes, codes.ctypes.data if self.n_ev else None

    def _fn(self, name):
        """The C entry point `name`, or its `_f64` twin for a float64 program."""
        return getattr(load(), name + "_f64" if self.f64 else name)

    def run(self, codes: np.ndarray, n_rows: int, out: np.ndarray | None = None) -> np.ndarray:
        """Host path: evidence codes uint8 [n_ev, n_rows] in, posterior float32
        [Q, n_rows] out (copies H2D, every step, D2H, synchronises)."""
        n_rows = int(n_rows)
        codes, ev_ptr = self._evidence(codes, n_rows)
        if out is None:
            out = np.empty((self.Q, n_rows), dtype=self.dtype)
        elif out.shape != (self.Q, n_rows) or out.dtype != self.dtype or not out.flags.c_contiguous:
            raise ValueError(f"out must be a C-contiguous {self.dtype.__name__} [Q, n_rows] array")
        _check(self._fn("sbn_program_run_host")(self._h, ev_ptr, n_rows, n_rows, out.ctypes.data, n_rows))
        return out

    def run_soft(self, codes: np.ndarray, lik, n_rows: int, log_evidence: bool = False):
        """Host path of a program with soft evidence (planner `soft=`): evidence codes uint8 [n_ev, n_rows] and
        likelihoods [n_rows, n_lik] (one column per state of every soft variable, `plan.soft` order) in,
        posterior [Q, n_rows] out, and with `log_evidence` also log P(e, lik) float64 [n_rows] (posterior
        programs).  `lik` is a numpy array or a torch tensor; a CUDA tensor on the program's device is read
        in place, with no host round trip."""
        n_rows = int(n_rows)
        codes, ev_ptr = self._evidence(codes, n_rows)
        lik, lik_args = self._likelihoods(lik, n_rows)
        out = np.empty((self.Q, n_rows), dtype=self.dtype)
        log_ev = np.empty(n_rows, dtype=np.float64) if log_evidence else None
        _check(self._fn("sbn_program_run_soft_host")(self._h, ev_ptr, n_rows, n_rows, *lik_args, out.ctypes.data, n_rows,
                                                      None if log_ev is None else log_ev.ctypes.data))
        return (out, log_ev) if log_evidence else out

    def _array(self, a, dtype, shape, what):
        """(the array argument `a` as a C-contiguous `dtype` array, to keep alive until the call returns; its
        pointer; whether it is on the device) of a numpy array or a torch tensor.  A CUDA tensor on the program's
        device is read in place, with no host round trip.  ValueError for another `shape` or device; `what` names
        the argument."""
        on_device = type(a).__module__.startswith("torch") and a.is_cuda
        if on_device:
            import torch

            if a.device.index != self.device:
                raise ValueError(f"{what} on cuda:{a.device.index}; the program runs on cuda:{self.device}")
            a = a.to(torch.float64 if dtype == np.float64 else torch.float32).contiguous()
            torch.cuda.current_stream(a.device).synchronize()  # the program's stream reads it next
        else:
            a = np.ascontiguousarray(a.detach().numpy() if type(a).__module__.startswith("torch") else a, dtype=dtype)
        if tuple(a.shape) != shape:
            raise ValueError(f"{what} have shape {tuple(a.shape)}, expected {shape}")
        return a, a.data_ptr() if on_device else a.ctypes.data, on_device

    def _likelihoods(self, lik, n_rows):
        """(the likelihoods [n_rows, n_lik] as `_array` keeps them, and the call's (pointer, ld_lik, on-device
        flag)).  The likelihoods take the program's type, except that the float32 MPE and MAP programs take them in
        float64: their pack takes the log of each ratio in double, and no float64 twin would rescue a row whose
        scale float32 cannot hold."""
        n_lik = sum(int(self.plan._card[v]) for v in self.plan.soft)
        f64 = self.f64 or self.plan.version in (8, 9)
        lik, ptr, on_device = self._array(lik, np.float64 if f64 else np.float32, (n_rows, n_lik), "likelihoods")
        return lik, (ptr, n_lik, int(on_device))

    def _program_likelihoods(self, lik, n_rows, kind):
        """`_likelihoods` of a call that takes programs with and without soft variables (`kind` "gradient" or
        "joint"): the first need their likelihoods, the second take none."""
        if not self.plan.soft:
            if lik is not None:
                raise ValueError(f"likelihoods given to a {kind} program without soft variables")
            return None, (None, 0, 0)
        if lik is None:
            raise ValueError(f"a {kind} program with soft variables needs their likelihoods")
        return self._likelihoods(lik, n_rows)

    def evidence(self, codes: np.ndarray, n_rows: int) -> np.ndarray:
        """P(event) per evidence row (the normaliser of the posterior), host path."""
        n_rows = int(n_rows)
        codes, ev_ptr = self._evidence(codes, n_rows)
        out = np.empty(n_rows, dtype=self.dtype)
        _check(self._fn("sbn_program_evidence_host")(self._h, ev_ptr, n_rows, n_rows, out.ctypes.data))
        return out

    def counts(self, codes: np.ndarray, n_rows: int, lik=None, log_evidence: bool = False):
        """Counts programs (planner.build_counts_plan): (expected counts float64 [n_counts] summed over the
        rows, P(observed) [n_rows], NaN for a row the float32 range rule flags), host path.  A program with soft
        evidence (planner.build_pattern_plan) takes likelihoods `lik` as `run_soft` does; P(observed) is then
        P(observed, lik / max), and `log_evidence` appends log P(observed, lik) float64 [n_rows]."""
        n_rows = int(n_rows)
        codes, ev_ptr = self._evidence(codes, n_rows)
        counts = np.zeros(int(self.plan.n_counts), dtype=np.float64)
        prob = np.empty(n_rows, dtype=self.dtype)
        if lik is None:
            _check(self._fn("sbn_program_counts_host")(self._h, ev_ptr, n_rows, n_rows, counts.ctypes.data, counts.size,
                                                       prob.ctypes.data))
            return counts, prob
        lik, lik_args = self._likelihoods(lik, n_rows)
        log_ev = np.empty(n_rows, dtype=np.float64) if log_evidence else None
        _check(self._fn("sbn_program_counts_soft_host")(self._h, ev_ptr, n_rows, n_rows, *lik_args, counts.ctypes.data,
                                                        counts.size, prob.ctypes.data,
                                                        None if log_ev is None else log_ev.ctypes.data))
        return (counts, prob, log_ev) if log_evidence else (counts, prob)

    def grad_forward(self, codes: np.ndarray, n_rows: int, lik=None):
        """Gradient programs (planner.build_pattern_plan kind "grad"): (P(observed, lik / max) [n_rows], NaN for a
        row the float32 range rule flags; log P(observed, lik) float64 [n_rows]).  Only the launches P(observed)
        depends on run.  `lik` as in `run_soft`, for a program with soft variables."""
        n_rows = int(n_rows)
        codes, ev_ptr = self._evidence(codes, n_rows)
        lik, lik_args = self._program_likelihoods(lik, n_rows, "gradient")
        prob = np.empty(n_rows, dtype=self.dtype)
        log_prob = np.empty(n_rows, dtype=np.float64)
        _check(self._fn("sbn_program_grad_forward_host")(self._h, ev_ptr, n_rows, n_rows, *lik_args, prob.ctypes.data,
                                                         log_prob.ctypes.data))
        return prob, log_prob

    def grad_backward(self, codes: np.ndarray, n_rows: int, weights, lik=None):
        """Gradient programs: (weighted counts float64 [n_counts] = sum_b w_b * P(family entry | observed, lik),
        derivative readouts [n_lik, n_rows] = d log P(observed, lik / max) / d (lik / max), P(observed, lik / max)
        [n_rows]), NaN readouts and P(observed) for a flagged row, which adds nothing.  `weights` [n_rows] is a
        numpy array or a torch tensor; a CUDA tensor on the program's device is read in place, as `lik` is."""
        n_rows = int(n_rows)
        codes, ev_ptr = self._evidence(codes, n_rows)
        lik, lik_args = self._program_likelihoods(lik, n_rows, "gradient")
        weights, w_ptr, w_on_device = self._array(weights, np.float64, (n_rows,), "weights")
        n_lik = self.Q - 1
        counts = np.zeros(int(self.plan.n_counts), dtype=np.float64)
        deriv = np.empty((n_lik, n_rows), dtype=self.dtype)
        prob = np.empty(n_rows, dtype=self.dtype)
        _check(self._fn("sbn_program_grad_backward_host")(
            self._h, ev_ptr, n_rows, n_rows, *lik_args, w_ptr, int(w_on_device), counts.ctypes.data, counts.size,
            deriv.ctypes.data if n_lik else None, n_rows, prob.ctypes.data))
        return counts, deriv, prob

    def joint(self, codes: np.ndarray, n_rows: int, lik=None):
        """Joint programs (planner.build_joint_plan): (output [Q, n_rows], whose rows `plan.group_rows[k] ..` hold
        the joint posterior of group k's unobserved members (the first one fastest); P(observed, lik / max)
        [n_rows]), NaN throughout for a row the float32 range rule flags, host path.  `lik` as in `run_soft`, for
        a program with soft variables (and None otherwise)."""
        n_rows = int(n_rows)
        codes, ev_ptr = self._evidence(codes, n_rows)
        lik, lik_args = self._program_likelihoods(lik, n_rows, "joint")
        out = np.empty((self.Q, n_rows), dtype=self.dtype)
        prob = np.empty(n_rows, dtype=self.dtype)
        _check(self._fn("sbn_program_joint_host")(self._h, ev_ptr, n_rows, n_rows, *lik_args, out.ctypes.data, n_rows,
                                                  prob.ctypes.data))
        return out, prob

    def set_tables(self, blob: np.ndarray):
        """Replace a counts or gradient program's tables (planner.refresh_tables gives the blob of new CPTs)."""
        blob = np.ascontiguousarray(blob, dtype=self.dtype)
        _check(self._fn("sbn_program_set_tables")(self._h, blob.ctypes.data, blob.size))

    def sample(self, codes: np.ndarray, n_rows: int, n_draws: int, seed: int, row_base: int = 0, lik=None,
               log_evidence: bool = False):
        """Sample programs (planner.build_sample_plan): (drawn codes uint8 [n_sampled, n_draws, n_rows] in
        the order of `plan.sampled`, P(observed) [n_rows], NaN for a row the float32 range rule flags), host
        path.  Row b's draws depend only on (seed, row_base + b, draw index).  `lik` and `log_evidence` are
        those of `counts`, for a program with soft evidence."""
        n_rows, n_draws = int(n_rows), int(n_draws)
        codes, ev_ptr = self._evidence(codes, n_rows)
        out = np.empty((len(self.plan.sampled), n_draws, n_rows), dtype=np.uint8)
        prob = np.empty(n_rows, dtype=self.dtype)
        seed = int(seed) & (2**64 - 1)
        if lik is None:
            _check(self._fn("sbn_program_sample_host")(self._h, ev_ptr, n_rows, n_rows, n_draws, seed, int(row_base),
                                                       out.ctypes.data, prob.ctypes.data))
            return out, prob
        lik, lik_args = self._likelihoods(lik, n_rows)
        log_ev = np.empty(n_rows, dtype=np.float64) if log_evidence else None
        _check(self._fn("sbn_program_sample_soft_host")(self._h, ev_ptr, n_rows, n_rows, *lik_args, n_draws, seed,
                                                        int(row_base), out.ctypes.data, prob.ctypes.data,
                                                        None if log_ev is None else log_ev.ctypes.data))
        return (out, prob, log_ev) if log_evidence else (out, prob)

    def mpe(self, codes: np.ndarray, n_rows: int, lik=None):
        """MPE programs (planner.build_mpe_plan): (decoded codes uint8 [n_decoded, n_rows] in the order of
        `plan.sampled`, max log P(x, e) float32 [n_rows], -inf for a row of probability zero), host path.  A
        program with soft evidence takes likelihoods `lik` as `run_soft` does; its max log P(x, e, lik) comes
        back in float64, on the caller's scale of `lik`."""
        n_rows = int(n_rows)
        codes, ev_ptr = self._evidence(codes, n_rows)
        out = np.empty((len(self.plan.sampled), n_rows), dtype=np.uint8)
        if lik is None:
            log_prob = np.empty(n_rows, dtype=np.float32)
            _check(load().sbn_program_mpe_host(self._h, ev_ptr, n_rows, n_rows, out.ctypes.data, log_prob.ctypes.data))
            return out, log_prob
        lik, lik_args = self._likelihoods(lik, n_rows)
        log_prob = np.empty(n_rows, dtype=np.float64)
        _check(load().sbn_program_mpe_soft_host(self._h, ev_ptr, n_rows, n_rows, *lik_args, out.ctypes.data,
                                                log_prob.ctypes.data))
        return out, log_prob

    def map(self, codes: np.ndarray, n_rows: int, lik=None):
        """Marginal MAP programs (planner.build_map_plan): (decoded codes uint8 [n_map, n_rows] of the MAP
        variables in the order of `plan.sampled`, max log P(x_MAP, e) float32 [n_rows], -inf for a row of
        probability zero), host path.  The engine runs them through the MPE entry point, `lik` included."""
        if self.plan.version != 9:
            raise ValueError(f"a version-{self.plan.version} program is not a marginal MAP program")
        return self.mpe(codes, n_rows, lik=lik)

    def run_device(self, d_ev: int, ld_ev: int, n_rows: int, d_out: int, ld_out: int, stream: int = 0):
        """Device path: raw device pointers, asynchronous on `stream`."""
        _check(load().sbn_program_run_device(self._h, ctypes.c_void_p(d_ev), int(ld_ev), int(n_rows),
                                             ctypes.c_void_p(d_out), int(ld_out), ctypes.c_void_p(stream)))

    def step_roles(self) -> np.ndarray:
        """Per program step: 0 ran once at creation, 1 own launch, 2 / 3 first / second step of a paired launch,
        4 / 5 expanding product / its consumer as one launch, 6 inside an on-chip segment."""
        roles = np.zeros(len(self.plan.steps), dtype=np.int32)
        _check(load().sbn_program_step_roles(self._h, roles.ctypes.data, roles.size))
        return roles

    def profile(self, d_ev: int, ld_ev: int, n_rows: int, d_out: int, ld_out: int, stream: int = 0) -> np.ndarray:
        n = len(self.plan.steps) + 1
        ms = np.zeros(n, dtype=np.float32)
        _check(load().sbn_program_profile(self._h, ctypes.c_void_p(d_ev), int(ld_ev), int(n_rows),
                                          ctypes.c_void_p(d_out), int(ld_out), ctypes.c_void_p(stream),
                                          ms.ctypes.data, n))
        return ms


class GibbsSampler:
    """Device Gibbs sampler for one (query variables, evidence variables) pair: one chain per
    evidence row (csrc/sbn_gibbs.cuh; the reference: bayes_net.py:665-737)."""

    def __init__(self, net, query_ids, evidence_ids, cycle_ids, device: int | None = None):
        lib = load()
        self.device = default_device() if device is None else int(device)
        n = len(net.names)
        card = np.ascontiguousarray(net.card, dtype=np.int32)
        self._card = [int(c) for c in card]
        par_ptr = np.zeros(n + 1, dtype=np.int32)
        par_idx = []
        offsets = np.zeros(n, dtype=np.int32)
        blob = []
        off = 0
        for v in range(n):
            par_idx.extend(net.parents[v])
            par_ptr[v + 1] = len(par_idx)
            t = np.ascontiguousarray(net.cpt[v], dtype=np.float32).reshape(-1)
            offsets[v] = off
            blob.append(t)
            off += t.size
        self._tables = np.concatenate(blob)
        par_idx = np.ascontiguousarray(par_idx, dtype=np.int32)
        self.query = np.ascontiguousarray(query_ids, dtype=np.int32)
        self.evidence = np.ascontiguousarray(evidence_ids, dtype=np.int32)
        # the cycle is only walked by Gibbs; keep the C side's "non-empty" contract when all is observed
        cycle = np.ascontiguousarray(cycle_ids if len(cycle_ids) else query_ids, dtype=np.int32)
        self.Q = int(np.prod([net.card[q] for q in query_ids]))
        self.n_ev = len(evidence_ids)
        self._h = ctypes.c_void_p()
        _check(lib.sbn_gibbs_create(
            self.device, n, card.ctypes.data, par_ptr.ctypes.data, par_idx.ctypes.data if par_idx.size else None,
            offsets.ctypes.data, self._tables.ctypes.data, self._tables.size, len(self.query), self.query.ctypes.data,
            self.n_ev, self.evidence.ctypes.data if self.n_ev else None, len(cycle), cycle.ctypes.data,
            ctypes.byref(self._h)))

    ALGORITHMS = {"gibbs": 0, "likelihood": 1, "rejection": 2, "gibbs_generic": 3}

    def run(self, codes: np.ndarray, n_chains: int, n_iterations: int, seed: int, algorithm: str = "gibbs") -> np.ndarray:
        """uint8 codes [n_ev, n_rows] -> estimated posterior float32 [Q, n_rows] (one Gibbs
        chain, or n_iterations forward samples, per evidence row)."""
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        if self.n_ev and codes.shape != (self.n_ev, n_chains):
            raise ValueError(f"evidence codes have shape {codes.shape}, expected {(self.n_ev, n_chains)}")
        out = np.empty((self.Q, n_chains), dtype=np.float32)
        _check(load().sbn_sampler_run_host(self._h, self.ALGORITHMS[algorithm], codes.ctypes.data if self.n_ev else None,
                                           n_chains, n_chains, int(n_iterations),
                                           ctypes.c_uint64(int(seed) & (2**64 - 1)), out.ctypes.data, n_chains))
        return out

    def conditional(self, var: int, joint) -> np.ndarray:
        """P(var | Markov blanket) for one joint state (uint8 codes per variable id), as the chain
        evaluates it (bayes_net.py:699-712 precomputes the same table)."""
        joint = np.ascontiguousarray(joint, dtype=np.uint8)
        out = np.zeros(self._card[var], dtype=np.float32)
        _check(load().sbn_gibbs_conditional(self._h, int(var), joint.ctypes.data, out.ctypes.data))
        return out

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            load().sbn_gibbs_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


TALLY_MAX_TABLE = 1 << 22     # SBN_TALLY_MAX_TABLE: entries of one family's table
TALLY_SMEM_BINS = 32768       # SBN_TALLY_SMEM_BINS: a larger table counts with global atomics


class Tally:
    """A complete discrete data set resident on one GPU, and the counting passes of structure learning over it
    (csrc/sbn_tally.cu).  `codes` is uint8 [n_vars, n_rows], every code of column v below `cards[v]`; it is
    uploaded once.  A family is a sequence of column ids, the child first and its parents after it."""

    SCORES = {"bic": 0, "bdeu": 1}
    TESTS = {"g2": 0, "chi2": 1}

    def __init__(self, codes, cards, device: int | None = None):
        lib = load()
        self.device = default_device() if device is None else int(device)
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        if codes.ndim != 2:
            raise ValueError(f"codes have shape {codes.shape}, expected [n_vars, n_rows]")
        self.cards = np.ascontiguousarray(cards, dtype=np.int32)
        if self.cards.shape != (codes.shape[0],):
            raise ValueError(f"{self.cards.size} cardinalities for {codes.shape[0]} columns")
        self.n_vars, self.n_rows = codes.shape
        self._h = ctypes.c_void_p()
        _check(lib.sbn_tally_create(self.device, codes.ctypes.data, self.n_rows, self.n_vars, self.n_rows,
                                    self.cards.ctypes.data, ctypes.byref(self._h)))

    @staticmethod
    def _words(families):
        words = []
        for fam in families:
            words.append(len(fam))
            words.extend(int(v) for v in fam)
        return np.ascontiguousarray(words, dtype=np.int32)

    def counts(self, families) -> list:
        """The contingency table of every family, exact: uint64 [prod of the members' cards] each, the child
        fastest, then the first parent, and so on."""
        sizes = [int(np.prod([int(self.cards[v]) for v in fam])) for fam in families]
        words = self._words(families)
        out = np.zeros(sum(sizes), dtype=np.uint64)
        _check(load().sbn_tally_counts(self._h, words.ctypes.data, words.size, out.ctypes.data, out.size))
        return np.split(out, np.cumsum(sizes)[:-1])

    def scores(self, families, kind: str = "bic", ess: float = 1.0) -> np.ndarray:
        """The decomposable score ("bic" or "bdeu" with equivalent sample size `ess`) of every family, float64;
        only the scores leave the device."""
        words = self._words(families)
        out = np.empty(len(families), dtype=np.float64)
        _check(load().sbn_tally_scores(self._h, words.ctypes.data, words.size, self.SCORES[kind], float(ess),
                                       out.ctypes.data, out.size))
        return out

    def tests(self, tests, kind: str = "g2") -> np.ndarray:
        """Conditional-independence tests x _|_ y | S, each a sequence of column ids x, y, *S: float64 [n, 3] of
        (statistic, degrees of freedom, p-value), with the G^2 ("g2") or Pearson X^2 ("chi2") statistic; only
        these leave the device (include/sorobn_b200.h, sbn_tally_tests)."""
        words = self._words(tests)
        out = np.empty((len(tests), 3), dtype=np.float64)
        _check(load().sbn_tally_tests(self._h, words.ctypes.data, words.size, self.TESTS[kind], out.ctypes.data,
                                      len(tests)))
        return out

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            load().sbn_tally_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BeliefPropagation:
    """Loopy belief propagation over one compiled factor graph on one GPU (csrc/sbn_bp.cu): `words` and `tables` are
    those of `bp.compile_graph` (sum-product, `run`), of `bp.compile_mpe_graph` (max-product, `mpe`) or of
    `bp.compile_counts_graph` (expected counts, `counts`); the algorithm is defined in sorobn_b200/bp.py."""

    def __init__(self, words, tables, device: int | None = None):
        lib = load()
        self.device = default_device() if device is None else int(device)
        words = np.ascontiguousarray(words, dtype=np.int32)
        tables = np.ascontiguousarray(tables, dtype=np.float32)
        self.n_ev, self.n_var, self.Q = int(words[2]), int(words[4]), int(words[7])
        self.n_table_floats = int(words[8])
        self._h = ctypes.c_void_p()
        _check(lib.sbn_bp_create(self.device, words.ctypes.data, words.size, tables.ctypes.data if tables.size else None,
                                 tables.size, ctypes.byref(self._h)))

    def run(self, codes, n_rows: int, n_iterations: int, damping: float, tol: float):
        """uint8 evidence codes [n_ev, n_rows] -> (beliefs float32 [Q, n_rows], NaN for a row that met a zero sum;
        iterations int32 [n_rows]: the sweep at which each row converged or met a zero, n_iterations + 1 when it
        did not converge)."""
        n_rows = int(n_rows)
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        if self.n_ev and codes.shape != (self.n_ev, n_rows):
            raise ValueError(f"evidence codes have shape {codes.shape}, expected {(self.n_ev, n_rows)}")
        out = np.empty((self.Q, n_rows), dtype=np.float32)
        iters = np.empty(n_rows, dtype=np.int32)
        _check(load().sbn_bp_run_host(self._h, codes.ctypes.data if self.n_ev else None, n_rows, n_rows,
                                      int(n_iterations), float(damping), float(tol), out.ctypes.data, n_rows,
                                      iters.ctypes.data))
        return out, iters

    def mpe(self, codes, n_rows: int, n_iterations: int, damping: float, tol: float):
        """uint8 evidence codes [n_ev, n_rows] -> (decoded codes uint8 [n_var, n_rows] in var id order, 0 for a dead
        row; log P(decode, e) float64 [n_rows], -inf for a decode of probability 0, NaN for a row that met a zero
        sum; iterations int32 [n_rows] as `run`, 0 when there is nothing to decode)."""
        n_rows = int(n_rows)
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        if self.n_ev and codes.shape != (self.n_ev, n_rows):
            raise ValueError(f"evidence codes have shape {codes.shape}, expected {(self.n_ev, n_rows)}")
        out = np.empty((self.n_var, n_rows), dtype=np.uint8)
        log_p = np.empty(n_rows, dtype=np.float64)
        iters = np.empty(n_rows, dtype=np.int32)
        _check(load().sbn_bp_mpe_host(self._h, codes.ctypes.data if self.n_ev else None, n_rows, n_rows,
                                      int(n_iterations), float(damping), float(tol),
                                      out.ctypes.data if self.n_var else None, n_rows, log_p.ctypes.data,
                                      iters.ctypes.data))
        return out, log_p, iters

    def counts(self, codes, n_rows: int, n_iterations: int, damping: float, tol: float):
        """uint8 evidence codes [n_ev, n_rows] -> (expected counts float64 [n_table_floats] in blob order, summed
        over the live rows (`Graph.perm` maps them to the dense CPTs); Bethe log-likelihood float64 [n_rows], NaN for
        a dead row; iterations int32 [n_rows] as `run`, 0 for a row dead before its first sweep and when every node
        is observed)."""
        n_rows = int(n_rows)
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        if self.n_ev and codes.shape != (self.n_ev, n_rows):
            raise ValueError(f"evidence codes have shape {codes.shape}, expected {(self.n_ev, n_rows)}")
        counts = np.empty(self.n_table_floats, dtype=np.float64)
        log_z = np.empty(n_rows, dtype=np.float64)
        iters = np.empty(n_rows, dtype=np.int32)
        _check(load().sbn_bp_counts_host(self._h, codes.ctypes.data if self.n_ev else None, n_rows, n_rows,
                                         int(n_iterations), float(damping), float(tol),
                                         counts.ctypes.data if counts.size else None, log_z.ctypes.data,
                                         iters.ctypes.data))
        return counts, log_z, iters

    def set_tables(self, tables):
        """Replace the float32 table blob by `tables` of the same size (the words stay)."""
        tables = np.ascontiguousarray(tables, dtype=np.float32)
        _check(load().sbn_bp_set_tables(self._h, tables.ctypes.data if tables.size else None, tables.size))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            load().sbn_bp_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
