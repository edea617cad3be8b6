"""Python face of libhector_mpc_b200.so (ctypes over the C-ABI in include/hector_mpc_b200.h).

Mirrors the reference's boundary, hector_control/ConvexMPC/convexMPC_interface.h:39-43 — same names,
argument order and semantics — and adds the batched calls.  All numerical work happens in the CUDA
library; this module only marshals pointers.  There is no CPU fallback: if the shared library or an
H100 (sm_90a) is missing, calls raise.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

from .scenarios import COMMAND_DTYPE, STATE_DTYPE, UPDATE_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libhector_mpc_b200.so")

HMPC_OK, HMPC_ERR_ARG, HMPC_ERR_CUDA, HMPC_ERR_NOT_CONVERGED = 0, 1, 2, 3
ST_OK, ST_ITER_CAP, ST_WS_CAP, ST_INFEASIBLE, ST_NOT_SPD = 0, 1, 2, 3, 4

EXPORTS = [
    "setup_problem", "get_solution", "update_solver_settings", "update_problem_data",
    "hmpc_record_bytes", "hmpc_pack_records", "hmpc_create", "hmpc_destroy", "hmpc_last_error",
    "hmpc_set_problem", "hmpc_solve_batch", "hmpc_solve_device", "hmpc_launches_per_solve",
    "hmpc_assemble_device", "hmpc_class_config", "hmpc_solve_batch_ex", "hmpc_solve_device_ex",
    "hmpc_prepare_device", "hmpc_solve_batch_states", "hmpc_rollout_device", "hmpc_reset_warm_start",
    "hmpc_shard_unique_id", "hmpc_shard_init", "hmpc_solve_batch_sharded", "hmpc_shard_wait",
    "hmpc_pin_host_buffer", "hmpc_unpin_host_buffer", "hmpc_swing_device",
    "hmpc_reference_last_status", "hmpc_reference_last_rc",
    "hmpc_solve_device_warm", "hmpc_solve_batch_warm", "hmpc_reference_set_warm_start",
    "hmpc_set_refinement", "hmpc_reference_set_refinement",
    "hmpc_solve_device_masked", "hmpc_solve_batch_masked",
    "hmpc_solve_states_device_masked", "hmpc_solve_batch_states_warm", "hmpc_solve_batch_states_masked",
    "hmpc_solve_batch_sharded_warm", "hmpc_solve_batch_states_sharded_warm",
    "hmpc_predict_device", "hmpc_predict_batch", "hmpc_certify_device", "hmpc_certify_batch",
    "hmpc_solve_device_multi", "hmpc_solve_batch_multi",
    "hmpc_solve_states_device_multi", "hmpc_solve_batch_states_multi",
]
# hmpc_certificate_t, and its flag bits (include/hector_mpc_b200.h)
CERTIFICATE_DTYPE = np.dtype([("cost", "<f8"), ("stationarity", "<f8"), ("primal", "<f8"), ("complementarity", "<f8"),
                              ("n_active", "<i4"), ("flags", "<i4")])
CERT_PASS, CERT_NONFINITE, CERT_SWING, CERT_STATIONARITY, CERT_PRIMAL, CERT_COMPLEMENTARITY = 1, 2, 4, 8, 16, 32
REFINEMENT_CLASS = 3  # hmpc_class_config index of the refinement class (HMPC_REFINEMENT_CLASS)

SETUP_DTYPE = np.dtype([("dt", "<f4"), ("mu", "<f4"), ("f_max", "<f4"), ("horizon", "<i4")], align=True)

_lib = None


class HmpcError(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    """Load the CUDA library; raises if it has not been built (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise HmpcError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = ctypes.CDLL(LIB_PATH)
        L.setup_problem.argtypes = [ctypes.c_double, ctypes.c_int, ctypes.c_double, ctypes.c_double]
        L.setup_problem.restype = None
        L.get_solution.argtypes = [ctypes.c_int]
        L.get_solution.restype = ctypes.c_double
        L.update_solver_settings.argtypes = [ctypes.c_int] + [ctypes.c_double] * 5
        L.update_solver_settings.restype = None
        dp = ctypes.POINTER(ctypes.c_double)
        L.update_problem_data.argtypes = [dp, dp, dp, dp, dp, dp, ctypes.c_double, dp, dp, dp, ctypes.POINTER(ctypes.c_int)]
        L.update_problem_data.restype = None
        L.hmpc_record_bytes.argtypes = [ctypes.c_int]
        L.hmpc_record_bytes.restype = ctypes.c_size_t
        L.hmpc_pack_records.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        L.hmpc_pack_records.restype = ctypes.c_int
        L.hmpc_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.hmpc_create.restype = ctypes.c_void_p
        L.hmpc_destroy.argtypes = [ctypes.c_void_p]
        L.hmpc_destroy.restype = None
        L.hmpc_last_error.restype = ctypes.c_char_p
        L.hmpc_set_problem.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.hmpc_set_problem.restype = ctypes.c_int
        L.hmpc_solve_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.hmpc_solve_batch.restype = ctypes.c_int
        L.hmpc_solve_device.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.hmpc_solve_device.restype = ctypes.c_int
        L.hmpc_launches_per_solve.argtypes = [ctypes.c_void_p]
        L.hmpc_launches_per_solve.restype = ctypes.c_int
        L.hmpc_assemble_device.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int] + [ctypes.c_void_p] * 6
        L.hmpc_assemble_device.restype = ctypes.c_int
        L.hmpc_reference_last_status.restype = ctypes.c_int
        L.hmpc_reference_last_rc.restype = ctypes.c_int
        L.hmpc_solve_batch_ex.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 3
        L.hmpc_solve_batch_ex.restype = ctypes.c_int
        L.hmpc_solve_device_ex.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 4
        L.hmpc_solve_device_ex.restype = ctypes.c_int
        L.hmpc_prepare_device.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p]
        L.hmpc_prepare_device.restype = ctypes.c_int
        L.hmpc_solve_batch_states.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_double] + [ctypes.c_void_p] * 3
        L.hmpc_solve_batch_states.restype = ctypes.c_int
        L.hmpc_rollout_device.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                          ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.hmpc_rollout_device.restype = ctypes.c_int
        L.hmpc_reset_warm_start.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.hmpc_reset_warm_start.restype = ctypes.c_int
        L.hmpc_shard_unique_id.argtypes = [ctypes.c_void_p]
        L.hmpc_shard_unique_id.restype = ctypes.c_int
        L.hmpc_shard_init.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        L.hmpc_shard_init.restype = ctypes.c_int
        L.hmpc_solve_batch_sharded.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.hmpc_solve_batch_sharded.restype = ctypes.c_int
        L.hmpc_shard_wait.argtypes = [ctypes.c_void_p]
        L.hmpc_shard_wait.restype = ctypes.c_int
        L.hmpc_pin_host_buffer.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
        L.hmpc_pin_host_buffer.restype = ctypes.c_int
        L.hmpc_unpin_host_buffer.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.hmpc_unpin_host_buffer.restype = ctypes.c_int
        L.hmpc_swing_device.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p]
        L.hmpc_swing_device.restype = ctypes.c_int
        L.hmpc_class_config.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        L.hmpc_class_config.restype = ctypes.c_int
        L.hmpc_solve_device_warm.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 5
        L.hmpc_solve_device_warm.restype = ctypes.c_int
        L.hmpc_solve_batch_warm.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 4
        L.hmpc_solve_batch_warm.restype = ctypes.c_int
        L.hmpc_reference_set_warm_start.argtypes = [ctypes.c_int]
        L.hmpc_reference_set_warm_start.restype = None
        L.hmpc_set_refinement.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.hmpc_set_refinement.restype = ctypes.c_int
        L.hmpc_reference_set_refinement.argtypes = [ctypes.c_int]
        L.hmpc_reference_set_refinement.restype = None
        L.hmpc_solve_device_masked.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 6
        L.hmpc_solve_device_masked.restype = ctypes.c_int
        L.hmpc_solve_batch_masked.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 5
        L.hmpc_solve_batch_masked.restype = ctypes.c_int
        L.hmpc_solve_states_device_masked.argtypes = ([ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_double]
                                                      + [ctypes.c_void_p] * 6)
        L.hmpc_solve_states_device_masked.restype = ctypes.c_int
        L.hmpc_solve_batch_states_warm.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_double] + [ctypes.c_void_p] * 4
        L.hmpc_solve_batch_states_warm.restype = ctypes.c_int
        L.hmpc_solve_batch_states_masked.argtypes = ([ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_double]
                                                     + [ctypes.c_void_p] * 4)
        L.hmpc_solve_batch_states_masked.restype = ctypes.c_int
        L.hmpc_solve_batch_sharded_warm.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 6
        L.hmpc_solve_batch_sharded_warm.restype = ctypes.c_int
        L.hmpc_solve_batch_states_sharded_warm.argtypes = ([ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_double]
                                                           + [ctypes.c_void_p] * 5)
        L.hmpc_solve_batch_states_sharded_warm.restype = ctypes.c_int
        L.hmpc_predict_device.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 4
        L.hmpc_predict_device.restype = ctypes.c_int
        L.hmpc_predict_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 3
        L.hmpc_predict_batch.restype = ctypes.c_int
        L.hmpc_certify_device.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 5
        L.hmpc_certify_device.restype = ctypes.c_int
        L.hmpc_certify_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 4
        L.hmpc_certify_batch.restype = ctypes.c_int
        L.hmpc_solve_device_multi.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 6
        L.hmpc_solve_device_multi.restype = ctypes.c_int
        L.hmpc_solve_batch_multi.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 5
        L.hmpc_solve_batch_multi.restype = ctypes.c_int
        L.hmpc_solve_states_device_multi.argtypes = ([ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 2
                                                     + [ctypes.c_double] + [ctypes.c_void_p] * 8)
        L.hmpc_solve_states_device_multi.restype = ctypes.c_int
        L.hmpc_solve_batch_states_multi.argtypes = ([ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 2
                                                    + [ctypes.c_double] + [ctypes.c_void_p] * 5)
        L.hmpc_solve_batch_states_multi.restype = ctypes.c_int
        _lib = L
    return _lib


def last_error() -> str:
    return lib().hmpc_last_error().decode()


def _check(rc: int, allow_not_converged: bool = False) -> int:
    if rc == HMPC_OK or (allow_not_converged and rc == HMPC_ERR_NOT_CONVERGED):
        return rc
    raise HmpcError(f"libhector_mpc_b200 rc={rc}: {last_error()}")


# ---------------------------------------------------------------------------------------------------
# Part 1: the reference's own entry points (convexMPC_interface.h:39-43)
# ---------------------------------------------------------------------------------------------------
def setup_problem(dt: float, horizon: int, mu: float, f_max: float) -> None:
    lib().setup_problem(dt, horizon, mu, f_max)


def update_problem_data(p, v, q, w, r, joint_angles, yaw, weights, state_trajectory, Alpha_K, gait) -> None:
    """Blocks until the solve is done (convexMPC_interface.cpp:83-103)."""
    def d(a):
        a = np.ascontiguousarray(a, dtype=np.float64)
        return a, a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    keep = [d(a) for a in (p, v, q, w, r, joint_angles, weights, state_trajectory, Alpha_K)]
    g = np.ascontiguousarray(gait, dtype=np.int32)
    ptr = [k[1] for k in keep]
    lib().update_problem_data(ptr[0], ptr[1], ptr[2], ptr[3], ptr[4], ptr[5], float(yaw), ptr[6], ptr[7], ptr[8],
                              g.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))


def get_solution(index: int) -> float:
    return lib().get_solution(index)


def update_solver_settings(max_iter, rho, sigma, solver_alpha, terminate, use_jcqp) -> None:
    lib().update_solver_settings(max_iter, rho, sigma, solver_alpha, terminate, use_jcqp)


def reference_last_status() -> int:
    return lib().hmpc_reference_last_status()


def reference_last_rc() -> int:
    """Result of the last update_problem_data: 0, HMPC_ERR_NOT_CONVERGED, or the error the tick failed with."""
    return lib().hmpc_reference_last_rc()


def reference_set_warm_start(on: bool) -> None:
    """update_problem_data proposes the previous call's working set, moved one step (hmpc_reference_set_warm_start);
    off by default, like the reference's cold start."""
    lib().hmpc_reference_set_warm_start(1 if on else 0)


def reference_set_refinement(on: bool) -> None:
    """update_problem_data solves robots beyond the conditioning limit (e.g. lying on their side) through the refinement
    class instead of reporting them as not solved (hmpc_reference_set_refinement); off by default."""
    lib().hmpc_reference_set_refinement(1 if on else 0)


# ---------------------------------------------------------------------------------------------------
# Part 2: batched interface
# ---------------------------------------------------------------------------------------------------
def record_bytes(horizon: int) -> int:
    return int(lib().hmpc_record_bytes(horizon))


def pack_records(records: np.ndarray, horizon: int) -> np.ndarray:
    """reference records -> packed device layout (uint8 [B, stride]); pure byte shuffling in C."""
    records = np.ascontiguousarray(records, dtype=UPDATE_DTYPE)
    out = np.zeros((records.shape[0], record_bytes(horizon)), dtype=np.uint8)
    _check(lib().hmpc_pack_records(records.ctypes.data, records.shape[0], horizon, out.ctypes.data))
    return out


def unpack_records(packed: np.ndarray, horizon: int) -> np.ndarray:
    """Inverse of pack_records (numpy): packed device records -> `update_data_t` records, e.g. to hand what a device
    loop logged to another consumer of the reference's record format."""
    packed = np.ascontiguousarray(packed, dtype=np.uint8).reshape(-1, record_bytes(horizon))
    n = packed.shape[0]
    f = packed[:, : (54 + 12 * horizon) * 4].copy().view(np.float32)
    out = np.zeros(n, dtype=UPDATE_DTYPE)
    out["p"], out["v"], out["q"], out["w"], out["r"] = f[:, 0:3], f[:, 3:6], f[:, 6:10], f[:, 10:13], f[:, 13:19]
    out["joint_angles"], out["yaw"], out["weights"], out["Alpha_K"] = f[:, 19:29], f[:, 29], f[:, 30:42], f[:, 42:54]
    out["traj"][:, : 12 * horizon] = f[:, 54: 54 + 12 * horizon]
    g0 = (54 + 12 * horizon) * 4
    out["gait"][:, : 2 * horizon] = packed[:, g0: g0 + 2 * horizon]
    return out


def status_code(s):
    return np.asarray(s) & 0xFF


def status_iters(s):
    return (np.asarray(s) >> 8) & 0xFFF


def status_nactive(s):
    return (np.asarray(s) >> 20) & 0xFF


def status_refined(s):
    """1 where the refinement class solved the instance (HMPC_STATUS_REFINED, bit 28)."""
    return (np.asarray(s) >> 28) & 1


def page_aligned(shape, dtype) -> np.ndarray:
    """A zeroed array that owns whole memory pages (start aligned, size rounded up): what a control loop should hand to
    BatchedMPC.pin / hmpc_pin_host_buffer — a C caller uses posix_memalign the same way."""
    page = os.sysconf("SC_PAGESIZE") if hasattr(os, "sysconf") else 4096
    dt = np.dtype(dtype)
    nbytes = int(np.prod(shape)) * dt.itemsize
    raw = np.zeros((nbytes + page - 1) // page * page + page, dtype=np.uint8)
    off = (-raw.ctypes.data) % page
    return raw[off:off + nbytes].view(dt).reshape(shape)


class BatchedMPC:
    """Context for `max_batch` robots of `horizon` steps on one GPU (hmpc_create / hmpc_destroy)."""

    def __init__(self, max_batch: int, horizon: int = 10, device: int = 0, dt: float = 0.04, mu: float = 0.25,
                 f_max: float = 500.0):
        self._h = lib().hmpc_create(max_batch, horizon, device)
        if not self._h:
            raise HmpcError(f"hmpc_create failed: {last_error()}")
        self.max_batch, self.horizon, self.device = max_batch, horizon, device
        self.set_problem(dt, mu, f_max)

    def set_problem(self, dt: float, mu: float, f_max: float) -> None:
        s = np.zeros(1, dtype=SETUP_DTYPE)
        s["dt"], s["mu"], s["f_max"], s["horizon"] = dt, mu, f_max, self.horizon
        _check(lib().hmpc_set_problem(self._h, s.ctypes.data))

    def set_refinement(self, on: bool) -> None:
        """Solve robots beyond the conditioning limit of the sweep inversion (scaled condition number above 1.5e4, e.g. a
        robot lying on its side) in the refinement class instead of returning code 4 (hmpc_set_refinement).  Off by
        default.  A refined instance has code 0 and status_refined() == 1; one the class cannot solve keeps code 4."""
        _check(lib().hmpc_set_refinement(self._h, 1 if on else 0))

    @property
    def launches_per_solve(self) -> int:
        return lib().hmpc_launches_per_solve(self._h)

    def class_config(self, cls: int) -> dict:
        out = np.zeros(6, dtype=np.int32)
        _check(lib().hmpc_class_config(self._h, cls, out.ctypes.data))
        return dict(zip(("threads", "smem_bytes", "qmax", "grid_cap", "nb_cap", "strip"), (int(v) for v in out)))

    def pin(self, *arrays: np.ndarray) -> None:
        """Register caller-owned arrays (records or states, wrench, status) for the in-place mode of solve_batch and
        solve_batch_states (and their _warm and _masked calls), and of predict_batch and certify_batch: the GPU then reads the records or states where they lie and writes the results where the caller wants them (hmpc_pin_host_buffer).
        The arrays must stay alive until unpin()/close().  Registration pins whole pages: allocate the arrays with
        page_aligned() so that no unrelated heap object shares their pages (a later cudaMemcpy of such a neighbour, partly
        inside a registered page range, fails with cudaErrorInvalidValue)."""
        for a in arrays:
            assert a.flags.c_contiguous
            _check(lib().hmpc_pin_host_buffer(self._h, a.ctypes.data, a.nbytes))

    def unpin(self, *arrays: np.ndarray) -> None:
        for a in arrays:
            _check(lib().hmpc_unpin_host_buffer(self._h, a.ctypes.data))

    def _host_call(self, fn, x, dtype, strict, out, torques=False, mask=None, dt_mpc=None, warm=False, shift=None,
                   sharded=False, d_all=None):
        """One host-buffer call fn(ctx, x, B, [mask], [dt_mpc], wrench, [tau], status, [shift], [d_all]): `mask` and `dt_mpc`
        are passed when given, `shift` with warm=True, `tau` unless torques is None, and with sharded=True the mask (or
        NULL) and `d_all` (or NULL) always.  -> (wrench, status), or (wrench, tau, status) with torques=True."""
        if x.dtype != dtype or not x.flags.c_contiguous:
            x = np.ascontiguousarray(x, dtype=dtype)
        B = x.shape[0]
        if out is not None:
            wrench, status = out
            assert wrench.dtype == np.float64 and wrench.shape == (B, 12 * self.horizon) and wrench.flags.c_contiguous
            assert status.dtype == np.int32 and status.shape == (B,)
        else:
            wrench = np.zeros((B, 12 * self.horizon), dtype=np.float64)
            status = np.zeros(B, dtype=np.int32)
        tau = np.zeros((B, 10), dtype=np.float64) if torques else None
        args = [self._h, x.ctypes.data, B]
        if mask is not None:
            mask = np.ascontiguousarray(np.asarray(mask) != 0).view(np.uint8)
            assert mask.shape == (B,)
            args.append(mask.ctypes.data)
        elif sharded:
            args.append(None)
        if dt_mpc is not None:
            args.append(dt_mpc)
        args.append(wrench.ctypes.data)
        if torques is not None:
            args.append(tau.ctypes.data if torques else None)
        args.append(status.ctypes.data)
        if warm:
            if shift is not None:
                shift = np.ascontiguousarray(shift, dtype=np.int32)
                assert shift.shape == (B,)
            args.append(shift.ctypes.data if shift is not None else None)
        if sharded:
            args.append(ctypes.c_void_p(d_all.data_ptr()) if d_all is not None else None)
        _check(fn(*args), allow_not_converged=not strict)
        return (wrench, tau, status) if torques else (wrench, status)

    def solve_batch(self, records: np.ndarray, strict: bool = True, out=None):
        """Host-buffer path: H2D + kernels + D2H inside.  -> (wrench [B,12N] f64, status [B] i32).
        `out=(wrench, status)` reuses caller-owned result arrays (what a C caller in a control loop does)."""
        return self._host_call(lib().hmpc_solve_batch, records, UPDATE_DTYPE, strict, out, torques=None)

    def solve_batch_warm(self, records: np.ndarray, shift=None, torques: bool = False, strict: bool = True, out=None):
        """solve_batch warm-started from each robot's working set of its last warm call (hmpc_solve_batch_warm).
        `shift` int32 [B]: steps robot i's horizon moved since then (None: all 1; 0: same horizon; < 0: no history).
        -> (wrench, status), or (wrench, tau, status) with torques=True."""
        return self._host_call(lib().hmpc_solve_batch_warm, records, UPDATE_DTYPE, strict, out, torques, warm=True, shift=shift)

    def solve_batch_masked(self, records: np.ndarray, mask, shift=None, torques: bool = False, strict: bool = True, out=None):
        """solve_batch_warm of the robots with mask[i] != 0 only (hmpc_solve_batch_masked): `mask` bool or uint8 [B], `shift`
        int32 [B] read for listed robots only (None: 1 each).  Only listed rows of the results are written.  With out=None the
        arrays are new and unlisted rows hold zeros (a status of 0 there means "not solved", not "optimal"); with
        `out=(wrench, status)` they keep what the caller's arrays held.  strict: raise when a listed robot did not converge.
        -> (wrench, status), or (wrench, tau, status) with torques=True."""
        return self._host_call(lib().hmpc_solve_batch_masked, records, UPDATE_DTYPE, strict, out, torques, mask, warm=True, shift=shift)

    def solve_batch_torques(self, records: np.ndarray, strict: bool = True):
        """Host path with the leg-controller epilogue: -> (wrench [B,12N], tau [B,10], status [B])."""
        return self._host_call(lib().hmpc_solve_batch_ex, records, UPDATE_DTYPE, strict, None, torques=True)

    def solve_batch_states(self, states: np.ndarray, strict: bool = True, torques: bool = False, out=None, dt_mpc: float = 0.04):
        """Row f-1: `hmpc_state_t` records in, data preparation on the device.  In place when the states, wrench and status
        arrays are pinned (pin()).  -> (wrench, [tau,] status)."""
        return self._host_call(lib().hmpc_solve_batch_states, states, STATE_DTYPE, strict, out, torques, dt_mpc=dt_mpc)

    def solve_batch_states_warm(self, states: np.ndarray, shift=None, torques: bool = False, strict: bool = True, out=None,
                                dt_mpc: float = 0.04):
        """solve_batch_states warm-started from each robot's working set of its last warm call (hmpc_solve_batch_states_warm).
        `shift` int32 [B]: steps robot i's horizon moved since then (None: all 1; 0: same horizon; < 0: no history).
        In place when the states, wrench and status arrays are pinned (pin()).  -> (wrench, status), or (wrench, tau, status)
        with torques=True."""
        return self._host_call(lib().hmpc_solve_batch_states_warm, states, STATE_DTYPE, strict, out, torques, dt_mpc=dt_mpc,
                               warm=True, shift=shift)

    def solve_batch_states_masked(self, states: np.ndarray, mask, shift=None, torques: bool = False, strict: bool = True,
                                  out=None, dt_mpc: float = 0.04):
        """solve_batch_states_warm of the robots with mask[i] != 0 only (hmpc_solve_batch_states_masked): `mask` bool or uint8
        [B], `shift` int32 [B] read for listed robots only (None: 1 each).  Only listed rows of the results are written.  With
        out=None the arrays are new and unlisted rows hold zeros (a status of 0 there means "not solved", not "optimal");
        with `out=(wrench, status)` they keep what the caller's arrays held.  strict: raise when a listed robot did not
        converge.  -> (wrench, status), or (wrench, tau, status) with torques=True."""
        return self._host_call(lib().hmpc_solve_batch_states_masked, states, STATE_DTYPE, strict, out, torques, mask,
                               dt_mpc=dt_mpc, warm=True, shift=shift)

    def prepare_device(self, d_states, B: int, d_records, stream=None, dt_mpc: float = 0.04) -> None:
        """Row f-1 on device-resident data: torch uint8 [B,352] states -> packed records [B,stride].
        Capturable in a CUDA graph (torch.cuda.graph; include/hector_mpc_b200.h, "CUDA graphs")."""
        import torch

        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_prepare_device(self._h, d_states.data_ptr(), B, dt_mpc, d_records.data_ptr(), ctypes.c_void_p(st)))

    def rollout_device(self, d_states, d_loop, B: int, ticks: int, d_wrench_log=None, d_record_log=None, stream=None,
                       dt_mpc: float = 0.04) -> None:
        """Row f-3: `ticks` closed-loop ticks (prepare -> solve -> advance) enqueued on one stream, no host in the
        loop.  torch CUDA tensors: states uint8 [B,352], loop uint8 [B,80], logs f32 [ticks,B,12] / uint8 [ticks,B,stride].
        Capturable in a CUDA graph: every replay advances the states and the loop by `ticks` ticks."""
        import torch

        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_rollout_device(self._h, d_states.data_ptr(), d_loop.data_ptr(), B, ticks, dt_mpc,
                                         d_wrench_log.data_ptr() if d_wrench_log is not None else None,
                                         d_record_log.data_ptr() if d_record_log is not None else None, ctypes.c_void_p(st)))

    # ---- multi-GPU: one process per GPU, batch sharded (hmpc_shard_*) ----
    @staticmethod
    def shard_unique_id() -> bytes:
        buf = ctypes.create_string_buffer(128)
        _check(lib().hmpc_shard_unique_id(buf))
        return buf.raw

    def shard_init(self, rank: int, world: int, unique_id: bytes) -> None:
        assert len(unique_id) == 128
        _check(lib().hmpc_shard_init(self._h, rank, world, ctypes.c_char_p(unique_id)))

    def solve_batch_sharded(self, records: np.ndarray, out, d_all=None, strict: bool = True):
        """This rank's slice through hmpc_solve_batch_sharded: results of the slice into `out` = (wrench f64 [b,12N], status
        i32 [b]) like solve_batch(out=...); `d_all` (torch CUDA f32 [world*b, 12N]) receives the one all-gather."""
        w, s = out
        rc = lib().hmpc_solve_batch_sharded(self._h, records.ctypes.data, len(records), w.ctypes.data, s.ctypes.data,
                                            ctypes.c_void_p(d_all.data_ptr()) if d_all is not None else None)
        _check(rc, allow_not_converged=not strict)
        return w, s

    def solve_batch_sharded_warm(self, x: np.ndarray, out, d_all=None, mask=None, shift=None, torques: bool = False,
                                 strict: bool = True, dt_mpc: float = 0.04):
        """This rank's slice warm-started, optionally masked (hmpc_solve_batch_sharded_warm, or
        hmpc_solve_batch_states_sharded_warm when `x` holds hmpc_state_t states): mask None is solve_batch_warm on the slice,
        a mask is solve_batch_masked.  `out` = (wrench f64 [b,12N], status i32 [b]); `d_all` (torch CUDA f32 [world*b, 12N])
        receives the all-gather, in which every robot's row is its latest result (zeros before its first solve).
        -> (wrench, status), or (wrench, tau, status) with torques=True."""
        if x.dtype == STATE_DTYPE:
            return self._host_call(lib().hmpc_solve_batch_states_sharded_warm, x, STATE_DTYPE, strict, out, torques, mask,
                                   dt_mpc=dt_mpc, warm=True, shift=shift, sharded=True, d_all=d_all)
        return self._host_call(lib().hmpc_solve_batch_sharded_warm, x, UPDATE_DTYPE, strict, out, torques, mask, warm=True,
                               shift=shift, sharded=True, d_all=d_all)

    def shard_wait(self) -> None:
        _check(lib().hmpc_shard_wait(self._h))

    def reset_warm_start(self, stream=None) -> None:
        """Forget the working sets the closed loop keeps between ticks (a new loop on this context starts cold).
        Capturable in a CUDA graph: every replay clears them."""
        import torch

        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_reset_warm_start(self._h, ctypes.c_void_p(st)))

    def swing_device(self, d_states, d_loop, d_phase, d_swing, B: int, d_cmd, dt: float = 0.001, dt_swing: float = 0.04,
                     stream=None) -> None:
        """Row f-4: one swingLegController::updateSwingLeg per robot on the device.  torch CUDA tensors: states uint8
        [B,352], loop uint8 [B,80], phase f64 [B], swing uint8 [B,72] (updated in place), cmd uint8 [B,232].
        Capturable in a CUDA graph: every replay updates `d_swing`."""
        import torch

        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_swing_device(self._h, d_states.data_ptr(), d_loop.data_ptr(), d_phase.data_ptr(), d_swing.data_ptr(),
                                       B, dt, dt_swing, d_cmd.data_ptr(), ctypes.c_void_p(st)))

    def solve_device(self, d_records, B: int, d_wrench, d_status, stream=None) -> None:
        """Device-resident path.  Arguments are torch CUDA tensors (uint8 [B,stride], f32 [B,12N], i32 [B]).
        Capturable in a CUDA graph: a replay solves what the captured tensors hold at that time."""
        import torch

        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_solve_device(self._h, d_records.data_ptr(), B, d_wrench.data_ptr(), d_status.data_ptr(),
                                       ctypes.c_void_p(st)))

    def solve_device_warm(self, d_records, B: int, d_wrench, d_status, d_tau=None, d_shift=None, stream=None) -> None:
        """solve_device warm-started from each robot's working set of its last warm call (hmpc_solve_device_warm).
        `d_tau` f32 [B,10] or None; `d_shift` i32 [B] on the GPU or None (every robot moved one step).
        Capturable in a CUDA graph: every replay proposes and records working sets, reading `d_shift` when it runs."""
        import torch

        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_solve_device_warm(self._h, d_records.data_ptr(), B, d_wrench.data_ptr(), d_status.data_ptr(),
                                            d_tau.data_ptr() if d_tau is not None else None,
                                            d_shift.data_ptr() if d_shift is not None else None, ctypes.c_void_p(st)))

    def solve_device_masked(self, d_records, B: int, d_mask, d_wrench, d_status, d_tau=None, d_shift=None, stream=None) -> None:
        """solve_device_warm of the robots with d_mask[i] != 0 only (hmpc_solve_device_masked).  `d_mask` torch bool or uint8
        [B] on the GPU, read on the device: no host synchronisation.  Unlisted rows of d_wrench, d_status, d_tau and their
        working sets keep their bytes.  Capturable in a CUDA graph: a replay solves the robots the captured mask lists
        when it runs."""
        import torch

        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_solve_device_masked(self._h, d_records.data_ptr(), B, d_mask.data_ptr(), d_wrench.data_ptr(),
                                              d_status.data_ptr(), d_tau.data_ptr() if d_tau is not None else None,
                                              d_shift.data_ptr() if d_shift is not None else None, ctypes.c_void_p(st)))

    def solve_states_device_masked(self, d_states, B: int, d_mask, d_records, d_wrench, d_status, d_tau=None, d_shift=None,
                                   stream=None, dt_mpc: float = 0.04) -> None:
        """solve_device_masked on robot states (hmpc_solve_states_device_masked): one chain prepares the listed robots'
        records into `d_records` (uint8 [B,stride]; unlisted rows keep their bytes) and solves them.  `d_states` torch uint8
        [B,352] on the GPU, the other arguments as in solve_device_masked.  Capturable in a CUDA graph: a replay prepares
        and solves the robots the captured mask lists from the states the captured tensor holds when it runs."""
        import torch

        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_solve_states_device_masked(self._h, d_states.data_ptr(), B, d_mask.data_ptr(), dt_mpc,
                                                     d_records.data_ptr(), d_wrench.data_ptr(), d_status.data_ptr(),
                                                     d_tau.data_ptr() if d_tau is not None else None,
                                                     d_shift.data_ptr() if d_shift is not None else None, ctypes.c_void_p(st)))

    def predict_device(self, d_records, B: int, d_wrench, d_pred, d_mask=None, stream=None) -> None:
        """The MPC's plan on the device (hmpc_predict_device): robot i's predicted states under the discrete model its QP was
        built from, d_pred[i, k] = x_{k+1} (rpy, p, omega, v: the layout of a record's traj).  torch CUDA tensors: records
        uint8 [B,stride] (what the solve read), wrench f32 [B,12N] (what it wrote), d_pred f32 [B,N,12]; `d_mask` bool or
        uint8 [B] or None (every robot): unlisted rows of d_pred keep their bytes.  A robot whose status code is not 0 has an
        untrusted wrench, so its plan is untrusted too.  Enqueued on the current stream; capturable in a CUDA graph."""
        import torch

        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_predict_device(self._h, d_records.data_ptr(), B, d_mask.data_ptr() if d_mask is not None else None,
                                         d_wrench.data_ptr(), d_pred.data_ptr(), ctypes.c_void_p(st)))

    def predict_batch(self, records: np.ndarray, wrench: np.ndarray, mask=None, out=None) -> np.ndarray:
        """The MPC's plan from host buffers (hmpc_predict_batch): `records` update_data_t [B], `wrench` f64 [B,12N] as the
        host solves return it -> f64 [B,N,12].  In place when records, wrench and `out` are pinned (pin()).  With a mask,
        unlisted rows are not written: zeros in a new array, the caller's bytes in `out`."""
        records = np.ascontiguousarray(records, dtype=UPDATE_DTYPE)
        B, N = records.shape[0], self.horizon
        wrench = np.ascontiguousarray(wrench, dtype=np.float64)
        assert wrench.shape == (B, 12 * N)
        if out is None:
            out = np.zeros((B, N, 12), dtype=np.float64)
        assert out.dtype == np.float64 and out.shape == (B, N, 12) and out.flags.c_contiguous
        m = None
        if mask is not None:
            mask = np.ascontiguousarray(np.asarray(mask) != 0).view(np.uint8)
            assert mask.shape == (B,)
            m = mask.ctypes.data
        _check(lib().hmpc_predict_batch(self._h, records.ctypes.data, B, m, wrench.ctypes.data, out.ctypes.data))
        return out

    def certify_device(self, d_records, B: int, d_wrench, d_cert, d_lambda=None, d_mask=None, stream=None) -> None:
        """The certificate on the device (hmpc_certify_device): is robot i's wrench a KKT point of its record's QP?  torch
        CUDA tensors: records uint8 [B,stride], wrench f32 [B,12N], d_cert uint8 [B,40] (view as CERTIFICATE_DTYPE on the
        host), d_lambda f32 [B,N,2,8] or None; `d_mask` bool or uint8 [B] or None (every robot): unlisted rows keep their
        bytes.  Enqueued on the current stream; capturable in a CUDA graph."""
        import torch

        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_certify_device(self._h, d_records.data_ptr(), B, d_mask.data_ptr() if d_mask is not None else None,
                                         d_wrench.data_ptr(), d_cert.data_ptr(),
                                         d_lambda.data_ptr() if d_lambda is not None else None, ctypes.c_void_p(st)))

    def certify_batch(self, records: np.ndarray, wrench: np.ndarray, mask=None, out=None, lam=None):
        """The certificate from host buffers (hmpc_certify_batch): `records` update_data_t [B], `wrench` f64 [B,12N] ->
        CERTIFICATE_DTYPE [B] (`out`), and with `lam` (f64 [B,N,2,8], or True for a new array) the multipliers:
        -> (cert, lam).  In place when records, wrench, out and lam are pinned (pin()).  With a mask, unlisted rows are not
        written."""
        records = np.ascontiguousarray(records, dtype=UPDATE_DTYPE)
        B, N = records.shape[0], self.horizon
        wrench = np.ascontiguousarray(wrench, dtype=np.float64)
        assert wrench.shape == (B, 12 * N)
        if out is None:
            out = np.zeros(B, CERTIFICATE_DTYPE)
        assert out.dtype == CERTIFICATE_DTYPE and out.shape == (B,) and out.flags.c_contiguous
        want_lam = lam is not None and lam is not False
        if lam is True:
            lam = np.zeros((B, N, 2, 8), np.float64)
        if want_lam:
            assert lam.dtype == np.float64 and lam.shape == (B, N, 2, 8) and lam.flags.c_contiguous
        m = None
        if mask is not None:
            mask = np.ascontiguousarray(np.asarray(mask) != 0).view(np.uint8)
            assert mask.shape == (B,)
            m = mask.ctypes.data
        _check(lib().hmpc_certify_batch(self._h, records.ctypes.data, B, m, wrench.ctypes.data, out.ctypes.data,
                                        lam.ctypes.data if want_lam else None))
        return (out, lam) if want_lam else out

    def solve_device_multi(self, d_records, B: int, d_traj, d_wrench, d_status, d_cost=None, d_mask=None, stream=None) -> None:
        """Robot i's MPC for K candidate reference trajectories at once (hmpc_solve_device_multi).  torch CUDA tensors:
        records uint8 [B,stride]; d_traj f32 [B,K,12N] (laid out like the record's traj, which is not read); results d_wrench
        f32 [B,K,12N], d_status i32 [B,K], d_cost f64 [B,K] or None: the tracking cost J of certify_device, for ranking the
        candidates.  Candidate (i,k) equals solve_device on robot i's record with traj k, bit for bit.  `d_mask` bool or uint8
        [B] or None: unlisted robots' rows keep their bytes.  Cold, enqueued on the current stream, capturable."""
        import torch

        K = d_traj.shape[1]
        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_solve_device_multi(self._h, d_records.data_ptr(), B, K, d_traj.data_ptr(),
                                             d_mask.data_ptr() if d_mask is not None else None, d_wrench.data_ptr(),
                                             d_status.data_ptr(), d_cost.data_ptr() if d_cost is not None else None,
                                             ctypes.c_void_p(st)))

    def solve_batch_multi(self, records: np.ndarray, traj: np.ndarray, mask=None, cost: bool = True, strict: bool = True,
                          out=None):
        """solve_device_multi from host buffers (hmpc_solve_batch_multi): `records` update_data_t [B], `traj` f32 [B,K,12N]
        -> (wrench f64 [B,K,12N], status i32 [B,K], cost f64 [B,K] or None).  `out=(wrench, status, cost)` reuses the
        caller's arrays (cost may be None); in place when records, traj and every output are pinned (pin()).  With a mask
        only listed robots' rows are written.  strict: raise when a listed candidate did not converge."""
        records = np.ascontiguousarray(records, dtype=UPDATE_DTYPE)
        traj = np.ascontiguousarray(traj, dtype=np.float32)
        B, N = records.shape[0], self.horizon
        assert traj.ndim == 3 and traj.shape[0] == B and traj.shape[2] == 12 * N
        K = traj.shape[1]
        if out is None:
            out = (np.zeros((B, K, 12 * N), np.float64), np.zeros((B, K), np.int32), np.zeros((B, K), np.float64) if cost else None)
        w, st, c = out
        assert w.dtype == np.float64 and w.shape == (B, K, 12 * N) and w.flags.c_contiguous
        assert st.dtype == np.int32 and st.shape == (B, K) and st.flags.c_contiguous
        assert c is None or (c.dtype == np.float64 and c.shape == (B, K) and c.flags.c_contiguous)
        m = None
        if mask is not None:
            mask = np.ascontiguousarray(np.asarray(mask) != 0).view(np.uint8)
            assert mask.shape == (B,)
            m = mask.ctypes.data
        _check(lib().hmpc_solve_batch_multi(self._h, records.ctypes.data, B, K, traj.ctypes.data, m, w.ctypes.data,
                                            st.ctypes.data, c.ctypes.data if c is not None else None),
               allow_not_converged=not strict)
        return w, st, c

    def solve_states_device_multi(self, d_states, B: int, d_cmd, d_records, d_traj, d_wrench, d_status, d_cost, d_best,
                                  d_tau=None, d_mask=None, stream=None, dt_mpc: float = 0.04) -> None:
        """Robot i's MPC for K candidate commands from its state, the cheapest converged one picked on the device
        (hmpc_solve_states_device_multi).  torch CUDA tensors: d_states uint8 [B,352], d_cmd uint8 [B,K,56] or f64 [B,K,7]
        (COMMAND_DTYPE: state_des, world_position_desired); d_records uint8 [B,stride] receives the record of the chosen
        command, d_traj f32 [B,K,12N] the candidates' trajectories; results d_wrench f32 [B,K,12N], d_status i32 [B,K], d_cost
        f64 [B,K], d_best i32 [B] (-1: no candidate converged), d_tau f32 [B,10] or None (the chosen candidate's torques).
        Each equals the expanded batch's prepare_device / solve_device_ex / certify_device, bit for bit.  `d_mask` bool or
        uint8 [B] or None: unlisted robots' rows keep their bytes.  Cold, enqueued on the current stream, capturable."""
        import torch

        K = d_traj.shape[1]
        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_solve_states_device_multi(self._h, d_states.data_ptr(), B, K, d_cmd.data_ptr(),
                                                    d_mask.data_ptr() if d_mask is not None else None, dt_mpc,
                                                    d_records.data_ptr(), d_traj.data_ptr(), d_wrench.data_ptr(),
                                                    d_status.data_ptr(), d_cost.data_ptr(), d_best.data_ptr(),
                                                    d_tau.data_ptr() if d_tau is not None else None, ctypes.c_void_p(st)))

    def solve_batch_states_multi(self, states: np.ndarray, cmd: np.ndarray, mask=None, torques: bool = True,
                                 strict: bool = True, out=None, dt_mpc: float = 0.04):
        """solve_states_device_multi from host buffers (hmpc_solve_batch_states_multi): `states` STATE_DTYPE [B], `cmd`
        COMMAND_DTYPE [B,K] -> (wrench f64 [B,K,12N], status i32 [B,K], cost f64 [B,K], best i32 [B], tau f64 [B,10] or
        None).  `out=(wrench, status, cost, best, tau)` reuses the caller's arrays (tau may be None); in place when states,
        cmd and every output but tau are pinned (pin()).  With a mask only listed robots' rows are written.  strict: raise
        when a listed robot has no converged candidate (best == -1)."""
        states = np.ascontiguousarray(states, dtype=STATE_DTYPE)
        cmd = np.ascontiguousarray(cmd, dtype=COMMAND_DTYPE)
        B, N = states.shape[0], self.horizon
        assert cmd.ndim == 2 and cmd.shape[0] == B
        K = cmd.shape[1]
        if out is None:
            out = (np.zeros((B, K, 12 * N), np.float64), np.zeros((B, K), np.int32), np.zeros((B, K), np.float64),
                   np.zeros(B, np.int32), np.zeros((B, 10), np.float64) if torques else None)
        w, st, c, best, tau = out
        assert w.dtype == np.float64 and w.shape == (B, K, 12 * N) and w.flags.c_contiguous
        assert st.dtype == np.int32 and st.shape == (B, K) and st.flags.c_contiguous
        assert c.dtype == np.float64 and c.shape == (B, K) and c.flags.c_contiguous
        assert best.dtype == np.int32 and best.shape == (B,) and best.flags.c_contiguous
        assert tau is None or (tau.dtype == np.float64 and tau.shape == (B, 10) and tau.flags.c_contiguous)
        m = None
        if mask is not None:
            mask = np.ascontiguousarray(np.asarray(mask) != 0).view(np.uint8)
            assert mask.shape == (B,)
            m = mask.ctypes.data
        _check(lib().hmpc_solve_batch_states_multi(self._h, states.ctypes.data, B, K, cmd.ctypes.data, m, dt_mpc,
                                                   w.ctypes.data, st.ctypes.data, c.ctypes.data, best.ctypes.data,
                                                   tau.ctypes.data if tau is not None else None),
               allow_not_converged=not strict)
        return w, st, c, best, tau

    def assemble_device(self, d_records, B: int, stream=None) -> dict:
        """Parity hook: un-reduced fp32 QP data of B packed records (torch tensors on the GPU)."""
        import torch

        N = self.horizon
        dev = torch.device("cuda", self.device)
        out = dict(
            H=torch.zeros((B, 12 * N, 12 * N), dtype=torch.float32, device=dev),
            g=torch.zeros((B, 12 * N), dtype=torch.float32, device=dev),
            Fblk=torch.zeros((B, 16, 12), dtype=torch.float32, device=dev),
            lb=torch.zeros((B, 16 * N), dtype=torch.float32, device=dev),
            ub=torch.zeros((B, 16 * N), dtype=torch.float32, device=dev),
        )
        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        _check(lib().hmpc_assemble_device(self._h, d_records.data_ptr(), B, out["H"].data_ptr(), out["g"].data_ptr(),
                                          out["Fblk"].data_ptr(), out["lb"].data_ptr(), out["ub"].data_ptr(),
                                          ctypes.c_void_p(st)))
        return out

    def close(self) -> None:
        if getattr(self, "_h", None):
            lib().hmpc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
