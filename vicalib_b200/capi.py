"""ctypes binding of libvcgpu.so (include/vcgpu.h) — the reference-facing boundary.

`Calibrator` mirrors the slice of `ViCalibrator` (include/vicalib/vicalibrator.h:119-1086) that
the calibration solve needs, on top of the C-ABI: upload cameras / frames / observations / IMU,
set the optimisation flags, solve, read the state back.  There is NO CPU fallback: if the CUDA
library is missing or no GPU is present this raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvcgpu.so")
_LIB = None

EXPORTS = [
    "vcgpu_create", "vcgpu_destroy", "vcgpu_last_error", "vcgpu_set_cameras", "vcgpu_set_frames",
    "vcgpu_set_observations", "vcgpu_set_imu", "vcgpu_set_imu_params", "vcgpu_set_flags",
    "vcgpu_set_options", "vcgpu_default_flags", "vcgpu_default_options", "vcgpu_register_mirrors",
    "vcgpu_solve", "vcgpu_iterate", "vcgpu_evaluate", "vcgpu_cost", "vcgpu_remove_outliers",
    "vcgpu_get_obs_active", "vcgpu_update_imu_weights", "vcgpu_get_imu_weights", "vcgpu_set_imu_weights",
    "vcgpu_get_state", "vcgpu_num_residuals", "vcgpu_frame_dim", "vcgpu_num_globals", "vcgpu_eval_reproj",
    "vcgpu_eval_imu", "vcgpu_normal_equations", "vcgpu_solve_arrow", "vcgpu_comm_unique_id", "vcgpu_comm_init",
    "vcgpu_set_profiling", "vcgpu_get_stage_times", "vcgpu_fp64_peak", "vcgpu_get_phase_clocks", "vcgpu_get_covariance", "vcgpu_pose_pnp_ransac",
]


class Flags(C.Structure):
    _fields_ = [("inertial", C.c_int), ("rotation_only", C.c_int), ("bias_active", C.c_int),
                ("scale_active", C.c_int), ("optimize_ts", C.c_int), ("fix_intrinsics", C.c_int),
                ("visual", C.c_int), ("visual_mult", C.c_double), ("imu_mult", C.c_double)]


class Options(C.Structure):
    _fields_ = [("max_iters", C.c_int), ("function_tol", C.c_double), ("gradient_tol", C.c_double),
                ("param_tol", C.c_double), ("init_radius", C.c_double), ("strategy", C.c_int),
                ("jacobi_scaling", C.c_int), ("update_imu_weights", C.c_int),
                ("update_state_every_iteration", C.c_int)]


class Iteration(C.Structure):
    _fields_ = [("iteration", C.c_int), ("step_is_successful", C.c_int), ("cost", C.c_double),
                ("cost_change", C.c_double), ("gradient_max_norm", C.c_double), ("gradient_norm", C.c_double),
                ("step_norm", C.c_double), ("relative_decrease", C.c_double), ("trust_region_radius", C.c_double)]


class Summary(C.Structure):
    _fields_ = [("iterations", C.c_int), ("successful_steps", C.c_int), ("termination", C.c_int),
                ("num_residuals", C.c_int), ("initial_cost", C.c_double), ("final_cost", C.c_double),
                ("device_seconds", C.c_double), ("kernel_launches", C.c_int)]


class Config(C.Structure):
    _fields_ = [("device", C.c_int)]


ITER_CB = C.CFUNCTYPE(C.c_int, C.POINTER(Iteration), C.c_void_p)


class VcgpuError(RuntimeError):
    pass


def lib():
    """Load libvcgpu.so; fails loudly when it has not been built (no fallback path exists)."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise VcgpuError(f"{LIB_PATH} is missing: build it with __graft_entry__.build() "
                             "(make -C vicalib_b200/csrc); there is no CPU fallback")
        L = C.CDLL(LIB_PATH)
        L.vcgpu_last_error.restype = C.c_char_p
        L.vcgpu_last_error.argtypes = [C.c_void_p]
        _LIB = L
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _c(a, dt=np.float64):
    return np.ascontiguousarray(a, dtype=dt)


class Calibrator:
    """Host-side mirror of the ViCalibrator solve API over the C-ABI."""

    def __init__(self, device: int = -1):
        self.L = lib()
        self.h = C.c_void_p()
        rc = self.L.vcgpu_create(C.byref(Config(device)), C.byref(self.h))
        if rc != 0:
            raise VcgpuError(f"vcgpu_create failed ({rc}): a CUDA device is required; there is no CPU fallback")
        self.flags = Flags()
        self.opts = Options()
        self.L.vcgpu_default_flags(C.byref(self.flags))
        self.L.vcgpu_default_options(C.byref(self.opts))
        self.n_cams = self.n_frames = self.n_obs = 0
        self._keep = []

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.vcgpu_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc):
        if rc != 0:
            raise VcgpuError(f"vcgpu error {rc}: {self.L.vcgpu_last_error(self.h).decode()}")

    # ---- uploads (AddCamera / AddFrame / AddObservation / AddImuMeasurements, vicalibrator.h:332-468)
    def set_cameras(self, models, intr, q_ck, p_ck):
        self.n_cams = len(models)
        self._chk(self.L.vcgpu_set_cameras(self.h, C.c_int(self.n_cams), _p(_c(models, np.int32)), _p(_c(intr)),
                                           _p(_c(q_ck)), _p(_c(p_ck))))

    def set_frames(self, T_wp, v_w, ftime):
        self.n_frames = len(ftime)
        self._chk(self.L.vcgpu_set_frames(self.h, C.c_int(self.n_frames), _p(_c(T_wp)), _p(_c(v_w)), _p(_c(ftime))))

    def set_observations(self, frame_id, cam_id, p_w, p_c):
        self.n_obs = len(frame_id)
        self._chk(self.L.vcgpu_set_observations(self.h, C.c_int64(self.n_obs), _p(_c(frame_id, np.int32)),
                                                _p(_c(cam_id, np.int32)), _p(_c(p_w)), _p(_c(p_c))))

    def set_imu(self, t, w, a, sigma_g, sigma_a):
        self._chk(self.L.vcgpu_set_imu(self.h, C.c_int(len(t)), _p(_c(t)), _p(_c(w)), _p(_c(a)),
                                       C.c_double(sigma_g), C.c_double(sigma_a)))

    def set_imu_params(self, g, b, sf, ts):
        self._chk(self.L.vcgpu_set_imu_params(self.h, _p(_c(g)), _p(_c(b)), _p(_c(sf)), C.c_double(ts)))

    def load(self, p):
        """Upload a vicalib_b200.synth.Problem (or anything with the same fields)."""
        from .synth import ACCEL_SIGMA, GYRO_SIGMA

        self.set_cameras(p.models, p.intr, p.q_ck, p.p_ck)
        self.set_frames(p.T_wp, p.v_w, p.ftime)
        self.set_observations(p.obs_frame, p.obs_cam, p.p_w, p.p_c)
        self.set_imu(p.imu_t, p.imu_w, p.imu_a, GYRO_SIGMA, ACCEL_SIGMA)
        self.set_imu_params(p.g, p.b, p.sf, p.ts)

    def set_flags(self, **kw):
        for k, v in kw.items():
            setattr(self.flags, k, v)
        self._chk(self.L.vcgpu_set_flags(self.h, C.byref(self.flags)))

    def set_options(self, **kw):
        for k, v in kw.items():
            setattr(self.opts, k, v)
        self._chk(self.L.vcgpu_set_options(self.h, C.byref(self.opts)))

    # ---- multi-GPU (one process per GPU; frames sharded; NCCL all-reduce of the reduced system)
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        if lib().vcgpu_comm_unique_id(buf) != 0:
            raise VcgpuError("ncclGetUniqueId failed")
        return bytes(buf)

    def comm_init(self, unique_id: bytes, rank: int, nranks: int):
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        self._chk(self.L.vcgpu_comm_init(self.h, buf, C.c_int(rank), C.c_int(nranks)))

    # ---- hot path
    def solve(self, callback=None, free_running=False):
        """Solve; `rows` holds one row per iteration.  free_running: no iteration callback at all, so the device runs
        the loop in batches without a host round trip per iteration (no rows; `callback` must be None)."""
        s = Summary()
        rows = []

        def _cb(itp, _user):
            it = itp.contents
            rows.append([it.iteration, it.cost, it.cost_change, it.gradient_max_norm, it.gradient_norm,
                         it.step_norm, it.relative_decrease, it.trust_region_radius, it.step_is_successful])
            return int(callback(it)) if callback else 0

        if free_running and callback is not None:
            raise ValueError("a free-running solve takes no callback")
        cb = None if free_running else ITER_CB(_cb)
        self._chk(self.L.vcgpu_solve(self.h, cb, None, C.byref(s)))
        out = {f[0]: getattr(s, f[0]) for f in Summary._fields_}
        out["rows"] = np.array(rows)
        return out

    def iterate(self, n):
        s = Summary()
        self._chk(self.L.vcgpu_iterate(self.h, C.c_int(n), C.byref(s)))
        return {f[0]: getattr(s, f[0]) for f in Summary._fields_}

    def cost(self):
        c = C.c_double()
        self._chk(self.L.vcgpu_cost(self.h, C.byref(c)))
        return c.value

    def evaluate(self, cam=-1, residuals=False):
        c = C.c_double()
        n = C.c_int64()
        res = np.zeros(2 * self.n_obs) if residuals else None
        self._chk(self.L.vcgpu_evaluate(self.h, C.c_int(cam), C.byref(c), _p(res), C.byref(n)))
        return (c.value, res[: 2 * n.value], n.value) if residuals else (c.value, n.value)

    def remove_outliers(self, rmse, threshold):
        n = C.c_int64()
        self._chk(self.L.vcgpu_remove_outliers(self.h, _p(_c(rmse)), C.c_double(threshold), C.byref(n)))
        return n.value

    def obs_active(self):
        a = np.zeros(self.n_obs, dtype=np.uint8)
        self._chk(self.L.vcgpu_get_obs_active(self.h, _p(a)))
        return a

    def state(self):
        s = dict(intr=np.zeros((self.n_cams, 10)), q_ck=np.zeros((self.n_cams, 4)), p_ck=np.zeros((self.n_cams, 3)),
                 T_wp=np.zeros((self.n_frames, 7)), v_w=np.zeros((self.n_frames, 3)), g=np.zeros(2), b=np.zeros(6),
                 sf=np.zeros(6))
        ts = C.c_double()
        self._chk(self.L.vcgpu_get_state(self.h, _p(s["intr"]), _p(s["q_ck"]), _p(s["p_ck"]), _p(s["T_wp"]),
                                         _p(s["v_w"]), _p(s["g"]), _p(s["b"]), _p(s["sf"]), C.byref(ts)))
        s["ts"] = ts.value
        return s

    @property
    def fd(self):
        v = C.c_int()
        self._chk(self.L.vcgpu_frame_dim(self.h, C.byref(v)))
        return v.value

    @property
    def G(self):
        v = C.c_int()
        self._chk(self.L.vcgpu_num_globals(self.h, C.byref(v)))
        return v.value

    def num_residuals(self):
        v = C.c_int()
        self._chk(self.L.vcgpu_num_residuals(self.h, C.byref(v)))
        return v.value

    # ---- inspection hooks (parity tests)
    def eval_reproj(self, jac=True):
        r = np.zeros((self.n_obs, 2))
        J = np.zeros((self.n_obs, 2, 22)) if jac else None
        self._chk(self.L.vcgpu_eval_reproj(self.h, _p(r), _p(J)))
        return r, J

    def eval_imu(self, jac=True):
        n = max(self.n_frames - 1, 0)
        r = np.zeros((n, 9))
        J = np.zeros((n, 9, 33)) if jac else None
        self._chk(self.L.vcgpu_eval_imu(self.h, _p(r), _p(J)))
        return r, J

    def normal_equations(self):
        nf, fd, G = self.n_frames, self.fd, self.G
        out = dict(B=np.zeros((nf, fd, fd)), U=np.zeros((nf, fd, fd)), E=np.zeros((nf, fd, G)),
                   gf=np.zeros((nf, fd)), C=np.zeros((G, G)), gc=np.zeros(G))
        c = C.c_double()
        self._chk(self.L.vcgpu_normal_equations(self.h, _p(out["B"]), _p(out["U"]), _p(out["E"]), _p(out["gf"]),
                                                _p(out["C"]), _p(out["gc"]), C.byref(c)))
        out["cost"] = c.value
        return out

    def solve_arrow(self, scale, D2):
        x = np.zeros(self.n_frames * self.fd + self.G)
        self._chk(self.L.vcgpu_solve_arrow(self.h, _p(_c(scale)), _p(_c(D2)), _p(x)))
        return x

    STAGES = ["diag", "frame_solve", "global_solve", "backsub", "eval_reproj", "build_frames", "reduce_globals",
              "finalize", "imu_eval", "imu_weights", "grid_sync", "eval_tasks", "imu_accumulate"]

    def set_profiling(self, profile=True, flush_l2=False):
        self._chk(self.L.vcgpu_set_profiling(self.h, C.c_int(int(profile)), C.c_int(int(flush_l2))))

    def fp64_peak(self, device=0):
        """Measured FP64 throughput (TFLOP/s): (vector DFMA, tensor DMMA m8n8k4)."""
        a, b = C.c_double(0.0), C.c_double(0.0)
        self._chk(self.L.vcgpu_fp64_peak(C.c_int(device), C.byref(a), C.byref(b)))
        return a.value, b.value

    def stage_times(self):
        ms = np.zeros(16)
        n = np.zeros(16, dtype=np.int64)
        self._chk(self.L.vcgpu_get_stage_times(self.h, _p(ms), _p(n)))
        return {name: (float(ms[i]), int(n[i])) for i, name in enumerate(self.STAGES)}

    def pose_pnp_ransac(self, cam_id, start, count, pix, pw, robust_its=0, robust_tol=0.0):
        """batched PosePnPRansac: one (camera, correspondence range) per view -> (T_cw [n, 7], rmse [n], n_used [n])"""
        n = len(cam_id)
        T = np.zeros((n, 7))
        rmse = np.zeros(n)
        used = np.zeros(n, dtype=np.int32)
        self._chk(self.L.vcgpu_pose_pnp_ransac(self.h, C.c_int(n), _p(_c(cam_id, np.int32)), _p(_c(start, np.int64)),
                                               _p(_c(count, np.int32)), _p(_c(pix)), _p(_c(pw)), C.c_int(robust_its),
                                               C.c_double(robust_tol), _p(T), _p(rmse), _p(used)))
        return T, rmse, used

    def covariance(self):
        """GetSolutionCovariance: tangent covariance of the globals, G x G"""
        G = self.G
        cov = np.zeros((G, G))
        self._chk(self.L.vcgpu_get_covariance(self.h, _p(cov)))
        return cov

    def phase_clocks(self):
        """raw phase clocks (ns) of the persistent inertial kernels, see vcgpu_get_phase_clocks"""
        ns = np.zeros(64, dtype=np.uint64)
        self._chk(self.L.vcgpu_get_phase_clocks(self.h, _p(ns)))
        return ns

    def update_imu_weights(self):
        self._chk(self.L.vcgpu_update_imu_weights(self.h))

    def imu_weights(self):
        w = np.zeros((max(self.n_frames - 1, 0), 9, 9))
        self._chk(self.L.vcgpu_get_imu_weights(self.h, _p(w)))
        return w

    def set_imu_weights(self, w):
        self._chk(self.L.vcgpu_set_imu_weights(self.h, _p(_c(w))))
