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
    "vcgpu_solve", "vcgpu_solve_batch", "vcgpu_batch_plan", "vcgpu_solve_batch_inertial", "vcgpu_batch_plan_inertial", "vcgpu_iterate", "vcgpu_evaluate", "vcgpu_cost", "vcgpu_remove_outliers",
    "vcgpu_get_obs_active", "vcgpu_update_imu_weights", "vcgpu_get_imu_weights", "vcgpu_set_imu_weights",
    "vcgpu_get_state", "vcgpu_num_residuals", "vcgpu_frame_dim", "vcgpu_num_globals", "vcgpu_eval_reproj",
    "vcgpu_eval_imu", "vcgpu_normal_equations", "vcgpu_solve_arrow", "vcgpu_comm_unique_id", "vcgpu_comm_init",
    "vcgpu_set_profiling", "vcgpu_get_stage_times", "vcgpu_fp64_peak", "vcgpu_get_phase_clocks", "vcgpu_get_covariance", "vcgpu_get_covariance_batch",
    "vcgpu_get_frame_covariance", "vcgpu_get_frame_covariance_batch", "vcgpu_evaluate_batch", "vcgpu_remove_outliers_batch",
    "vcgpu_pose_pnp_ransac", "vcgpu_pose_pnp_ransac_batch", "vcgpu_calibrate_batch",
    "vcgpu_get_frame_cross_covariance", "vcgpu_get_frame_cross_covariance_batch",
    "vcgpu_get_imu_mahalanobis", "vcgpu_get_imu_mahalanobis_batch",
    "vcgpu_get_integration_poses", "vcgpu_get_integration_poses_batch",
    "vcgpu_get_projection_covariance", "vcgpu_get_projection_covariance_batch",
    "vcgpu_get_view_information", "vcgpu_get_view_information_batch",
    "vcgpu_get_observation_influence", "vcgpu_get_observation_influence_batch",
    "vcgpu_get_imu_influence", "vcgpu_get_imu_influence_batch",
    "vcgpu_align_imu", "vcgpu_align_imu_batch",
]

CHI2_95_9 = 16.9190  # chi2inv(0.95, 9): the bound UpdateImuWeights logs each interval's distance against


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


class PnpViews(C.Structure):
    """vcgpu_pnp_views: one rig's views and outputs of vcgpu_pose_pnp_ransac_batch"""
    _fields_ = [("n_views", C.c_int), ("cam_id", C.c_void_p), ("start", C.c_void_p), ("count", C.c_void_p),
                ("pix", C.c_void_p), ("pw", C.c_void_p), ("T_cw", C.c_void_p), ("rmse_or_null", C.c_void_p),
                ("n_used_or_null", C.c_void_p)]


class ProjPoints(C.Structure):
    """vcgpu_proj_points: one rig's points and outputs of vcgpu_get_projection_covariance(_batch)"""
    _fields_ = [("n", C.c_int64), ("cam_id", C.c_void_p), ("pix", C.c_void_p), ("depth", C.c_void_p), ("frame", C.c_int),
                ("cov", C.c_void_p), ("ray_or_null", C.c_void_p)]


# vcgpu_proj_points::frame
PROJ_FRAMES = {"camera": 0, "rig": 1}


def _proj_points(cam_id, pix, depth, frame, rays):
    """the arrays of one rig's points and a ProjPoints over them (the arrays must outlive the call)"""
    if frame not in PROJ_FRAMES:
        raise ValueError(f"frame must be one of {sorted(PROJ_FRAMES)}, not {frame!r}")
    cam = _c(np.atleast_1d(cam_id), np.int32)
    n = len(cam)
    px = _c(pix).reshape(n, 2)
    d = None if depth is None else _c(np.broadcast_to(np.asarray(depth, dtype=np.float64), (n,)))
    cov = np.zeros((max(n, 1), 3))
    ray = np.zeros((max(n, 1), 3)) if rays else None
    pts = ProjPoints(n, cam.ctypes.data, px.ctypes.data, None if d is None else d.ctypes.data, PROJ_FRAMES[frame],
                     cov.ctypes.data, None if ray is None else ray.ctypes.data)
    return (cam, px, d, cov, ray), pts


def _proj_result(keep, n):
    cov, ray = keep[3][:n], keep[4]
    return cov if ray is None else (cov, ray[:n])


class ViewCandidates(C.Structure):
    """vcgpu_view_candidates: one rig's candidate views, target and outputs of vcgpu_get_view_information(_batch)"""
    _fields_ = [("n_cand", C.c_int64), ("T_wp", C.c_void_p), ("n_pts", C.c_int), ("p_w", C.c_void_p),
                ("facing", C.c_void_p), ("width", C.c_void_p), ("height", C.c_void_p), ("n_seen", C.c_void_p),
                ("gain", C.c_void_p), ("var_or_null", C.c_void_p), ("post_or_null", C.c_void_p)]


def _view_candidates(T_wp, p_w, width, height, facing, var, post, n_cams, G):
    """the arrays of one rig's candidates and a ViewCandidates over them (the arrays must outlive the call)"""
    T = _c(T_wp).reshape(-1, 7)
    pw = _c(p_w).reshape(-1, 3)
    n = len(T)
    wd = _c(np.broadcast_to(np.asarray(width), (n_cams,)), np.int32)
    ht = _c(np.broadcast_to(np.asarray(height), (n_cams,)), np.int32)
    fc = None if facing is None else _c(facing).reshape(3)
    seen = np.zeros((max(n, 1), n_cams), np.int32)
    gain = np.zeros(max(n, 1))
    vr = np.zeros((max(n, 1), G)) if var else None
    ps = np.zeros((max(n, 1), G, G)) if post else None
    v = ViewCandidates(n, T.ctypes.data, len(pw), pw.ctypes.data, None if fc is None else fc.ctypes.data, wd.ctypes.data,
                       ht.ctypes.data, seen.ctypes.data, gain.ctypes.data, None if vr is None else vr.ctypes.data,
                       None if ps is None else ps.ctypes.data)
    return (T, pw, wd, ht, fc, seen, gain, vr, ps), v


def _view_result(keep, n):
    """dict(gain, n_seen[, var][, post]) of one rig's call"""
    out = dict(gain=keep[6][:n], n_seen=keep[5][:n])
    if keep[7] is not None:
        out["var"] = keep[7][:n]
    if keep[8] is not None:
        out["post"] = keep[8][:n]
    return out


class ObsInfluence(C.Structure):
    """vcgpu_obs_influence: one rig's outputs of vcgpu_get_observation_influence(_batch), any of them NULL"""
    _fields_ = [("h", C.c_void_p), ("stud", C.c_void_p), ("infl", C.c_void_p)]


def _obs_influence(n_obs, h, stud, infl):
    """the output arrays of one rig and an ObsInfluence over them (the arrays must outlive the call)"""
    m = max(n_obs, 1)
    keep = (np.zeros((m, 3)) if h else None, np.zeros(m) if stud else None, np.zeros(m) if infl else None)
    return keep, ObsInfluence(*[None if a is None else a.ctypes.data for a in keep])


def _obs_influence_result(keep, n_obs):
    """dict(h[, stud][, infl]) of one rig's call"""
    return {k: a[:n_obs] for k, a in zip(("h", "stud", "infl"), keep) if a is not None}


class ImuInfluence(C.Structure):
    """vcgpu_imu_influence: one rig's outputs of vcgpu_get_imu_influence(_batch), any of them NULL"""
    _fields_ = [("h", C.c_void_p), ("stud", C.c_void_p), ("infl", C.c_void_p)]


def _imu_influence(ni, h, stud, infl):
    """the output arrays of one rig's intervals and an ImuInfluence over them (the arrays must outlive the call)"""
    m = max(ni, 1)
    keep = (np.zeros((m, 9, 9)) if h else None, np.zeros(m) if stud else None, np.zeros(m) if infl else None)
    return keep, ImuInfluence(*[None if a is None else a.ctypes.data for a in keep])


def _imu_influence_result(keep, ni, obs_keep, n_obs):
    """dict(h[, stud][, infl][, observations]) of one rig's call"""
    out = {k: a[:ni] for k, a in zip(("h", "stud", "infl"), keep) if a is not None}
    if obs_keep is not None:
        out["observations"] = _obs_influence_result(obs_keep, n_obs)
    return out


class ImuAlignOpts(C.Structure):
    """vcgpu_imu_align_opts"""
    _fields_ = [("ts_lo", C.c_double), ("ts_hi", C.c_double), ("n_ts", C.c_int), ("find_time_offset", C.c_int),
                ("max_iters", C.c_int), ("apply", C.c_int)]


class ImuAlignment(C.Structure):
    """vcgpu_imu_alignment"""
    _fields_ = [("Q", C.c_double * 4), ("ts", C.c_double), ("b_g", C.c_double * 3), ("rms", C.c_double),
                ("excitation", C.c_double * 3), ("n_intervals", C.c_int), ("iterations", C.c_int),
                ("curve_or_null", C.c_void_p)]


def _align_args(ts_lo, ts_hi, n_ts, find_time_offset, max_iters, apply, curve):
    """the opts, the output struct and the curve array of one rig (the array must outlive the call)"""
    c = np.full(max(int(n_ts), 1), np.nan) if curve else None
    o = ImuAlignOpts(float(ts_lo), float(ts_hi), int(n_ts), int(bool(find_time_offset)), int(max_iters), int(bool(apply)))
    return o, ImuAlignment(curve_or_null=None if c is None else c.ctypes.data), c


def _align_result(a, c, status):
    """dict(Q, ts, b_g, rms, excitation, n_intervals, iterations, status[, curve]) of one rig"""
    out = dict(Q=np.array(a.Q[:]), ts=a.ts, b_g=np.array(a.b_g[:]), rms=a.rms, excitation=np.array(a.excitation[:]),
               n_intervals=a.n_intervals, iterations=a.iterations, status=int(status))
    if c is not None:
        out["curve"] = c
    return out


class Flow(C.Structure):
    """vcgpu_flow: the switches of ViCalibrator::SolveThread's stage machine (vcgpu_calibrate_batch)"""
    _fields_ = [("calibrate_imu", C.c_int), ("remove_outliers", C.c_int), ("outlier_threshold", C.c_double),
                ("block_duplication", C.c_int), ("gravity_initialized", C.c_int), ("max_solves", C.c_int)]


class FlowSummary(C.Structure):
    _fields_ = [("solves", C.c_int), ("iterations", C.c_int), ("finished", C.c_int), ("stage", C.c_int),
                ("outliers_removed", C.c_int64), ("mse", C.c_double), ("last", Summary), ("flags", Flags)]


# vcgpu_flow_summary::stage
FLOW_VISION, FLOW_ROTATION, FLOW_TRANSLATION, FLOW_SCALE, FLOW_FINISHED = range(5)


class Config(C.Structure):
    _fields_ = [("device", C.c_int)]


ITER_CB = C.CFUNCTYPE(C.c_int, C.POINTER(Iteration), C.c_void_p)


class VcgpuError(RuntimeError):
    """A negative return code of the library.  covariance_batch and frame_covariance_batch also set `status` (one code
    per rig) and `covariances` (the arrays written, None for the rigs whose system is not positive definite)."""

    status = None
    covariances = None


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

    def batch_plan(self):
        """(CTAs per cluster, warps per CTA, clusters of that shape resident at once) of this rig in solve_batch"""
        a, b, c = C.c_int(), C.c_int(), C.c_int()
        self._chk(self.L.vcgpu_batch_plan(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def batch_plan_inertial(self):
        """(CTAs per cluster, clusters of that size resident at once) of this rig in solve_batch_inertial"""
        a, c = C.c_int(), C.c_int()
        self._chk(self.L.vcgpu_batch_plan_inertial(self.h, C.byref(a), C.byref(c)))
        return a.value, c.value

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
        """profile bits: 1 stage events (multi-launch engine), 4 multi-launch engine, 8 persistent-kernel phase clocks;
        any other bit raises VcgpuError and leaves the handle as it was"""
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

    def frame_covariance(self):
        """GetCovarianceBlock(t_wp, t_wp) (and (v_w, v_w) with the inertial terms on) of every frame:
        (n_frames, fd, fd), each frame's tangent in the order of its rows in normal_equations()' B"""
        fd = self.fd
        cov = np.zeros((self.n_frames, fd, fd))
        self._chk(self.L.vcgpu_get_frame_covariance(self.h, _p(cov)))
        return cov

    def frame_cross_covariance(self):
        """GetCovarianceBlock(t_wp[f], globals) and (t_wp[f], t_wp[f+1]) of every frame (with v_w likewise when the
        inertial terms are on): (fg [n_frames, fd, G], fn [n_frames - 1, fd, fd]); rows as frame_covariance()'s,
        columns of fg as covariance()'s"""
        fd, nf = self.fd, self.n_frames
        fg, fn = np.zeros((nf, fd, self.G)), np.zeros((max(nf - 1, 0), fd, fd))
        self._chk(self.L.vcgpu_get_frame_cross_covariance(self.h, _p(fg), _p(fn)))
        return fg, fn

    def imu_mahalanobis(self, residuals=False):
        """Each IMU interval's Mahalanobis distance as UpdateImuWeights logs it against CHI2_95_9 (vicalibrator.h:786-794),
        at the current state: (n_frames - 1,) distances, NaN where an interval has no measurements or its covariance
        is not positive definite; residuals=True also returns the reference's 9-vector residuals, (n_frames - 1, 9)
        (NaN rows without measurements).  Nothing on the handle changes."""
        n = max(self.n_frames - 1, 0)
        d = np.zeros(max(n, 1))
        r = np.zeros((max(n, 1), 9)) if residuals else None
        self._chk(self.L.vcgpu_get_imu_mahalanobis(self.h, _p(d), _p(r)))
        return (d[:n], r[:n]) if residuals else d[:n]

    def integration_poses(self):
        """GetIntegrationPoses(k) of every interval k (vicalibrator.h:508-533) at the current state: n_frames - 1 arrays
        of (count_k, 14) rows q (x y z w) | t (3) | v_w (3) | w_w (3) | time, the frame's own pose first, count_k the
        interval's number of IMU measurements (0 without any).  Computed in rotation-only stages too.  Nothing on the
        handle changes."""
        start = np.zeros(max(self.n_frames, 1), dtype=np.int64)
        self._chk(self.L.vcgpu_get_integration_poses(self.h, _p(start), None))
        poses = np.zeros((max(int(start[-1]), 1), 14))
        self._chk(self.L.vcgpu_get_integration_poses(self.h, _p(start), _p(poses)))
        return _split_poses(start, poses)

    def projection_covariance(self, cam_id, pix, depth=None, frame="camera", cov=None, rays=False):
        """The pixel covariance the calibration leaves at projected points (vcgpu_get_projection_covariance): point i is
        pixel pix[i] (n, 2) of camera cam_id[i] at distance depth[i] along its ray (None or 0: at infinity), fixed in
        the camera frame ("camera": only the intrinsics move it) or in the rig frame ("rig": q_ck and p_ck too).
        Returns (n, 3) rows S_uu, S_uv, S_vv for unit observation variance (scale by the residual variance), NaN
        outside the lens model's domain; rays=True also returns the (n, 3) unit rays.  cov: the G x G matrix of
        covariance() to use instead of computing it.  Nothing on the handle changes."""
        keep, pts = _proj_points(cam_id, pix, depth, frame, rays)
        S = None if cov is None else _c(cov).reshape(self.G, self.G)
        self._chk(self.L.vcgpu_get_projection_covariance(self.h, _p(S), C.byref(pts)))
        return _proj_result(keep, pts.n)

    def view_information(self, T_wp, p_w, width, height, facing=None, cov=None, var=False, post=False):
        """The information candidate views of the target would add to the globals (vcgpu_get_view_information):
        T_wp (n, 7) candidate rig poses (q | t), p_w (m, 3) the target's points in the world frame, width / height
        each camera's image size (a scalar for all), facing the target's front normal or None.  Returns a dict:
        gain (n,) the entropy in nats the view removes from the globals (NaN: the view does not fix its pose),
        n_seen (n, n_cams), and with var=True the posterior variances (n, G), with post=True the posterior matrices
        (n, G, G).  cov: the G x G prior to use instead of covariance(), e.g. an earlier post.  Nothing on the handle
        changes."""
        keep, v = _view_candidates(T_wp, p_w, width, height, facing, var, post, self.n_cams, self.G)
        S = None if cov is None else _c(cov).reshape(self.G, self.G)
        self._chk(self.L.vcgpu_get_view_information(self.h, _p(S), C.byref(v)))
        return _view_result(keep, v.n_cand)

    def observation_influence(self, h=True, stud=True, infl=True):
        """Regression diagnostics of every reprojection observation, active or removed, in upload order
        (vcgpu_get_observation_influence): h (n, 3) the leverage H_uu, H_uv, H_vv; stud (n,) the studentized (deleted)
        residual, or for a removed observation its predictive residual; infl (n,) the shift of the globals its deletion
        (or re-admission) causes, measured in the globals' covariance.  stud and infl assume unit observation variance:
        divide by the residual variance before reading them against chi-square quantiles.  NaN where the observation's
        camera or vision frame is not determined.  Only the outputs asked for are returned.  Nothing on the handle
        changes."""
        keep, o = _obs_influence(self.n_obs, h, stud, infl)
        self._chk(self.L.vcgpu_get_observation_influence(self.h, C.byref(o)))
        return _obs_influence_result(keep, self.n_obs)

    def imu_influence(self, h=True, stud=True, infl=True, observations=False):
        """Regression diagnostics of every IMU interval k = 0 .. n_frames - 2 (vcgpu_get_imu_influence): h (n, 9, 9) the
        leverage H_k; stud (n,) the studentized (deleted) residual; infl (n,) the shift of the globals the interval's
        deletion causes, measured in the globals' covariance (the observation call's metric).  stud and infl assume unit
        observation variance.  NaN in all three for an interval with no measurements; stud and infl NaN where I - H_k is
        not positive definite.  observations=True adds "observations", observation_influence()'s dict from the same
        elimination.  Only the outputs asked for are returned.  Nothing on the handle changes."""
        ni = max(self.n_frames - 1, 0)
        keep, o = _imu_influence(ni, h, stud, infl)
        okeep, oo = _obs_influence(self.n_obs, True, True, True) if observations else (None, None)
        self._chk(self.L.vcgpu_get_imu_influence(self.h, C.byref(o), C.byref(oo) if observations else None))
        return _imu_influence_result(keep, ni, okeep, self.n_obs)

    def align_imu(self, ts_lo=-0.1, ts_hi=0.1, n_ts=401, find_time_offset=True, max_iters=20, apply=False, curve=False):
        """vcgpu_align_imu: the rotation Q (IMU axes to the current rig axes, x y z w with w >= 0), time offset ts and
        gyro bias b_g that align the gyro stream with the frame poses' turns, from a grid of n_ts offsets in
        [ts_lo, ts_hi] and a Gauss-Newton refinement.  Returns dict(Q, ts, b_g, rms, excitation, n_intervals, iterations,
        status[, curve]); status is 0, or -3 (VCGPU_ERR_NUMERIC: fewer than 3 usable intervals or a singular fit; Q, ts,
        b_g and rms are then NaN and nothing is applied).  apply=True puts the result on the handle: q_ck and every
        frame's rotation right-multiplied by Q, ts and b_g replaced.  The inertial flag is not required."""
        o, a, c = _align_args(ts_lo, ts_hi, n_ts, find_time_offset, max_iters, apply, curve)
        rc = self.L.vcgpu_align_imu(self.h, C.byref(o), C.byref(a))
        if rc not in (0, -3):
            self._chk(rc)
        return _align_result(a, c, rc)

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


def solve_batch(calibrators):
    """vcgpu_solve_batch: solve every Calibrator of the list in one call, each rig in its own thread-block cluster
    (free-running: no callback, no rows).  Returns one summary dict per calibrator, in order."""
    return _solve_many(lib().vcgpu_solve_batch, calibrators)


def solve_batch_inertial(calibrators):
    """vcgpu_solve_batch_inertial: solve_batch for rigs with inertial terms on (each rig in its own thread-block cluster
    of the persistent inertial kernels).  Returns one summary dict per calibrator, in order."""
    return _solve_many(lib().vcgpu_solve_batch_inertial, calibrators)


def calibrate_batch(calibrators, calibrate_imu=True, remove_outliers=True, outlier_threshold=2.0, block_duplication=True,
                    gravity_initialized=False, max_solves=100):
    """vcgpu_calibrate_batch: ViCalibrator::SolveThread's staged flow for every Calibrator of the list in one call,
    each rig from the stage its flags describe.  Returns one (summary dict, per-camera RMSE array) per calibrator, in
    order; the dict holds solves, iterations, finished, stage (FLOW_*), outliers_removed, mse, `last` (the last
    solve's summary dict) and `flags` (a dict of the handle's flags at return, which also become the calibrator's)."""
    n = len(calibrators)
    L = lib()
    flow = Flow(int(calibrate_imu), int(remove_outliers), float(outlier_threshold), int(block_duplication),
                int(gravity_initialized), int(max_solves))
    hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in calibrators])
    out = (FlowSummary * max(n, 1))()
    rmse = [np.zeros(max(g.n_cams, 1)) if g is not None else np.zeros(1) for g in calibrators]
    rp = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in rmse])
    _batch_check(L, L.vcgpu_calibrate_batch(hs, C.c_int(n), C.byref(flow), out, rp), calibrators)
    res = []
    for i, g in enumerate(calibrators):
        s = out[i]
        d = {f[0]: getattr(s, f[0]) for f in FlowSummary._fields_ if f[0] not in ("last", "flags")}
        d["last"] = {f[0]: getattr(s.last, f[0]) for f in Summary._fields_}
        d["flags"] = {f[0]: getattr(s.flags, f[0]) for f in Flags._fields_}
        C.memmove(C.byref(g.flags), C.byref(s.flags), C.sizeof(Flags))
        res.append((d, rmse[i][: g.n_cams].copy()))
    return res


def _solve_many(entry, calibrators):
    n = len(calibrators)
    L = lib()
    hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in calibrators])
    out = (Summary * max(n, 1))()
    rc = entry(hs, C.c_int(n), out)
    if rc != 0:
        msg = next((L.vcgpu_last_error(g.h).decode() for g in calibrators if g is not None and g.h.value), "")
        raise VcgpuError(f"vcgpu error {rc}: {msg}")
    return [{f[0]: getattr(out[i], f[0]) for f in Summary._fields_} for i in range(n)]


def covariance_batch(calibrators, out=None):
    """vcgpu_get_covariance_batch: the covariance of the globals of every Calibrator of the list (vision and inertial
    rigs may be mixed), each rig in its own thread-block cluster.  Returns one G x G array per calibrator, in order;
    out: optional list of C-contiguous float64 (G, G) arrays to write into.  Raises VcgpuError; where some rigs' systems
    are not positive definite, the error's `status` gives every rig's code and `covariances` the other rigs' matrices."""
    if out is None:
        out = [None if g is None else np.zeros((g.G, g.G)) for g in calibrators]
    return _covariances(lib().vcgpu_get_covariance_batch, "covariance_batch", calibrators, out)


def frame_covariance_batch(calibrators, out=None):
    """vcgpu_get_frame_covariance_batch: Calibrator.frame_covariance() of every Calibrator of the list (vision and
    inertial rigs may be mixed), each rig in its own thread-block cluster.  Returns one (n_frames, fd, fd) array per
    calibrator, in order; out: optional list of C-contiguous float64 arrays of that shape to write into.  Raises
    VcgpuError as covariance_batch does."""
    if out is None:
        out = [None if g is None else np.zeros((g.n_frames, g.fd, g.fd)) for g in calibrators]
    return _covariances(lib().vcgpu_get_frame_covariance_batch, "frame_covariance_batch", calibrators, out)


def frame_cross_covariance_batch(calibrators):
    """vcgpu_get_frame_cross_covariance_batch: Calibrator.frame_cross_covariance() of every Calibrator of the list
    (vision and inertial rigs may be mixed), each rig in its own thread-block cluster.  Returns one (fg, fn) per
    calibrator, in order.  Raises VcgpuError as covariance_batch does; its `covariances` then holds (fg, fn) or None."""
    n = len(calibrators)
    L = lib()
    fg = [None if g is None else np.zeros((g.n_frames, g.fd, g.G)) for g in calibrators]
    fn = [None if g is None else np.zeros((max(g.n_frames - 1, 0), g.fd, g.fd)) for g in calibrators]
    hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in calibrators])
    pg = (C.c_void_p * max(n, 1))(*[None if a is None else a.ctypes.data for a in fg])
    pn = (C.c_void_p * max(n, 1))(*[None if a is None else a.ctypes.data for a in fn])
    status = (C.c_int * max(n, 1))()
    rc = L.vcgpu_get_frame_cross_covariance_batch(hs, C.c_int(n), pg, pn, status)
    out = list(zip(fg, fn))
    if rc != 0:
        msg = next((L.vcgpu_last_error(g.h).decode() for g in calibrators if g is not None and g.h.value), "")
        e = VcgpuError(f"vcgpu error {rc}: {msg}")
        if rc == -3:
            e.status = [status[i] for i in range(n)]
            e.covariances = [out[i] if status[i] == 0 else None for i in range(n)]
        raise e
    return out


def imu_mahalanobis_batch(calibrators, residuals=False):
    """vcgpu_get_imu_mahalanobis_batch: Calibrator.imu_mahalanobis() of every Calibrator of the list in one launch; each
    rig's values are the bits its own call returns.  Returns one distance array per calibrator, in order, or with
    residuals=True one (distances, residuals) pair."""
    n = len(calibrators)
    L = lib()
    ni = [0 if g is None else max(g.n_frames - 1, 0) for g in calibrators]
    d = [np.zeros(max(k, 1)) for k in ni]
    r = [np.zeros((max(k, 1), 9)) for k in ni] if residuals else None
    hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in calibrators])
    dp = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in d])
    rp = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in r]) if residuals else None
    _batch_check(L, L.vcgpu_get_imu_mahalanobis_batch(hs, C.c_int(n), dp, rp), calibrators)
    if residuals:
        return [(d[i][: ni[i]], r[i][: ni[i]]) for i in range(n)]
    return [d[i][: ni[i]] for i in range(n)]


def projection_covariance_batch(calibrators, points):
    """vcgpu_get_projection_covariance_batch: Calibrator.projection_covariance() of every Calibrator of the list, the
    matrices by covariance_batch's cluster kernels and one point launch for all.  points: one dict per calibrator with
    cam_id, pix and optionally depth, frame ("camera") and rays (False).  Returns one result per calibrator, in order,
    as projection_covariance() returns it.  Raises VcgpuError as covariance_batch does; its `covariances` then holds
    the results of the rigs that were written and None for the others."""
    n = len(calibrators)
    L = lib()
    keeps, arr = [], (ProjPoints * max(n, 1))()
    for i, p in enumerate(points):
        keep, arr[i] = _proj_points(p["cam_id"], p["pix"], p.get("depth"), p.get("frame", "camera"), p.get("rays", False))
        keeps.append(keep)
    hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in calibrators])
    st = (C.c_int * max(n, 1))()
    rc = L.vcgpu_get_projection_covariance_batch(hs, C.c_int(n), arr, st)
    out = [_proj_result(keeps[i], arr[i].n) for i in range(n)]
    if rc != 0:
        msg = next((L.vcgpu_last_error(g.h).decode() for g in calibrators if g is not None and g.h.value), "")
        e = VcgpuError(f"vcgpu error {rc}: {msg}")
        if rc == -3:
            e.status = [st[i] for i in range(n)]
            e.covariances = [out[i] if st[i] == 0 else None for i in range(n)]
        raise e
    return out


def view_information_batch(calibrators, views):
    """vcgpu_get_view_information_batch: Calibrator.view_information() of every Calibrator of the list, the priors by
    covariance_batch's cluster kernels and one candidate launch for all.  views: one dict per calibrator with T_wp,
    p_w, width, height and optionally facing, var and post.  Returns one dict per calibrator, in order, as
    view_information() returns it.  Raises VcgpuError as covariance_batch does; its `results` then holds the results
    of the rigs that were written and None for the others."""
    n = len(calibrators)
    if len(views) != n:
        raise ValueError(f"{len(views)} views for {n} calibrators")
    L = lib()
    keeps, arr = [], (ViewCandidates * max(n, 1))()
    for i, v in enumerate(views):
        g = calibrators[i]
        keep, arr[i] = _view_candidates(v["T_wp"], v["p_w"], v["width"], v["height"], v.get("facing"), v.get("var", False),
                                        v.get("post", False), g.n_cams if g is not None else 1, g.G if g is not None else 1)
        keeps.append(keep)
    hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in calibrators])
    st = (C.c_int * max(n, 1))()
    rc = L.vcgpu_get_view_information_batch(hs, C.c_int(n), arr, st)
    out = [_view_result(keeps[i], arr[i].n_cand) for i in range(n)]
    if rc != 0:
        msg = next((L.vcgpu_last_error(g.h).decode() for g in calibrators if g is not None and g.h.value), "")
        e = VcgpuError(f"vcgpu error {rc}: {msg}")
        if rc == -3:
            e.status = [st[i] for i in range(n)]
            e.results = [out[i] if st[i] == 0 else None for i in range(n)]
        raise e
    return out


def observation_influence_batch(calibrators, h=True, stud=True, infl=True):
    """vcgpu_get_observation_influence_batch: Calibrator.observation_influence() of every Calibrator of the list (vision
    and inertial rigs may be mixed), the covariance blocks from one elimination per rig by the cluster kernels and one launch of
    each influence kernel for all.  Returns one dict per calibrator, in order.  Raises VcgpuError as covariance_batch
    does; its `results` then holds the results of the rigs that were written and None for the others."""
    n = len(calibrators)
    L = lib()
    keeps, arr = [], (ObsInfluence * max(n, 1))()
    for i, g in enumerate(calibrators):
        keep, arr[i] = _obs_influence(g.n_obs if g is not None else 0, h, stud, infl)
        keeps.append(keep)
    hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in calibrators])
    st = (C.c_int * max(n, 1))()
    rc = L.vcgpu_get_observation_influence_batch(hs, C.c_int(n), arr, st)
    out = [_obs_influence_result(keeps[i], calibrators[i].n_obs if calibrators[i] is not None else 0) for i in range(n)]
    if rc != 0:
        msg = next((L.vcgpu_last_error(g.h).decode() for g in calibrators if g is not None and g.h.value), "")
        e = VcgpuError(f"vcgpu error {rc}: {msg}")
        if rc == -3:
            e.status = [st[i] for i in range(n)]
            e.results = [out[i] if st[i] == 0 else None for i in range(n)]
        raise e
    return out


def imu_influence_batch(calibrators, h=True, stud=True, infl=True, observations=False):
    """vcgpu_get_imu_influence_batch: Calibrator.imu_influence() of every Calibrator of the list (inertial rigs), the
    covariance blocks from one elimination per rig by the cluster kernels and one launch of each influence kernel for
    all.  Returns one dict per calibrator, in order.  Raises VcgpuError as covariance_batch does; its `results` then
    holds the results of the rigs that were written and None for the others."""
    n = len(calibrators)
    L = lib()
    ni = [max(g.n_frames - 1, 0) if g is not None else 0 for g in calibrators]
    no = [g.n_obs if g is not None else 0 for g in calibrators]
    keeps, okeeps = [], []
    arr, oarr = (ImuInfluence * max(n, 1))(), (ObsInfluence * max(n, 1))()
    for i in range(n):
        keep, arr[i] = _imu_influence(ni[i], h, stud, infl)
        keeps.append(keep)
        okeep = None
        if observations:
            okeep, oarr[i] = _obs_influence(no[i], True, True, True)
        okeeps.append(okeep)
    hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in calibrators])
    st = (C.c_int * max(n, 1))()
    rc = L.vcgpu_get_imu_influence_batch(hs, C.c_int(n), arr, oarr if observations else None, st)
    out = [_imu_influence_result(keeps[i], ni[i], okeeps[i], no[i]) for i in range(n)]
    if rc != 0:
        msg = next((L.vcgpu_last_error(g.h).decode() for g in calibrators if g is not None and g.h.value), "")
        e = VcgpuError(f"vcgpu error {rc}: {msg}")
        if rc == -3:
            e.status = [st[i] for i in range(n)]
            e.results = [out[i] if st[i] == 0 else None for i in range(n)]
        raise e
    return out


def align_imu_batch(calibrators, ts_lo=-0.1, ts_hi=0.1, n_ts=401, find_time_offset=True, max_iters=20, apply=False,
                    curve=False):
    """vcgpu_align_imu_batch: Calibrator.align_imu() of every Calibrator of the list in one call, each rig's result the
    bits its own call returns.  Any option may be one value or a list with one value per calibrator.  Returns one dict
    per calibrator, in order, as align_imu() returns it (status -3 marks a rig whose fit failed)."""
    n = len(calibrators)
    L = lib()
    per = [v if isinstance(v, (list, tuple)) else [v] * n for v in (ts_lo, ts_hi, n_ts, find_time_offset, max_iters, apply, curve)]
    args = [_align_args(*(v[i] for v in per)) for i in range(n)]
    hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in calibrators])
    opts = (ImuAlignOpts * max(n, 1))(*[a[0] for a in args])
    outs = (ImuAlignment * max(n, 1))(*[a[1] for a in args])
    status = (C.c_int * max(n, 1))()
    rc = L.vcgpu_align_imu_batch(hs, C.c_int(n), opts, outs, status)
    if rc not in (0, -3):
        _batch_check(L, rc, calibrators)
    return [_align_result(outs[i], args[i][2], status[i]) for i in range(n)]


def _split_poses(start, poses):
    return [poses[start[k]: start[k + 1]] for k in range(len(start) - 1)]


def integration_poses_batch(calibrators):
    """vcgpu_get_integration_poses_batch: Calibrator.integration_poses() of every Calibrator of the list, one count pass
    and one fill pass for all; each rig's poses are the bits its own call returns.  Returns one list of (count_k, 14)
    arrays per calibrator, in order."""
    n = len(calibrators)
    L = lib()
    start = [np.zeros(max(0 if g is None else g.n_frames, 1), dtype=np.int64) for g in calibrators]
    hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in calibrators])
    sp = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in start])
    _batch_check(L, L.vcgpu_get_integration_poses_batch(hs, C.c_int(n), sp, None), calibrators)
    poses = [np.zeros((max(int(a[-1]), 1), 14)) for a in start]
    pp = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in poses])
    _batch_check(L, L.vcgpu_get_integration_poses_batch(hs, C.c_int(n), sp, pp), calibrators)
    return [_split_poses(a, b) for a, b in zip(start, poses)]


def _covariances(entry, name, calibrators, out):
    n = len(calibrators)
    L = lib()
    for a in out:
        if a is not None and (a.dtype != np.float64 or not a.flags.c_contiguous):
            raise ValueError(f"{name}: out arrays must be C-contiguous float64")
    hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in calibrators])
    ptrs = (C.c_void_p * max(n, 1))(*[None if a is None else a.ctypes.data for a in out])
    status = (C.c_int * max(n, 1))()
    rc = entry(hs, C.c_int(n), ptrs, status)
    if rc != 0:
        msg = next((L.vcgpu_last_error(g.h).decode() for g in calibrators if g is not None and g.h.value), "")
        e = VcgpuError(f"vcgpu error {rc}: {msg}")
        if rc == -3:  # VCGPU_ERR_NUMERIC: the other rigs' matrices are written
            e.status = [status[i] for i in range(n)]
            e.covariances = [out[i] if status[i] == 0 else None for i in range(n)]
        raise e
    return list(out)


def evaluate_batch(calibrators, residuals=False):
    """vcgpu_evaluate_batch: Calibrator.evaluate(c) of every camera of every Calibrator of the list, in one launch.
    Returns one (cost[n_cams], blocks[n_cams]) per calibrator, in order; residuals=True adds a third entry, the
    residuals of Calibrator.evaluate(-1, residuals=True)."""
    n = len(calibrators)
    L = lib()
    cost = [np.zeros(max(g.n_cams, 1)) for g in calibrators]
    blocks = [np.zeros(max(g.n_cams, 1), dtype=np.int64) for g in calibrators]
    res = [np.zeros(max(2 * g.n_obs, 1)) for g in calibrators] if residuals else None
    hs = (C.c_void_p * max(n, 1))(*[g.h for g in calibrators])
    cp = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in cost])
    bp = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in blocks])
    rp = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in res]) if residuals else None
    _batch_check(L, L.vcgpu_evaluate_batch(hs, C.c_int(n), cp, bp, rp), calibrators)
    out = []
    for g, c, b, k in zip(calibrators, cost, blocks, range(n)):
        c, b = c[: g.n_cams], b[: g.n_cams]
        out.append((c, b, res[k][: 2 * int(b.sum())]) if residuals else (c, b))
    return out


def remove_outliers_batch(calibrators, rmses, threshold):
    """vcgpu_remove_outliers_batch: Calibrator.remove_outliers(rmses[i], threshold) of every Calibrator of the list,
    in one launch.  Returns the removed counts, in order."""
    n = len(calibrators)
    L = lib()
    rmse = [_c(r) for r in rmses]
    hs = (C.c_void_p * max(n, 1))(*[g.h for g in calibrators])
    rp = (C.c_void_p * max(n, 1))(*[r.ctypes.data for r in rmse])
    removed = np.zeros(max(n, 1), dtype=np.int64)
    _batch_check(L, L.vcgpu_remove_outliers_batch(hs, C.c_int(n), rp, C.c_double(threshold), _p(removed)), calibrators)
    return [int(x) for x in removed[:n]]


def pose_pnp_batch(entries, robust_its=0, robust_tol=0.0):
    """vcgpu_pose_pnp_ransac_batch: Calibrator.pose_pnp_ransac of every rig in one launch.  entries: one
    (Calibrator, (cam_id, start, count, pix, pw)) per rig, the view arguments of Calibrator.pose_pnp_ransac.  Returns one
    (T_cw [n, 7], rmse [n], n_used [n]) per rig, in order; each is the bits the rig's own call returns."""
    n = len(entries)
    L = lib()
    keep, outs = [], []
    views = (PnpViews * max(n, 1))()
    for k, (g, (cam_id, start, count, pix, pw)) in enumerate(entries):
        ins = [_c(cam_id, np.int32), _c(start, np.int64), _c(count, np.int32), _c(pix), _c(pw)]
        m = len(ins[0])
        out = (np.zeros((m, 7)), np.zeros(m), np.zeros(m, dtype=np.int32))
        keep.append(ins)
        outs.append(out)
        views[k] = PnpViews(m, *[a.ctypes.data for a in ins], *[a.ctypes.data for a in out])
    hs = (C.c_void_p * max(n, 1))(*[g.h for g, _ in entries])
    _batch_check(L, L.vcgpu_pose_pnp_ransac_batch(hs, C.c_int(n), views, C.c_int(robust_its), C.c_double(robust_tol)),
                 [g for g, _ in entries])
    return outs


def _batch_check(L, rc, calibrators):
    if rc != 0:
        msg = next((L.vcgpu_last_error(g.h).decode() for g in calibrators if g is not None and g.h.value), "")
        raise VcgpuError(f"vcgpu error {rc}: {msg}")
