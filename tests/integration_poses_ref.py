"""Reference values of ViCalibrator::GetIntegrationPoses(k) (vicalibrator.h:508-533) for every interval k of a problem:
the poses the double RK4 of IntegrateResidual (types.h:611-687) passes through from frame k over GetRange(t_k, t_k+1, ts),
14 doubles each, q (x y z w) | t (3) | v_w (3) | w_w (3) | time.
  ref_poses     ref_integration_poses of oracle/_ref/libvicalib_ref_poses.so (oracle/ref_poses.cc): the reference's
                own headers (None where not built)
  oracle_poses  the oracle's GetRange and IntegrateImuD
  mirror_poses  the host mirror's GetIntegrationPoses (vicalib_b200/host/vicalibrator.h)
Each returns a list of (count_k, 14) arrays, count_k the number of measurements GetRange yields.

The oracle and mirror entry points live in tests/cpp/integration_poses_oracle.cc, compiled here into a temporary
directory with the oracle's compiler flags (oracle/Makefile), so the tree stays as it was."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libvicalib_ref_poses.so")
POSE = 14
_LIB = None
_DIR = None


def lib():
    global _LIB, _DIR
    if _LIB is None:
        _DIR = tempfile.TemporaryDirectory(prefix="vo_integration_poses_")
        so = os.path.join(_DIR.name, "libvo_integration_poses.so")
        subprocess.run([os.environ.get("CXX", "g++"), "-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-shared",
                        "-I", os.path.join(ROOT, "oracle"), "-o", so,
                        os.path.join(ROOT, "tests", "cpp", "integration_poses_oracle.cc"), "-lpthread"],
                       check=True, timeout=300)
        _LIB = C.CDLL(so)
    return _LIB


def ref_lib():
    if not os.path.exists(REF_SO):
        return None
    return C.CDLL(REF_SO)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _c(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _state(p, state):
    s = state or {}
    return {k: _c(s.get(k, getattr(p, k))) for k in ("T_wp", "v_w", "g", "b", "sf")}, float(s.get("ts", p.ts))


def _poses(fn, p, state):
    n = len(p.imu_t)
    # a one-element placeholder keeps the pointers valid for an empty stream (n = 0 is passed)
    t, w, a = (_c(p.imu_t) if n else np.zeros(1), _c(p.imu_w) if n else np.zeros((1, 3)),
               _c(p.imu_a) if n else np.zeros((1, 3)))
    s, ts = _state(p, state)
    ft = _c(p.ftime)
    cap = n + 2  # GetRange yields at most every sample and the two ends
    out = []
    for k in range(len(ft) - 1):
        buf = np.zeros((cap, POSE))
        m = fn(C.c_int(n), _p(t), _p(w), _p(a), C.c_double(ft[k]), C.c_double(ft[k + 1]), _p(_c(s["T_wp"][k])),
               _p(_c(s["v_w"][k])), _p(s["g"]), _p(s["b"]), _p(s["sf"]), C.c_double(ts), _p(buf), C.c_int(cap))
        assert 0 <= m <= cap
        out.append(buf[:m].copy())
    return out


def ref_poses(ref, p, state=None):
    """[n_frames - 1] arrays from ref_integration_poses at p's state (or at `state`, a Calibrator.state()-like dict)"""
    return _poses(ref.ref_integration_poses, p, state)


def oracle_poses(p, state=None):
    return _poses(lib().vo_integration_poses, p, state)


def mirror_poses(p, state=None):
    return _poses(lib().mirror_integration_poses, p, state)


def worst(a, b):
    """largest difference of two intervals' poses per column group, relative to the group's scale in `b` over the interval
    (1 for the quaternion; the largest |value|, at least 1e-3, for t, v_w and w_w): (q, t, v, w)"""
    if len(b) == 0:
        return np.zeros(4)
    out = []
    for lo, hi, floor in ((0, 4, 1.0), (4, 7, 1e-3), (7, 10, 1e-3), (10, 13, 1e-3)):
        scale = 1.0 if lo == 0 else max(floor, np.abs(b[:, lo:hi]).max())
        out.append(np.abs(a[:, lo:hi] - b[:, lo:hi]).max() / scale)
    return np.array(out)


def mirror_all_timed(p, state=None):
    """the mirror's GetIntegrationPoses(k) for every k on one object: (total poses, seconds of the loop)"""
    n = len(p.imu_t)
    t, w, a = _c(p.imu_t), _c(p.imu_w), _c(p.imu_a)
    s, ts = _state(p, state)
    sec = C.c_double()
    L = lib()
    L.mirror_all_integration_poses.restype = C.c_int64
    total = L.mirror_all_integration_poses(C.c_int(n), _p(t), _p(w), _p(a), C.c_int(p.n_frames), _p(_c(p.ftime)),
                                           _p(s["T_wp"]), _p(s["v_w"]), _p(s["g"]), _p(s["b"]), _p(s["sf"]),
                                           C.c_double(ts), C.byref(sec))
    return int(total), sec.value
