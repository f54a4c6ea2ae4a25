"""Reference values of each IMU interval's Mahalanobis distance, the one UpdateImuWeights logs against chi2inv(0.95, 9)
(vicalibrator.h:786-794):
  oracle_dist     the oracle's UpdateOneImuWeight (oracle/imu_weights.h) with its `mahalanobis` output, every interval
  oracle_interval the oracle's P = Jt C Jt^T and residual r of one interval, as the loop body forms them
  ref_dist        oracle/_ref's ref_update_weight: the reference's own headers, its `dist` (None where not built)
  eig_dist        the device formula in numpy: sum_k (V[:,k] . r)^2 / lambda_k from eigh(sym P), NaN where lambda <= 0
NaN marks an interval with no measurements, where the reference `continue`s and logs nothing (:731-733).

The oracle entry points live in tests/cpp/imu_mahalanobis_oracle.cc, compiled here into a temporary directory with the
oracle's compiler flags (oracle/Makefile), so the tree stays as it was."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from vicalib_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libvicalib_ref.so")
CHI2_95_9 = 16.9190  # chi2inv(0.95, 9), the bound the reference logs against
_LIB = None
_DIR = None


def lib():
    global _LIB, _DIR
    if _LIB is None:
        _DIR = tempfile.TemporaryDirectory(prefix="vo_mahalanobis_")
        so = os.path.join(_DIR.name, "libvo_mahalanobis.so")
        subprocess.run([os.environ.get("CXX", "g++"), "-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-shared",
                        "-I", os.path.join(ROOT, "oracle"), "-o", so,
                        os.path.join(ROOT, "tests", "cpp", "imu_mahalanobis_oracle.cc")], check=True, timeout=300)
        L = C.CDLL(so)
        L.vo_imu_interval.restype = C.c_int
        _LIB = L
    return _LIB


def ref_lib():
    if not os.path.exists(REF_SO):
        return None
    L = C.CDLL(REF_SO)
    L.ref_update_weight.restype = C.c_int
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _c(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _imu(p):
    # a one-element placeholder keeps the pointers valid for an empty stream (n = 0 is passed)
    n = len(p.imu_t)
    keep = (_c(p.imu_t) if n else np.zeros(1), _c(p.imu_w) if n else np.zeros((1, 3)), _c(p.imu_a) if n else np.zeros((1, 3)))
    return (C.c_int(n), *[_p(x) for x in keep]), keep


def _state(p, state):
    s = state or {}
    return {k: _c(s.get(k, getattr(p, k))) for k in ("T_wp", "v_w", "g", "b", "sf")}, float(s.get("ts", p.ts))


def oracle_dist(p, state=None, sigma_g=synth.GYRO_SIGMA, sigma_a=synth.ACCEL_SIGMA):
    """[n_frames - 1] distances at p's state (or at `state`, a Calibrator.state()-like dict)"""
    args, _keep = _imu(p)
    s, ts = _state(p, state)
    d = np.zeros(p.n_frames - 1)
    lib().vo_imu_mahalanobis(*args, C.c_int(p.n_frames), _p(_c(p.ftime)), _p(s["T_wp"]), _p(s["v_w"]), _p(s["g"]),
                             _p(s["b"]), _p(s["sf"]), C.c_double(ts), C.c_double(sigma_g), C.c_double(sigma_a), _p(d))
    return d


def oracle_interval(p, k, state=None, sigma_g=synth.GYRO_SIGMA, sigma_a=synth.ACCEL_SIGMA):
    """(P 9 x 9, r 9, number of measurements) of interval k; (None, None, 0) without measurements"""
    args, _keep = _imu(p)
    s, ts = _state(p, state)
    P, r = np.zeros((9, 9)), np.zeros(9)
    m = lib().vo_imu_interval(*args, C.c_double(p.ftime[k]), C.c_double(p.ftime[k + 1]), _p(_c(s["T_wp"][k])),
                              _p(_c(s["v_w"][k])), _p(_c(s["T_wp"][k + 1])), _p(_c(s["v_w"][k + 1])), _p(s["g"]),
                              _p(s["b"]), _p(s["sf"]), C.c_double(ts), C.c_double(sigma_g), C.c_double(sigma_a), _p(P),
                              _p(r))
    return (P, r, m) if m else (None, None, 0)


def ref_dist(ref, p, state=None, sigma_g=synth.GYRO_SIGMA, sigma_a=synth.ACCEL_SIGMA):
    """[n_frames - 1] distances from ref_update_weight (the reference's `dist`), NaN where it returns 0"""
    args, _keep = _imu(p)
    s, ts = _state(p, state)
    d = np.full(p.n_frames - 1, np.nan)
    for k in range(p.n_frames - 1):
        W, m = np.zeros((9, 9)), C.c_double()
        rc = ref.ref_update_weight(*args, C.c_double(p.ftime[k]), C.c_double(p.ftime[k + 1]), _p(_c(s["T_wp"][k])),
                                   _p(_c(s["v_w"][k])), _p(_c(s["T_wp"][k + 1])), _p(_c(s["v_w"][k + 1])), _p(s["g"]),
                                   _p(s["b"]), _p(s["sf"]), C.c_double(ts), C.c_double(sigma_g), C.c_double(sigma_a),
                                   _p(W), C.byref(m))
        if rc:
            d[k] = m.value
    return d


def eig_dist(P, r):
    lam, V = np.linalg.eigh(0.5 * (P + P.T))
    if not np.all(lam > 0):
        return np.nan
    z = V.T @ r
    return float(np.sum(z * z / lam))
