"""CPU: the oracle on the IMU streams of imu_streams.py (jittered, gapped, slow, partial, frame-tied, dropped frames,
0-2 samples), against the classification the builders assert and against oracle/_ref, the reference's own headers
(see test_cpu_oracle_ref.py): GetRange on every interval, the functor's residual and 9 x 33 Jacobian, UpdateImuWeights
on every interval with at least two RK4 steps.

On a single-step interval (no interior sample) the 9 x 9 covariance has rank <= 6, so the weight is decided by
rounding, in the reference too: W is finite but not positive definite to working precision, and is not compared."""
import ctypes as C
import os

import numpy as np
import pytest

import imu_streams
from vicalib_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "oracle", "_ref", "libvicalib_ref.so")
needs_ref = pytest.mark.skipif(not os.path.exists(SO), reason="oracle/_ref is built only where the reference tree exists")
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
MAX_RANGE = 2048


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _c(a):
    return np.ascontiguousarray(a, dtype=np.float64)


@pytest.fixture(scope="module")
def ref():
    L = C.CDLL(SO)
    for f in ("ref_get_range", "ref_imu_eval", "ref_update_weight"):
        getattr(L, f).restype = C.c_int
    return L


@pytest.fixture(scope="module", params=imu_streams.NAMES)
def stream(request):
    s = imu_streams.build(request.param)
    s.p = imu_streams.perturbed(s.p)
    return s


def _imu(p):
    # a one-element placeholder keeps the pointers valid for an empty stream (n = 0 is passed)
    t = _c(p.imu_t) if len(p.imu_t) else np.zeros(1)
    w = _c(p.imu_w) if len(p.imu_t) else np.zeros((1, 3))
    a = _c(p.imu_a) if len(p.imu_t) else np.zeros((1, 3))
    return (C.c_int(len(p.imu_t)), _p(t), _p(w), _p(a)), (t, w, a)


def test_classification_matches_get_range(stream):
    """The builders' classification against the oracle's GetRange: no rows where HasElement is false; otherwise rows
    from ftime[k] to min(ftime[k+1], t_last + ts) with `steps` nonzero-length steps."""
    from oracle.binding import Oracle

    p, c = stream.p, stream.cls
    o = Oracle(p, **ALL_ON)
    tt_last = p.imu_t[-1] + p.ts if len(p.imu_t) else None
    for k in range(p.n_frames - 1):
        rows = o.imu_get_range(p.ftime[k], p.ftime[k + 1], p.ts, max_n=MAX_RANGE)
        assert len(rows) < MAX_RANGE
        if not c["covered"][k]:
            assert len(rows) == 0, k
            continue
        t = rows[:, 0]
        assert t[0] == p.ftime[k] and t[-1] == min(p.ftime[k + 1], tt_last), k
        assert np.all(np.diff(t) >= 0) and np.count_nonzero(np.diff(t)) == c["steps"][k], (k, t)


@needs_ref
def test_get_range_matches_ref(ref, stream):
    from oracle.binding import Oracle

    p = stream.p
    o = Oracle(p, **ALL_ON)
    args, _keep = _imu(p)
    for k in range(p.n_frames - 1):
        out = np.zeros((MAX_RANGE, 7))
        n = ref.ref_get_range(*args, C.c_double(p.ftime[k]), C.c_double(p.ftime[k + 1]), C.c_double(p.ts), _p(out), MAX_RANGE)
        mine = o.imu_get_range(p.ftime[k], p.ftime[k + 1], p.ts, max_n=MAX_RANGE)
        assert n == len(mine), k
        assert np.allclose(out[:n], mine, rtol=1e-14, atol=1e-15), k


@needs_ref
def test_functor_matches_ref(ref, stream):
    """Residual and 9 x 33 Jacobian of every interval at 1e-11 relative; exact zeros without measurements."""
    from oracle.binding import Oracle

    p, c = stream.p, stream.cls
    o = Oracle(p, **ALL_ON)
    rng = np.random.default_rng(7)
    W = rng.standard_normal((p.n_frames - 1, 9, 9)) + 30 * np.eye(9)
    W = 0.5 * (W + W.transpose(0, 2, 1))
    o.set_imu_weights(W)
    r_o, J_o = o.eval_imu()
    args, _keep = _imu(p)
    for k in range(p.n_frames - 1):
        r, J = np.zeros(9), np.zeros((9, 33))
        rc = ref.ref_imu_eval(*args, C.c_double(p.ftime[k]), C.c_double(p.ftime[k + 1]), _p(_c(W[k])), C.c_int(0),
                              _p(_c(p.T_wp[k + 1])), _p(_c(p.T_wp[k])), _p(_c(p.v_w[k + 1])), _p(_c(p.v_w[k])), _p(_c(p.g)),
                              _p(_c(p.b)), _p(_c(p.sf)), C.c_double(p.ts), _p(r), _p(J))
        assert rc == 0
        if not c["covered"][k]:
            assert not r_o[k].any() and not J_o[k].any() and not r.any() and not J.any(), k
            continue
        assert np.abs(r - r_o[k]).max() <= 1e-11 * max(1.0, np.abs(r_o[k]).max()), k
        assert np.abs(J - J_o[k]).max() <= 1e-11 * np.abs(J_o[k]).max(), k


def _ref_weight(ref, p, k):
    args, _keep = _imu(p)
    W = np.zeros((9, 9))
    m = C.c_double()
    rc = ref.ref_update_weight(*args, C.c_double(p.ftime[k]), C.c_double(p.ftime[k + 1]), _p(_c(p.T_wp[k])),
                               _p(_c(p.v_w[k])), _p(_c(p.T_wp[k + 1])), _p(_c(p.v_w[k + 1])), _p(_c(p.g)), _p(_c(p.b)),
                               _p(_c(p.sf)), C.c_double(p.ts), C.c_double(synth.GYRO_SIGMA),
                               C.c_double(synth.ACCEL_SIGMA), _p(W), C.byref(m))
    return rc, W


@needs_ref
def test_update_imu_weights_matches_ref(ref, stream):
    """Intervals with >= 2 steps: the reference's weight_sqrt_ at 1e-8 relative.  Intervals without measurements:
    the weights stay as they were, bit for bit, and the reference skips them.  Single-step intervals: finite in both,
    and the oracle's W is not positive definite to working precision (cond > 1e15): decided by rounding."""
    from oracle.binding import Oracle

    p, c = stream.p, stream.cls
    o = Oracle(p, **ALL_ON)
    W0 = np.broadcast_to(np.diag(np.arange(400.0, 409.0)), (p.n_frames - 1, 9, 9)).copy()
    o.set_imu_weights(W0)
    o.update_imu_weights()
    W_o = o.imu_weights()
    for k in range(p.n_frames - 1):
        if c["covered"][k] and c["steps"][k] == 0:
            continue  # a zero-step interval (one sample, on a frame time): the covariance is exactly 0
        rc, W = _ref_weight(ref, p, k)
        if not c["covered"][k]:
            assert rc == 0 and np.array_equal(W_o[k], W0[k]), k
        elif c["single"][k]:
            assert rc == 1 and np.isfinite(W).all() and np.isfinite(W_o[k]).all(), k
            ev = np.abs(np.linalg.eigvalsh(0.5 * (W_o[k] + W_o[k].T)))
            assert ev.max() / ev.min() > 1e15, (k, ev.max() / ev.min())
        else:
            assert rc == 1
            assert np.abs(W - W_o[k]).max() <= 1e-8 * np.abs(W_o[k]).max(), (k, np.abs(W - W_o[k]).max() / np.abs(W_o[k]).max())
