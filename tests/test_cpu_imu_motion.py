"""CPU: the inertial path under vigorous motion and across the quaternion double cover (imu_motion.py,
tests/golden/imu_vigorous_kat.npz).

- The builders' regimes, and synth.make_problem's default trajectory unchanged bit for bit (the benchmark and every
  other test build on it).
- The oracle against imu_vigorous_kat.npz (60-digit mpmath, rotation matrices, exact central differences) at the bars of
  test_cpu_oracle_golden.py: |w| dt up to 0.03 per RK4 step, where an error of 4th order in the per-step angle is ~1e-6
  instead of the ~1e-9 it is on the gentle trajectory; end-residual quaternions with w ~ -1, w ~ -0.1 and angles of
  2.6-2.95 rad.
- The oracle against oracle/_ref (the reference's own headers; skipped where it is absent, as test_cpu_oracle_ref.py
  is) on every builder and on flipped variants: the functor's residual and 9 x 33 Jacobian, and UpdateImuWeights' W,
  whose derivative tables (dLog_dq, dLog_dSE3) see w < 0 here.  This pins the weights at high rates, where no exact
  KAT exists: the reference's truncated d exp(w)/dw series departs from the exact derivative there on purpose.
- The oracle's invariance under q -> -q: residuals, Jacobians, normal equations and weights of flipped(p) against p.
"""
import ctypes as C
import dataclasses
import hashlib
import os

import numpy as np
import pytest

import imu_motion
import imu_streams
from vicalib_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
SO = os.path.join(ROOT, "oracle", "_ref", "libvicalib_ref.so")
needs_ref = pytest.mark.skipif(not os.path.exists(SO), reason="oracle/_ref is built only where the reference tree exists")
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)


# ------------------------------------------------------------------ builders, and the default trajectory unchanged
@pytest.mark.parametrize("name", imu_motion.NAMES)
def test_builder_regime(name):
    m = imu_motion.build(name)  # asserts its own regime
    r = m.regime
    print(f"\n{name}: max |w| {r['w']:.2f} rad/s, max |w| dt {r['wdt']:.4f}, max ||a| - g| {r['accel']:.1f} m/s^2, "
          f"steps {m.cls['steps'].min()}-{m.cls['steps'].max()}, opposite-sign pairs {r['sign_flips'].tolist()}")
    g = imu_motion.regime(synth.make_problem(models=("poly3",), n_frames=90, inertial=True, seed=15))
    assert r["w"] > 4 * g["w"] and r["accel"] > 50 * g["accel"] and len(g["sign_flips"]) == 0  # the gentle default


def _digest(p):
    h = hashlib.sha256()
    for f in dataclasses.fields(p):
        v = getattr(p, f.name)
        for a in ([v[k] for k in sorted(v)] if isinstance(v, dict) else [v]):
            h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


# sha256 of every array of the Problem (truth included), as the default trajectory made them before motion= existed
DEFAULT_DIGESTS = [
    (dict(), "3c65745ec8c9b44f54ef9e0d0ce9e6976f6cf12806e77e0a96c350e30f15d809"),
    (dict(models=("poly3", "kb4"), n_frames=30, inertial=True, seed=3, ts_truth=0.003),
     "f39ae673db90538e41d06e56fed291ef0874195be38713ee0239e795e76591d7"),
    (dict(models=("fov",), n_frames=20, grid=(10, 7), inertial=True, seed=31, imu_rate=1000.0),
     "5ae72220a2db93fb7839998f29e4c9fe43d6303122335a6c73c287a5e838433d"),
]


def test_default_trajectory_unchanged():
    for kw, want in DEFAULT_DIGESTS:
        assert _digest(synth.make_problem(**kw)) == want, kw
        assert _digest(synth.make_problem(motion="gentle", **kw)) == want, kw
    assert _digest(synth.make_config("config3", n_frames=40)) == \
        "d2351cb67f2de8e7e0ed7ffae0cad0717948f1c8e4f5158ccc100741baa9726e"
    with pytest.raises(ValueError):
        synth.make_problem(motion="wild")


# ------------------------------------------------------------------ the oracle against the vigorous KAT
def kat_problem(z):
    """a Problem carrying the fixture's stream, frames and IMU parameters (one linear camera, no observations)"""
    nf = len(z["ftime"])
    p = synth.make_problem(models=("linear",), n_frames=nf, inertial=True, seed=1)
    p.T_wp, p.v_w, p.ftime = z["T_wp"].copy(), z["v_w"].copy(), z["ftime"].copy()
    p.imu_t, p.imu_w, p.imu_a = z["imu_t"].copy(), z["imu_w"].copy(), z["imu_a"].copy()
    p.g, p.b, p.sf, p.ts = z["g"].copy(), z["b"].copy(), z["sf"].copy(), float(z["ts"])
    return p


def test_vigorous_kat_regime():
    """the fixture has what it is for: fast rotation and large accelerations, 20-50 steps, frame quaternions of both
    signs, end-residual quaternions with w < 0 (one converged, w ~ -1), rotations of 2.5-3.0 rad, no sample on a frame"""
    z = np.load(os.path.join(GOLD, "imu_vigorous_kat.npz"))
    p = kat_problem(z)
    w = np.linalg.norm(p.imu_w, axis=1)
    assert w.max() >= 7.5 and (w[1:] * np.diff(p.imu_t)).max() >= 0.03
    assert np.linalg.norm(p.imu_a, axis=1).max() >= 22.0
    assert not np.any(p.sf == 1) and np.all(p.b != 0) and p.ts != 0
    c = imu_streams.classify(p)
    assert c["comparable"].all() and c["steps"].min() >= 20 and c["steps"].max() <= 50
    assert not imu_streams.ts_kinks(z).any()
    assert (p.T_wp[:, 3] < 0).any() and (p.T_wp[:, 3] > 0).any()
    raw = np.linalg.solve(z["W"].T, z["r"][0].T).T  # r = W^T raw
    ang = np.linalg.norm(raw[:, 3:6], axis=1)
    assert ang.min() < 1e-9 and ((ang > 2.5) & (ang < 3.0)).sum() >= 2 and ang.max() < 3.0


@pytest.mark.parametrize("switch", [0, 1])
def test_oracle_vs_vigorous_kat(switch):
    from oracle.binding import Oracle

    z = np.load(os.path.join(GOLD, "imu_vigorous_kat.npz"))
    p = kat_problem(z)
    o = Oracle(p, inertial=1, rotation_only=switch, bias_active=1, scale_active=1, optimize_ts=1)
    o.set_imu_weights(np.broadcast_to(z["W"], (p.n_frames - 1, 9, 9)).copy())
    r, J = o.eval_imu()
    err_r = np.abs(r - z["r"][switch]).max() / np.abs(z["r"][switch]).max()
    err_J = np.abs(J - z["J"][switch]).max() / np.abs(z["J"][switch]).max()
    print(f"\noracle vs vigorous KAT, switch {switch}: r {err_r:.1e}, J {err_J:.1e}")
    assert err_r <= 1e-9 and err_J <= 1e-9


# ------------------------------------------------------------------ the oracle against the reference's own headers
def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _c(a):
    return np.ascontiguousarray(a, dtype=np.float64)


@pytest.fixture(scope="module")
def ref():
    L = C.CDLL(SO)
    for f in ("ref_imu_eval", "ref_update_weight"):
        getattr(L, f).restype = C.c_int
    return L


def _variants():
    out = []
    for name in imu_motion.NAMES:
        out.append((name, False))
        out.append((name, True))
    return out


def _variant(name, flip):
    m = imu_motion.build(name)
    if flip:
        m.p = imu_motion.flipped(m.p, imu_motion.scattered(m.p.n_frames), cams=[0])
    return m


@needs_ref
@pytest.mark.parametrize("name,flip", _variants(), ids=[f"{n}-{'flipped' if f else 'canonical'}" for n, f in _variants()])
def test_functor_and_weights_match_ref(ref, name, flip):
    """ref_imu_eval: residual and 9 x 33 Jacobian at test_imu_cost_functor_and_jacobian's 1e-11; ref_update_weight: W at
    test_update_imu_weights' 1e-8 relative, on every interval"""
    from oracle.binding import Oracle

    m = _variant(name, flip)
    p = m.p
    o = Oracle(p, **ALL_ON)
    rng = np.random.default_rng(3)
    W = rng.standard_normal((p.n_frames - 1, 9, 9)) + 30 * np.eye(9)
    W = 0.5 * (W + W.transpose(0, 2, 1))
    o.set_imu_weights(W)
    r_o, J_o = o.eval_imu()
    o.update_imu_weights()
    W_o = o.imu_weights()
    t, w, a = _c(p.imu_t), _c(p.imu_w), _c(p.imu_a)
    imu = (C.c_int(len(t)), _p(t), _p(w), _p(a))
    worst = [0.0, 0.0, 0.0]
    for k in range(p.n_frames - 1):
        r, J = np.zeros(9), np.zeros((9, 33))
        T2, T1, v2, v1 = _c(p.T_wp[k + 1]), _c(p.T_wp[k]), _c(p.v_w[k + 1]), _c(p.v_w[k])
        gg, b, sf = _c(p.g), _c(p.b), _c(p.sf)
        assert ref.ref_imu_eval(*imu, C.c_double(p.ftime[k]), C.c_double(p.ftime[k + 1]), _p(_c(W[k])), C.c_int(0),
                                _p(T2), _p(T1), _p(v2), _p(v1), _p(gg), _p(b), _p(sf), C.c_double(p.ts), _p(r), _p(J)) == 0
        Wr = np.zeros((9, 9))
        mm = C.c_double()
        assert ref.ref_update_weight(*imu, C.c_double(p.ftime[k]), C.c_double(p.ftime[k + 1]), _p(T1), _p(v1), _p(T2),
                                     _p(v2), _p(gg), _p(b), _p(sf), C.c_double(p.ts), C.c_double(synth.GYRO_SIGMA),
                                     C.c_double(synth.ACCEL_SIGMA), _p(Wr), C.byref(mm)) == 1
        e = (np.abs(r - r_o[k]).max() / max(1.0, np.abs(r_o[k]).max()), np.abs(J - J_o[k]).max() / np.abs(J_o[k]).max(),
             np.abs(Wr - W_o[k]).max() / np.abs(W_o[k]).max())
        worst = [max(x, y) for x, y in zip(worst, e)]
        assert e[0] <= 1e-11 and e[1] <= 1e-11, (k, e)
        assert e[2] <= 1e-8, (k, e)
    print(f"\n{name} {'flipped' if flip else 'canonical'}: oracle vs reference r {worst[0]:.1e} J {worst[1]:.1e} "
          f"W {worst[2]:.1e}")


# ------------------------------------------------------------------ the oracle's sign invariance
def _oracle_all(p, inertial):
    from oracle.binding import Oracle

    flags = ALL_ON if inertial else {}
    o = Oracle(p, **flags)
    out = {}
    out["r_reproj"], out["J_reproj"] = o.eval_reproj()
    if inertial:
        W = imu_motion_weights(p.n_frames - 1)
        o.set_imu_weights(W)
        out["r_imu"], out["J_imu"] = o.eval_imu()
    ne = o.normal_equations()
    for k in ("B", "U", "E", "gf", "C", "gc"):
        out["ne_" + k] = ne[k]
    if inertial:
        o.update_imu_weights()
        out["W"] = o.imu_weights()
    return out


def imu_motion_weights(ni):
    """a non-default symmetric positive definite weight per interval (test_gpu_imu_streams._weights0)"""
    rng = np.random.default_rng(11)
    W = 3.0 * rng.standard_normal((ni, 9, 9))
    return 0.5 * (W + W.transpose(0, 2, 1)) + np.arange(400.0, 409.0) * np.eye(9)


@pytest.mark.parametrize("name", imu_motion.NAMES + ("vision",))
def test_oracle_sign_invariance(name):
    """flipped(p) against p, to 1e-12 of each quantity's largest entry"""
    inertial = name != "vision"
    p = imu_motion.build(name).p if inertial else imu_motion.vision()
    q = imu_motion.flipped(p, imu_motion.scattered(p.n_frames), cams=[p.n_cams - 1])
    a, b = _oracle_all(p, inertial), _oracle_all(q, inertial)
    same = []
    for k in a:
        err = np.abs(a[k] - b[k]).max() / max(np.abs(a[k]).max(), 1e-300)
        assert err <= 1e-12, (k, err)
        if np.array_equal(a[k], b[k]):
            same.append(k)
    print(f"\n{name}: bit-identical under q -> -q: {same}")
