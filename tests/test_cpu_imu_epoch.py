"""CPU: the inertial path on Unix-time stamps (imu_epoch.py, tests/golden/imu_epoch_kat.npz).

- Every builder's regime: the realistic problems' rounded sums and midpoint weights, the rounding tie, the twins.
- The oracle against imu_epoch_kat.npz (60-digit mpmath with the reference's binary64 time sums) at
  test_cpu_oracle_golden.test_imu_kat's 1e-9, and more than 1e3 x that bar away from the exact-sum residual.
- The oracle against oracle/_ref (the reference's own functor and UpdateImuWeights; skipped where it is absent) on every
  realistic problem and on the rounding tie, at test_cpu_imu_motion.test_functor_and_weights_match_ref's bars.
- Twin invariance, bit for bit: the oracle's residuals, Jacobians, normal equations and one cold UpdateImuWeights, and
  the reference functor's residuals and Jacobians, at the small origin and at E on the 2^-21 s grid.
"""
import ctypes as C
import os

import numpy as np
import pytest

import imu_epoch
import imu_streams
from test_cpu_imu_motion import ALL_ON, SO, imu_motion_weights, kat_problem, needs_ref
from vicalib_b200 import synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KAT_BAR = 1e-9  # test_cpu_oracle_golden.test_imu_kat


# ------------------------------------------------------------------ the builders' regimes
@pytest.mark.parametrize("name", imu_epoch.REALISTIC)
def test_realistic_regime(name):
    e = imu_epoch.realistic(name)  # asserts its own regime
    print(f"\n{name}: {len(e.p.imu_t)} samples, inexact t_i + ts {e.inexact:.0%}, max |alpha_mid - 0.5| {e.alpha:.1e}, "
          f"classification changed at E: {e.changed or 'nowhere'}")


def test_rounding_tie_regime():
    e = imu_epoch.rounding_tie()  # asserts its own regime
    assert e.changed["covered"] == [0]  # HasElement at frame 0 holds by rounding alone
    assert e.changed["tie_start"] == e.changed["tie_end"] == list(range(e.p.n_frames - 1))


@pytest.mark.parametrize("name", imu_epoch.TWINS)
def test_twin_regime(name):
    small, epoch = imu_epoch.twin(imu_epoch.twin_source(name))  # asserts the grid and equal classifications
    assert small.ts != 0.0 and np.all(epoch.imu_t >= 2.0 ** 30)


# ------------------------------------------------------------------ the oracle against the Unix-time KAT
def test_epoch_kat_regime():
    """the fixture has what it is for: stamps at E, sums that round, no sample near a frame, r far from r_exact"""
    z = np.load(os.path.join(GOLD, "imu_epoch_kat.npz"))
    p = kat_problem(z)
    assert np.all((p.imu_t >= 2.0 ** 30) & (p.imu_t < 2.0 ** 31)) and np.all(p.ftime >= 2.0 ** 30)
    assert imu_epoch.inexact_fraction(p) >= 0.9 and imu_epoch.alpha_departure(p)[0] >= 1e-5
    c = imu_streams.classify(p)
    assert c["comparable"].all() and not imu_streams.ts_kinks(z).any()
    for s in (0, 1):
        assert np.abs(z["r"][s] - z["r_exact"][s]).max() >= 1e3 * KAT_BAR * np.abs(z["r"][s]).max()


@pytest.mark.parametrize("switch", [0, 1])
def test_oracle_vs_epoch_kat(switch):
    from oracle.binding import Oracle

    z = np.load(os.path.join(GOLD, "imu_epoch_kat.npz"))
    p = kat_problem(z)
    o = Oracle(p, inertial=1, rotation_only=switch, bias_active=1, scale_active=1, optimize_ts=1)
    o.set_imu_weights(np.broadcast_to(z["W"], (p.n_frames - 1, 9, 9)).copy())
    r, J = o.eval_imu()
    scale = np.abs(z["r"][switch]).max()
    err_r = np.abs(r - z["r"][switch]).max() / scale
    err_J = np.abs(J - z["J"][switch]).max() / np.abs(z["J"][switch]).max()
    exact = np.abs(r - z["r_exact"][switch]).max() / scale
    print(f"\noracle vs epoch KAT, switch {switch}: r {err_r:.1e}, J {err_J:.1e}; from the exact-sum residual {exact:.1e}")
    assert err_r <= KAT_BAR and err_J <= KAT_BAR
    assert exact >= 1e3 * KAT_BAR  # the oracle does the reference's rounding, not exact time arithmetic


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


def _ref_intervals(ref, p, W):
    """ref_imu_eval (r, 9 x 33 J) and ref_update_weight (W, None without measurements) of every interval"""
    t, w, a = _c(p.imu_t), _c(p.imu_w), _c(p.imu_a)
    imu = (C.c_int(len(t)), _p(t), _p(w), _p(a))
    gg, b, sf = _c(p.g), _c(p.b), _c(p.sf)
    rs, Js, Ws = [], [], []
    for k in range(p.n_frames - 1):
        r, J = np.zeros(9), np.zeros((9, 33))
        T2, T1, v2, v1 = _c(p.T_wp[k + 1]), _c(p.T_wp[k]), _c(p.v_w[k + 1]), _c(p.v_w[k])
        rc = ref.ref_imu_eval(*imu, C.c_double(p.ftime[k]), C.c_double(p.ftime[k + 1]), _p(_c(W[k])), C.c_int(0),
                              _p(T2), _p(T1), _p(v2), _p(v1), _p(gg), _p(b), _p(sf), C.c_double(p.ts), _p(r), _p(J))
        Wr = np.zeros((9, 9))
        mm = C.c_double()
        has = ref.ref_update_weight(*imu, C.c_double(p.ftime[k]), C.c_double(p.ftime[k + 1]), _p(T1), _p(v1), _p(T2),
                                    _p(v2), _p(gg), _p(b), _p(sf), C.c_double(p.ts), C.c_double(synth.GYRO_SIGMA),
                                    C.c_double(synth.ACCEL_SIGMA), _p(Wr), C.byref(mm))
        assert rc == 0, k
        rs.append(r)
        Js.append(J)
        Ws.append(Wr if has == 1 else None)
    return np.array(rs), np.array(Js), Ws


def _epoch_case(name):
    return imu_epoch.rounding_tie() if name == "rounding_tie" else imu_epoch.realistic(name)


@needs_ref
@pytest.mark.parametrize("name", imu_epoch.REALISTIC + ("rounding_tie",))
def test_functor_and_weights_match_ref(ref, name):
    """at E: the residual and Jacobian at 1e-11, W at 1e-8 relative where the interval has >= 2 RK4 steps (single-step
    weights are decided by rounding, DESIGN.md UpdateImuWeights); intervals without measurements 0 in both"""
    from oracle.binding import Oracle

    e = _epoch_case(name)
    p = e.p
    o = Oracle(p, **ALL_ON)
    W = imu_motion_weights(p.n_frames - 1)
    o.set_imu_weights(W)
    r_o, J_o = o.eval_imu()
    o.update_imu_weights()
    W_o = o.imu_weights()
    r_r, J_r, W_r = _ref_intervals(ref, p, W)
    c = e.cls
    worst = [0.0, 0.0, 0.0]
    for k in range(p.n_frames - 1):
        if not c["covered"][k]:
            assert W_r[k] is None and not r_r[k].any() and not J_r[k].any(), k  # no measurements: zero rows, no weight
            assert not r_o[k].any() and not J_o[k].any() and np.array_equal(W_o[k], W[k]), k
            continue
        ek = [np.abs(r_r[k] - r_o[k]).max() / max(1.0, np.abs(r_o[k]).max()),
              np.abs(J_r[k] - J_o[k]).max() / np.abs(J_o[k]).max()]
        assert ek[0] <= 1e-11 and ek[1] <= 1e-11, (k, ek)
        if c["comparable"][k]:
            ek.append(np.abs(W_r[k] - W_o[k]).max() / np.abs(W_o[k]).max())
            assert ek[2] <= 1e-8, (k, ek)
        worst[:len(ek)] = [max(x, y) for x, y in zip(worst, ek)]
    print(f"\n{name} at E: oracle vs reference r {worst[0]:.1e} J {worst[1]:.1e} W {worst[2]:.1e}")


# ------------------------------------------------------------------ twin invariance
def _oracle_all(p):
    from oracle.binding import Oracle

    o = Oracle(p, **ALL_ON)
    o.set_imu_weights(imu_motion_weights(p.n_frames - 1))
    out = {}
    out["r_imu"], out["J_imu"] = o.eval_imu()
    ne = o.normal_equations()
    for k in ("B", "U", "E", "gf", "C", "gc"):
        out["ne_" + k] = ne[k]
    out["cost"] = np.array(ne["cost"])
    o.update_imu_weights()
    out["W"] = o.imu_weights()
    return out


@pytest.mark.parametrize("name", imu_epoch.TWINS)
def test_oracle_twin_invariance(name):
    small, epoch = imu_epoch.twin(imu_epoch.twin_source(name))
    a, b = _oracle_all(small), _oracle_all(epoch)
    assert np.abs(a["r_imu"]).max() > 0 and np.abs(a["W"] - imu_motion_weights(small.n_frames - 1)).max() > 1.0
    for k in a:
        assert np.array_equal(a[k], b[k]), k


@needs_ref
@pytest.mark.parametrize("name", imu_epoch.TWINS)
def test_ref_twin_invariance(ref, name):
    small, epoch = imu_epoch.twin(imu_epoch.twin_source(name))
    W = imu_motion_weights(small.n_frames - 1)
    (r0, J0, W0), (r1, J1, W1) = _ref_intervals(ref, small, W), _ref_intervals(ref, epoch, W)
    assert np.array_equal(r0, r1) and np.array_equal(J0, J1)
    for k, (x, y) in enumerate(zip(W0, W1)):
        assert (x is None) == (y is None) and (x is None or np.array_equal(x, y)), k
