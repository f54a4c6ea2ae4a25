"""CPU: the reference of vcgpu_get_imu_influence (tests/imu_influence_ref.py) against the dense problem.
  hat matrix   H_k is the 9 x 9 diagonal block of A (A^T A)^-1 A^T, A the weighted rows of every active corner and every
               interval (so A^T A is the oracle's whole system): the weights are the solve's.  Correlation-scaled
               where the system is too ill-conditioned for an absolute bar (see the test)
  trace        sum tr(H_obs) + sum tr(H_imu) = the kept tangents, 9 per frame (6 rotation-only) plus |F|
  refit        one Gauss-Newton step with interval k taken out, from g = 0: the globals' shift in Sigma_F is infl, and
               r~ . r~_after is stud
  exact        H = I on the last interval when the last frame has no active corner
Rigs: all IMU globals on, imu_mult = 2, rotation-only, and bias / scale / ts off."""
import dataclasses

import numpy as np
import pytest

import dense_cov
import imu_influence_ref as R
import influence_ref as OR
from oracle.binding import Oracle
from test_cpu_observation_influence import _converged

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
CASES = {
    "all_on": (("poly2",), dict(ALL_ON)),
    "imu_mult_2": (("poly3",), dict(ALL_ON, imu_mult=2.0, visual_mult=1.5)),
    "rotation_only": (("poly2",), dict(ALL_ON, rotation_only=1, bias_active=0, scale_active=0)),
    "bias_scale_ts_off": (("poly3", "kb4"), dict(ALL_ON, bias_active=0, scale_active=0, optimize_ts=0)),
}


def _setup(models, flags):
    p, o, flags = _converged(models, True, flags)
    live = 6 if flags.get("rotation_only") else o.fd
    used = np.ones(p.n_frames, bool)
    Hi, keep = dense_cov.dense_inverse(o, used, live)
    act = o.obs_active()
    imu = R.influence(o, Hi, p.models, flags.get("imu_mult", 1.0))
    obs = OR.influence(o, Hi, p.models, p.obs_frame, p.obs_cam, act, used, flags.get("visual_mult", 1.0))
    return p, o, flags, Hi, keep, act, imu, obs


def _all_rows(o, p, flags, act):
    """every weighted row of the problem: (A, the rows of each interval in A)"""
    ob = OR.rows(o, p.models, p.obs_frame, p.obs_cam, flags.get("visual_mult", 1.0))
    im = R.rows(o, p.models, flags.get("imu_mult", 1.0))
    n = p.n_frames * o.fd + o.G
    blocks, at = [], []
    for i, (P, Jt, _) in enumerate(ob):
        if act[i]:
            b = np.zeros((2, n))
            b[:, P] = Jt
            blocks.append(b)
    n0 = 2 * len(blocks)
    for k, (P, Jt, _, _) in enumerate(im):
        b = np.zeros((9, n))
        b[:, P] = Jt
        blocks.append(b)
        at.append(n0 + 9 * k)
    return np.vstack(blocks), at


@pytest.mark.parametrize("name", list(CASES))
def test_hat_matrix_and_trace(name):
    models, flags = CASES[name]
    p, o, flags, Hi, keep, act, imu, obs = _setup(models, flags)
    A, at = _all_rows(o, p, flags, act)
    # A^T A is the oracle's system: the weights applied here are the solve's
    H, _, keep2 = OR.dense_system(o, np.ones(p.n_frames, bool), 6 if flags.get("rotation_only") else o.fd)
    kk = np.flatnonzero(keep)
    assert np.array_equal(keep, keep2)
    AtA = A[:, kk].T @ A[:, kk]
    assert np.abs(AtA - H[np.ix_(kk, kk)]).max() <= 1e-9 * np.abs(H).max()
    # the hat matrix Q Q^T from a QR of the column-equilibrated rows: the normal equations of an inertial rig are too
    # ill-conditioned to form it from (A^T A)^-1 to 1e-9
    Ak = A[:, kk]
    Q, _ = np.linalg.qr(Ak / np.linalg.norm(Ak, axis=0)[None, :])
    d = np.stack([Q[a:a + 9] @ Q[a:a + 9].T for a in at])
    # 1e-9 correlation-scaled (sc_h: the first-order change of H when every Sigma_ij moves by sqrt(Sigma_ii Sigma_jj)), and
    # 1e-9 absolute where the system allows it.  With every IMU global free the Jacobi-scaled J^T J has a condition number
    # of 1e11: inverting it and A^T A, equal to 3e-15 correlation-scaled, gives H 1.4e-6 apart (imu_mult = 2: 2.3e-7),
    # while the correlation-scaled difference is 6.7e-12.  Rotation-only (condition 2e6) and bias / scale / ts off (4e9)
    # agree to 8.5e-12 and 6.3e-10 absolute.
    e = np.abs(d - imu["h"])
    sc = imu["sc_h"]
    assert (e[sc == 0.0] == 0.0).all() and (e[sc > 0.0] / sc[sc > 0.0]).max() < 1e-9
    if flags.get("rotation_only") or not flags.get("bias_active"):
        assert e.max() < 1e-9, e.max()
    if flags.get("rotation_only"):
        off = np.r_[0, 1, 2, 6, 7, 8]
        assert (imu["h"][:, off, :] == 0.0).all() and (imu["h"][:, :, off] == 0.0).all()
    tr = np.trace(imu["h"], axis1=1, axis2=2).sum() + (obs["h"][act > 0, 0] + obs["h"][act > 0, 2]).sum()
    # the same conditioning bounds the trace: with every IMU global free, sum tr(Hi J~^T J~) = tr(I) holds to 5.4e-8
    # relative (Hi the dense inverse, accurate to condition x eps), so that bar is 1e-6 there; 1e-8 elsewhere
    bar = 1e-8 if flags.get("rotation_only") or not flags.get("bias_active") else 1e-6
    assert abs(tr - keep.sum()) < bar * keep.sum(), (tr, keep.sum())


@pytest.mark.parametrize("name", ["all_on", "imu_mult_2", "rotation_only"])
def test_refit(name):
    models, flags = CASES[name]
    p, o, flags, Hi, keep, act, imu, obs = _setup(models, flags)
    live = 6 if flags.get("rotation_only") else o.fd
    H, g, _ = OR.dense_system(o, np.ones(p.n_frames, bool), live)
    nfp = p.n_frames * o.fd
    Sg = Hi[nfp:, nfp:]
    F = np.flatnonzero(np.diag(Sg) != 0.0)
    SF = Sg[np.ix_(F, F)]
    rows = R.rows(o, p.models, flags.get("imu_mult", 1.0))
    ok = np.flatnonzero(np.isfinite(imu["infl"]))
    assert len(ok) >= len(rows) - 2  # an end interval may have no measurements
    # 1e-6 relative, as the observation refit; 1e-5 with every IMU global free, where both sides rest on a system
    # conditioned 1e11 (measured 2.1e-6 on interval 1 of "all_on", 1e-8 or less elsewhere)
    bar = 1e-5 if flags.get("bias_active") and flags.get("imu_mult", 1.0) == 1.0 else 1e-6
    for k in ok[[0, 3, 11, 20, -1]]:
        P, Jt, rt, _ = rows[k]
        # the inertial solve stops with a gradient the IMU terms leave well above rounding: step from g = 0
        dg, r_after = R.refit(H, 0.0 * g, keep, P, Jt, rt, nfp, F)
        infl = dg @ np.linalg.solve(SF, dg)
        stud = rt @ r_after
        assert abs(infl - imu["infl"][k]) <= bar * max(abs(infl), 1e-12) + 1e-14, (k, infl, imu["infl"][k])
        assert abs(stud - imu["stud"][k]) <= bar * max(abs(stud), 1e-12) + 1e-14, (k, stud, imu["stud"][k])


def test_last_frame_without_corners_has_unit_leverage():
    """every corner of the last frame moved and removed: interval nf - 2 alone fixes that frame, so H = I and I - H has
    no Cholesky factor"""
    p, o, _ = _converged(("poly3",), True, ALL_ON, n_frames=30)
    pc = p.p_c.copy()
    last = p.obs_frame == p.n_frames - 1
    pc[last] += 50.0
    st = o.state()
    p2 = dataclasses.replace(p, p_c=pc, intr=st["intr"], q_ck=st["q_ck"], p_ck=st["p_ck"], T_wp=st["T_wp"], v_w=st["v_w"],
                             g=st["g"], b=st["b"], sf=st["sf"], ts=st["ts"])
    o = Oracle(p2, **ALL_ON)
    o.remove_outliers(np.array([1.0]), 5.0)
    act = o.obs_active()
    assert not act[last].any() and act[~last].all()
    Hi, _ = dense_cov.dense_inverse(o, np.ones(p.n_frames, bool), o.fd)
    imu = R.influence(o, Hi, p.models)
    assert np.abs(imu["h"][-1] - np.eye(9)).max() < 1e-6
    assert np.isnan(imu["stud"][-1]) and np.isnan(imu["infl"][-1])
    # the interval before it alone fixes the velocity of the frame between: three unit leverages, so NaN too
    assert np.isnan(imu["stud"][-2]) and np.sort(np.linalg.eigvalsh(imu["h"][-2]))[-3:].min() > 1.0 - 1e-6
    assert np.isfinite(imu["stud"][1:-2]).all()
