"""CPU: the reference of vcgpu_get_observation_influence (tests/influence_ref.py) against the dense problem.
  hat matrix   H_i is the 2 x 2 diagonal block of J~ (J~^T J~)^-1 J~^T, J~ the weighted rows of every active
               observation (vision rigs, so J~^T J~ is the whole system): the weights are the solve's
  trace        on vision rigs the sum of tr(H_i) over the active observations is 6 per used frame plus |F|
  refit        one Gauss-Newton step with the observation taken out (or a removed one put back) at a tightly converged
               state: the globals' shift in Sigma_F is infl, and r~ . r~_after is stud
Five models, 1, 2 and 4 cameras, visual_mult = 2, removed observations, and one inertial rig."""
import dataclasses

import numpy as np
import pytest

import dense_cov
import influence_ref as R
from oracle.binding import Oracle
from vicalib_b200 import synth

INERTIAL = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)


def _converged(models, inertial=False, flags=None, n_frames=None, remove=False, seed=31):
    flags = dict(flags or {})
    nf = n_frames or (40 if inertial else 12)
    p = synth.make_problem(models=models, n_frames=nf, grid=(7, 5), inertial=inertial, seed=seed)
    o = Oracle(p, **flags)
    # IMU weights held fixed, so the solve reaches a stationary point of one problem
    o.set_options(max_iters=60, function_tol=1e-16, gradient_tol=1e-16, param_tol=1e-16, update_imu_weights=0)
    o.solve()
    if remove:  # a few observations out, then converge again without them
        r, _ = o.eval_reproj(jac=False)
        rmse = np.array([np.sqrt(np.mean((r[p.obs_cam == c] ** 2).sum(1))) for c in range(p.n_cams)])
        o.remove_outliers(rmse, 1.6)
        o.solve()
    return p, o, flags


def _ref(p, o, flags):
    fd = o.fd
    used = np.ones(p.n_frames, bool)
    live = 6 if flags.get("rotation_only") else fd
    Hi, keep = dense_cov.dense_inverse(o, used, live)
    act = o.obs_active()
    out = R.influence(o, Hi, p.models, p.obs_frame, p.obs_cam, act, used, flags.get("visual_mult", 1.0))
    return out, Hi, keep, act


CASES = {
    "linear": (("linear",), {}),
    "fov": (("fov",), {}),
    "poly2": (("poly2",), {}),
    "poly3": (("poly3",), dict(visual_mult=2.0)),
    "kb4": (("kb4",), {}),
    "poly3_kb4": (("poly3", "kb4"), {}),
    "four_cams": (("poly3", "fov", "kb4", "linear"), dict(fix_intrinsics=1)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_hat_matrix_and_trace(name):
    models, flags = CASES[name]
    p, o, flags = _converged(models, flags=flags)
    out, Hi, keep, act = _ref(p, o, flags)
    rows = R.rows(o, p.models, p.obs_frame, p.obs_cam, flags.get("visual_mult", 1.0))
    n = len(keep)
    A = np.zeros((2 * int(act.sum()), n))
    k = 0
    for i, (P, Jt, _) in enumerate(rows):
        if act[i]:
            A[2 * k:2 * k + 2, P] = Jt
            k += 1
    kk = np.flatnonzero(keep)
    Ak = A[:, kk]
    hat = Ak @ np.linalg.solve(Ak.T @ Ak, Ak.T)
    ia = np.flatnonzero(act)
    d = np.stack([hat[0::2, 0::2].diagonal(), hat[0::2, 1::2].diagonal(), hat[1::2, 1::2].diagonal()], 1)
    assert np.abs(d - out["h"][ia]).max() < 1e-9
    tr = (out["h"][ia, 0] + out["h"][ia, 2]).sum()
    assert abs(tr - keep.sum()) < 1e-8 * keep.sum(), (tr, keep.sum())


@pytest.mark.parametrize("models,inertial,flags,remove", [
    (("poly3",), False, {}, False),
    (("kb4", "fov"), False, dict(visual_mult=2.0), True),
    (("poly2",), True, INERTIAL, False),
], ids=["poly3", "kb4_fov_removed", "inertial"])
def test_refit(models, inertial, flags, remove):
    p, o, flags = _converged(models, inertial, flags, remove=remove)
    out, Hi, keep, act = _ref(p, o, flags)
    live = 6 if flags.get("rotation_only") else o.fd
    H, g, keep2 = R.dense_system(o, np.ones(p.n_frames, bool), live)
    assert np.array_equal(keep, keep2)
    nfp = p.n_frames * o.fd
    Sg = Hi[nfp:, nfp:]
    F = np.flatnonzero(np.diag(Sg) != 0.0)
    SF = Sg[np.ix_(F, F)]
    rows = R.rows(o, p.models, p.obs_frame, p.obs_cam, flags.get("visual_mult", 1.0))
    rng = np.random.default_rng(3)
    pick = list(rng.choice(np.flatnonzero(act), 12, replace=False)) + list(np.flatnonzero(act == 0)[:6])
    assert not remove or (act == 0).any()
    for i in pick:
        P, Jt, rt = rows[i]
        # the inertial solve stops with a gradient the IMU terms leave well above rounding: step from g = 0 there
        dg, r_after = R.refit(H, 0.0 * g if inertial else g, keep, P, Jt, rt, act[i] > 0, nfp, F)
        infl = dg @ np.linalg.solve(SF, dg)
        stud = rt @ r_after
        assert abs(infl - out["infl"][i]) <= 1e-6 * max(abs(infl), 1e-12) + 1e-14, (i, infl, out["infl"][i])
        assert abs(stud - out["stud"][i]) <= 1e-6 * max(abs(stud), 1e-12) + 1e-14, (i, stud, out["stud"][i])
