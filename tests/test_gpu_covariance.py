"""GPU: solution covariance of the global parameters (SURVEY §8 f4; GetSolutionCovariance, vicalibrator.h:802-857) from the
device's frame elimination vs a dense numpy inverse of the oracle's J^T J on small problems, on rigs only the per-handle
call serves, with no side effect on the handle, and on systems whose frame columns are empty."""
import numpy as np
import pytest

import chain_plan
import target_views as tv
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu


def _dense_cov(o):
    """[globals, globals] block of inv(J^T J) from the oracle's block normal equations, constant columns removed"""
    ne = o.normal_equations()
    nf, fd, G = ne["B"].shape[0], o.fd, o.G
    n = nf * fd + G
    H = np.zeros((n, n))
    for f in range(nf):
        s = slice(f * fd, (f + 1) * fd)
        H[s, s] = ne["B"][f]
        H[s, nf * fd:] = ne["E"][f]
        H[nf * fd:, s] = ne["E"][f].T
        if f > 0:
            sp = slice((f - 1) * fd, f * fd)
            H[sp, s] = ne["U"][f]
            H[s, sp] = ne["U"][f].T
    H[nf * fd:, nf * fd:] = ne["C"]
    mask = o.global_mask() != 0
    keep = np.concatenate([np.ones(nf * fd, bool), mask])
    Hi = np.linalg.inv(H[np.ix_(keep, keep)])
    cov = np.zeros((G, G))
    idx = np.where(mask)[0]
    cov[np.ix_(idx, idx)] = Hi[nf * fd:, nf * fd:]
    return cov


ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
BAR = {False: 1e-6, True: 1e-4}
NUMERIC = -3


def _solved(models, inertial, flags, seed=15, nf=None, **kw):
    """a handle solved on synth.make_problem(models, ...), and the oracle at the state it converged to"""
    from oracle.binding import Oracle
    from vicalib_b200.capi import Calibrator

    # inertial problems need a few seconds of motion before biases / gravity are observable (else J^T J is singular to
    # working precision and neither inverse means anything)
    nf = nf or (90 if inertial else 18)
    p = synth.make_problem(models=models, n_frames=nf, inertial=inertial, seed=seed, **kw)
    g = Calibrator()
    g.load(p)
    g.set_flags(**flags)
    g.set_options(function_tol=1e-12, max_iters=15)
    g.solve()
    st = g.state()
    # the oracle evaluates J^T J at the state the device converged to
    p2 = synth.make_problem(models=models, n_frames=nf, inertial=inertial, seed=seed, **kw)
    p2.intr, p2.q_ck, p2.p_ck, p2.T_wp, p2.v_w = st["intr"], st["q_ck"], st["p_ck"], st["T_wp"], st["v_w"]
    p2.g, p2.b, p2.sf, p2.ts = st["g"], st["b"], st["sf"], st["ts"]
    o = Oracle(p2, **flags)
    if inertial:
        o.set_imu_weights(g.imu_weights())
    return g, o


def _check(g, o, inertial):
    cov_o = _dense_cov(o)
    cov_g = g.covariance()
    assert cov_g.shape == cov_o.shape
    sd = np.sqrt(np.maximum(np.diag(cov_o), 1e-300))
    corr_err = np.abs(cov_g - cov_o) / np.outer(sd, sd).clip(1e-300)
    live = np.diag(cov_o) > 0
    # every entry relative to the two standard deviations; both inverses lose cond(J^T J) * eps digits, and the inertial
    # systems are conditioned ~1e10 even after Jacobi scaling
    assert corr_err[np.ix_(live, live)].max() <= BAR[inertial]
    assert np.array_equal(cov_g[~live], np.zeros_like(cov_g[~live]))  # constant blocks: zero rows (ceres::Covariance)
    assert np.array_equal(~live, o.global_mask() == 0)
    assert np.array_equal(cov_g, cov_g.T)  # exactly symmetric
    # a second solve after the covariance call is unaffected by it
    c0 = g.cost()
    assert abs(c0 - o.cost()) <= 1e-9 * c0


@pytest.mark.parametrize("models,inertial,flags", [
    (("poly3",), False, {}),
    (("fov", "kb4"), False, {}),
    (("poly3", "poly2"), True, dict(inertial=1, bias_active=1, scale_active=1, optimize_ts=1)),
    (("poly3",), True, dict(inertial=1, bias_active=1, scale_active=0, optimize_ts=0)),
    # fixed intrinsics: 4-10 constant columns per camera whose damped pivots are the LM floor alone
    (("poly3", "fov"), False, dict(fix_intrinsics=1)),
    (("kb4",), True, dict(inertial=1, bias_active=1, scale_active=1, optimize_ts=1, fix_intrinsics=1)),
])
def test_covariance_matches_dense_inverse(models, inertial, flags):
    g, o = _solved(models, inertial, flags)
    _check(g, o, inertial)


@pytest.mark.parametrize("models,inertial,G,kw", [
    # G = 68: past the persistent inertial kernels and the batch call
    (chain_plan.rig_with_globals(68), True, 68, dict(grid=(8, 6))),
    # G = 112: past the persistent vision kernel and the batch call; at 18 frames its scaled J^T J is conditioned 5e10,
    # too close to singular for two inverses to agree to the bar, at 40 frames 1e9
    (("kb4",) * 8, False, 112, dict(nf=40)),
], ids=["inertial_G68", "vision_G112"])
def test_rigs_only_the_per_handle_call_serves(models, inertial, G, kw):
    g, o = _solved(models, inertial, dict(ALL_ON) if inertial else {}, seed=G, **kw)
    assert g.G == G
    _check(g, o, inertial)


def _same_solve(s, s0, st, st0):
    for k in ("iterations", "successful_steps", "termination", "num_residuals", "initial_cost", "final_cost", "kernel_launches"):
        assert s[k] == s0[k], (k, s[k], s0[k])
    for k in st0:
        assert np.array_equal(np.asarray(st[k]), np.asarray(st0[k])), k


@pytest.mark.parametrize("inertial", [False, True], ids=["vision", "inertial"])
def test_no_side_effects(inertial):
    """state and IMU weights are left bit for bit, and a following solve (and, inertial, batch solve) gives the bits a
    fresh handle gives"""
    from vicalib_b200.capi import Calibrator, solve_batch_inertial

    def make():
        p = synth.make_problem(models=("poly3", "kb4"), n_frames=60 if inertial else 20, inertial=inertial, seed=8)
        g = Calibrator()
        g.load(p)
        g.set_flags(**(ALL_ON if inertial else {}))
        g.set_options(max_iters=4)
        return g

    def snapshot(g):
        W = g.imu_weights() if inertial else np.zeros(0)
        return {k: np.asarray(v).tobytes() for k, v in g.state().items()}, W.tobytes()

    g, fresh = make(), make()
    g.solve()
    fresh.solve()
    before = snapshot(g)
    g.covariance()
    assert snapshot(g) == before
    _same_solve(g.solve(free_running=True), fresh.solve(free_running=True), g.state(), fresh.state())
    assert snapshot(g) == snapshot(fresh)
    if inertial:
        g.covariance()
        (s,), (s0,) = solve_batch_inertial([g]), solve_batch_inertial([fresh])
        _same_solve(s, s0, g.state(), fresh.state())
        assert snapshot(g) == snapshot(fresh)


@pytest.mark.parametrize("case,expect", [("unseen_frames", NUMERIC), ("rotation_only", NUMERIC)])
def test_empty_frame_columns(case, expect):
    """frames whose columns of the undamped J^T J are empty: a vision frame no active observation sees, and the
    velocities of a rotation-only run.  The globals' call takes no frame damping, so J^T J is singular there"""
    from vicalib_b200.capi import Calibrator, _p

    if case == "unseen_frames":
        v = tv.build("unseen_runs")
        p, flags = v.p, v.flags
    else:
        p = synth.make_problem(models=("poly3",), n_frames=90, inertial=True, seed=15)
        flags = dict(inertial=1, rotation_only=1, bias_active=0, scale_active=0, optimize_ts=1)
    g = Calibrator()
    g.load(p)
    g.set_flags(**flags)
    g.set_options(function_tol=1e-12, max_iters=15)
    g.solve()
    out = np.full((g.G, g.G), np.nan)
    assert g.L.vcgpu_get_covariance(g.h, _p(out)) == expect
