"""GPU: the reprojection build and the solves on the target views real recordings produce (target_views.py).

- The build of vcgpu_normal_equations (fused_build_kernel; eval_mega_kernel too for inertial rigs) against the
  long-double reference of target_views.reproj_blocks, entry by entry and reported per frame and per (frame, camera)
  block: |dev - ref| <= 1e-11 of the same sum over absolute values.  One dropped or doubled corner moves a block by far
  more; E columns of a camera that does not see a frame must be exactly 0.
- build_frame_warp is reachable only through the persistent and batch solves: one LM iteration on the persistent and
  multi-launch engines against one long-double damped step from the reference blocks, then 6 iterations persistent
  against multi-launch (test_gpu_persistent's bars) and 8 against the oracle, and one DOGLEG solve.
- Batches mixing these rigs: every rig as its own vcgpu_solve / vcgpu_get_covariance (the bars of test_gpu_batch*.py
  and test_gpu_covariance_batch.py).
- A camera no active observation sees, from the upload or emptied by vcgpu_remove_outliers: its blocks come back bit
  for bit from every engine, the parameter tolerance stops where the oracle does, and both covariance entry points
  return zero rows and columns for it and the dense inverse elsewhere.
- PnP on views of 4, 5, 32, 33 and 600 corners and on cropped views, against oracle/pnp.py.
"""
import numpy as np
import pytest

import constant_blocks as cb
import dogleg_ref
import target_views as tv
from test_gpu_covariance import _dense_cov
from test_gpu_covariance_batch import BAR as COV_BAR, _check_matrix, _corr_err
from test_gpu_persistent import _agree
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

MULTI_LAUNCH = 4  # vcgpu_set_profiling bit 2
TOL0 = dict(function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
STATE_KEYS = ("T_wp", "v_w", "q_ck", "p_ck", "intr", "g", "b", "sf")
VISION_KEYS = ("intr", "q_ck", "p_ck", "T_wp")
_VIEWS = {}


def _view(name):
    """each builder once per session (they are deterministic; the tests never change a view's problem)"""
    if name not in _VIEWS:
        _VIEWS[name] = tv.build(name)
    return _VIEWS[name]


def _calibrator(v, mode=0, **opts):
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.load(v.p)
    if v.flags:
        g.set_flags(**v.flags)
    g.set_profiling(mode, False)
    if opts:
        g.set_options(**opts)
    return g


def _oracle(v, **opts):
    from oracle.binding import Oracle

    o = Oracle(v.p, **v.flags)
    if opts:
        o.set_options(**opts)
    return o


def _engine_ran(s, inertial, persistent):
    per = 2 if inertial else 1
    return (s["kernel_launches"] <= per * s["iterations"] + 12) == persistent


def _reference(v, o=None):
    """the long-double reprojection blocks at the uploaded state, plus (inertial) the oracle's IMU blocks; returns
    (ref, abs sums, per-key allowance for the IMU part)"""
    o = o if o is not None else _oracle(v)
    r, J = o.eval_reproj()
    ref, ab = tv.reproj_blocks(v.p, r, J, o.global_mask(), o.fd, o.G)
    extra, imu = {}, None
    if v.inertial:
        o.set_flags(**v.flags, visual=0)
        imu = o.normal_equations()
        o.set_flags(**v.flags)
        for k in ("B", "E", "gf", "C", "gc"):
            ref[k] = ref[k] + imu[k].astype(np.longdouble)
            # the IMU terms are not what these views change: test_gpu_imu_parity's family-wide bar
            extra[k] = 1e-10 * np.abs(imu[k]).max()
        ref["U"] = imu["U"]
        ref["cost"] = ref["cost"] + imu["cost"]
    return ref, ab, extra


# ------------------------------------------------------------------ 1. the build, against the long-double reference
BUILD_CASES = [(n, 0) for n in tv.VISION] + [(n, m) for n in tv.INERTIAL for m in (0, MULTI_LAUNCH)]


@pytest.mark.parametrize("name,mode", BUILD_CASES,
                         ids=[f"{n}-{'fused' if not n.endswith('inertial') else ('eval_mega' if m == 0 else 'fused')}"
                              for n, m in BUILD_CASES])
def test_build_matches_long_double_reference(name, mode):
    v = _view(name)
    g = _calibrator(v, mode)
    ne = g.normal_equations()
    ref, ab, extra = _reference(v)
    assert abs(ne["cost"] - float(ref["cost"])) <= 1e-11 * float(ref["cost"])
    bad = tv.block_errors(ne, ref, ab, v.p.models, 1e-11, extra)
    assert not bad, bad[:8]
    if v.inertial:
        assert np.abs(ne["U"] - ref["U"]).max() <= 1e-10 * np.abs(ref["U"]).max()
    # a camera that does not see a frame: its columns of that frame's E exactly 0
    n = tv.counts(v.p)
    for c, o in enumerate(tv.cam_offsets(v.p.models)):
        cols = slice(o, o + 6 + synth.NUM_INTR[int(v.p.models[c])])
        assert not ne["E"][n[c] == 0][:, :, cols].any(), c


# ------------------------------------------------------------------ 2. solves: build_frame_warp
def _step_reference(v):
    """the state after one LM iteration from the long-double blocks: Jacobi scale, D2 = clamp(diag, 1e-6, 1e32) / radius
    at the initial radius, dogleg_ref.gauss_newton's refined solve, then the oracle's Plus"""
    o = _oracle(v)
    ref, _, _ = _reference(v, o)
    ne = {k: np.asarray(ref[k], dtype=np.float64) for k in ("B", "E", "gf", "C", "gc")}
    ne["U"] = np.asarray(ref["U"], dtype=np.float64) if "U" in ref else np.zeros_like(ne["B"])
    radius = 1e4  # vcgpu_default_options' and the oracle's init_radius
    scale = dogleg_ref.jacobi_scale(ne)
    diag = dogleg_ref._diag(ne) * scale * scale
    D2 = np.clip(diag, 1e-6, 1e32) / radius
    x = dogleg_ref.gauss_newton(ne, scale, D2)
    o.plus(scale * x)
    return o.state()


VISION_SOLVES = [n for n in tv.VISION]


@pytest.mark.parametrize("name", VISION_SOLVES)
def test_one_lm_step_matches_reference(name):
    """measured on an H100: the device's step is within 5e-12 of the reference's (relative to the step)"""
    v = _view(name)
    ref = _step_reference(v)
    launches = []
    for mode in (0, MULTI_LAUNCH):
        g = _calibrator(v, mode, max_iters=1, **TOL0)
        assert g.opts.init_radius == 1e4
        s = g.solve()
        assert s["iterations"] == 1 and s["successful_steps"] == 1
        launches.append(s["kernel_launches"])
        st = g.state()
        for k in VISION_KEYS:
            moved = np.abs(ref[k] - getattr(v.p, k)).max()
            err = np.abs(st[k] - ref[k]).max()
            assert err <= 1e-9 * moved + 1e-15 * np.abs(ref[k]).max(), (mode, k, err, moved)
    assert launches[0] < launches[1], launches  # the persistent kernel ran


@pytest.mark.parametrize("name", VISION_SOLVES)
def test_persistent_matches_multi_launch(name):
    _agree(_view(name).p)


def _against_oracle(v, mode=0, strategy=0, iters=8):
    """test_gpu_persistent.test_persistent_matches_oracle's bars (inertial: fixed IMU weights)"""
    opts = dict(max_iters=iters, strategy=strategy, **TOL0)
    if v.inertial:
        opts["update_imu_weights"] = 0
    o, g = _oracle(v, num_threads=8, **opts), _calibrator(v, mode, **opts)
    so, sg = o.solve(), g.solve()
    assert _engine_ran(sg, v.inertial, mode == 0), sg["kernel_launches"]
    assert sg["iterations"] == so["iterations"] == iters
    # These rigs converge within 6-8 iterations (test_persistent_matches_oracle's does not).  Measured on an H100: past
    # convergence the cost changes by ~1e-13 and its sign, hence the step's acceptance, is rounding; so the accepted
    # steps are compared over the iterations whose cost change is above 1e-10 of the cost, where both must agree.
    live = [it for it in range(1, iters + 1) if abs(so["rows"][it, 2]) > 1e-10 * so["rows"][it, 1]]
    assert len(live) >= 5
    assert np.array_equal(sg["rows"][live, 8], so["rows"][live, 8])
    assert np.allclose(sg["rows"][live, 1], so["rows"][live, 1], rtol=1e-9)
    assert abs(sg["final_cost"] - so["final_cost"]) <= 1e-9 * so["final_cost"]
    xo, st = o.state(), g.state()
    for k in (STATE_KEYS if v.inertial else VISION_KEYS):
        assert np.abs(st[k] - xo[k]).max() <= 1e-6 * max(np.abs(xo[k]).max(), 1.0), k
    return g, st


ORACLE_CASES = [(n, 0) for n in tv.VISION] + [(n, m) for n in tv.INERTIAL for m in (0, MULTI_LAUNCH)]


@pytest.mark.parametrize("name,mode", ORACLE_CASES,
                         ids=[f"{n}-{'persistent' if m == 0 else 'multi_launch'}" for n, m in ORACLE_CASES])
def test_solve_matches_oracle(name, mode):
    v = _view(name)
    _, st = _against_oracle(v, mode)
    if v.unseen_cam >= 0:
        _unseen_bits(v, st)


@pytest.mark.parametrize("name", ["cropped", "counts", "unseen_camera"])
def test_dogleg_persistent(name):
    v = _view(name)
    _, st = _against_oracle(v, 0, strategy=1)
    if v.unseen_cam >= 0:
        _unseen_bits(v, st)


# ------------------------------------------------------------------ 3. batches mixing these rigs
def _solo_and_batch(names, entry):
    from vicalib_b200 import capi

    solo, batch = [], []
    for n in names:
        v = _view(n)
        g = _calibrator(v, max_iters=6, **TOL0)
        s = g.solve(free_running=True)
        solo.append((s, g.state()))
        batch.append(_calibrator(v, max_iters=6, **TOL0))
    sums = getattr(capi, entry)(batch)
    return solo, [(s, g.state()) for s, g in zip(sums, batch)], batch


def _agree_solo(got, ref, keys, what):
    (s, st), (s0, st0) = got, ref
    for k in ("iterations", "successful_steps", "termination", "num_residuals"):
        assert s[k] == s0[k], (what, k, s[k], s0[k])
    assert abs(s["final_cost"] - s0["final_cost"]) <= 1e-10 * s0["final_cost"], what
    for k in keys:
        assert np.abs(st[k] - st0[k]).max() <= 1e-8 * max(np.abs(st0[k]).max(), 1.0), (what, k)


def test_solve_batch_mixed():
    names = list(tv.VISION)
    solo, batch, _ = _solo_and_batch(names, "solve_batch")
    for n, a, b in zip(names, batch, solo):
        _agree_solo(a, b, VISION_KEYS, n)
        if _view(n).unseen_cam >= 0:
            _unseen_bits(_view(n), a[1])


def test_solve_batch_inertial_mixed():
    names = list(tv.INERTIAL)
    solo, batch, _ = _solo_and_batch(names, "solve_batch_inertial")
    for n, a, b in zip(names, batch, solo):
        _agree_solo(a, b, STATE_KEYS, n)
        if _view(n).unseen_cam >= 0:
            _unseen_bits(_view(n), a[1])


# ------------------------------------------------------------------ 4. a camera no active observation sees
def _unseen_bits(v, st):
    c = v.unseen_cam
    for k in ("q_ck", "p_ck", "intr"):
        assert np.array_equal(st[k][c], getattr(v.p, k)[c]), (v.name, k)


def _cam_cols(p, c):
    o = tv.cam_offsets(p.models)[c]
    return np.arange(o, o + 6 + synth.NUM_INTR[int(p.models[c])])


@pytest.mark.parametrize("mode", [0, MULTI_LAUNCH], ids=["persistent", "multi_launch"])
@pytest.mark.parametrize("name", ["unseen_camera", "unseen_camera_inertial"])
def test_unseen_camera_param_tol(name, mode):
    """the tolerance under which the free-block x_norm stops at iteration k and the all-block one earlier: the device
    stops at k with the oracle's state"""
    v = _view(name)
    rows, norms, win = cb.param_tol_case(v.p, v.flags)
    assert win is not None
    tol, k, j = win
    o = _oracle(v, max_iters=k + 5, function_tol=0.0, gradient_tol=0.0, param_tol=tol)
    g = _calibrator(v, mode, max_iters=k + 5, function_tol=0.0, gradient_tol=0.0, param_tol=tol)
    s_o, s_g = o.solve(), g.solve()
    assert s_o["termination"] == 3 and s_o["iterations"] == k
    assert (s_g["termination"], s_g["iterations"], s_g["successful_steps"]) == (3, k, s_o["successful_steps"])
    st = g.state()
    _unseen_bits(v, st)
    for key in STATE_KEYS:
        assert np.abs(st[key] - o.state()[key]).max() <= 1e-6 * max(1.0, np.abs(o.state()[key]).max()), key


def _solved(v, mode=0):
    """a handle solved to convergence, and the oracle at its state"""
    import dataclasses

    g = _calibrator(v, mode, function_tol=1e-12, max_iters=15)
    g.solve()
    st = g.state()
    p2 = dataclasses.replace(v.p, intr=st["intr"], q_ck=st["q_ck"], p_ck=st["p_ck"], T_wp=st["T_wp"], v_w=st["v_w"],
                             g=st["g"], b=st["b"], sf=st["sf"], ts=st["ts"])
    from oracle.binding import Oracle

    o = Oracle(p2, **v.flags)
    if v.inertial:
        o.set_imu_weights(g.imu_weights())
    return g, o, st


def _check_unseen_cov(v, cov, o, c, batch):
    cols = _cam_cols(v.p, c)
    assert not cov[cols].any() and not cov[:, cols].any()
    if batch:
        _check_matrix(cov, o.global_mask())
    else:  # solved column by column: symmetric to rounding
        live = o.global_mask() != 0
        assert np.all(np.diag(cov)[live] > 0) and not cov[~live].any() and not cov[:, ~live].any()
    e = _corr_err(cov, _dense_cov(o))
    print(f"\n{v.name}: covariance vs dense inverse {e:.1e}")
    assert e <= COV_BAR[v.inertial], e


@pytest.mark.parametrize("name", ["unseen_camera", "unseen_camera_inertial"])
def test_unseen_camera_covariance(name):
    from vicalib_b200.capi import covariance_batch

    v = _view(name)
    g, o, st = _solved(v)
    _unseen_bits(v, st)
    _check_unseen_cov(v, g.covariance(), o, v.unseen_cam, False)
    other = _calibrator(_view("cropped") if not v.inertial else _view("one_camera2_inertial"))
    covs = covariance_batch([other, g])
    _check_unseen_cov(v, covs[1], o, v.unseen_cam, True)
    assert _corr_err(covs[0], other.covariance()) <= COV_BAR[v.inertial]


EMPTIED = [(False, 0), (False, MULTI_LAUNCH), (True, 0)]


@pytest.mark.parametrize("inertial,mode", EMPTIED, ids=["vision-persistent", "vision-multi_launch", "inertial-persistent"])
def test_camera_emptied_by_remove_outliers(inertial, mode):
    """unseen_camera's camera, uploaded with its corners and given an rmse of 0: vcgpu_remove_outliers takes every
    corner it has, the groups are rebuilt, and the camera leaves the solve as a never-seen one does"""
    p, c, flags = tv.unseen_camera_rig(inertial)
    w = tv.View("emptied", p, flags, unseen_cam=c)
    g, o = _calibrator(w, mode), _oracle(w)
    assert o.global_mask()[_cam_cols(p, c)].all()
    rmse = np.full(p.n_cams, np.inf)
    rmse[c] = 0.0
    n = g.remove_outliers(rmse, 1.0)
    assert n == o.remove_outliers(rmse, 1.0) == int((p.obs_cam == c).sum())
    assert not o.global_mask()[_cam_cols(p, c)].any()
    opts = dict(max_iters=8, **TOL0)
    if inertial:
        opts["update_imu_weights"] = 0
    g.set_options(**opts)
    o.set_options(**opts)
    s_g, s_o = g.solve(), o.solve()
    assert _engine_ran(s_g, inertial, mode == 0), s_g["kernel_launches"]
    assert s_g["successful_steps"] == s_o["successful_steps"]
    assert abs(s_g["final_cost"] - s_o["final_cost"]) <= 1e-9 * s_o["final_cost"]
    st, xo = g.state(), o.state()
    _unseen_bits(w, st)
    for k in (STATE_KEYS if inertial else VISION_KEYS):
        assert np.abs(st[k] - xo[k]).max() <= 1e-6 * max(np.abs(xo[k]).max(), 1.0), k
    cov = g.covariance()
    assert not cov[_cam_cols(p, c)].any() and not cov[:, _cam_cols(p, c)].any()
    assert np.all(np.diag(cov)[o.global_mask() != 0] > 0)


# ------------------------------------------------------------------ 5. PnP on partial views
def _groups(p):
    key = p.obs_cam.astype(np.int64) * p.n_frames + p.obs_frame
    start = np.flatnonzero(np.r_[True, key[1:] != key[:-1]])
    count = np.diff(np.r_[start, len(key)])
    return p.obs_cam[start].astype(np.int32), start.astype(np.int64), count.astype(np.int32)


def _pnp_check(p, cam, start, count, pix, **kw):
    from oracle import pnp
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.set_cameras(p.models, p.intr, p.q_ck, p.p_ck)
    T, rmse, used = g.pose_pnp_ransac(cam, start, count, pix, p.p_w, **kw)
    for i in range(len(cam)):
        sl = slice(start[i], start[i] + count[i])
        To, ro, no = pnp.pnp_planar(int(p.models[cam[i]]), p.intr[cam[i]], pix[sl], p.p_w[sl], view=i, **kw)
        assert used[i] == no, (i, count[i])
        assert np.abs(T[i] - To).max() <= 1e-8, (i, count[i], np.abs(T[i] - To).max())
        assert abs(rmse[i] - ro) <= 1e-10, (i, count[i])
    return used


def test_pnp_boundary_counts():
    import dataclasses

    v = _view("counts")
    p = dataclasses.replace(v.p, intr=v.p.truth["intr"].copy())
    cam, start, count = _groups(p)
    sel = np.isin(count, (4, 5, 32, 33, 600))
    assert set(count[sel].tolist()) == {4, 5, 32, 33, 600}
    used = _pnp_check(p, cam[sel], start[sel], count[sel], p.p_c)
    assert np.array_equal(used, count[sel])


@pytest.mark.parametrize("robust", [False, True], ids=["plain", "ransac"])
def test_pnp_cropped_views(robust):
    import dataclasses

    v = _view("cropped")
    p = dataclasses.replace(v.p, intr=v.p.truth["intr"].copy())
    cam, start, count = _groups(p)
    ok = np.array([len(np.unique(p.grid_idx[s:s + n, 0])) >= 3 and len(np.unique(p.grid_idx[s:s + n, 1])) >= 3
                   for s, n in zip(start, count)])
    assert ok.sum() >= 30 and count[ok].min() <= 12
    pix = p.p_c.copy()
    kw = {}
    if robust:
        pix[::11] += 25.0  # wrong associations
        kw = dict(robust_its=40, robust_tol=3.0 / 300)
    _pnp_check(p, cam[ok], start[ok], count[ok], pix, **kw)
