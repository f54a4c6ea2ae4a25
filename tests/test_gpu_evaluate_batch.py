"""GPU: vcgpu_evaluate_batch and vcgpu_remove_outliers_batch (eval_batch_kernel, one launch over tiles of every rig),
and the per-handle vcgpu_evaluate and vcgpu_remove_outliers, which run it as a batch of one.  The reference is code
they do not share: the residuals of vcgpu_eval_reproj at the active observations, their per-camera costs summed in
numpy and the outlier sets formed from them in numpy.  Residuals and counts must be the same bits, costs within 1e-13
relative (the device sums in another order), removal sets equal.  A rig's tiling is a function of the rig alone, so
its outputs must not move, bit for bit, with the rest of the batch.  Not covered: handles on different devices and
frame-sharded handles (both need more than one GPU); their refusals are argument checks next to the ones tested here.
"""
import ctypes as C

import numpy as np
import pytest

from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
COST_BAR = 1e-13
TOL0 = dict(function_tol=0.0, gradient_tol=0.0, param_tol=0.0)


def _rig(models, n_frames, seed, inertial=False, grid=(10, 7), problem=None):
    from vicalib_b200.capi import Calibrator

    p = problem if problem is not None else synth.make_problem(models=models, n_frames=n_frames, grid=grid, inertial=inertial, seed=seed)
    g = Calibrator()
    g.load(p)
    if inertial:
        g.set_flags(**ALL_ON)
    g.obs_cam = np.asarray(p.obs_cam)  # for _reference
    return g, p


def _reference(g, obs_cam):
    """(cost[n_cams], blocks[n_cams], residuals) of the active observations, caller order, from vcgpu_eval_reproj"""
    act = g.obs_active().astype(bool)
    r = g.eval_reproj(jac=False)[0][act]
    cam = np.asarray(obs_cam)[act]
    cost = np.array([0.5 * np.sum(r[cam == c, 0] * r[cam == c, 0] + r[cam == c, 1] * r[cam == c, 1]) for c in range(g.n_cams)])
    return cost, np.array([(cam == c).sum() for c in range(g.n_cams)], dtype=np.int64), r.ravel()


def _outliers(g, obs_cam, rmse, threshold):
    """the active observations RemoveOutliers drops, formed in numpy from the residuals of vcgpu_eval_reproj"""
    r = g.eval_reproj(jac=False)[0]
    err = np.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1])
    return g.obs_active().astype(bool) & (err > threshold * np.asarray(rmse)[np.asarray(obs_cam)])


def _per_handle(g):
    """(cost[n_cams], blocks[n_cams], residuals) through vcgpu_evaluate"""
    per = [g.evaluate(c) for c in range(g.n_cams)]
    _, res, _ = g.evaluate(-1, residuals=True)
    return np.array([c for c, _ in per]), np.array([n for _, n in per], dtype=np.int64), res


def _check(got, ref, what):
    (c, b, r), (c0, b0, r0) = got, ref
    assert np.array_equal(b, b0), (what, b, b0)
    assert r.tobytes() == r0.tobytes(), what
    for k in range(len(c0)):
        if b0[k] == 0:
            assert c[k] == 0.0 and c0[k] == 0.0, (what, k)
        else:
            assert abs(c[k] - c0[k]) <= COST_BAR * c0[k], (what, k, c[k], c0[k])


def _mixed_rigs(seed):
    """vision rigs of all five models (one with two cameras), poly3 + IMU rigs, a rig whose camera 1 lost every
    observation to vcgpu_remove_outliers, and a rig with no active observation"""
    rigs = [_rig((m,), 12, seed + k)[0] for k, m in enumerate(("linear", "fov", "poly2", "poly3", "kb4"))]
    rigs.append(_rig(("fov", "kb4"), 16, seed + 5)[0])
    rigs.append(_rig(("poly3",), 40, seed + 6, inertial=True)[0])
    rigs.append(_rig(("poly3", "poly2"), 24, seed + 7, inertial=True)[0])
    emptied, p = _rig(("poly3", "poly3"), 14, seed + 8)
    assert emptied.remove_outliers(np.array([np.inf, 0.0]), 1.0) == int((p.obs_cam == 1).sum())
    rigs.append(emptied)
    empty, p = _rig(("poly3",), 10, seed + 9)
    assert empty.remove_outliers(np.array([0.0]), 1.0) == len(p.obs_cam)
    rigs.append(empty)
    return rigs


# ------------------------------------------------------------------ 1. against the per-handle calls, one mixed call
def test_parity_mixed_batch():
    from vicalib_b200.capi import evaluate_batch

    rigs = _mixed_rigs(100)
    for state in ("upload point", "after solve iterations"):
        if state != "upload point":
            for g in rigs[:-1]:  # a few iterations, so that the accepted point may sit in either buffer
                g.set_options(max_iters=3, **TOL0)
                g.solve(free_running=True)
        got = evaluate_batch(rigs, residuals=True)
        for k, (g, out) in enumerate(zip(rigs, got)):
            ref = _reference(g, g.obs_cam)
            _check(out, ref, (state, k))
            _check(_per_handle(g), ref, (state, k, "per handle"))
        assert got[-1][1].sum() == 0 and got[-2][1][1] == 0 and got[-2][1][0] > 0
    # without residuals, the same costs
    plain = evaluate_batch(rigs)
    for (c, b), (c0, b0, _) in zip(plain, got):
        assert c.tobytes() == c0.tobytes() and np.array_equal(b, b0)


# ------------------------------------------------------------------ 2. a rig's outputs do not depend on the batch
def test_independence():
    from vicalib_b200.capi import evaluate_batch

    target = _rig(("poly3", "kb4"), 30, 200)[0]
    others = [_rig(("poly3",) if k % 3 else ("fov", "poly2"), 6 + 3 * k, 210 + k, inertial=k % 4 == 1)[0] for k in range(39)]
    alone = evaluate_batch([target], residuals=True)[0]

    def bits(out):
        return tuple(a.tobytes() for a in out)

    many = others[:20] + [target] + others[20:]
    assert bits(evaluate_batch(many, residuals=True)[20]) == bits(alone)
    assert bits(evaluate_batch(many[::-1], residuals=True)[len(many) - 1 - 20]) == bits(alone)
    assert bits(evaluate_batch(many, residuals=True)[20]) == bits(alone)
    assert bits(evaluate_batch([target], residuals=True)[0]) == bits(alone)


# ------------------------------------------------------------------ 3. outliers
def _with_outliers(models, n_frames, seed, inertial=False, n_bad=12):
    """a problem whose pixels at n_bad known observations are off by 100 px"""
    p = synth.make_problem(models=models, n_frames=n_frames, grid=(10, 7), inertial=inertial, seed=seed)
    bad = np.random.default_rng(seed).choice(len(p.obs_cam), n_bad, replace=False)
    p.p_c = p.p_c.copy()
    p.p_c[bad] += 100.0
    return p, bad


def _rmse(g):
    return np.array([np.sqrt(2.0 * c / n) if n else 0.0 for c, n in (g.evaluate(k) for k in range(g.n_cams))])


def _margin(g, p, rmse, threshold):
    """smallest relative distance of an active observation's |r| from its threshold"""
    act = g.obs_active().astype(bool)
    _, res, _ = g.evaluate(-1, residuals=True)
    err = np.hypot(res[0::2], res[1::2])
    lim = threshold * rmse[p.obs_cam[act]]
    return float((np.abs(err - lim) / lim).min())


def test_outliers_match_per_handle():
    from vicalib_b200.capi import remove_outliers_batch

    specs = [(("poly3", "kb4"), 20, 300, False), (("fov",), 16, 301, False), (("poly3",), 40, 302, True)]
    batch, solo, ps, bads = [], [], [], []
    for models, nf, seed, inertial in specs:
        p, bad = _with_outliers(models, nf, seed, inertial)
        batch.append(_rig(models, nf, seed, inertial, problem=p)[0])
        solo.append(_rig(models, nf, seed, inertial, problem=p)[0])
        ps.append(p)
        bads.append(bad)
    for g, s in zip(batch, solo):  # a solve first, as a station evaluates after one
        for x in (g, s):
            x.set_options(max_iters=10, **TOL0)
            x.solve(free_running=True)
    threshold = 3.0
    rmses = [_rmse(g) for g in batch]
    for g, s, r, p in zip(batch, solo, rmses, ps):
        assert np.array_equal(r, _rmse(s))
        assert _margin(g, p, r, threshold) > 1e-12
    drop = [_outliers(g, p.obs_cam, r, threshold) for g, r, p in zip(batch, rmses, ps)]
    keep = [g.obs_active().astype(bool) & ~d for g, d in zip(batch, drop)]
    counts = remove_outliers_batch(batch, rmses, threshold)
    for g, s, r, bad, n, d, k in zip(batch, solo, rmses, bads, counts, drop, keep):
        assert n == s.remove_outliers(r, threshold) == d.sum() and n >= len(bad)
        act = g.obs_active()
        assert np.array_equal(act, s.obs_active())
        assert np.array_equal(act.astype(bool), k)
        assert not act[bad].any()


def test_outliers_nothing_removed_leaves_handle():
    from vicalib_b200.capi import remove_outliers_batch

    def make():
        return [_rig(("poly3", "poly2"), 18, 310)[0], _rig(("poly3",), 40, 311, inertial=True)[0]]

    rigs, twins = make(), make()
    assert remove_outliers_batch(rigs, [_rmse(g) for g in rigs], 1e6) == [0, 0]
    for g, t in zip(rigs, twins):
        assert g.obs_active().all()
        g.set_options(max_iters=5, **TOL0)
        t.set_options(max_iters=5, **TOL0)
        _same_solve(g.solve(free_running=True), t.solve(free_running=True), g.state(), t.state())


# ------------------------------------------------------------------ 4. no side effects
def _snapshot(g):
    st = g.state()
    W = g.imu_weights() if g.flags.inertial else np.zeros(0)
    return {k: np.asarray(v).tobytes() for k, v in st.items()}, W.tobytes(), g.obs_active().tobytes()


def _same_solve(s, s0, st, st0):
    for k in ("iterations", "successful_steps", "termination", "num_residuals", "initial_cost", "final_cost", "kernel_launches"):
        assert s[k] == s0[k], (k, s[k], s0[k])
    for k in st0:
        assert np.array_equal(np.asarray(st[k]), np.asarray(st0[k])), k


def test_no_side_effects():
    from vicalib_b200.capi import evaluate_batch, solve_batch, solve_batch_inertial

    def make():
        return [_rig(("poly3",), 20, 321)[0], _rig(("poly3", "kb4"), 30, 322)[0],
                _rig(("poly3",), 40, 323, inertial=True)[0], _rig(("poly3",), 90, 324, inertial=True)[0]]

    rigs, fresh = make(), make()
    for g in rigs + fresh:
        g.set_options(max_iters=6, **TOL0)
    before = [_snapshot(g) for g in rigs]
    evaluate_batch(rigs, residuals=True)
    assert [_snapshot(g) for g in rigs] == before
    for g, f in zip(rigs, fresh):
        _same_solve(g.solve(free_running=True), f.solve(free_running=True), g.state(), f.state())
        if g.flags.inertial:
            assert np.array_equal(g.imu_weights(), f.imu_weights())
    # the batch solves, too, after a second call
    evaluate_batch(rigs)
    for solve, part in ((solve_batch, slice(0, 2)), (solve_batch_inertial, slice(2, 4))):
        sums, sums0 = solve(rigs[part]), solve(fresh[part])
        for g, f, s, s0 in zip(rigs[part], fresh[part], sums, sums0):
            _same_solve(s, s0, g.state(), f.state())


# ------------------------------------------------------------------ 5. the station: solve, evaluate, outliers, solve again
def test_station_flow():
    from vicalib_b200.capi import evaluate_batch, remove_outliers_batch, solve_batch, solve_batch_inertial

    threshold = 3.0
    specs = {False: [(("poly3",), 20, 400), (("poly3", "fov"), 30, 401)],
             True: [(("poly3",), 40, 402), (("poly3", "poly2"), 40, 403)]}
    for inertial, rigs in specs.items():
        solve = solve_batch_inertial if inertial else solve_batch
        batch, solo = [], []
        for models, nf, seed in rigs:
            p, _ = _with_outliers(models, nf, seed, inertial)
            for out in (batch, solo):
                g = _rig(models, nf, seed, inertial, problem=p)[0]
                g.set_options(max_iters=8, **TOL0)
                out.append(g)
        solve(batch)
        evals = evaluate_batch(batch)
        rmses = [np.array([np.sqrt(2.0 * c / n) if n else 0.0 for c, n in zip(cost, blocks)]) for cost, blocks in evals]
        counts = remove_outliers_batch(batch, rmses, threshold)
        after = solve(batch)
        for g, r, n, s_b in zip(solo, rmses, counts, after):
            g.solve(free_running=True)
            r0 = _rmse(g)
            assert np.abs(r - r0).max() <= 1e-8 * r0.max(), (r, r0)
            assert g.remove_outliers(r0, threshold) == n and n > 0
            s = g.solve(free_running=True)
            for k in ("iterations", "successful_steps", "termination", "num_residuals"):
                assert s[k] == s_b[k], (inertial, k)
            assert abs(s["final_cost"] - s_b["final_cost"]) <= 1e-10 * s["final_cost"]
        for g, b in zip(solo, batch):
            assert np.array_equal(g.obs_active(), b.obs_active())
            st, st0 = b.state(), g.state()
            rel = max(float(np.abs(st[k] - st0[k]).max() / max(np.abs(st0[k]).max(), 1.0))
                      for k in ("T_wp", "v_w", "q_ck", "p_ck", "intr", "g", "b", "sf"))
            assert rel <= 1e-8, (inertial, rel)


# ------------------------------------------------------------------ 6. a rig above 500 000 observations
def test_north_star_sized_rig():
    from vicalib_b200.capi import Calibrator, evaluate_batch, remove_outliers_batch

    p = synth.make_config("target")
    assert len(p.obs_cam) > 500_000
    gs = []
    for _ in range(2):
        g = Calibrator()
        g.load(p)
        g.set_flags(**ALL_ON)
        g.set_options(max_iters=2, **TOL0)
        g.solve(free_running=True)
        gs.append(g)
    g, twin = gs
    ref = _reference(g, p.obs_cam)
    _check(evaluate_batch([g], residuals=True)[0], ref, "target")
    _check(_per_handle(g), ref, "target, per handle")
    rmse = _rmse(g)
    threshold = 2.5
    assert _margin(g, p, rmse, threshold) > 1e-12
    drop = _outliers(g, p.obs_cam, rmse, threshold)
    keep = g.obs_active().astype(bool) & ~drop
    n = remove_outliers_batch([g], [rmse], threshold)[0]
    assert n == twin.remove_outliers(rmse, threshold) == drop.sum() and n > 0
    assert np.array_equal(g.obs_active(), twin.obs_active())
    assert np.array_equal(g.obs_active().astype(bool), keep)


# ------------------------------------------------------------------ 7. refusals
def test_refusals():
    from vicalib_b200.capi import lib

    L = lib()
    good = [_rig(("poly3",), 20, 501)[0], _rig(("poly3", "kb4"), 16, 502, inertial=True)[0]]
    fresh = [_rig(("poly3",), 20, 501)[0], _rig(("poly3", "kb4"), 16, 502, inertial=True)[0]]

    def arr(kind, xs):
        return (kind * max(len(xs), 1))(*xs)

    def refused(call, gs, index, **kw):
        assert call(gs, **kw) == -1
        if index is not None:
            for g in gs:
                if g is not None:
                    assert f"handle {index}:" in L.vcgpu_last_error(g.h).decode(), L.vcgpu_last_error(g.h).decode()

    def evaluate(gs, cost_null=None):
        costs = [np.full(8, np.nan) for _ in gs]
        blocks = [np.full(8, -7, dtype=np.int64) for _ in gs]
        cp = [None if i == cost_null else c.ctypes.data for i, c in enumerate(costs)]
        rc = L.vcgpu_evaluate_batch(arr(C.c_void_p, [None if g is None else g.h for g in gs]), C.c_int(len(gs)),
                                    arr(C.c_void_p, cp), arr(C.c_void_p, [b.ctypes.data for b in blocks]), None)
        assert all(np.isnan(c).all() for c in costs) and all((b == -7).all() for b in blocks)
        return rc

    def outliers(gs, rmse_null=None, array_null=False):
        rm = [np.zeros(2) for _ in gs]
        removed = np.full(max(len(gs), 1), -7, dtype=np.int64)
        rp = None if array_null else arr(C.c_void_p, [None if i == rmse_null else r.ctypes.data for i, r in enumerate(rm)])
        rc = L.vcgpu_remove_outliers_batch(arr(C.c_void_p, [None if g is None else g.h for g in gs]), C.c_int(len(gs)),
                                           rp, C.c_double(0.5), removed.ctypes.data_as(C.c_void_p))
        assert (removed == -7).all()
        return rc

    before = [_snapshot(g) for g in good]
    for fn in (evaluate, outliers):
        refused(fn, [], None)                                           # n = 0
        refused(fn, [good[0], good[1], None], 2)                        # a null handle
        refused(fn, [None, good[0]], 0)
        refused(fn, [good[0], good[1], good[0]], 2)                     # a repeated handle
    refused(evaluate, good, 1, cost_null=1)                             # a null cam_cost[i]
    refused(outliers, good, 1, rmse_null=1)                             # a null rmse[i]
    refused(outliers, good, 0, array_null=True)                         # a null rmse array
    assert [_snapshot(g) for g in good] == before
    for g, f in zip(good, fresh):
        g.set_options(max_iters=4, **TOL0)
        f.set_options(max_iters=4, **TOL0)
        _same_solve(g.solve(free_running=True), f.solve(free_running=True), g.state(), f.state())
