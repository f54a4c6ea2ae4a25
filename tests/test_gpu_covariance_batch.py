"""GPU: vcgpu_get_covariance_batch (one thread-block cluster per rig: cov_mega_batch_kernel for vision rigs,
chain_cov_batch_kernel for inertial rigs) against the dense inverse of the oracle's J^T J and against
vcgpu_get_covariance on the same handle, with the bars test_gpu_covariance.py uses (correlation-scaled error 1e-6
vision, 1e-4 inertial).  A rig's cluster size is a function of the rig alone, so its matrix must not move, bit for bit,
with the rest of the batch.  Not covered: handles on different devices and frame-sharded handles (both need more than
one GPU); their refusals are argument checks next to the ones tested here.
"""
import numpy as np
import pytest

import batch_imu_plan
import batch_plan
import chain_plan
from test_gpu_covariance import _dense_cov
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
BAR = {False: 1e-6, True: 1e-4}
NUMERIC = -3

# the six cases of test_gpu_covariance.py
CASES = [
    (("poly3",), False, {}),
    (("fov", "kb4"), False, {}),
    (("poly3", "poly2"), True, dict(inertial=1, bias_active=1, scale_active=1, optimize_ts=1)),
    (("poly3",), True, dict(inertial=1, bias_active=1, scale_active=0, optimize_ts=0)),
    (("poly3", "fov"), False, dict(fix_intrinsics=1)),
    (("kb4",), True, dict(inertial=1, bias_active=1, scale_active=1, optimize_ts=1, fix_intrinsics=1)),
]


def _solved_case(models, inertial, flags):
    """a handle solved as test_gpu_covariance.py solves it, and the oracle at the state it converged to"""
    from oracle.binding import Oracle
    from vicalib_b200.capi import Calibrator

    nf = 90 if inertial else 18
    p = synth.make_problem(models=models, n_frames=nf, inertial=inertial, seed=15)
    g = Calibrator()
    g.load(p)
    g.set_flags(**flags)
    g.set_options(function_tol=1e-12, max_iters=15)
    g.solve()
    st = g.state()
    p2 = synth.make_problem(models=models, n_frames=nf, inertial=inertial, seed=15)
    p2.intr, p2.q_ck, p2.p_ck, p2.T_wp, p2.v_w = st["intr"], st["q_ck"], st["p_ck"], st["T_wp"], st["v_w"]
    p2.g, p2.b, p2.sf, p2.ts = st["g"], st["b"], st["sf"], st["ts"]
    o = Oracle(p2, **flags)
    if inertial:
        o.set_imu_weights(g.imu_weights())
    return g, o


def _corr_err(cov, ref):
    """largest entry error relative to the two standard deviations, over the free globals of ref"""
    sd = np.sqrt(np.maximum(np.diag(ref), 1e-300))
    live = np.diag(ref) > 0
    err = np.abs(cov - ref) / np.outer(sd, sd).clip(1e-300)
    return float(err[np.ix_(live, live)].max())


def _check_matrix(cov, mask):
    """exactly symmetric, rows and columns of constant globals exactly 0"""
    assert np.array_equal(cov, cov.T)
    const = mask == 0
    assert np.all(cov[const] == 0.0) and np.all(cov[:, const] == 0.0)
    assert np.all(np.diag(cov)[~const] > 0.0)


def _cov_batch(gs):
    """covariance_batch that also returns the statuses: (matrices or None, statuses)"""
    from vicalib_b200.capi import VcgpuError, covariance_batch

    try:
        return covariance_batch(gs), [0] * len(gs)
    except VcgpuError as e:
        if e.status is None:
            raise
        return e.covariances, e.status


# ------------------------------------------------------------------ 1. parity, all six cases in one mixed call
def test_parity_mixed_batch():
    from vicalib_b200.capi import covariance_batch

    cases = [_solved_case(*c) for c in CASES]
    gs = [g for g, _ in cases]
    covs = covariance_batch(gs)
    for (models, inertial, flags), (g, o), cov in zip(CASES, cases, covs):
        _check_matrix(cov, o.global_mask())
        e_dense = _corr_err(cov, _dense_cov(o))
        e_solo = _corr_err(cov, g.covariance())
        print(f"\n{models} inertial={inertial} {flags}: vs dense inverse {e_dense:.1e}, vs vcgpu_get_covariance {e_solo:.1e}")
        assert e_dense <= BAR[inertial], (models, flags, e_dense)
        assert e_solo <= BAR[inertial], (models, flags, e_solo)


# ------------------------------------------------------------------ 2. shapes: every cluster size of both kinds, bits
def _vision(n_frames, seed, models=("poly3",)):
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.load(synth.make_problem(models=models, n_frames=n_frames, grid=(10, 7), seed=seed))
    return g


def _inertial(n_frames, seed, models=("poly3",), grid=(10, 7)):
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.load(synth.make_problem(models=models, n_frames=n_frames, grid=grid, inertial=True, seed=seed))
    g.set_flags(**ALL_ON)
    return g


def _shape_rigs(seed):
    w = batch_plan.batch_warps(chain_plan.rig_globals(("poly3",), False), 1)
    rigs, sizes = [], []
    for size in (1, 2, 4, 8):
        rigs.append(_vision(size * w, seed + size))
        sizes.append(("vision", size))
    for size in (1, 2, 4, 8):
        nf = chain_plan.GROUPS * chain_plan.CHUNK * size
        assert batch_imu_plan.cluster_size(nf) == size
        rigs.append(_inertial(nf, seed + 10 + size))
        sizes.append(("inertial", size))
    g67 = _inertial(48, seed + 30, models=chain_plan.rig_with_globals(67), grid=(14, 10))
    assert g67.G == 67
    rigs.append(g67)
    sizes.append(("inertial", batch_imu_plan.cluster_size(48)))
    for g, (kind, size) in zip(rigs, sizes):
        assert (g.batch_plan()[0] if kind == "vision" else g.batch_plan_inertial()[0]) == size, (kind, size)
    return rigs


def _bits(a, b):
    return (a is None and b is None) or (a is not None and b is not None and a.tobytes() == b.tobytes())


def test_shapes_and_bits():
    rigs = _shape_rigs(400)
    n = len(rigs)
    alone = [_cov_batch([g]) for g in rigs]
    alone = [(c[0], s[0]) for c, s in alone]
    mixed, st = _cov_batch(rigs)
    rev, st_r = _cov_batch(rigs[::-1])
    others = _shape_rigs(500)
    beside, st_b = _cov_batch([g for pair in zip(rigs, others) for g in pair])
    for i, (c0, s0) in enumerate(alone):
        assert st[i] == s0 and st_r[n - 1 - i] == s0 and st_b[2 * i] == s0
        assert _bits(mixed[i], c0), f"rig {i}: mixed batch"
        assert _bits(rev[n - 1 - i], c0), f"rig {i}: reversed"
        assert _bits(beside[2 * i], c0), f"rig {i}: beside other rigs"
    # the vision rigs, whose systems are well conditioned at the start point, against the per-handle call
    for g, (c0, s0) in zip(rigs[:4], alone[:4]):
        assert s0 == 0
        _check_matrix(c0, np.diag(c0) != 0)
        assert _corr_err(c0, g.covariance()) <= BAR[False]
    print(f"\nshapes: statuses {[s for _, s in alone]}")


# ------------------------------------------------------------------ 3. the handles are left as they were
def _snapshot(g):
    st = g.state()
    W = g.imu_weights() if g.flags.inertial else np.zeros(0)
    return {k: np.asarray(v).tobytes() for k, v in st.items()}, W.tobytes()


def _same_solve(s, s0, st, st0):
    for k in ("iterations", "successful_steps", "termination", "num_residuals", "initial_cost", "final_cost", "kernel_launches"):
        assert s[k] == s0[k], (k, s[k], s0[k])
    for k in st0:
        assert np.array_equal(np.asarray(st[k]), np.asarray(st0[k])), k


def test_no_side_effects():
    from vicalib_b200.capi import covariance_batch, solve_batch_inertial

    def make():
        return [_vision(20, 61), _vision(40, 62, models=("poly3", "kb4")), _inertial(40, 63), _inertial(90, 64)]

    rigs, fresh = make(), make()
    for g in rigs:  # options the call ignores
        g.set_options(update_state_every_iteration=1, max_iters=3)
    rigs[0].set_options(strategy=1)
    rigs[2].set_options(strategy=1)
    before = [_snapshot(g) for g in rigs]
    covariance_batch(rigs)
    assert [_snapshot(g) for g in rigs] == before
    for g in rigs + fresh:
        g.set_options(update_state_every_iteration=0, strategy=0, max_iters=6)
    for g, f in zip(rigs[:2], fresh[:2]):
        _same_solve(g.solve(free_running=True), f.solve(free_running=True), g.state(), f.state())
    for g, f in zip(rigs[2:], fresh[2:]):
        _same_solve(g.solve(free_running=True), f.solve(free_running=True), g.state(), f.state())
        assert np.array_equal(g.imu_weights(), f.imu_weights())
    # the batch inertial solve, too (sync-word parity), after a second call
    covariance_batch(rigs)
    sums, sums0 = solve_batch_inertial(rigs[2:]), solve_batch_inertial(fresh[2:])
    for g, f, s, s0 in zip(rigs[2:], fresh[2:], sums, sums0):
        _same_solve(s, s0, g.state(), f.state())


# ------------------------------------------------------------------ 4. the station: batch solve, then batch covariance
def test_station_flow():
    from vicalib_b200.capi import covariance_batch, solve_batch_inertial

    def make():
        out = []
        for i in range(4):
            g = _inertial(90, 80 + i, models=("poly3",) if i % 2 else ("poly3", "poly2"), grid=(14, 10))
            g.set_options(function_tol=1e-12, max_iters=15)
            out.append(g)
        return out

    batch, solo = make(), make()
    solve_batch_inertial(batch)
    covs = covariance_batch(batch)
    for g, cov in zip(solo, covs):
        g.solve(free_running=True)
        err = _corr_err(cov, g.covariance())
        print(f"\nstation rig: vs vcgpu_solve + vcgpu_get_covariance {err:.1e}")
        assert err <= BAR[True]


# ------------------------------------------------------------------ 5. refusals
def test_refusals():
    from vicalib_b200.capi import VcgpuError, covariance_batch

    def refused(gs, index, out=None):
        bufs = out if out is not None else [None if g is None else np.full((g.G, g.G), np.nan) for g in gs]
        with pytest.raises(VcgpuError) as e:
            covariance_batch(gs, out=bufs)
        assert "vcgpu error -1" in str(e.value), str(e.value)
        if index is not None:
            assert f"handle {index}:" in str(e.value), str(e.value)
        for b in bufs:
            assert b is None or np.isnan(b).all()

    good = [_vision(20, 71), _inertial(40, 72)]
    fresh = [_vision(20, 71), _inertial(40, 72)]

    def bad(kind, profiling=None, flush=False, **kw):
        g = _vision(20, 73, **kw) if kind == "vision" else _inertial(24, 74, **kw)
        if profiling is not None or flush:
            g.set_profiling(profiling or 0, flush)
        return g

    specs = [("vision", dict(profiling=p)) for p in (1, 2, 4, 8)] + [("inertial", dict(profiling=p)) for p in (1, 2, 4, 8)]
    specs += [("vision", dict(flush=True)), ("inertial", dict(flush=True)),
              ("inertial", dict(models=chain_plan.rig_with_globals(68), grid=(14, 10))),  # G = 68
              ("vision", dict(models=("kb4",) * 8))]                                        # G = 112
    bads = [bad(k, **s) for k, s in specs]
    assert bads[-2].G == 68 and bads[-1].G == 112
    novis = _vision(20, 75)
    novis.set_flags(visual=0)  # no active observation
    bads.append(novis)
    refused([], None)                                          # n = 0
    refused([good[0], good[1], None], 2)                       # a null handle
    refused([None, good[0]], 0)
    refused([good[0], good[1], good[0]], 2)                    # a repeated handle
    bufs = [np.full((g.G, g.G), np.nan) for g in good]
    refused(good, 1, out=[bufs[0], None])                      # a null cov pointer
    assert np.isnan(bufs[0]).all()
    for b in bads:
        refused([good[0], good[1], b], 2)
        refused([b, good[0], good[1]], 0)
    # nothing ran: the handles solve as fresh ones do
    for g, f in zip(good, fresh):
        _same_solve(g.solve(free_running=True), f.solve(free_running=True), g.state(), f.state())


# ------------------------------------------------------------------ 6. a singular rig among healthy ones
def test_singular_rig_among_healthy():
    from vicalib_b200.capi import VcgpuError

    # every reprojection residual weighted 0: the frames' and the free globals' columns are empty, so J^T J is singular
    # (a camera that loses every observation is not: it leaves the problem, test_emptied_camera_rig_among_healthy)
    sing = _vision(18, 90, models=("poly3", "poly3"))
    sing.set_flags(visual_mult=0.0)
    with pytest.raises(VcgpuError) as e:
        sing.covariance()
    assert "vcgpu error -3" in str(e.value)
    healthy = [_vision(18, 91), _inertial(90, 92)]
    gs = [healthy[0], sing, healthy[1]]
    bufs = [np.full((g.G, g.G), np.nan) for g in gs]
    from vicalib_b200.capi import covariance_batch

    with pytest.raises(VcgpuError) as e:
        covariance_batch(gs, out=bufs)
    assert "vcgpu error -3" in str(e.value) and "handle(s) 1" in str(e.value), str(e.value)
    assert e.value.status == [0, NUMERIC, 0]
    assert np.isnan(bufs[1]).all() and e.value.covariances[1] is None
    for i in (0, 2):
        _check_matrix(bufs[i], np.diag(bufs[i]) != 0)
        assert _corr_err(bufs[i], gs[i].covariance()) <= BAR[i == 2]


# ------------------------------------------------------------------ 7. a camera emptied by remove_outliers
def test_emptied_camera_rig_among_healthy():
    """Camera 1 loses every observation to vcgpu_remove_outliers: it is in no residual any more, so its blocks leave the
    problem (as Ceres removes them) and both entry points return VCGPU_OK, exact-zero rows and columns for it, and the
    dense inverse of the oracle's J^T J (which drops it the same way) elsewhere."""
    from oracle.binding import Oracle
    from vicalib_b200.capi import covariance_batch

    p = synth.make_problem(models=("poly3", "poly3"), n_frames=18, grid=(10, 7), seed=90)
    rmse = np.array([np.inf, 0.0])
    emptied = _vision(18, 90, models=("poly3", "poly3"))
    assert emptied.remove_outliers(rmse, 1.0) == int((p.obs_cam == 1).sum())
    o = Oracle(p)
    o.remove_outliers(rmse, 1.0)
    mask = o.global_mask()
    cam1 = np.arange(13, 26)
    assert mask[:13].any() and not mask[cam1].any()
    solo = emptied.covariance()
    healthy = [_vision(18, 91), _inertial(90, 92)]
    gs = [healthy[0], emptied, healthy[1]]
    covs = covariance_batch(gs)
    _check_matrix(covs[1], mask)
    assert not solo[cam1].any() and not solo[:, cam1].any()
    ref = _dense_cov(o)
    assert _corr_err(covs[1], ref) <= BAR[False] and _corr_err(solo, ref) <= BAR[False]
    for i in (0, 2):
        _check_matrix(covs[i], np.diag(covs[i]) != 0)
        assert _corr_err(covs[i], gs[i].covariance()) <= BAR[i == 2]
