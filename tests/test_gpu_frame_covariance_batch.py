"""GPU: vcgpu_get_frame_covariance_batch (one thread-block cluster per rig: cov_frame_mega_batch_kernel for vision rigs,
chain_frame_cov_batch_kernel for inertial rigs) against the frame blocks of the dense inverse of the oracle's J^T J
(test_gpu_frame_covariance.py's correlation-scaled bars: 1e-6 vision, 1e-4 inertial) and against
vcgpu_get_frame_covariance on the same handle (1e-8 vision, 1e-5 inertial: the two calls factor an inertial system
differently, the multi-launch elimination and a Cholesky against the cluster's elimination and an L D L^T, and on
systems conditioned near 1e11 after scaling they differ by a few 1e-6, as much as either differs from the dense
inverse).  A rig's cluster size is a function of the rig alone, so its blocks must not move, bit for bit, with the rest
of the batch.  Not covered: handles on different devices and frame-sharded handles (both need more than one GPU); their
refusals are the argument checks of vcgpu_get_covariance_batch."""
import numpy as np
import pytest

import chain_plan
import target_views as tv
from test_gpu_covariance_batch import _bits, _inertial, _same_solve, _snapshot, _vision
from test_gpu_frame_covariance import ALL_ON, BAR, LEVEL_CASES, NUMERIC, _dense_frame_cov, _solved
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

SOLO_BAR = {False: 1e-8, True: 1e-5}


def _fcov_batch(gs, out=None):
    """frame_covariance_batch that also returns the statuses: (blocks or None, statuses)"""
    from vicalib_b200.capi import VcgpuError, frame_covariance_batch

    try:
        return frame_covariance_batch(gs, out=out), [0] * len(gs)
    except VcgpuError as e:
        if e.status is None:
            raise
        return e.covariances, e.status


def _corr(cov, ref, keep):
    """largest error of the kept blocks relative to the two standard deviations of ref"""
    sd = np.sqrt(np.einsum("fii->fi", ref[keep]))
    assert np.all(sd > 0)
    return float((np.abs(cov[keep] - ref[keep]) / (sd[:, :, None] * sd[:, None, :])).max())


def _check(g, o, inertial, cov, used=None):
    """one rig's blocks of a batch: exactly symmetric, exact zeros where vcgpu_get_frame_covariance has them, and within
    the bars of the dense inverse and of vcgpu_get_frame_covariance"""
    nf, fd = g.n_frames, 9 if inertial else 6
    used = np.ones(nf, bool) if used is None else used
    live = 6 if inertial and g.flags.rotation_only else fd
    assert cov.shape == (nf, fd, fd)
    assert np.array_equal(cov, cov.transpose(0, 2, 1))
    assert not cov[~used].any() and not cov[:, live:].any()
    solo = g.frame_covariance()
    assert np.all(cov[solo == 0.0] == 0.0)
    ref = _dense_frame_cov(o, used, live)[:, :live, :live]
    e_dense = _corr(cov[:, :live, :live], ref, used)
    e_solo = _corr(cov[:, :live, :live], solo[:, :live, :live], used)
    print(f"\n{nf} frames, fd {fd}, G {g.G}: vs dense inverse {e_dense:.1e}, vs vcgpu_get_frame_covariance {e_solo:.1e}")
    assert e_dense <= BAR[inertial], e_dense
    assert e_solo <= SOLO_BAR[inertial], e_solo


# ------------------------------------------------------------------ 1. parity, every case of the per-handle tests in one call
MATCH_CASES = [
    (("poly3",), False, {}),
    (("fov", "kb4"), False, {}),
    (("poly3", "poly2"), True, dict(ALL_ON)),
    (("poly3",), True, dict(inertial=1, rotation_only=1, bias_active=0, scale_active=0, optimize_ts=1)),
    (("poly3", "fov"), False, dict(fix_intrinsics=1)),
    (("kb4",), True, dict(ALL_ON, fix_intrinsics=1)),
]


def _missing_cameras_rig():
    """test_inertial_frames_missing_cameras' rig: a chunk no camera sees and a run one camera of two sees"""
    p = synth.make_problem(models=("poly3", "poly3"), n_frames=90, grid=(10, 7), inertial=True, seed=45)
    c = chain_plan.CHUNK
    gone = ((p.obs_frame >= 40) & (p.obs_frame < 40 + c)) | ((p.obs_frame >= 60) & (p.obs_frame < 76) & (p.obs_cam == 1))
    return tv.keep(p, ~gone)


def test_parity_mixed_batch():
    from vicalib_b200.capi import frame_covariance_batch

    rigs = []  # (handle, oracle, inertial, used)
    for models, inertial, flags in MATCH_CASES:
        p = synth.make_problem(models=models, n_frames=90 if inertial else 18, inertial=inertial, seed=15)
        rigs.append((*_solved(p, flags), inertial, None))
    v = tv.build("unseen_runs")
    rigs.append((*_solved(v.p, v.flags), False, tv.counts(v.p).sum(0) > 0))
    v = tv.build("unseen_camera_inertial")
    rigs.append((*_solved(v.p, v.flags), True, None))
    rigs.append((*_solved(_missing_cameras_rig(), dict(ALL_ON)), True, None))
    covs = frame_covariance_batch([r[0] for r in rigs])
    for (g, o, inertial, used), cov in zip(rigs, covs):
        _check(g, o, inertial, cov, used)


# ------------------------------------------------------------------ 2. the level shapes and G = 67 in one call; G = 68 refused
def test_level_shapes_batched():
    from vicalib_b200.capi import VcgpuError, frame_covariance_batch

    rigs = []
    for nf in LEVEL_CASES:
        p = synth.make_problem(models=("poly3",), n_frames=nf, grid=(8, 6), inertial=True, seed=100 + nf,
                               frame_rate=min(30.0, nf / 3.0))
        rigs.append(_solved(p, dict(ALL_ON)))
    p = synth.make_problem(models=chain_plan.rig_with_globals(67), n_frames=90, grid=(8, 6), inertial=True, seed=67)
    rigs.append(_solved(p, dict(ALL_ON)))
    assert rigs[-1][0].G == 67
    covs = frame_covariance_batch([g for g, _ in rigs])
    for (g, o), cov in zip(rigs, covs):
        _check(g, o, True, cov)
    g68 = _inertial(24, 68, models=chain_plan.rig_with_globals(68), grid=(14, 10))
    assert g68.G == 68
    with pytest.raises(VcgpuError) as e:
        frame_covariance_batch([rigs[0][0], g68])
    assert "vcgpu error -1" in str(e.value) and "handle 1:" in str(e.value), str(e.value)


# ------------------------------------------------------------------ 3. bits: alone, mixed, reversed, with clusters queued
def _shape_rigs(seed):
    return [_vision(18, seed), _vision(60, seed + 1, models=("poly3", "kb4")), _vision(300, seed + 2),
            _inertial(24, seed + 3), _inertial(90, seed + 4), _inertial(600, seed + 5, grid=(8, 6)),
            _inertial(48, seed + 6, models=chain_plan.rig_with_globals(67), grid=(14, 10))]


def test_bits_whatever_the_batch():
    rigs = _shape_rigs(400)
    n = len(rigs)
    alone = [_fcov_batch([g]) for g in rigs]
    alone = [(c[0], s[0]) for c, s in alone]
    mixed, st = _fcov_batch(rigs)
    rev, st_r = _fcov_batch(rigs[::-1])
    for i, (c0, s0) in enumerate(alone):
        assert st[i] == s0 and st_r[n - 1 - i] == s0
        assert _bits(mixed[i], c0), f"rig {i}: mixed batch"
        assert _bits(rev[n - 1 - i], c0), f"rig {i}: reversed"
    print(f"\nbits: statuses {[s for _, s in alone]}")
    # more rigs than the device holds clusters of at once: the last ones queue behind the first
    resident = rigs[3].batch_plan_inertial()[1]
    many = [rigs[3]] + [_inertial(24, 900 + k) for k in range(resident)] + [rigs[0]]
    covs, sts = _fcov_batch(many)
    assert sts[0] == alone[3][1] and sts[-1] == alone[0][1]
    assert _bits(covs[0], alone[3][0]) and _bits(covs[-1], alone[0][0])
    again, _ = _fcov_batch(many[1:3])
    assert _bits(again[0], covs[1]) and _bits(again[1], covs[2])


# ------------------------------------------------------------------ 4. the handles are left as they were
def test_no_side_effects():
    from vicalib_b200.capi import frame_covariance_batch, solve_batch_inertial

    def make():
        return [_vision(20, 61), _vision(40, 62, models=("poly3", "kb4")), _inertial(40, 63), _inertial(90, 64)]

    rigs, fresh = make(), make()
    for g in rigs:  # options the call ignores
        g.set_options(update_state_every_iteration=1, max_iters=3)
    rigs[0].set_options(strategy=1)
    rigs[2].set_options(strategy=1)
    before = [_snapshot(g) for g in rigs]
    frame_covariance_batch(rigs)
    assert [_snapshot(g) for g in rigs] == before
    for g in rigs + fresh:
        g.set_options(update_state_every_iteration=0, strategy=0, max_iters=6)
    for g, f in zip(rigs, fresh):
        _same_solve(g.solve(free_running=True), f.solve(free_running=True), g.state(), f.state())
    for g, f in zip(rigs[2:], fresh[2:]):
        assert np.array_equal(g.imu_weights(), f.imu_weights())
    # the batch inertial solve, too (sync-word parity), after a second call
    frame_covariance_batch(rigs)
    sums, sums0 = solve_batch_inertial(rigs[2:]), solve_batch_inertial(fresh[2:])
    for g, f, s, s0 in zip(rigs[2:], fresh[2:], sums, sums0):
        _same_solve(s, s0, g.state(), f.state())
        assert np.array_equal(g.imu_weights(), f.imu_weights())


# ------------------------------------------------------------------ 5. the station: batch solve, covariance, frame covariance
def test_station_flow():
    from vicalib_b200.capi import covariance_batch, frame_covariance_batch, solve_batch_inertial

    def make():
        out = []
        for i in range(4):
            g = _inertial(90, 80 + i, models=("poly3",) if i % 2 else ("poly3", "poly2"), grid=(14, 10))
            g.set_options(function_tol=1e-12, max_iters=15)
            out.append(g)
        return out

    batch, solo = make(), make()
    solve_batch_inertial(batch)
    covariance_batch(batch)
    fcovs = frame_covariance_batch(batch)
    for g, fcov in zip(solo, fcovs):
        g.solve(free_running=True)
        g.covariance()
        ref = g.frame_covariance()
        err = _corr(fcov, ref, np.ones(g.n_frames, bool))
        print(f"\nstation rig: vs vcgpu_solve + vcgpu_get_frame_covariance {err:.1e}")
        assert err <= BAR[True]


# ------------------------------------------------------------------ 6. failures: a singular rig among healthy ones, refusals
def test_singular_rig_among_healthy():
    from vicalib_b200.capi import VcgpuError, frame_covariance_batch

    # every reprojection residual weighted 0: the frames' columns are empty, so J^T J is singular
    sing = _vision(18, 90, models=("poly3", "poly3"))
    sing.set_flags(visual_mult=0.0)
    healthy = [_vision(18, 91), _inertial(90, 92)]
    gs = [healthy[0], sing, healthy[1]]
    bufs = [np.full((g.n_frames, g.fd, g.fd), np.nan) for g in gs]
    with pytest.raises(VcgpuError) as e:
        frame_covariance_batch(gs, out=bufs)
    assert "vcgpu error -3" in str(e.value) and "handle(s) 1" in str(e.value), str(e.value)
    assert e.value.status == [0, NUMERIC, 0]
    assert np.isnan(bufs[1]).all() and e.value.covariances[1] is None
    for i in (0, 2):
        ref = gs[i].frame_covariance()
        assert np.array_equal(bufs[i], bufs[i].transpose(0, 2, 1))
        assert _corr(bufs[i], ref, np.ones(gs[i].n_frames, bool)) <= SOLO_BAR[i == 2]


def test_refusals():
    from vicalib_b200.capi import VcgpuError, frame_covariance_batch

    def refused(gs, index, out=None):
        bufs = out if out is not None else [None if g is None else np.full((g.n_frames, g.fd, g.fd), np.nan) for g in gs]
        with pytest.raises(VcgpuError) as e:
            frame_covariance_batch(gs, out=bufs)
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

    specs = [("vision", dict(profiling=p)) for p in (1, 4, 8)] + [("inertial", dict(profiling=p)) for p in (1, 4, 8)]
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
    bufs = [np.full((g.n_frames, g.fd, g.fd), np.nan) for g in good]
    refused(good, 1, out=[bufs[0], None])                      # a null cov pointer
    assert np.isnan(bufs[0]).all()
    for b in bads:
        refused([good[0], good[1], b], 2)
        refused([b, good[0], good[1]], 0)
    # nothing ran: the handles solve as fresh ones do
    for g, f in zip(good, fresh):
        _same_solve(g.solve(free_running=True), f.solve(free_running=True), g.state(), f.state())
