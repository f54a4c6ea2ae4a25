"""GPU: vcgpu_get_frame_cross_covariance_batch (one thread-block cluster per rig: cov_frame_cross_mega_batch_kernel for
vision rigs, chain_frame_cross_cov_batch_kernel for inertial rigs) against the dense inverse of the oracle's J^T J (the
frame call's correlation-scaled bars, 1e-6 vision and 1e-4 inertial) and against vcgpu_get_frame_cross_covariance on
the same handle (test_gpu_frame_covariance_batch.py's bars, 1e-8 vision and 1e-5 inertial: the two calls factor an
inertial system differently, and on systems conditioned near 1e11 after scaling they differ by a few 1e-6).  A rig's
cluster size is a function of the rig alone, so its blocks must not move, bit for bit, with the rest of the batch."""
import numpy as np
import pytest

import chain_plan
import target_views as tv
from dense_cov import corr_errors
from test_gpu_covariance_batch import _inertial, _same_solve, _snapshot, _vision
from test_gpu_frame_covariance import ALL_ON, NUMERIC, _solved
from test_gpu_frame_covariance_batch import MATCH_CASES, SOLO_BAR, _missing_cameras_rig
from test_gpu_frame_cross_covariance import check
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu


def _xcov_batch(gs):
    """frame_cross_covariance_batch that also returns the statuses: (blocks or None per rig, statuses)"""
    from vicalib_b200.capi import VcgpuError, frame_cross_covariance_batch

    try:
        return frame_cross_covariance_batch(gs), [0] * len(gs)
    except VcgpuError as e:
        if e.status is None:
            raise
        return e.covariances, e.status


def _bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def _vs_solo(g, fg, fn, sd_g=None):
    """the correlation-scaled distance of (fg, fn) from vcgpu_get_frame_cross_covariance on the same handle, the same
    exact zeros; scaled by the standard deviations of vcgpu_get_frame_covariance and sd_g (default: those of
    vcgpu_get_covariance, which a rotation-only rig does not have: its velocities are in no residual)"""
    sfg, sfn = g.frame_cross_covariance()
    assert np.array_equal(fg == 0.0, sfg == 0.0) and np.array_equal(fn == 0.0, sfn == 0.0)
    sd_f = np.sqrt(np.einsum("fii->fi", g.frame_covariance()))
    sd_g = np.sqrt(np.diag(g.covariance())) if sd_g is None else sd_g
    keep_f, keep_g = sd_f > 0, sd_g > 0
    return corr_errors(fg, fn, sfg, sfn, np.where(keep_f, sd_f, 1.0), np.where(keep_g, sd_g, 1.0), keep_f, keep_g)


# ------------------------------------------------------------------ 1. parity: the per-handle cases in one mixed call
def test_parity_mixed_batch():
    from vicalib_b200.capi import frame_cross_covariance_batch

    rigs = []  # (handle, oracle, inertial, used)
    for models, inertial, flags in MATCH_CASES:
        p = synth.make_problem(models=models, n_frames=90 if inertial else 18, inertial=inertial, seed=15)
        rigs.append((*_solved(p, flags), inertial, None))
    v = tv.build("unseen_runs")
    rigs.append((*_solved(v.p, v.flags), False, tv.counts(v.p).sum(0) > 0))
    v = tv.build("unseen_camera_inertial")
    rigs.append((*_solved(v.p, v.flags), True, None))
    rigs.append((*_solved(_missing_cameras_rig(), dict(ALL_ON)), True, None))
    outs = frame_cross_covariance_batch([r[0] for r in rigs])
    worst = {False: 0.0, True: 0.0}
    for (g, o, inertial, used), (fg, fn) in zip(rigs, outs):
        *_, sd_g = check(g, o, inertial, fg, fn, used)
        e = max(_vs_solo(g, fg, fn, sd_g))
        worst[inertial] = max(worst[inertial], e)
        assert e <= SOLO_BAR[inertial], e
    print(f"\nvs vcgpu_get_frame_cross_covariance: vision {worst[False]:.1e}, inertial {worst[True]:.1e}")


# ------------------------------------------------------------------ 2. bits: alone, mixed, reversed, with clusters queued
def _shape_rigs(seed):
    return [_vision(18, seed), _vision(60, seed + 1, models=("poly3", "kb4")), _vision(300, seed + 2),
            _inertial(24, seed + 3), _inertial(90, seed + 4), _inertial(600, seed + 5, grid=(8, 6)),
            _inertial(48, seed + 6, models=chain_plan.rig_with_globals(67), grid=(14, 10))]


def test_bits_whatever_the_batch():
    rigs = _shape_rigs(400)
    n = len(rigs)
    alone = [_xcov_batch([g]) for g in rigs]
    alone = [(c[0], s[0]) for c, s in alone]
    mixed, st = _xcov_batch(rigs)
    rev, st_r = _xcov_batch(rigs[::-1])
    for i, (c0, s0) in enumerate(alone):
        assert st[i] == s0 and st_r[n - 1 - i] == s0
        assert _bits(mixed[i], c0), f"rig {i}: mixed batch"
        assert _bits(rev[n - 1 - i], c0), f"rig {i}: reversed"
    print(f"\nbits: statuses {[s for _, s in alone]}")
    # more rigs than the device holds clusters of at once: the last ones queue behind the first
    resident = rigs[3].batch_plan_inertial()[1]
    many = [rigs[3]] + [_inertial(24, 900 + k) for k in range(resident)] + [rigs[0]]
    outs, sts = _xcov_batch(many)
    assert sts[0] == alone[3][1] and sts[-1] == alone[0][1]
    assert _bits(outs[0], alone[3][0]) and _bits(outs[-1], alone[0][0])
    again, _ = _xcov_batch(many[1:3])
    assert _bits(again[0], outs[1]) and _bits(again[1], outs[2])


# ------------------------------------------------------------------ 3. the handles are left as they were
def test_no_side_effects():
    from vicalib_b200.capi import frame_cross_covariance_batch

    def make():
        return [_vision(20, 61), _vision(40, 62, models=("poly3", "kb4")), _inertial(40, 63), _inertial(90, 64)]

    rigs, fresh = make(), make()
    before = [_snapshot(g) for g in rigs]
    frame_cross_covariance_batch(rigs)
    assert [_snapshot(g) for g in rigs] == before
    for g, f in zip(rigs, fresh):
        assert g.frame_covariance().tobytes() == f.frame_covariance().tobytes()
        _same_solve(g.solve(free_running=True), f.solve(free_running=True), g.state(), f.state())


# ------------------------------------------------------------------ 4. the station: staged calibration, then this call
def test_station_flow():
    from vicalib_b200.capi import calibrate_batch, frame_cross_covariance_batch

    gs = []
    for i in range(4):
        g = _inertial(90, 80 + i, models=("poly3",) if i % 2 else ("poly3", "poly2"), grid=(14, 10))
        g.set_options(function_tol=1e-12, max_iters=15)
        gs.append(g)
    calibrate_batch(gs, remove_outliers=False)
    outs = frame_cross_covariance_batch(gs)
    for g, (fg, fn) in zip(gs, outs):
        inertial = bool(g.flags.inertial)
        e = max(_vs_solo(g, fg, fn))
        print(f"\nstation rig (inertial {inertial}): vs vcgpu_get_frame_cross_covariance {e:.1e}")
        assert e <= SOLO_BAR[inertial], e


# ------------------------------------------------------------------ 5. failures: a singular rig among healthy ones, refusals
def test_singular_rig_among_healthy():
    from vicalib_b200.capi import VcgpuError, frame_cross_covariance_batch

    sing = _vision(18, 90, models=("poly3", "poly3"))
    sing.set_flags(visual_mult=0.0)  # every reprojection residual weighted 0: J^T J is singular
    gs = [_vision(18, 91), sing, _inertial(90, 92)]
    with pytest.raises(VcgpuError) as e:
        frame_cross_covariance_batch(gs)
    assert "vcgpu error -3" in str(e.value) and "handle(s) 1" in str(e.value), str(e.value)
    assert e.value.status == [0, NUMERIC, 0]
    assert e.value.covariances[1] is None
    for i in (0, 2):
        fg, fn = e.value.covariances[i]
        assert max(_vs_solo(gs[i], fg, fn)) <= SOLO_BAR[i == 2]


def test_singular_rig_writes_nothing():
    import ctypes as C

    from vicalib_b200.capi import lib

    sing = _vision(18, 93, models=("poly3", "poly3"))
    sing.set_flags(visual_mult=0.0)
    fg, fn = np.full((18, 6, sing.G), np.nan), np.full((17, 6, 6), np.nan)
    hs = (C.c_void_p * 1)(sing.h)
    pg, pn = (C.c_void_p * 1)(fg.ctypes.data), (C.c_void_p * 1)(fn.ctypes.data)
    status = (C.c_int * 1)()
    assert lib().vcgpu_get_frame_cross_covariance_batch(hs, 1, pg, pn, status) == NUMERIC
    assert status[0] == NUMERIC and np.isnan(fg).all() and np.isnan(fn).all()


def test_refusals():
    """vcgpu_get_frame_covariance_batch's refusals, each naming the index; nothing is written and nothing runs"""
    import ctypes as C

    from vicalib_b200.capi import lib

    L = lib()

    def refused(gs, index, fg=True, fn=True, null_rig=None):
        n = len(gs)
        bg = [None if g is None else np.full((g.n_frames, g.fd, g.G), np.nan) for g in gs]
        bn = [None if g is None else np.full((g.n_frames - 1, g.fd, g.fd), np.nan) for g in gs]
        if null_rig is not None:
            bg[null_rig] = bn[null_rig] = None
        hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in gs])
        pg = (C.c_void_p * max(n, 1))(*[None if a is None else a.ctypes.data for a in bg]) if fg else None
        pn = (C.c_void_p * max(n, 1))(*[None if a is None else a.ctypes.data for a in bn]) if fn else None
        assert L.vcgpu_get_frame_cross_covariance_batch(hs, C.c_int(n), pg, pn, None) == -1
        if index is not None:
            msg = next(L.vcgpu_last_error(g.h).decode() for g in gs if g is not None)
            assert f"handle {index}:" in msg, msg
        for b in bg + bn:
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
    refused([], None)                                   # n = 0
    refused([good[0], good[1], None], 2)                # a null handle
    refused([None, good[0]], 0)
    refused([good[0], good[1], good[0]], 2)             # a repeated handle
    refused(good, 1, null_rig=1)                        # both pointers of a rig null
    refused(good, 0, fg=False, fn=False)                # both arrays null
    for b in bads:
        refused([good[0], good[1], b], 2)
        refused([b, good[0], good[1]], 0)
    # one array null: the other is written, the same bits as both
    from vicalib_b200.capi import frame_cross_covariance_batch

    both = frame_cross_covariance_batch(good)
    g0 = good[0]
    fg = np.zeros((g0.n_frames, g0.fd, g0.G))
    hs = (C.c_void_p * 1)(g0.h)
    assert L.vcgpu_get_frame_cross_covariance_batch(hs, 1, (C.c_void_p * 1)(fg.ctypes.data), None, None) == 0
    assert fg.tobytes() == both[0][0].tobytes()
    for g, f in zip(good, fresh):
        _same_solve(g.solve(free_running=True), f.solve(free_running=True), g.state(), f.state())
