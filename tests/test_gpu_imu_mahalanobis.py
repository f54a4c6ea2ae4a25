"""GPU: vcgpu_get_imu_mahalanobis(_batch), each IMU interval's Mahalanobis distance as UpdateImuWeights logs it
(vicalibrator.h:786-794), computed by imu_mahalanobis_kernel from the weight update's covariance chain and a cold-started
Jacobi eigen-decomposition.
  parity     d against the oracle's UpdateOneImuWeight and the reference's own ref_update_weight, r against the oracle, on
             the problems of test_cpu_imu_mahalanobis.py; NaN exactly where nothing is measured
  no effect  weights, state and a following solve are the bits they would have been without the call; the call's bits
             do not depend on the weight history or the flags
  diagnosis  a gyro step in a few intervals of a clean rig stands out
  batch      the bits of the per-handle calls in any order and subset; refusals name the index and write nothing
Single-step intervals are not compared (their P has rank <= 6: test_cpu_imu_mahalanobis.py)."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import imu_mahalanobis_ref as M
import test_cpu_imu_mahalanobis as T
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
# Bars measured on an H100 80GB HBM3 (700 W).  d against the oracle and the reference, relative to d: largest 1.3e-10
# (stream imu20, cond(P) up to 4.3e5), 6.3e-10 at the true state (base_truth, d of order ten); r against the oracle,
# relative to the interval's max |r|: largest 1.4e-11 (base_truth), 3.5e-14 elsewhere.  Each bar leaves a factor of 7 to 16.
D_BAR, D_TRUTH_BAR, R_BAR = 1e-9, 1e-8, 1e-10


def _calibrator(p, **flags):
    from vicalib_b200.capi import Calibrator

    g = Calibrator(device=0)
    g.load(p)
    g.set_flags(**(flags or ALL_ON))
    return g


@pytest.fixture(scope="module")
def ref():
    return M.ref_lib()  # None where oracle/_ref was not built: the oracle alone is compared


@pytest.mark.parametrize("name", list(T.CASES))
def test_parity(ref, name):
    p = T.CASES[name]
    g = _calibrator(p)
    d, r = g.imu_mahalanobis(residuals=True)
    cmp, covered = T._comparable(p)
    assert np.isnan(d[~covered]).all() and np.isnan(r[~covered]).all(), name
    assert np.isfinite(d[cmp]).all() and np.isfinite(r[covered]).all(), name
    if not cmp.any():
        return
    d_o = M.oracle_dist(p)
    bar = D_TRUTH_BAR if name.endswith("_truth") else D_BAR
    rel_o = np.abs(d[cmp] - d_o[cmp]) / np.abs(d_o[cmp])
    rel_r = 0.0
    if ref is not None:
        d_r = M.ref_dist(ref, p)
        rel_r = (np.abs(d[cmp] - d_r[cmp]) / np.abs(d_r[cmp])).max()
    rel_res = 0.0
    for k in np.flatnonzero(covered):
        _P, r_o, _m = M.oracle_interval(p, k)
        rel_res = max(rel_res, np.abs(r[k] - r_o).max() / np.abs(r_o).max())
    print(f"{name}: d vs oracle {rel_o.max():.2e}, vs reference {rel_r:.2e}; r vs oracle {rel_res:.2e}")
    assert rel_o.max() <= bar and rel_r <= bar and rel_res <= R_BAR, (name, rel_o.max(), rel_r, rel_res)


def _solve(g, iters):
    g.set_options(max_iters=iters, function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
    return g.solve()


def _state_bits(g):
    return b"".join(v.tobytes() if isinstance(v, np.ndarray) else np.float64(v).tobytes() for v in g.state().values())


def test_no_side_effects():
    """weights and state bits unchanged by the call, and a following solve gives the rows and state bits of a handle
    that never made it"""
    p = T.CASES["stream_jittered"]
    a, b = _calibrator(p), _calibrator(p)
    _solve(a, 3)
    _solve(b, 3)
    W0, S0 = a.imu_weights(), _state_bits(a)
    a.imu_mahalanobis(residuals=True)
    assert a.imu_weights().tobytes() == W0.tobytes() and _state_bits(a) == S0
    sa, sb = _solve(a, 4), _solve(b, 4)
    assert sa["rows"].tobytes() == sb["rows"].tobytes() and sa["final_cost"] == sb["final_cost"]
    assert _state_bits(a) == _state_bits(b) and a.imu_weights().tobytes() == b.imu_weights().tobytes()


def test_same_bits_after_set_or_after_a_solve():
    """the call's bits depend on the state alone: right after set_* at a solved state, after the solve that reached it
    (with its weight history), and with rotation_only set, which the distance does not read"""
    p = T.CASES["motion_imu400"]
    a = _calibrator(p)
    _solve(a, 4)
    s = a.state()
    da, ra = a.imu_mahalanobis(residuals=True)
    q = dataclasses.replace(p, T_wp=s["T_wp"], v_w=s["v_w"], g=s["g"], b=s["b"], sf=s["sf"], ts=s["ts"])
    for flags in (ALL_ON, dict(ALL_ON, rotation_only=1)):
        b = _calibrator(q, **flags)
        db, rb = b.imu_mahalanobis(residuals=True)
        assert db.tobytes() == da.tobytes() and rb.tobytes() == ra.tobytes(), flags


def _clean_rig():
    p = synth.make_problem(models=("poly3",), n_frames=40, grid=(10, 7), inertial=True, seed=5)
    return T._truth(p)


def test_corrupted_gyro_intervals_stand_out():
    """a 0.05 rad/s step on the gyro samples inside intervals 10 and 25 of a clean rig: their distances exceed 16.919 and
    100 x the median of the intervals whose samples are untouched"""
    p = _clean_rig()
    d0 = _calibrator(p).imu_mahalanobis()
    print(f"clean rig: {np.mean(d0 > M.CHI2_95_9):.3f} of {len(d0)} intervals above {M.CHI2_95_9} (observation), "
          f"median {np.median(d0):.2f}")
    bad = [10, 25]
    w = p.imu_w.copy()
    tt = p.imu_t + p.ts
    for k in bad:
        w[(tt > p.ftime[k]) & (tt < p.ftime[k + 1]), 2] += 0.05
    d = _calibrator(dataclasses.replace(p, imu_w=w)).imu_mahalanobis()
    near = {j for k in bad for j in (k - 1, k, k + 1)}  # a neighbour interpolates its end from a step sample
    clean = np.array([k for k in range(len(d)) if k not in near])
    med = np.median(d[clean])
    print(f"corrupted: {d[bad]}, median of the untouched {med:.2f}")
    assert np.all(d[bad] > M.CHI2_95_9) and np.all(d[bad] > 100 * med)


def _raw_batch(gs, r_mask, sentinel=None):
    """vcgpu_get_imu_mahalanobis_batch with r[i] NULL where not r_mask[i]: (rc, d per rig, r per rig or None)"""
    from vicalib_b200.capi import lib

    ni = [max(g.n_frames - 1, 1) if g is not None else 1 for g in gs]
    fill = np.nan if sentinel is None else sentinel
    d = [np.full(k, fill) for k in ni]
    r = [np.full((k, 9), fill) if m else None for k, m in zip(ni, r_mask)]
    n = len(gs)
    hs = (C.c_void_p * max(n, 1))(*[None if g is None else g.h for g in gs])
    dp = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in d])
    rp = (C.c_void_p * max(n, 1))(*[None if a is None else a.ctypes.data for a in r])
    rc = lib().vcgpu_get_imu_mahalanobis_batch(hs, C.c_int(n), dp, rp)
    return rc, d, r


def _batch_rigs():
    ps = [T.CASES[k] for k in ("base", "stream_jittered", "motion_imu400", "epoch_dropped", "stream_samples2")]
    ps.append(synth.make_problem(models=("poly3",), n_frames=131, grid=(8, 6), inertial=True, seed=9))
    return [_calibrator(p) for p in ps]


def test_batch_bits_match_per_handle():
    from vicalib_b200.capi import imu_mahalanobis_batch

    gs = _batch_rigs()
    solo = [g.imu_mahalanobis(residuals=True) for g in gs]
    orders = [list(range(len(gs))), list(reversed(range(len(gs)))), [3, 1], [5], [2, 0, 4]]
    for order in orders:
        sub = [gs[i] for i in order]
        for i, (d, r) in zip(order, imu_mahalanobis_batch(sub, residuals=True)):
            assert d.tobytes() == solo[i][0].tobytes() and r.tobytes() == solo[i][1].tobytes(), (order, i)
        mask = [j % 2 == 0 for j in range(len(sub))]
        rc, d, r = _raw_batch(sub, mask)
        assert rc == 0
        for j, i in enumerate(order):
            assert d[j].tobytes() == solo[i][0].tobytes(), (order, i)
            if mask[j]:
                assert r[j].tobytes() == solo[i][1].tobytes(), (order, i)


def test_refusals_name_the_index_and_write_nothing():
    from vicalib_b200.capi import VcgpuError, imu_mahalanobis_batch, lib

    gs = _batch_rigs()[:3]
    off = _calibrator(T.CASES["base"], inertial=0)
    p = T.CASES["base"]
    one = _calibrator(p)
    one.set_frames(p.T_wp[:1], p.v_w[:1], p.ftime[:1])
    with pytest.raises(VcgpuError, match="inertial terms are off"):
        off.imu_mahalanobis()
    with pytest.raises(VcgpuError, match="fewer than two frames"):
        one.imu_mahalanobis()
    for rigs, index, why in (([gs[0], off, gs[1]], 1, "the inertial terms are off"),
                             ([gs[0], gs[1], one], 2, "fewer than two frames"),
                             ([gs[0], gs[1], gs[0]], 2, "the same handle as 0"),
                             ([gs[0], None, gs[1]], 1, "null handle")):
        rc, d, r = _raw_batch(rigs, [True] * len(rigs), sentinel=-7.0)
        assert rc == -1
        assert all((a == -7.0).all() for a in d) and all((a == -7.0).all() for a in r)
        msg = lib().vcgpu_last_error(gs[0].h).decode()
        assert f"handle {index}: {why}" in msg, msg
        with pytest.raises(VcgpuError, match=f"handle {index}:"):
            imu_mahalanobis_batch(rigs)
    # a null dist entry
    hs = (C.c_void_p * 2)(gs[0].h, gs[1].h)
    keep = np.full(gs[0].n_frames - 1, -7.0)
    dp = (C.c_void_p * 2)(keep.ctypes.data, None)
    assert lib().vcgpu_get_imu_mahalanobis_batch(hs, C.c_int(2), dp, None) == -1
    assert "handle 1: null dist pointer" in lib().vcgpu_last_error(gs[0].h).decode() and (keep == -7.0).all()
    assert lib().vcgpu_get_imu_mahalanobis_batch(hs, C.c_int(0), dp, None) == -1
