"""GPU: vcgpu_get_imu_influence, the leverage, studentized residual and deletion influence of every IMU interval
(imu_eval_kernel into the call's buffers, infl_sgg_kernel, view_prior_kernel, imu_infl_kernel), against
tests/imu_influence_ref.py on the dense inverse of the oracle's J^T J at the state the device converged to.
  parity      poly3 and poly3 + kb4 with every IMU global free; bias / scale / ts off; rotation-only; fixed intrinsics;
              imu_mult = 2; weights after update_imu_weights; the imu_streams rigs partial (uncovered intervals: NaN),
              long_gap, jittered and tied; Unix-time stamps; vigorous motion; the kb4_poly3_inertial wide-lens rig; G = 67 and G = 68
  trace       sum tr(H_obs) + sum tr(H_imu) = the kept tangents, on the device's own combined output
  obs         the observation outputs of the same call are vcgpu_get_observation_influence's bits
  exact       H = I on the last interval when the last frame has no active corner (NaN stud and infl);
              VCGPU_ERR_NUMERIC with nothing written
  diagnosis   a gyro step in intervals 10 and 25 of a clean rig: the two largest stud fall there or next door
  handle      state, IMU weights and the bits of a following solve unchanged; null outputs and refusals; the C++
              method against the C-ABI"""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import chain_plan
import dense_cov
import imu_epoch
import imu_influence_ref as R
import imu_motion
import imu_streams
import test_cpu_imu_mahalanobis as TM
import wide_lenses as W
from test_gpu_frame_covariance import ALL_ON, NUMERIC
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu
INVALID = -1
ROT = dict(inertial=1, rotation_only=1, bias_active=0, scale_active=0, optimize_ts=1)


def _solved(p, flags, max_iters=15):
    """a handle solved from p with its IMU weights held at the identity (so it reaches a stationary point of one
    problem, as test_cpu_imu_influence.py's rigs), and the oracle at the state it converged to"""
    from oracle.binding import Oracle
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.load(p)
    g.set_flags(**flags)
    g.set_options(function_tol=1e-12, max_iters=max_iters, update_imu_weights=0)
    g.solve()
    st = g.state()
    p2 = dataclasses.replace(p, intr=st["intr"], q_ck=st["q_ck"], p_ck=st["p_ck"], T_wp=st["T_wp"], v_w=st["v_w"],
                             g=st["g"], b=st["b"], sf=st["sf"], ts=st["ts"])
    o = Oracle(p2, **flags)
    o.set_imu_weights(g.imu_weights())
    return g, o


def _device_sigma(g):
    """the device's own covariance blocks, assembled where the reference reads them; None where vcgpu_get_covariance
    refuses the rig (the velocities of a rotation-only run)"""
    from vicalib_b200.capi import VcgpuError

    try:
        Sgg = g.covariance()
    except VcgpuError:
        return None
    fg, fn = g.frame_cross_covariance()
    return R.assemble(g.n_frames, g.fd, Sgg, g.frame_covariance(), fg, fn)


def _rel(r, ref, k):
    ok = np.isfinite(ref["infl"]) & np.isfinite(r["infl"])
    return (np.abs(r[k][ok] - ref[k][ok]) / np.abs(ref[k][ok])).max(initial=0.0)


def _scaled(r, ref, k):
    ok = np.isfinite(ref[k]) & np.isfinite(r[k])
    sc = ref["sc_" + k][ok]
    e = np.abs(r[k][ok] - ref[k][ok])
    assert (e[sc == 0.0] == 0.0).all(), k  # exact zeros: the rows rotation-only runs drop
    return (e[sc > 0.0] / sc[sc > 0.0]).max(initial=0.0)


# Against the dense inverse of the oracle's J^T J and against the reference evaluated on the device's own Sigma blocks,
# all three are held to 1e-8 correlation-scaled (sc_* of imu_influence_ref, as influence_ref scales them).  The
# observation call's absolute bars on the device's own Sigma (h 1e-10, stud and infl 1e-8 relative) are not met by the
# intervals: measured on an H100 80GB HBM3 (700 W), h differs by up to 9.0e-10, stud by 7.0e-8 and infl by 5.3e-7.  The
# cause is the system, not the kernel: with every IMU global free the Jacobi-scaled J^T J has a condition number near
# 1e11, the Sigma blocks the three covariance calls return agree with the influence call's to that conditioning, and an
# interval's weighted rows are large (H is a difference of products of order 1e4), while stud and infl are amplified by
# 1 / lambda_min(I - H).  Those absolute errors are printed for the record.
CORR_BAR = 1e-8


def _clear(ref):
    """intervals the pivot test decides the same way on any rounding: empty ones, and those whose I - H has no
    eigenvalue within 1e-6 + 1e-8 max(sc_h) of 0.  A direction the interval alone fixes may fall either side of the test,
    and H is only as exact as the terms it cancels (sc_h, up to 1e9 on an interval next to a sparsely seen frame of the
    jittered stream, where H differs from the reference's by 3e-4 while lambda_min(I - H) is 3e-5)"""
    return np.array([not np.isfinite(x).all() or np.linalg.eigvalsh(np.eye(9) - x).min() > 1e-6 + 1e-8 * np.nanmax(sc)
                      for x, sc in zip(ref["h"], ref["sc_h"])])


def _same_nan(r, ref, c, k):
    bad = np.flatnonzero((np.isnan(r[k]) != np.isnan(ref[k])).reshape(len(c), -1).any(1) & c)
    for i in bad:
        lam = np.linalg.eigvalsh(np.eye(9) - ref["h"][i]).min() if np.isfinite(ref["h"][i]).all() else np.nan
        print(f"interval {i}: device {k} {r[k][i].ravel()[:3]}, reference {ref[k][i].ravel()[:3]}, lambda_min(I - H) {lam:.3e}, "
              f"|dh| {np.abs(r['h'][i] - ref['h'][i]).max():.3e}, r~ {np.abs(r['h'][i]).max():.3e}")
    assert len(bad) == 0, (k, bad)


def check(g, o, p, flags):
    r = g.imu_influence()
    im = flags.get("imu_mult", 1.0)
    Hd = _device_sigma(g)
    eh = es = ei = 0.0
    if Hd is not None:
        own = R.influence(o, Hd, p.models, im)
        c = _clear(own)
        for k in ("h", "stud", "infl"):
            _same_nan(r, own, c, k)
        eh = np.nanmax(np.abs(r["h"] - own["h"]), initial=0.0)
        es, ei = _rel(r, own, "stud"), _rel(r, own, "infl")
        oh, os_, oi = (_scaled(r, own, k) for k in ("h", "stud", "infl"))
        assert max(oh, os_, oi) <= CORR_BAR, (oh, os_, oi)
    live = 6 if flags.get("rotation_only") else o.fd
    Hi, _ = dense_cov.dense_inverse(o, np.ones(p.n_frames, bool), live)
    ref = R.influence(o, Hi, p.models, im)
    c = _clear(ref)
    for k in ("h", "stud", "infl"):
        _same_nan(r, ref, c, k)
    ch, cs, ci = (_scaled(r, ref, k) for k in ("h", "stud", "infl"))
    print(f"\n{p.n_frames} frames, G {g.G}, {int(np.isnan(r['stud']).sum())} NaN, {int((~c).sum())} near the pivot test: on the device's Sigma "
          f"{'(not taken) ' if Hd is None else ''}h {eh:.1e}, stud {es:.1e}, infl {ei:.1e}; vs the dense inverse, "
          f"correlation-scaled h {ch:.1e}, stud {cs:.1e}, infl {ci:.1e}")
    assert max(ch, cs, ci) <= CORR_BAR, (ch, cs, ci)
    if flags.get("rotation_only"):
        off = np.r_[0, 1, 2, 6, 7, 8]
        h = r["h"][np.isfinite(r["stud"])]
        assert (h[:, off, :] == 0.0).all() and (h[:, :, off] == 0.0).all()
    assert (r["h"] == np.swapaxes(r["h"], 1, 2))[np.isfinite(r["h"])].all()
    return r


def _stream(name):
    return imu_streams.build(name).p


CASES = {
    "poly3": lambda: (synth.make_problem(models=("poly3",), n_frames=60, inertial=True, seed=15), dict(ALL_ON)),
    "poly3_kb4": lambda: (synth.make_problem(models=("poly3", "kb4"), n_frames=60, inertial=True, seed=16), dict(ALL_ON)),
    "bias_scale_ts_off": lambda: (synth.make_problem(models=("poly3",), n_frames=50, inertial=True, seed=17),
                                  dict(ALL_ON, bias_active=0, scale_active=0, optimize_ts=0)),
    "rotation_only": lambda: (synth.make_problem(models=("poly3",), n_frames=50, inertial=True, seed=18), dict(ROT)),
    "fix_intrinsics": lambda: (synth.make_problem(models=("poly3", "fov"), n_frames=50, inertial=True, seed=19),
                               dict(ALL_ON, fix_intrinsics=1)),
    "imu_mult_2": lambda: (synth.make_problem(models=("kb4",), n_frames=50, inertial=True, seed=20), dict(ALL_ON, imu_mult=2.0)),
    "long_gap": lambda: (_stream("long_gap"), dict(ROT)),  # rotation-only: the gap leaves no velocity undetermined
    "partial": lambda: (_stream("partial"), dict(ROT)),
    "jittered": lambda: (_stream("jittered"), dict(ALL_ON)),
    "tied": lambda: (_stream("tied_ts"), dict(ROT)),
    "epoch": lambda: (imu_epoch.realistic("jittered").p, dict(ALL_ON)),
    "motion": lambda: (imu_motion.build("imu200").p, dict(ALL_ON)),
    "wide_lens": lambda: (W.build("kb4_poly3_inertial").p, W.build("kb4_poly3_inertial").flags),
}


@pytest.mark.parametrize("name", list(CASES))
def test_parity(name):
    p, flags = CASES[name]()
    g, o = _solved(p, flags)
    r = check(g, o, p, flags)
    if name == "partial":  # intervals the stream does not cover have no measurements
        empty = ~imu_streams.classify(p)["covered"]
        assert empty.any() and not empty.all()
        for k in ("h", "stud", "infl"):
            v = r[k].reshape(len(empty), -1)
            assert np.isnan(v[empty]).all() and np.isfinite(v[~empty]).all(), k


def test_updated_weights():
    """non-identity W: the weights update_imu_weights leaves, given to the oracle"""
    p = synth.make_problem(models=("poly3",), n_frames=50, inertial=True, seed=21)
    g, o = _solved(p, dict(ALL_ON))
    g.update_imu_weights()
    w = g.imu_weights()
    assert np.abs(w - np.eye(9)[None]).max() > 1e-3
    o.set_imu_weights(w)
    check(g, o, p, dict(ALL_ON))


@pytest.mark.parametrize("G", [67, 68])
def test_many_globals(G):
    p = synth.make_problem(models=chain_plan.rig_with_globals(G), n_frames=90, grid=(8, 6), inertial=True, seed=G)
    g, o = _solved(p, dict(ALL_ON))
    assert g.G == G
    check(g, o, p, dict(ALL_ON))


@pytest.mark.parametrize("flags", [dict(ALL_ON, bias_active=0, scale_active=0, optimize_ts=0), dict(ALL_ON)],
                         ids=["bias_scale_ts_off", "all_on"])
def test_trace_and_observations(flags):
    """sum tr(H_obs) + sum tr(H_imu) = 9 per frame + |F| on the device's own output; the observation outputs are the bits
    of vcgpu_get_observation_influence"""
    p = synth.make_problem(models=("poly3", "kb4"), n_frames=60, inertial=True, seed=29)
    g, _ = _solved(p, flags)
    r = g.imu_influence(observations=True)
    ob = g.observation_influence()
    assert all(r["observations"][k].tobytes() == ob[k].tobytes() for k in ob)
    act = g.obs_active() > 0
    keep = int((np.diag(g.covariance()) != 0).sum()) + 9 * p.n_frames
    tr = np.trace(r["h"], axis1=1, axis2=2).sum() + (ob["h"][act, 0] + ob["h"][act, 2]).sum()
    print(f"\nsum tr(H) {tr:.10f}, free tangents {keep}, relative {abs(tr - keep) / keep:.1e}")
    # 1e-8 relative; with every IMU global free the system is conditioned ~1e11 and the reference itself holds the
    # identity to 5.4e-8 (test_cpu_imu_influence.py), so 1e-6 there
    assert abs(tr - keep) <= (1e-6 if flags["bias_active"] else 1e-8) * keep, (tr, keep)


def test_last_frame_without_corners():
    """every corner of the last frame moved 50 px and removed: the last interval alone fixes that frame, so H = I, and
    the one before alone fixes the velocity of the frame between; both get NaN stud and infl"""
    from oracle.binding import Oracle
    from vicalib_b200.capi import Calibrator

    p = synth.make_problem(models=("poly3",), n_frames=40, inertial=True, seed=23)
    g, _ = _solved(p, dict(ALL_ON))
    st = g.state()
    pc = p.p_c.copy()
    last = p.obs_frame == p.n_frames - 1
    pc[last] += 50.0
    p2 = dataclasses.replace(p, p_c=pc, intr=st["intr"], q_ck=st["q_ck"], p_ck=st["p_ck"], T_wp=st["T_wp"], v_w=st["v_w"],
                             g=st["g"], b=st["b"], sf=st["sf"], ts=st["ts"])
    h = Calibrator()
    h.load(p2)
    h.set_flags(**ALL_ON)
    h.set_imu_weights(g.imu_weights())
    h.remove_outliers(np.array([1.0]), 5.0)
    act = h.obs_active()
    assert not act[last].any() and act[~last].all()
    r = h.imu_influence()
    assert np.abs(r["h"][-1] - np.eye(9)).max() < 1e-6, r["h"][-1]
    assert np.isnan(r["stud"][-2:]).all() and np.isnan(r["infl"][-2:]).all()
    assert np.isfinite(r["stud"][1:-2]).all()
    o = Oracle(p2, **ALL_ON)
    o.set_imu_weights(g.imu_weights())
    o.remove_outliers(np.array([1.0]), 5.0)
    check(h, o, p2, dict(ALL_ON))


def test_corrupted_gyro_intervals_stand_out():
    """a 0.05 rad/s step on the gyro samples inside intervals 10 and 25 of test_gpu_imu_mahalanobis.py's clean rig: the
    two largest stud fall in those intervals or their neighbours (a neighbour interpolates its end from a step sample)"""
    p = synth.make_problem(models=("poly3",), n_frames=40, grid=(10, 7), inertial=True, seed=5)
    p = TM._truth(p)
    bad = [10, 25]
    w = p.imu_w.copy()
    tt = p.imu_t + p.ts
    for k in bad:
        w[(tt > p.ftime[k]) & (tt < p.ftime[k + 1]), 2] += 0.05
    g, _ = _solved(dataclasses.replace(p, imu_w=w), dict(ALL_ON))
    s = g.imu_influence()["stud"]
    top = np.argsort(np.nan_to_num(s, nan=-1.0))[-2:]
    near = {j for k in bad for j in (k - 1, k, k + 1)}
    print(f"\nstud of intervals {bad}: {s[bad]}, largest at {sorted(top.tolist())}, median {np.nanmedian(s):.3g}")
    assert set(top.tolist()) <= near and {int(k) // 20 for k in top} == {0, 1}, top


def test_no_side_effects():
    p = synth.make_problem(models=("poly3",), n_frames=40, inertial=True, seed=24)
    g, _ = _solved(p, dict(ALL_ON), max_iters=4)
    s0, w0 = g.state(), g.imu_weights()
    a = g.imu_influence(observations=True)
    b = g.imu_influence(observations=True)
    assert all(a[k].tobytes() == b[k].tobytes() for k in ("h", "stud", "infl"))
    s1 = g.state()
    assert all(np.array_equal(s0[k], s1[k]) for k in s0) and np.array_equal(w0, g.imu_weights())
    from vicalib_b200.capi import Calibrator
    ref = Calibrator()
    ref.load(p)
    ref.set_flags(**ALL_ON)
    ref.set_options(function_tol=1e-12, max_iters=4, update_imu_weights=0)
    ref.solve()
    g.set_options(max_iters=3)
    ref.set_options(max_iters=3)
    g.solve()
    ref.solve()
    s2, s3 = g.state(), ref.state()
    assert all(np.asarray(s2[k]).tobytes() == np.asarray(s3[k]).tobytes() for k in s2)


def test_outputs_and_refusals():
    from vicalib_b200.capi import Calibrator, ImuInfluence, ObsInfluence

    p = synth.make_problem(models=("poly3",), n_frames=30, inertial=True, seed=25)
    g, _ = _solved(p, dict(ALL_ON))
    full = g.imu_influence()
    for h, s, i in [(True, False, False), (False, True, False), (False, False, True), (False, True, True)]:
        part = g.imu_influence(h=h, stud=s, infl=i)
        assert all(part[k].tobytes() == full[k].tobytes() for k in part)
    L = g.L
    none = ImuInfluence(None, None, None)
    assert L.vcgpu_get_imu_influence(g.h, None, None) == INVALID
    assert L.vcgpu_get_imu_influence(g.h, C.byref(none), None) == INVALID
    assert b"all null" in L.vcgpu_last_error(g.h)
    assert L.vcgpu_get_imu_influence(None, C.byref(none), None) == INVALID
    st = np.full(p.n_frames - 1, 7.0)
    one = ImuInfluence(None, st.ctypes.data, None)
    assert L.vcgpu_get_imu_influence(g.h, C.byref(one), C.byref(ObsInfluence(None, None, None))) == INVALID
    assert b"obs" in L.vcgpu_last_error(g.h)
    v = Calibrator()
    v.load(synth.make_problem(models=("poly3",), n_frames=12, seed=25))
    assert L.vcgpu_get_imu_influence(v.h, C.byref(one), None) == INVALID
    assert b"inertial" in L.vcgpu_last_error(v.h)
    assert (st == 7.0).all()
    s = Calibrator()
    s.load(p)
    s.set_flags(**dict(ALL_ON, visual_mult=0.0))
    hh = np.full((p.n_frames - 1, 81), np.nan)
    assert s.L.vcgpu_get_imu_influence(s.h, C.byref(ImuInfluence(hh.ctypes.data, None, None)), None) == NUMERIC
    assert np.isnan(hh).all()


def test_host_method(tmp_path):
    """ViCalibrator::GetImuInfluence against vcgpu_get_imu_influence on the same handle, through
    tests/cpp/imu_influence_main.cc: the same bits"""
    import os
    import subprocess

    from test_gpu_host_mirror import _write_problem

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "imu_influence")
    subprocess.run([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-Wall", "-o", exe,
                    os.path.join(root, "tests", "cpp", "imu_influence_main.cc"),
                    "-L" + os.path.join(root, "vicalib_b200"), "-lvcgpu", "-lpthread",
                    "-Wl,-rpath," + os.path.join(root, "vicalib_b200")], check=True, timeout=300)
    p = synth.make_problem(models=("poly3",), n_frames=24, inertial=True, seed=27)
    prob, res = str(tmp_path / "problem.bin"), str(tmp_path / "result.bin")
    _write_problem(prob, p, True, 15, 0)
    subprocess.run([exe, prob, res], check=True, timeout=600)
    out = np.fromfile(res, dtype=np.float64)
    n = int(out[:1].view(np.int64)[0])
    assert n == p.n_frames - 1 and len(out) == 1 + 2 * 83 * n
    a, b = out[1:1 + 83 * n], out[1 + 83 * n:]
    assert a.tobytes() == b.tobytes()
    assert np.isfinite(a).mean() > 0.9
