"""GPU: vcgpu_get_observation_influence, the leverage, studentized residual and deletion influence of every
reprojection observation (view_prior_kernel, infl_q_kernel, infl_obs_kernel), against tests/influence_ref.py on the
dense inverse of the oracle's J^T J at the state the device converged to.
  parity      five models, vision and inertial, rotation-only, fix_intrinsics, removed outliers (the inactive path),
              two wide-lens rigs, inertial G = 67 and G = 68 (the single call takes rigs the cluster kernels do not fit)
  trace       sum of tr(H_i) over the active observations = 6 per used frame + |F| on vision rigs, a config-2-sized
              rig included
  exact       NaN for a camera whose observations were all removed; VCGPU_ERR_NUMERIC with nothing written; a view
              left with 3 active corners has H_i = I on them
  handle      state, IMU weights and the bits of a following solve unchanged; null outputs and refusals"""
import dataclasses

import numpy as np
import pytest

import chain_plan
import dense_cov
import influence_ref as R
import wide_lenses as W
from test_gpu_frame_covariance import ALL_ON, NUMERIC, _solved
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu
INVALID = -1


def _frame_used(p, act):
    return np.bincount(p.obs_frame[act > 0], minlength=p.n_frames) > 0


def _ref(g, o, p, inertial, flags, Hi=None):
    """the reference on the dense inverse of the oracle's J^T J, or on Hi"""
    act = g.obs_active()
    assert np.array_equal(act, o.obs_active())
    used = np.ones(p.n_frames, bool) if inertial else _frame_used(p, act)
    live = 6 if inertial and flags.get("rotation_only") else o.fd
    keep = None
    if Hi is None:
        Hi, keep = dense_cov.dense_inverse(o, used, live)
    return R.influence(o, Hi, p.models, p.obs_frame, p.obs_cam, act, used, flags.get("visual_mult", 1.0)), keep, act


def _device_sigma(g):
    """the device's own covariance blocks, assembled where the reference reads them; None where vcgpu_get_covariance
    refuses the rig (its system keeps a frame no residual fixes: a vision frame no active observation sees, the
    velocities of a rotation-only run), which the frame calls and the influence call damp"""
    from vicalib_b200.capi import VcgpuError

    try:
        Sgg = g.covariance()
    except VcgpuError:
        return None
    fg, _ = g.frame_cross_covariance()
    return R.assemble(g.n_frames, g.fd, Sgg, g.frame_covariance(), fg)


def _rel(r, ref, k):
    ok = np.isfinite(ref["infl"])
    return (np.abs(r[k][ok] - ref[k][ok]) / np.abs(ref[k][ok])).max(initial=0.0)


def _scaled(r, ref, k):
    ok = np.isfinite(ref["infl"]) if k != "h" else np.isfinite(ref["h"][:, 0])
    return (np.abs(r[k][ok] - ref[k][ok]) / ref["sc_" + k][ok]).max(initial=0.0)


# h within 1e-10 absolute, stud and infl within 1e-8 relative, on the reference evaluated on the device's own Sigma
# blocks (the kernels' algebra).  Against the dense inverse of the oracle's J^T J, ill-conditioned on the inertial rigs,
# the errors are correlation-scaled (sc_* of influence_ref: the first-order change of each output when every Sigma_ij
# moves by sqrt(Sigma_ii Sigma_jj), as dense_cov.corr_errors scales Sigma) and held to 1e-8.  Measured on an H100 80GB
# HBM3 (700 W): on the device's Sigma h 3.9e-13, stud 4.5e-10, infl 5.1e-9 at most; correlation-scaled 5.5e-11 at most.
H_BAR, REL_BAR, CORR_BAR = 1e-10, 1e-8, 1e-8


def check(g, o, p, inertial, flags):
    r = g.observation_influence()
    Hd = _device_sigma(g)
    eh = es = ei = 0.0
    if Hd is not None:
        own, _, _ = _ref(g, o, p, inertial, flags, Hi=Hd)
        for k in ("h", "stud", "infl"):
            assert np.array_equal(np.isnan(r[k]), np.isnan(own[k])), k
        eh = np.nanmax(np.abs(r["h"] - own["h"]))
        es, ei = _rel(r, own, "stud"), _rel(r, own, "infl")
    ref, keep, act = _ref(g, o, p, inertial, flags)
    for k in ("h", "stud", "infl"):
        assert np.array_equal(np.isnan(r[k]), np.isnan(ref[k])), k
    ch, cs, ci = (_scaled(r, ref, k) for k in ("h", "stud", "infl"))
    print(f"\n{p.n_frames} frames, G {g.G}: on the device's Sigma {'(not taken) ' if Hd is None else ''}h {eh:.1e}, stud {es:.1e}, infl {ei:.1e}; "
          f"vs the dense inverse, correlation-scaled h {ch:.1e}, stud {cs:.1e}, infl {ci:.1e}")
    assert eh <= H_BAR and es <= REL_BAR and ei <= REL_BAR, (eh, es, ei)
    assert max(ch, cs, ci) <= CORR_BAR, (ch, cs, ci)
    if not inertial:
        tr = (r["h"][act > 0, 0] + r["h"][act > 0, 2]).sum()
        assert abs(tr - keep.sum()) <= 1e-8 * keep.sum(), (tr, keep.sum())
    return r


CASES = {
    "linear": (("linear",), False, {}),
    "fov": (("fov",), False, {}),
    "poly2": (("poly2",), False, dict(visual_mult=2.0)),
    "poly3": (("poly3",), False, {}),
    "kb4": (("kb4",), False, {}),
    "poly3_fov_fixed": (("poly3", "fov"), False, dict(fix_intrinsics=1)),
    "poly3_kb4_inertial": (("poly3", "kb4"), True, dict(ALL_ON)),
    "rotation_only": (("poly3",), True, dict(inertial=1, rotation_only=1, bias_active=0, scale_active=0, optimize_ts=1)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_parity(name):
    models, inertial, flags = CASES[name]
    p = synth.make_problem(models=models, n_frames=60 if inertial else 18, inertial=inertial, seed=15)
    g, o = _solved(p, flags)
    check(g, o, p, inertial, flags)


def test_removed_outliers():
    """the inactive path: predictive residuals of removed corners, the active ones without them"""
    p = synth.make_problem(models=("poly3", "kb4"), n_frames=18, seed=16)
    g, o = _solved(p, {})
    rmse = np.array([0.05, 0.05])
    g.remove_outliers(rmse, 2.0)
    o.remove_outliers(rmse, 2.0)
    act = g.obs_active()
    assert (act == 0).sum() > 10 and (act == 1).sum() > 100
    out = check(g, o, p, False, {})
    assert np.isfinite(out["stud"][act == 0]).all()


@pytest.mark.parametrize("name", ["fov_kb4", "kb4_poly3_inertial"])
def test_wide_lens_rig(name):
    lens = W.build(name)
    g, o = _solved(lens.p, lens.flags, max_iters=10)
    check(g, o, lens.p, bool(lens.flags.get("inertial", 0)), lens.flags)


@pytest.mark.parametrize("G", [67, 68])
def test_many_globals(G):
    p = synth.make_problem(models=chain_plan.rig_with_globals(G), n_frames=90, grid=(8, 6), inertial=True, seed=G)
    g, o = _solved(p, dict(ALL_ON))
    assert g.G == G
    check(g, o, p, True, dict(ALL_ON))


def test_trace_config2():
    """the trace identity on the GPU's own output on config 2 (one poly3 camera, 2000 frames, 280 000 corners)"""
    p = synth.make_config("config2")
    g, _ = _solved(p, {}, max_iters=10)
    r = g.observation_influence(stud=False, infl=False)
    act = g.obs_active() > 0
    keep = int((np.diag(g.covariance()) != 0).sum()) + 6 * int(_frame_used(p, act).sum())
    tr = (r["h"][act, 0] + r["h"][act, 2]).sum()
    print(f"\nconfig2: sum tr(H) {tr:.6f}, free tangents {keep}")
    assert abs(tr - keep) <= 1e-8 * keep, (tr, keep)


def _restarted(p, g, pc):
    """a handle and the oracle at g's state, on p with the detections pc"""
    from oracle.binding import Oracle
    from vicalib_b200.capi import Calibrator

    st = g.state()
    p2 = dataclasses.replace(p, p_c=pc, intr=st["intr"], q_ck=st["q_ck"], p_ck=st["p_ck"], T_wp=st["T_wp"], v_w=st["v_w"])
    h = Calibrator()
    h.load(p2)
    return h, Oracle(p2), p2


def test_frame_all_removed_is_nan():
    """every corner of vision frame 5 moved 50 px and removed: the frame is not determined, so its corners get NaN in all
    three, and the rest is as if it were not in the problem"""
    p = synth.make_problem(models=("poly3", "kb4"), n_frames=18, seed=26)
    g, _ = _solved(p, {})
    pc = p.p_c.copy()
    pc[p.obs_frame == 5] += 50.0
    h, o, p2 = _restarted(p, g, pc)
    for x in (h, o):
        x.remove_outliers(np.array([1.0, 1.0]), 5.0)
    act = h.obs_active()
    assert not act[p.obs_frame == 5].any() and act[p.obs_frame != 5].mean() > 0.95
    r = check(h, o, p2, False, {})
    for k in ("h", "stud", "infl"):
        v = r[k].reshape(len(act), -1)
        assert np.isnan(v[p.obs_frame == 5]).all() and np.isfinite(v[(p.obs_frame != 5) & (act > 0)]).all()


def test_camera_all_removed_is_nan():
    """every observation of camera 1 removed: that camera is not determined, so its corners get NaN in all three"""
    p = synth.make_problem(models=("poly3", "fov", "kb4"), n_frames=18, seed=22)
    g, o = _solved(p, {})
    g.remove_outliers(np.array([1e12, 1e-12, 1e12]), 1.0)
    o.remove_outliers(np.array([1e12, 1e-12, 1e12]), 1.0)
    act = g.obs_active()
    assert not act[p.obs_cam == 1].any() and act[p.obs_cam != 1].all()
    r = check(g, o, p, False, {})
    for k in ("h", "stud", "infl"):
        v = r[k].reshape(len(act), -1)
        assert np.isnan(v[p.obs_cam == 1]).all() and np.isfinite(v[p.obs_cam != 1]).all()


def test_three_corner_view_has_unit_leverage():
    """a view left with 3 active corners on a one-camera rig: those corners alone fix its pose, so H_i = I"""
    p = synth.make_problem(models=("poly3",), n_frames=18, seed=23)
    g, _ = _solved(p, {})
    # make every corner of frame 5 but three an outlier, then remove them; the three span the image (three collinear
    # corners would leave the rotation about their line free)
    sel = np.flatnonzero((p.obs_frame == 5) & (p.obs_cam == 0))
    u = p.p_c[sel]
    i0, i1 = int(np.argmin(u[:, 0])), int(np.argmax(u[:, 0]))
    d = np.abs(np.cross(u[i1] - u[i0], u - u[i0]))
    three = [i0, i1, int(np.argmax(d))]
    sel = np.r_[sel[three], np.delete(sel, three)]
    pc = p.p_c.copy()
    pc[sel[3:]] += 50.0
    h, _, _ = _restarted(p, g, pc)
    h.remove_outliers(np.array([1.0]), 5.0)
    act = h.obs_active()
    assert act[sel[:3]].all() and not act[sel[3:]].any()
    r = h.observation_influence()
    H = r["h"][sel[:3]]
    assert np.abs(H - np.array([1.0, 0.0, 1.0])).max() < 1e-6, H


def test_no_side_effects():
    p = synth.make_problem(models=("poly3",), n_frames=40, inertial=True, seed=24)
    g, _ = _solved(p, dict(ALL_ON), max_iters=4)
    s0, w0 = g.state(), g.imu_weights()
    a = g.observation_influence()
    b = g.observation_influence()
    assert all(a[k].tobytes() == b[k].tobytes() for k in a)
    s1 = g.state()
    assert all(np.array_equal(s0[k], s1[k]) for k in s0) and np.array_equal(w0, g.imu_weights())
    from vicalib_b200.capi import Calibrator
    ref = Calibrator()
    ref.load(p)
    ref.set_flags(**ALL_ON)
    ref.set_options(function_tol=1e-12, max_iters=4)
    ref.solve()
    g.set_options(max_iters=3)
    ref.set_options(max_iters=3)
    g.solve()
    ref.solve()
    s2, s3 = g.state(), ref.state()
    assert all(np.asarray(s2[k]).tobytes() == np.asarray(s3[k]).tobytes() for k in s2)


def test_outputs_and_refusals():
    from vicalib_b200.capi import Calibrator, ObsInfluence

    p = synth.make_problem(models=("poly3",), n_frames=18, seed=25)
    g, _ = _solved(p, {})
    full = g.observation_influence()
    for h, s, i in [(True, False, False), (False, True, False), (False, False, True), (False, True, True)]:
        part = g.observation_influence(h=h, stud=s, infl=i)
        assert all(part[k].tobytes() == full[k].tobytes() for k in part)
    assert g.L.vcgpu_get_observation_influence(g.h, None) == INVALID
    import ctypes as C
    assert g.L.vcgpu_get_observation_influence(g.h, C.byref(ObsInfluence(None, None, None))) == INVALID
    assert b"all null" in g.L.vcgpu_last_error(g.h)
    assert g.L.vcgpu_get_observation_influence(None, C.byref(ObsInfluence(None, None, None))) == INVALID
    s = Calibrator()
    s.load(p)
    s.set_flags(visual_mult=0.0)
    hh = np.full((p.n_obs, 3), np.nan)
    assert s.L.vcgpu_get_observation_influence(s.h, C.byref(ObsInfluence(hh.ctypes.data, None, None))) == NUMERIC
    assert np.isnan(hh).all()


def test_host_method(tmp_path):
    """ViCalibrator::GetObservationInfluence against vcgpu_get_observation_influence on the same handle, through
    tests/cpp/observation_influence_main.cc: the same bits"""
    import os
    import subprocess

    from test_gpu_host_mirror import _write_problem

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "observation_influence")
    subprocess.run([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-Wall", "-o", exe,
                    os.path.join(root, "tests", "cpp", "observation_influence_main.cc"),
                    "-L" + os.path.join(root, "vicalib_b200"), "-lvcgpu", "-lpthread",
                    "-Wl,-rpath," + os.path.join(root, "vicalib_b200")], check=True, timeout=300)
    p = synth.make_problem(models=("poly3", "kb4"), n_frames=18, seed=27)
    prob, res = str(tmp_path / "problem.bin"), str(tmp_path / "result.bin")
    _write_problem(prob, p, True, 15, 0)
    subprocess.run([exe, prob, res], check=True, timeout=600)
    out = np.fromfile(res, dtype=np.float64)
    n = int(out[:1].view(np.int64)[0])
    assert n == p.n_obs and len(out) == 1 + 2 * 5 * n
    a, b = out[1:1 + 5 * n], out[1 + 5 * n:]
    assert a.tobytes() == b.tobytes()
    assert np.isfinite(a).mean() > 0.99 and (a[:3 * n:3] > 0).all()
