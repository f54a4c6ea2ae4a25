"""GPU: vcgpu_align_imu and vcgpu_align_imu_batch against tests/imu_align_ref.py, the numpy restatement, on rigs started
as the reference starts without a cameras.xml (camera 0 as the rig frame, ts = 0, no gyro bias): the curve, its argmin
and the refined Q, ts, b_g and rms; bits under negated quaternions; no side effects without apply; the state apply leaves
and the solve that follows it; the batch's bits, order independence, refusals and failing rigs; find_time_offset = 0;
and the staged flow with the alignment between its vision and inertial halves."""
import ctypes as C

import numpy as np
import pytest

import imu_align_ref as R
import imu_motion
from oracle.binding import Oracle
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

GRID = dict(ts_lo=-0.05, ts_hi=0.05, n_ts=21)
GYRO_BIAS = np.array([0.05, -0.04, 0.03])
STATE_KEYS = ("intr", "q_ck", "p_ck", "T_wp", "v_w", "g", "b", "sf")


def rig(motion="gentle", ts_truth=0.013, seed=7, n_frames=40, models=("poly3",)):
    p = synth.make_problem(models=models, n_frames=n_frames, grid=(10, 7), inertial=True, seed=seed, ts_truth=ts_truth,
                           motion=motion)
    p.imu_w = p.imu_w - GYRO_BIAS / p.truth["sf"][:3]
    return R.camera0_start(p)


def calib(p, **flags):
    from vicalib_b200.capi import Calibrator

    g = Calibrator(device=0)
    g.load(p)
    if flags:
        g.set_flags(**flags)
    return g


def same(x, y):
    for k in ("Q", "ts", "b_g", "rms", "excitation", "n_intervals", "iterations", "status"):
        assert np.array_equal(np.asarray(x[k]), np.asarray(y[k]), equal_nan=True), (k, x[k], y[k])
    if "curve" in x or "curve" in y:
        assert np.array_equal(x["curve"], y["curve"], equal_nan=True)


# Parity bars.  The curve differs from the reference's only in summation order and the eigen-solver (cyclic Jacobi
# against LAPACK): 1e-9 relative.  The refined point is the same local minimum reached through different Jacobians (duals
# on the device, central differences in numpy) and stopped when a halved step no longer lowers the cost, so it agrees
# to the minimum's flatness: 1e-6 rad in Q, 1e-6 s in ts, 1e-5 rad/s in b_g and 1e-7 relative in rms.
@pytest.mark.parametrize("motion,ts_truth", [("gentle", 0.013), ("vigorous", -0.027)])
def test_parity_with_the_reference(motion, ts_truth):
    p = rig(motion, ts_truth)
    got = calib(p).align_imu(curve=True, **GRID)
    ref = R.align(p, Oracle(p), **GRID)
    assert got["status"] == 0 and got["n_intervals"] == ref["n_intervals"] == p.n_frames - 1
    assert np.abs(got["curve"] - ref["curve"]).max() <= 1e-9 * ref["curve"].max()
    assert np.argmin(got["curve"]) == np.argmin(ref["curve"])
    assert R.angle(got["Q"], ref["Q"]) < 1e-6 and got["Q"][3] >= 0
    assert abs(got["ts"] - ref["ts"]) < 1e-6
    assert np.abs(got["b_g"] - ref["b_g"]).max() < 1e-5
    assert abs(got["rms"] - ref["rms"]) <= 1e-7 * ref["rms"]
    assert np.abs(got["excitation"] - ref["excitation"]).max() <= 1e-6 * ref["excitation"].max()
    print(f"{motion}: iterations {got['iterations']} (numpy {ref['iterations']}), rotation error "
          f"{R.angle(got['Q'], p.truth['q_ck'][0]):.3e} rad, ts error {got['ts'] - ts_truth:.3e} s")


def test_same_bits_under_negated_quaternions():
    p = rig("vigorous", -0.027)
    f = imu_motion.flipped(p, frames=range(0, p.n_frames, 3), cams=[0])
    same(calib(p).align_imu(curve=True, **GRID), calib(f).align_imu(curve=True, **GRID))


def test_no_side_effects_without_apply():
    p = rig()
    flags = dict(inertial=1, rotation_only=1, optimize_ts=1)
    g, h = calib(p, **flags), calib(p, **flags)
    before = g.state()
    g.align_imu(**GRID)
    after = g.state()
    for k in STATE_KEYS:
        assert np.array_equal(before[k], after[k]), k
    assert before["ts"] == after["ts"]
    for c in (g, h):
        c.set_options(max_iters=3)
    sg, sh = g.solve(), h.solve()
    assert sg["final_cost"] == sh["final_cost"]
    for k in STATE_KEYS:
        assert np.array_equal(g.state()[k], h.state()[k]), k


def test_apply_sets_the_documented_state_and_the_next_solve_matches_a_fresh_handle():
    p = rig()
    g = calib(p)
    before = g.state()
    r = g.align_imu(apply=True, **GRID)
    assert r["status"] == 0
    after = g.state()
    Q = r["Q"]
    for c in range(p.n_cams):
        assert np.array_equal(after["q_ck"][c], R.qmul(before["q_ck"][c], Q))
    for f in range(p.n_frames):
        assert np.array_equal(after["T_wp"][f, :4], R.qmul(before["T_wp"][f, :4], Q))
    assert np.array_equal(after["T_wp"][:, 4:], before["T_wp"][:, 4:])
    for k in ("intr", "p_ck", "v_w", "g", "sf"):
        assert np.array_equal(after[k], before[k]), k
    assert np.array_equal(after["b"][3:], before["b"][3:]) and np.array_equal(after["b"][:3], r["b_g"])
    assert after["ts"] == r["ts"]
    # every camera pose T_wk T_ck^-1 is unchanged (to the rounding of the products)
    for f in range(p.n_frames):
        Rw0 = R.rot(before["T_wp"][f, :4]) @ R.rot(before["q_ck"][0]).T
        Rw1 = R.rot(after["T_wp"][f, :4]) @ R.rot(after["q_ck"][0]).T
        assert np.abs(Rw0 - Rw1).max() < 1e-14
    # a solve after apply gives the bits of a fresh handle uploaded with that state
    import dataclasses
    q = dataclasses.replace(p, q_ck=after["q_ck"], T_wp=after["T_wp"], b=after["b"], ts=after["ts"])
    flags = dict(inertial=1, rotation_only=1, optimize_ts=1, bias_active=1)
    fresh = calib(q, **flags)
    g.set_flags(**flags)
    for c in (g, fresh):
        c.set_options(max_iters=4)
    sg, sf = g.solve(), fresh.solve()
    assert sg["final_cost"] == sf["final_cost"] and sg["iterations"] == sf["iterations"]
    for k in STATE_KEYS:
        assert np.array_equal(g.state()[k], fresh.state()[k]), k


def test_without_find_time_offset_ts_keeps_its_bits():
    p = rig()
    p.ts = 0.0123456789
    g = calib(p)
    r = g.align_imu(find_time_offset=False, curve=True, **GRID)
    assert r["status"] == 0 and r["ts"] == p.ts and np.isnan(r["curve"]).all()
    ref = R.align(p, Oracle(p), find_time_offset=False, **GRID)
    assert R.angle(r["Q"], ref["Q"]) < 1e-6 and np.abs(r["b_g"] - ref["b_g"]).max() < 1e-5
    r = g.align_imu(find_time_offset=False, apply=True, **GRID)
    assert g.state()["ts"] == p.ts


def test_batch_bits_order_and_failing_rigs():
    from vicalib_b200.capi import align_imu_batch

    ps = [rig("gentle", 0.013), rig("vigorous", -0.027, seed=8, n_frames=30), rig("gentle", 0.0, seed=9, n_frames=300)]
    solo = [calib(p).align_imu(curve=True, **GRID) for p in ps]
    gs = [calib(p) for p in ps]
    got = align_imu_batch(gs, curve=True, **GRID)
    for a, b in zip(got, solo):
        same(a, b)
    got = align_imu_batch(gs[::-1], curve=True, **GRID)
    for a, b in zip(got, solo[::-1]):
        same(a, b)
    # a rig with two usable intervals fails alone: its curve and excitation are written, nothing is applied to it
    import dataclasses
    p = ps[0]
    keep = p.obs_frame < 3
    bad = calib(dataclasses.replace(p, obs_frame=p.obs_frame[keep], obs_cam=p.obs_cam[keep], p_w=p.p_w[keep],
                                    p_c=p.p_c[keep]))
    before = bad.state()
    out = align_imu_batch([gs[0], bad], curve=True, apply=[False, True], **GRID)
    same(out[0], solo[0])
    assert out[1]["status"] == -3 and out[1]["n_intervals"] == 2 and np.isnan(out[1]["Q"]).all()
    assert np.isfinite(out[1]["curve"]).all() and np.isfinite(out[1]["excitation"]).all()
    for k in STATE_KEYS:
        assert np.array_equal(bad.state()[k], before[k]), k


def test_batch_refusals_name_the_index_and_write_nothing():
    from vicalib_b200.capi import ImuAlignment, ImuAlignOpts, lib

    L = lib()
    gs = [calib(rig(seed=s, n_frames=20)) for s in (1, 2)]

    def call(handles, opts):
        n = len(handles)
        hs = (C.c_void_p * n)(*[None if g is None else g.h for g in handles])
        os_ = (ImuAlignOpts * n)(*opts)
        out = (ImuAlignment * n)()
        for o in out:
            o.ts = 12.5
        st = (C.c_int * n)(*[7] * n)
        rc = L.vcgpu_align_imu_batch(hs, C.c_int(n), os_, out, st)
        assert all(o.ts == 12.5 for o in out) and list(st) == [7] * n  # nothing written
        return rc, L.vcgpu_last_error(next(g for g in handles if g is not None).h).decode()

    good = ImuAlignOpts(-0.05, 0.05, 21, 1, 20, 0)
    for bad, why in ((ImuAlignOpts(-0.05, 0.05, 0, 1, 20, 0), "n_ts"), (ImuAlignOpts(-0.05, 0.05, 65537, 1, 20, 0), "n_ts"),
                     (ImuAlignOpts(0.05, -0.05, 21, 1, 20, 0), "ts_lo > ts_hi"),
                     (ImuAlignOpts(float("nan"), 0.05, 21, 1, 20, 0), "not finite")):
        rc, msg = call(gs, [good, bad])
        assert rc == -1 and "handle 1" in msg and why in msg, msg
    rc, msg = call([gs[0], gs[0]], [good, good])
    assert rc == -1 and "handle 1" in msg and "same handle" in msg
    rc, msg = call([gs[0], None], [good, good])
    assert rc == -1 and "handle 1" in msg
    from vicalib_b200.capi import Calibrator
    empty = Calibrator(device=0)
    p = rig(n_frames=20)
    empty.set_cameras(p.models, p.intr, p.q_ck, p.p_ck)
    empty.set_frames(p.T_wp, p.v_w, p.ftime)
    empty.set_observations(p.obs_frame, p.obs_cam, p.p_w, p.p_c)
    rc, msg = call([gs[0], empty], [good, good])
    assert rc == -1 and "handle 1: no IMU samples" in msg, msg
    assert L.vcgpu_align_imu(gs[0].h, None, None) == -1


# The staged flow from the reference's start: camera 0 as the rig frame, ts = 0 against ts_truth = 0.02 and gyro bias 0.
# The flow's own tests hold it to parity with the host mirror, not to the truth; the bars here are on the truth: 0.01 rad
# in camera 0's rotation, 1 ms in ts and 1 cm in camera 0's translation.  Measured on an H100: with the alignment the flow
# finishes after 4 solves, 5.4e-4 rad, 7.8e-5 s and 5.4e-4 m from the truth.  Without it (printed, not asserted) this
# rig's flow also finishes after 4 solves at the same point: here the rotation-only stage converges from the identity.
def test_flow_with_alignment_reaches_the_truth_from_the_reference_start():
    from vicalib_b200.capi import align_imu_batch, calibrate_batch

    p = synth.make_problem(models=("poly3", "poly3"), n_frames=120, grid=(14, 10), inertial=True, seed=11, ts_truth=0.02)
    p = R.camera0_start(p)
    truth_q = p.truth["q_ck"][0]
    inertial = dict(inertial=1, rotation_only=1, bias_active=0, scale_active=0, optimize_ts=1)

    def flow(align):
        g = calib(p, inertial=0, rotation_only=0)
        calibrate_batch([g], calibrate_imu=False)
        if align:
            r = align_imu_batch([g], apply=True, **GRID)[0]
            assert r["status"] == 0, r
        g.set_flags(**inertial)
        d, _ = calibrate_batch([g], calibrate_imu=True)[0]
        s = g.state()
        return d, s

    d, s = flow(True)
    rot_err = R.angle(s["q_ck"][0], truth_q)
    print(f"with the alignment: stage {d['stage']} after {d['solves']} solves, rotation error {rot_err:.2e} rad, "
          f"ts error {s['ts'] - 0.02:.2e} s, p_ck error {np.abs(s['p_ck'][0] - p.truth['p_ck'][0]).max():.2e} m")
    try:
        d0, s0 = flow(False)
        print(f"without it: stage {d0['stage']} after {d0['solves']} solves, rotation error "
              f"{R.angle(s0['q_ck'][0], truth_q):.2e} rad, ts error {s0['ts'] - 0.02:.2e} s")
    except Exception as e:  # recorded, not asserted
        print(f"without it: {e}")
    assert d["finished"]
    assert rot_err < 0.01
    assert abs(s["ts"] - 0.02) < 1e-3
    assert np.abs(s["p_ck"][0] - p.truth["p_ck"][0]).max() < 0.01


def test_host_method(tmp_path):
    """ViCalibrator::AlignImu against vcgpu_align_imu on the same handle after the mirror's vision-only flow, through
    tests/cpp/imu_align_main.cc: the same bits, and the mirror's camera, time offset and gyro bias take the result"""
    import os
    import subprocess

    from test_gpu_host_mirror import _write_problem

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "imu_align")
    subprocess.run([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-Wall", "-o", exe,
                    os.path.join(root, "tests", "cpp", "imu_align_main.cc"),
                    "-L" + os.path.join(root, "vicalib_b200"), "-lvcgpu", "-lpthread",
                    "-Wl,-rpath," + os.path.join(root, "vicalib_b200")], check=True, timeout=300)
    p = rig(n_frames=30)
    prob, res = str(tmp_path / "problem.bin"), str(tmp_path / "result.bin")
    _write_problem(prob, p, True, 30, 0)
    subprocess.run([exe, prob, res], check=True, timeout=600)
    out = np.fromfile(res, dtype=np.float64)
    a, b = out[:12], out[12:24]
    assert a.tobytes() == b.tobytes() and np.isfinite(a).all()
    Q = b[:4]
    qck = out[24:28]
    assert np.array_equal(qck, R.qmul(p.q_ck[0], Q))  # camera 0 is constant in the vision flow
    T = out[28:28 + 7 * p.n_frames].reshape(p.n_frames, 7)
    assert np.abs(np.linalg.norm(T[:, :4], axis=1) - 1).max() < 1e-12
    ts, bias = out[28 + 7 * p.n_frames], out[29 + 7 * p.n_frames:]
    assert ts == b[4] and np.array_equal(bias[:3], b[5:8]) and np.array_equal(bias[3:], np.zeros(3))
