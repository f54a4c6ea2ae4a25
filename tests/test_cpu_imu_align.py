"""CPU checks of tests/imu_align_ref.py, the numpy restatement of vcgpu_align_imu: Horn's closed form against an SVD
Kabsch fit and a brute-force rotation fit, recovery of the truth on synthetic rigs started as the reference starts without
a cameras.xml (camera 0 as the rig frame, ts = 0, no gyro bias), and the excitation of single-axis motion."""
import numpy as np
import pytest
from scipy.optimize import minimize

import imu_align_ref as R
from oracle.binding import Oracle
from vicalib_b200 import synth

GYRO_BIAS = np.array([0.05, -0.04, 0.03])  # rad/s, added to the stream's own bias
GRID = dict(ts_lo=-0.05, ts_hi=0.05, n_ts=21)


def rig(motion="gentle", ts_truth=0.0, seed=7, n_frames=40):
    """a one-camera inertial rig at truth + synth's pose noise, with GYRO_BIAS on the gyro, re-expressed with camera 0 as
    the rig frame; returns (problem, truth b_g)"""
    p = synth.make_problem(models=("poly3",), n_frames=n_frames, grid=(10, 7), inertial=True, seed=seed,
                           ts_truth=ts_truth, motion=motion)
    p.imu_w = p.imu_w - GYRO_BIAS / p.truth["sf"][:3]
    return R.camera0_start(p), p.truth["b"][:3] + GYRO_BIAS


def test_horn_matches_kabsch_and_a_brute_force_fit():
    p, _ = rig()
    o = Oracle(p)
    r = R.Rig(p, o, -0.05, 0.05)
    for s in (-0.02, 0.0, 0.01):
        b = r.turns(s, np.zeros(3))
        ch, Q = R.horn(r.a, b)
        ck, Rk = R.kabsch(r.a, b)
        assert abs(ch - ck) <= 1e-12 * ck
        assert np.abs(R.rot(Q) - Rk).max() < 1e-12
        # no rotation fits better than Horn's: a local search from Horn's answer and from three other starts
        f = lambda w: ((r.a - b @ synth.quat_to_mat(synth.so3_exp(w)).T) ** 2).sum(1).mean()  # noqa: E731
        best = min(minimize(f, w0, method="BFGS").fun for w0 in ([0, 0, 0], [2, 0, 0], [0, 2, 0], [0, 0, 2]))
        assert best >= ch * (1 - 1e-9)
        assert best <= ch * (1 + 1e-3)  # and BFGS, stopping at its gradient tolerance, comes within 5.3e-5 of it


# Bars measured on these rigs (seed 7, 40 frames, pose noise 2 mm / 5 mrad, the stream's sf left at 1 on the handle):
# gentle motion, whose turns span all three axes only weakly (excitation 1e-5 .. 6e-4), leaves 0.043 rad of rotation
# error, 0.013 rad/s of bias error and up to 4.1e-4 s of ts error (at ts = -0.027); vigorous motion 0.013 rad,
# 0.0076 rad/s and 1.1e-4 s.  The residual is the frame poses' 5 mrad noise (rms 0.0146 rad per interval).
BARS = {"gentle": (0.06, 6e-4, 0.02), "vigorous": (0.02, 2.5e-4, 0.012)}


@pytest.mark.parametrize("motion", ["gentle", "vigorous"])
@pytest.mark.parametrize("ts_truth", [0.0, 0.013, -0.027])
def test_recovers_the_truth_from_the_reference_start(motion, ts_truth):
    p, bg = rig(motion, ts_truth)
    r = R.align(p, Oracle(p), **GRID)
    assert r["status"] == 0 and r["n_intervals"] == p.n_frames - 1
    assert R.angle(p.q_ck[0], p.truth["q_ck"][0]) > 1.5  # the start is far from the answer (RDF over robotics axes)
    rot_bar, ts_bar, bg_bar = BARS[motion]
    assert R.angle(r["Q"], p.truth["q_ck"][0]) < rot_bar
    assert abs(r["ts"] - ts_truth) < ts_bar
    assert np.abs(r["b_g"] - bg).max() < bg_bar
    assert r["Q"][3] >= 0 and r["rms"] < 0.02
    # the grid's argmin is the candidate nearest the truth, and the refinement lowered the cost below it
    s = R.candidates(GRID["ts_lo"], GRID["ts_hi"], GRID["n_ts"])
    assert abs(s[np.argmin(r["curve"])] - ts_truth) <= 0.0051
    assert r["rms"] ** 2 < r["curve"].min()


def test_without_find_time_offset_ts_is_kept():
    p, _ = rig(ts_truth=0.013)
    p.ts = 0.012
    r = R.align(p, Oracle(p), find_time_offset=False, **GRID)
    assert r["ts"] == 0.012 and r["curve"] is None and r["status"] == 0


def test_single_axis_motion_has_two_null_excitations():
    p, _ = rig()
    p.imu_w = p.imu_w.copy()
    p.imu_w[:, :2] = 0.0  # the gyro turns about its z axis only
    r = R.align(p, Oracle(p), max_iters=0, **GRID)  # at the start point, before a fitted bias turns the other axes
    e = r["excitation"]
    assert e[2] > 1e-5 and e[0] <= 1e-15 * e[2] and e[1] <= 1e-15 * e[2], e


def test_too_few_usable_intervals_is_numeric():
    p, _ = rig()
    keep = p.obs_frame < 3  # frames 0 .. 2 seen: two usable intervals
    import dataclasses
    p = dataclasses.replace(p, obs_frame=p.obs_frame[keep], obs_cam=p.obs_cam[keep], p_w=p.p_w[keep], p_c=p.p_c[keep])
    r = R.align(p, Oracle(p), **GRID)
    assert r["status"] == -3 and r["n_intervals"] == 2 and np.isnan(r["Q"]).all()
