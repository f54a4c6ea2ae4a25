"""CPU: the staged flow of ViCalibrator::SolveThread as vcgpu_calibrate_batch runs it, restated in Python.

flow_step is the stage decision after a solve (the host mirror's SolveThread, vicalib_b200/host/vicalibrator.h:696-720),
flow_flags the multiplicities SetupProblem gives a stage (:615-622), gravity_from_accel the gravity initialisation
(:664-679).  They are checked here against a hand-written table of the mirror's transitions and against scipy's
rotations; test_gpu_calibrate_batch.py runs flow_reference, the whole machine with per-handle calls, against the batch.
"""
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

VISION, ROTATION, TRANSLATION, SCALE, FINISHED = range(5)  # vcgpu_flow_summary::stage


def stage_of(s):
    if s.get("finished"):
        return FINISHED
    if not s["inertial"]:
        return VISION
    if s["rotation_only"]:
        return ROTATION
    return SCALE if s["scale"] else TRANSLATION


def flow_step(s, converged, calibrate_imu, remove_outliers):
    """the decision after a solve: (new switches, remove outliers now, set the problem up again)"""
    s = dict(s)
    remove = setup = False
    if not converged:
        return s, remove, setup
    if calibrate_imu:
        if not s["inertial"]:
            s["inertial"] = True
        elif s["rotation_only"]:
            s["rotation_only"], s["bias"] = False, True
        elif not s["scale"]:
            s["scale"] = True
        elif remove_outliers and not s["outliers_removed"]:
            remove = True
        else:
            s["finished"] = True
        setup = not s["finished"]
    elif remove_outliers and not s["outliers_removed"]:
        remove = True
    else:
        s["finished"] = True
    if remove:
        s["outliers_removed"] = True
    return s, remove, setup


def flow_flags(s, adds, calibrate_imu, block_duplication):
    """SetupProblem's stage switches and multiplicities; adds = [visual, imu] blocks added so far, updated in place"""
    inertial = bool(calibrate_imu and s["inertial"])
    vm = im = 1.0
    if block_duplication:
        adds[0] += 1
        if inertial:
            adds[1] += 1
        vm, im = float(adds[0]), float(adds[1] if adds[1] > 0 else 1)
    return dict(inertial=int(inertial), rotation_only=int(s["rotation_only"]), bias_active=int(s["bias"]),
                scale_active=int(s["scale"]), visual_mult=vm, imu_mult=im)


def interpolate_accel(t, a, time):
    if not t[0] < time:
        return a[0]
    if not time < t[-1]:
        return a[-1]
    i = 0
    while i + 2 < len(t) and t[i + 1] < time:
        i += 1
    f = (time - t[i]) / (t[i + 1] - t[i])
    return np.array([a[i][k] * (1 - f) + a[i + 1][k] * f for k in range(3)])


def gravity_from_accel(q, a):
    """(pitch, roll) of the gravity direction R(q) a / |a| in the world, with the mirror's operations in its order"""
    x, y, z, w = q
    R = [1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
         2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
         2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]
    n = math.sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2])
    gb = [a[0] / n, a[1] / n, a[2] / n]
    gw = [R[0] * gb[0] + R[1] * gb[1] + R[2] * gb[2], R[3] * gb[0] + R[4] * gb[1] + R[5] * gb[2],
          R[6] * gb[0] + R[7] * gb[1] + R[8] * gb[2]]
    pp = math.asin(gw[1])
    return np.array([pp, math.asin(-gw[0] / math.cos(pp))])


def flow_reference(g, p, calibrate_imu, remove_outliers, outlier_threshold, block_duplication, gravity_initialized, max_solves):
    """the host mirror's SolveThread on one Calibrator g (problem p) with per-handle calls; returns the trace"""
    f = g.flags
    s = dict(inertial=bool(f.inertial), rotation_only=bool(f.rotation_only), bias=bool(f.bias_active), scale=bool(f.scale_active),
             outliers_removed=False, finished=False)
    gravity = bool(gravity_initialized)
    adds = [0, 0]
    setup = True
    trace = dict(solves=[], stages=[], removed=0)
    while not s["finished"] and len(trace["solves"]) < max_solves:
        if setup:
            st = g.state()
            g.set_cameras(p.models, st["intr"], st["q_ck"], st["p_ck"])
            g.set_frames(st["T_wp"], st["v_w"], p.ftime)
            g.set_imu_params(st["g"], st["b"], st["sf"], st["ts"])
            g.set_flags(**flow_flags(s, adds, calibrate_imu, block_duplication))
            if s["inertial"] and not s["rotation_only"] and not gravity and len(p.imu_t):
                mid = len(p.ftime) // 2
                grav = gravity_from_accel(st["T_wp"][mid][:4], interpolate_accel(p.imu_t, p.imu_a, p.ftime[mid]))
                gravity = True
                g.set_imu_params(grav, st["b"], st["sf"], st["ts"])
            setup = False
        if g.num_residuals() <= 0:
            break
        trace["stages"].append(stage_of(s))
        summary = g.solve(free_running=True)
        trace["solves"].append(summary)
        rmse = []
        for c in range(g.n_cams):
            cost, n = g.evaluate(c)
            rmse.append(math.sqrt(cost / n) if n > 0 else 0.0)
        s, remove, setup = flow_step(s, summary["termination"] != 0, calibrate_imu, remove_outliers)
        if remove:
            trace["removed"] += g.remove_outliers(np.array(rmse), outlier_threshold)
    trace["finished"] = int(s["finished"])
    trace["stage"] = stage_of(s)
    return trace


# ------------------------------------------------------------------ the mirror's transitions, by hand
def _s(inertial, rot, bias, scale, removed=False):
    return dict(inertial=inertial, rotation_only=rot, bias=bias, scale=scale, outliers_removed=removed, finished=False)


#   start                         calibrate_imu, remove_outliers ->  stage after, remove now, setup again
TABLE = [
    (_s(False, True, False, False), True, True, ROTATION, False, True),
    (_s(True, True, False, False), True, True, TRANSLATION, False, True),
    (_s(True, False, True, False), True, True, SCALE, False, True),
    (_s(True, False, True, True), True, True, SCALE, True, True),          # outlier removal, then the scale stage again
    (_s(True, False, True, True, True), True, True, FINISHED, False, False),
    (_s(True, False, True, True), True, False, FINISHED, False, False),
    (_s(False, True, False, False), False, True, VISION, True, False),     # vision flow: removal without a new setup
    (_s(False, True, False, False, True), False, True, FINISHED, False, False),
    (_s(False, True, False, False), False, False, FINISHED, False, False),
]


@pytest.mark.parametrize("row", range(len(TABLE)))
def test_transitions(row):
    s, imu, rem, stage, remove, setup = TABLE[row]
    t, r, u = flow_step(s, True, imu, rem)
    assert (stage_of(t), r, u) == (stage, remove, setup)
    assert flow_step(s, False, imu, rem) == (s, False, False)  # not converged: the same stage again


def test_multiplicities():
    """visual blocks 1, 2, 3, ... per setup; IMU blocks 1 until the first inertial stage, then 1, 2, 3, ..."""
    adds = [0, 0]
    seq = [_s(False, True, False, False), _s(True, True, False, False), _s(True, False, True, False), _s(True, False, True, True),
           _s(True, False, True, True, True)]
    got = [(f["visual_mult"], f["imu_mult"], f["inertial"]) for f in (flow_flags(s, adds, True, True) for s in seq)]
    assert got == [(1, 1, 0), (2, 1, 1), (3, 2, 1), (4, 3, 1), (5, 4, 1)]
    assert flow_flags(seq[2], [0, 0], True, False)["visual_mult"] == 1.0
    assert flow_flags(seq[2], [0, 0], False, True)["inertial"] == 0


def test_gravity_against_scipy():
    rng = np.random.default_rng(3)
    for _ in range(200):
        pitch, roll = rng.uniform(-1.2, 1.2, 2)
        gw = np.array([-math.sin(roll) * math.cos(pitch), math.sin(pitch), math.cos(roll) * math.cos(pitch)])
        rot = Rotation.random(random_state=rng)
        a = rot.as_matrix().T @ gw * rng.uniform(5, 15)  # the sample in the body frame of pose rot
        got = gravity_from_accel(rot.as_quat(), a)
        assert np.allclose(got, [pitch, roll], atol=1e-12)


def test_interpolate_accel():
    t = np.array([0.0, 1.0, 2.0])
    a = np.array([[0.0, 0, 0], [1, 2, 3], [3, 2, 1]])
    assert np.array_equal(interpolate_accel(t, a, -1.0), a[0])
    assert np.array_equal(interpolate_accel(t, a, 5.0), a[2])
    assert np.allclose(interpolate_accel(t, a, 1.5), [2, 2, 2])
