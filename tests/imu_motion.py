"""Problems with the motion of a handheld visual-inertial recording, cut from synth.make_problem(motion="vigorous"), each
of which asserts the regime it claims, so that a later change to synth cannot quietly remove it.

synth's default trajectory is gentle: |w| <= 1.2 rad/s, |w| dt <= 6e-3 per RK4 step at 200 Hz, ||a| - g| <= 0.21 m/s^2,
and the rig's attitude stays 1.5-2.6 rad from the world frame, so adjacent frames' quaternions (canonical, w >= 0) never
change sign.  A recording made to excite every axis turns at several rad/s and accelerates by many m/s^2.  The
vigorous trajectory (synth._vigorous_cam0_pose) keeps the grid in view and gives, at every IMU rate here:
  max |w| >= 6 rad/s, max ||a| - g| >= 10 m/s^2, the rig's attitude across pi from the world frame (adjacent frames whose
  canonical quaternions have opposite signs: the IMU end residual's quaternion has w < 0 there),
with 9 (200 Hz), 17 (400 Hz) and 51 (1 kHz) RK4 steps per interval and a per-step angle up to 0.031, 0.017 and 0.007.
Measured: max |w| 6.3 / 7.0 / 6.8 rad/s, max ||a| - g| 14.2 / 13.9 / 14.3 m/s^2, opposite-sign pairs at intervals
(21, 28) / (7,) / (0, 6).

flipped(p, frames, cams) is the same physical problem with chosen frame and camera quaternions negated.
"""
import dataclasses

import numpy as np

import imu_streams
from vicalib_b200 import synth

TS_TRUTH = 0.004  # the time offset the samples were drawn with
TS = 0.0025       # the offset the problems start from

# name: (IMU rate, frame rate, frames, models, seed, least max |w| dt per step, RK4 steps per interval)
SPECS = {
    "imu200": (200.0, 25.0, 30, ("poly3",), 41, 0.030, (8, 10)),
    "imu400": (400.0, 25.0, 26, ("poly3", "kb4"), 42, 0.016, (16, 18)),
    "imu1000": (1000.0, 20.0, 24, ("fov",), 44, 0.0065, (50, 52)),
}
NAMES = tuple(SPECS)


@dataclasses.dataclass
class Motion:
    name: str
    p: synth.Problem
    cls: dict
    regime: dict


def regime(p):
    """max |w|, max |w| dt over the stream, max ||a| - g|, and the intervals whose frames' quaternions have opposite
    signs (q_k . q_k+1 < 0)"""
    w = np.linalg.norm(p.imu_w, axis=1)
    a = np.linalg.norm(p.imu_a, axis=1)
    q = p.T_wp[:, :4]
    return dict(w=float(w.max()), wdt=float((w[1:] * np.diff(p.imu_t)).max()),
                accel=float(np.abs(a - synth.GRAVITY).max()),
                sign_flips=np.flatnonzero(np.einsum("ij,ij->i", q[:-1], q[1:]) < 0))


def build(name):
    rate, frame_rate, nf, models, seed, wdt, steps = SPECS[name]
    p = synth.make_problem(models=models, n_frames=nf, grid=(10, 7), inertial=True, seed=seed, imu_rate=rate,
                           frame_rate=frame_rate, ts_truth=TS_TRUTH, motion="vigorous")
    p.ts = TS
    p = imu_streams.perturbed(p)
    r = regime(p)
    assert r["w"] >= 6.0 and r["wdt"] >= wdt and r["accel"] >= 10.0, r
    assert len(r["sign_flips"]) >= 1, r  # the attitude crosses pi
    c = imu_streams.classify(p)
    assert c["covered"].all() and c["comparable"].all()
    assert c["steps"].min() >= steps[0] and c["steps"].max() <= steps[1], (c["steps"].min(), c["steps"].max())
    assert not c["tie_start"].any() and not c["tie_end"].any()
    return Motion(name, p, c, r)


def vision(seed=46, n_frames=20):
    """a two-camera rig on the vigorous trajectory for vision-only solves (inertial flags off; camera 0's extrinsics,
    the IMU frame's, are held constant there), with its attitude across pi as in the inertial rigs"""
    p = synth.make_problem(models=("poly3", "kb4"), n_frames=n_frames, grid=(10, 7), inertial=True, seed=seed,
                           frame_rate=25.0, motion="vigorous")
    assert len(regime(p)["sign_flips"]) >= 1
    return p


def flipped(p, frames=(), cams=()):
    """p with the quaternions of `frames` and of cameras `cams` negated: the same physical problem"""
    T, qc = p.T_wp.copy(), p.q_ck.copy()
    T[list(frames), :4] *= -1.0
    qc[list(cams)] *= -1.0
    return dataclasses.replace(p, T_wp=T, q_ck=qc)


def scattered(n_frames, seed=1):
    """a scattered third of the frames, the first and the last among them"""
    rng = np.random.default_rng(seed)
    f = set(rng.choice(np.arange(1, n_frames - 1), n_frames // 3 - 2, replace=False).tolist()) | {0, n_frames - 1}
    return sorted(f)
