"""CPU: ViCalibrator::GetIntegrationPoses(k) for every interval (vicalibrator.h:508-533), the oracle's integration rule
and the host mirror's own GetIntegrationPoses against the reference's (ref_integration_poses, oracle/ref_poses.cc), on a base
problem, the IMU streams of imu_streams.py (jittered, gapped, slow, partial, frame-tied: zero-length steps, 0 to 2
samples), the vigorous rigs of imu_motion.py with negated quaternions, stamps at Unix time (imu_epoch), a time offset
moving an interval end across a sample, intervals with no measurements and an interval ending past the last sample.

Counts and times are compared for equality; the poses to rounding (integration_poses_ref.worst: relative to each column
group's scale over the interval)."""
import dataclasses

import numpy as np
import pytest

import imu_epoch
import imu_motion
import imu_streams
import integration_poses_ref as R
from vicalib_b200 import synth

# oracle and mirror vs the reference: largest measured 1.8e-14 (stream_dropped, v_w); the bar leaves a factor of about 5
BAR = 1e-13


def _base():
    p = synth.make_problem(models=("poly3",), n_frames=12, grid=(14, 10), inertial=True, seed=77, ts_truth=0.003)
    return imu_streams.perturbed(p)


def _across(side):
    """the base problem with ts set so that the sample nearest the end of interval 4 lies 1e-7 s before (side -1) or
    after (+1) that end: GetRange moves it between intervals 4 and 5"""
    p = _base()
    t_end = p.ftime[5]
    i = int(np.argmin(np.abs(p.imu_t + p.ts - t_end)))
    return dataclasses.replace(p, ts=float(t_end - p.imu_t[i] + side * 1e-7))


def _cut():
    """samples only from the middle of interval 3 to the middle of interval 8: intervals 0-3 start before the stream (no
    measurements), interval 8 ends past the last sample (GetElement clamps it to that sample), 9 and 10 start after it"""
    p = _base()
    tt = p.imu_t + p.ts
    keep = (tt > 0.5 * (p.ftime[3] + p.ftime[4])) & (tt < 0.5 * (p.ftime[8] + p.ftime[9]))
    p = dataclasses.replace(p, imu_t=p.imu_t[keep].copy(), imu_w=p.imu_w[keep].copy(), imu_a=p.imu_a[keep].copy())
    c = imu_streams.classify(p)
    assert not c["covered"][[0, 1, 2, 3, 9, 10]].any() and c["covered"][4:9].all() and c["clamped"][8]
    return p


def _cases():
    out = [("base", _base()), ("ts_before_end", _across(-1)), ("ts_after_end", _across(+1)), ("cut", _cut())]
    out += [(f"stream_{n}", imu_streams.perturbed(imu_streams.build(n).p)) for n in imu_streams.NAMES]
    for n in imu_motion.NAMES:
        m = imu_motion.build(n)
        out.append((f"motion_{n}", m.p))
        out.append((f"motion_{n}_flipped", imu_motion.flipped(m.p, frames=imu_motion.scattered(m.p.n_frames))))
    out += [(f"epoch_{n}", imu_epoch.realistic(n).p) for n in ("jittered", "dropped", "samples2", "imu1000")]
    return out


CASES = dict(_cases())


@pytest.fixture(scope="module")
def ref():
    L = R.ref_lib()
    if L is None:
        pytest.skip("oracle/_ref is built only where the reference tree exists")
    return L


def check(got, want, name):
    """counts and times equal, poses within BAR; returns the worst (q, t, v, w) difference"""
    assert [len(x) for x in got] == [len(x) for x in want], name
    w = np.zeros(4)
    for k, (a, b) in enumerate(zip(got, want)):
        assert a[:, 13].tobytes() == b[:, 13].tobytes(), (name, k)
        w = np.maximum(w, R.worst(a, b))
    assert w.max() <= BAR, (name, w)
    return w


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_and_mirror_match_ref(ref, name):
    p = CASES[name]
    want = R.ref_poses(ref, p)
    covered = imu_streams.classify(p)["covered"]
    assert [len(x) > 0 for x in want] == covered.tolist(), name  # no measurements: no poses
    wo = check(R.oracle_poses(p), want, name)
    mirror = R.mirror_poses(p)
    # the mirror's GetRange finds the start element by a linear search, the reference's from its index guess: on an
    # interval whose start is a sample (t_i + ts == t_k) the mirror may also yield that sample, one more zero-length step
    tie = imu_streams.classify(p)["tie_start"]
    extra = [len(a) - len(b) for a, b in zip(mirror, want)]
    assert all(e in ((0, 1) if t else (0,)) for e, t in zip(extra, tie)), (name, extra)
    wm = check([_collapse(x) for x in mirror], [_collapse(x) for x in want], name)
    print(f"{name}: oracle {wo.max():.2e}, mirror {wm.max():.2e}")


def _collapse(x):
    """x without the poses that repeat their predecessor (zero-length steps)"""
    return x[np.r_[True, np.any(x[1:] != x[:-1], axis=1)]] if len(x) else x


def test_start_pose_is_the_frame(ref):
    """each interval starts from its frame's pose, velocity and time, with w_w = 0 (types.h:178-180)"""
    p = CASES["base"]
    for k, x in enumerate(R.ref_poses(ref, p)):
        assert x[0, :7].tobytes() == p.T_wp[k].tobytes() and x[0, 7:10].tobytes() == p.v_w[k].tobytes()
        assert (x[0, 10:13] == 0).all() and x[0, 13] == p.ftime[k]


def test_zero_length_steps_repeat_the_previous_pose(ref):
    """frame-tied streams: a sample on an interval end gives a step of dt == 0, whose pose repeats the previous one, its
    time and w_w included; w_w elsewhere is six times the step's mean world rate, so of the order of 6 |gyro|"""
    repeats = 0
    for name in ("stream_tied_ts0", "stream_tied_ts"):
        for x in R.ref_poses(ref, CASES[name]):
            same = np.all(x[1:] == x[:-1], axis=1)
            repeats += int(same.sum())
            if len(x) > 2:
                mean_rate = np.linalg.norm(x[1:, 10:13][~same], axis=1) / 6
                assert np.all(mean_rate < 10.0)
    assert repeats > 0


def test_time_offset_moves_a_sample_across_the_end(ref):
    before, after = R.ref_poses(ref, CASES["ts_before_end"]), R.ref_poses(ref, CASES["ts_after_end"])
    assert len(after[4]) == len(before[4]) - 1 and len(after[5]) == len(before[5]) + 1


def test_negated_quaternions_negate_only_the_quaternions():
    """the double cover: frames with negated quaternions give the same t, v_w, w_w and times, bit for bit, and the
    quaternions negated (the reference's pose update and rotation are odd and even in q)"""
    for n in imu_motion.NAMES:
        a, b = CASES[f"motion_{n}"], CASES[f"motion_{n}_flipped"]
        flipped = np.flatnonzero(np.any(a.T_wp[:, :4] != b.T_wp[:, :4], axis=1))
        assert len(flipped) > 0
        for pa, pb in ((R.oracle_poses(a), R.oracle_poses(b)), (R.mirror_poses(a), R.mirror_poses(b))):
            for k in range(a.n_frames - 1):
                x, y = pa[k], pb[k]
                assert x[:, 4:].tobytes() == y[:, 4:].tobytes(), (n, k)
                s = -1.0 if k in flipped else 1.0
                assert (x[:, :4] == s * y[:, :4]).all(), (n, k)
