"""GPU: the IMU Jacobian of vcgpu_eval_imu against the oracle, column by column, for each of the four ways the device
forms a column.  imu_eval_kernel evaluates three intervals per warp, a team of 10 lanes each: a lane carries one
attitude-coupled direction through the RK4 chain as a dual number; the (p, v)-only directions (pose1 translation, v1,
gravity, accelerometer bias and scale) ride beside it in plain doubles; the pose2 directions need only the end map;
the v2 columns are analytic.

Covered: interval counts 3k, 3k+1 and 3k+2 (the last warp holds one, two or three teams), warps whose intervals take
different numbers of RK4 steps (jittered and dropped-frame streams), the rotation-only switch, time offsets that move an
interval end across a sample, and masked IMU globals in the normal equations of both solve engines.
"""
import numpy as np
import pytest

import imu_streams
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
KINDS = {
    "attitude": (9, 10, 11, 20, 21, 22, 26, 27, 28, 32),  # pose1 rotation, gyro bias, gyro scale, ts
    "pv_only": (6, 7, 8, 15, 16, 17, 18, 19, 23, 24, 25, 29, 30, 31),  # pose1 translation, v1, g, accel bias, accel scale
    "end_map": (0, 1, 2, 3, 4, 5),  # pose2
    "analytic": (12, 13, 14),  # v2
}
assert sorted(c for cols in KINDS.values() for c in cols) == list(range(33))


def _weights(ni, seed=11):
    """symmetric, positive definite, distinct per interval and dense: every raw row reaches every weighted row"""
    rng = np.random.default_rng(seed)
    W = 3.0 * rng.standard_normal((ni, 9, 9))
    return 0.5 * (W + W.transpose(0, 2, 1)) + np.arange(400.0, 409.0) * np.eye(9)


def _pair(p, flags=ALL_ON):
    from oracle.binding import Oracle
    from vicalib_b200.capi import Calibrator

    o = Oracle(p, **flags)
    g = Calibrator()
    g.load(p)
    g.set_flags(**flags)
    W = _weights(p.n_frames - 1)
    o.set_imu_weights(W)
    g.set_imu_weights(W)
    return o, g


def _check_columns(o, g):
    r_o, J_o = o.eval_imu()
    r_g, J_g = g.eval_imu()
    assert np.abs(r_g - r_o).max() <= 1e-9 * max(np.abs(r_o).max(), 1.0)
    scale = np.abs(J_o).max()
    assert scale > 0.0
    for kind, cols in KINDS.items():
        for c in cols:
            ref = J_o[:, :, c]
            # each column against its own size (floored well below the Jacobian's: rows the weights leave tiny)
            tol = 1e-9 * max(np.abs(ref).max(), 1e-4 * scale)
            err = np.abs(J_g[:, :, c] - ref).max()
            assert err <= tol, f"{kind} column {c}: {err:.3e} > {tol:.3e}"
    return J_o, J_g


@pytest.mark.parametrize("n_frames", [10, 11, 12])  # 9, 10, 11 intervals: 3, 1 and 2 teams in the last warp
def test_columns_by_interval_count(n_frames):
    p = synth.make_problem(models=("poly3",), n_frames=n_frames, grid=(10, 7), inertial=True, seed=41, ts_truth=0.003)
    _check_columns(*_pair(p))


@pytest.mark.parametrize("name", ["jittered", "dropped"])
def test_columns_mixed_step_counts(name):
    s = imu_streams.build(name)
    p = imu_streams.perturbed(s.p)
    steps = np.asarray(imu_streams.classify(p)["steps"])
    ni = p.n_frames - 1
    warps = [steps[w: w + 3] for w in range(0, ni, 3)]
    assert any(len(set(w.tolist())) > 1 for w in warps), "no warp mixes step counts"
    _check_columns(*_pair(p))


def test_columns_rotation_only():
    p = synth.make_problem(models=("poly3",), n_frames=11, grid=(10, 7), inertial=True, seed=42, ts_truth=0.002)
    flags = dict(inertial=1, rotation_only=1, bias_active=0, scale_active=0, optimize_ts=1)
    _, J_g = _check_columns(*_pair(p, flags))
    assert not J_g[:, :3].any() and not J_g[:, 6:].any()  # rows 0-2 and 6-8 switched off


@pytest.mark.parametrize("mode", [0, 4], ids=["persistent", "multi_launch"])  # vcgpu_set_profiling bit 2
def test_masked_globals(mode):
    """vcgpu_eval_imu returns every column; the solve engines mask the inactive IMU globals (accelerometer and gyro
    biases, ts here) in the Jacobian before its products: their columns of E are zero, the blocks match the oracle"""
    p = synth.make_problem(models=("poly3",), n_frames=12, grid=(10, 7), inertial=True, seed=43, ts_truth=0.002)
    flags = dict(inertial=1, rotation_only=0, bias_active=0, scale_active=1, optimize_ts=0)
    o, g = _pair(p, flags)
    g.set_profiling(mode, False)
    ne_o, ne_g = o.normal_equations(), g.normal_equations()
    for k in ("B", "U", "E", "gf", "C", "gc"):
        assert np.abs(ne_g[k] - ne_o[k]).max() <= 1e-10 * np.abs(ne_o[k]).max(), k
    imu = ne_g["E"].shape[2] - 15  # the 15 IMU globals close the global block: g 2, b 6, sf 6, ts
    off = [imu + 2 + i for i in range(6)] + [imu + 14]
    assert not ne_g["E"][:, :, off].any()
    assert np.abs(ne_g["E"][:, :, imu + 8: imu + 14]).max() > 0.0


@pytest.mark.parametrize("ts", [-0.0049, 0.0, 0.00251, 0.0074])
def test_columns_time_offset_across_samples(ts):
    p = synth.make_problem(models=("poly3",), n_frames=10, grid=(10, 7), inertial=True, seed=5)
    p.ts = ts
    o, g = _pair(p)
    o.set_imu_params(p.g, p.b, p.sf, ts)
    g.set_imu_params(p.g, p.b, p.sf, ts)
    _check_columns(o, g)
