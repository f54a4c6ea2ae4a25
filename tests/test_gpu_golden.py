"""CUDA kernels vs the committed mpmath known-answer vectors (tests/golden/), through the C-ABI."""
import os

import numpy as np
import pytest

import imu_streams
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("fixture", ["reproj_kat.npz", "reproj_edge_kat.npz"])  # edge: model branches, centre, border
@pytest.mark.parametrize("name", ["linear", "fov", "poly2", "poly3", "kb4"])
def test_reprojection_kernel_vs_kat(name, fixture):
    from vicalib_b200.capi import Calibrator

    z = np.load(os.path.join(GOLD, fixture))
    model = synth.MODEL_IDS[name]
    K = synth.NUM_INTR[model]
    d = {k[len(name) + 1:]: z[k] for k in z.files if k.startswith(name + "_")}
    n = d["r"].shape[0]
    # one camera per KAT row would need n cameras (>8): evaluate row by row instead
    for i in range(n):
        g = Calibrator()
        g.set_cameras([model], d["intr"][i][None], d["q_ck"][i][None], d["p_ck"][i][None])
        g.set_frames(d["T_wk"][i][None], np.zeros((1, 3)), np.zeros(1))
        g.set_observations([0], [0], d["p_w"][i][None], d["z"][i][None])
        r, J = g.eval_reproj()
        assert np.abs(r[0] - d["r"][i]).max() <= 1e-10 * max(1.0, np.abs(d["r"][i]).max())
        assert np.abs(J[0][:, :12 + K] - d["J"][i]).max() <= 1e-10 * np.abs(d["J"][i]).max()
        g.close()


# imu_edge_kat.npz: the interpolation buffer's edges (ties, no interior sample, the end-of-buffer clamp), switch 0 only
@pytest.mark.parametrize("fixture,switch", [("imu_kat.npz", 0), ("imu_kat.npz", 1), ("imu_edge_kat.npz", 0)], ids=["0", "1", "edge"])
def test_imu_kernel_vs_kat(fixture, switch):
    from vicalib_b200.capi import Calibrator

    z = np.load(os.path.join(GOLD, fixture))
    nf = len(z["ftime"])
    g = Calibrator()
    g.set_cameras([0], np.array([[300, 300, 320, 240, 0, 0, 0, 0, 0, 0.0]]), np.array([[0, 0, 0, 1.0]]), np.zeros((1, 3)))
    g.set_frames(z["T_wp"], z["v_w"], z["ftime"])
    g.set_observations(np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros((0, 3)), np.zeros((0, 2)))
    g.set_imu(z["imu_t"], z["imu_w"], z["imu_a"], synth.GYRO_SIGMA, synth.ACCEL_SIGMA)
    g.set_imu_params(z["g"], z["b"], z["sf"], float(z["ts"]))
    g.set_flags(inertial=1, rotation_only=switch, bias_active=1, scale_active=1, optimize_ts=1)
    g.set_imu_weights(np.broadcast_to(z["W"], (nf - 1, 9, 9)).copy())
    r, J = g.eval_imu()
    assert np.abs(r - z["r"][switch]).max() <= 1e-9 * np.abs(z["r"][switch]).max()
    Jz = z["J"][switch].copy()
    kink = imu_streams.ts_kinks(z)  # column 32 (ts) of intervals with a sample on an end
    J[kink, :, 32] = Jz[kink, :, 32] = 0.0
    assert np.abs(J - Jz).max() <= 1e-9 * np.abs(Jz).max()


def test_imu_weights_kernel_vs_kat():
    """imu_weights_kernel against the independent mpmath covariance propagation (see test_cpu_oracle_golden.py)."""
    from vicalib_b200.capi import Calibrator

    z = np.load(os.path.join(GOLD, "imu_weights_kat.npz"))
    g = Calibrator()
    g.set_cameras([0], np.array([[300, 300, 320, 240, 0, 0, 0, 0, 0, 0.0]]), np.array([[0, 0, 0, 1.0]]), np.zeros((1, 3)))
    g.set_frames(z["T_wp"], z["v_w"], z["ftime"])
    g.set_observations(np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros((0, 3)), np.zeros((0, 2)))
    g.set_imu(z["imu_t"], z["imu_w"], z["imu_a"], float(z["sigma_g"]), float(z["sigma_a"]))
    g.set_imu_params(z["g"], z["b"], z["sf"], float(z["ts"]))
    g.set_flags(inertial=1, bias_active=1, scale_active=1, optimize_ts=1)
    g.update_imu_weights()
    W = g.imu_weights()[0]
    assert np.abs(W - z["W"]).max() <= 1e-8 * np.abs(z["W"]).max()
