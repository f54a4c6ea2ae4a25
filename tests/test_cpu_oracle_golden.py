"""Pins the oracle: CPU restatement (oracle/, float64 dual numbers, quaternion / Sophus-style code
paths) vs the committed known-answer vectors in tests/golden/, which come from an independent
60-digit mpmath restatement with rotation matrices and exact central differences
(tests/golden/make_golden.py).  The reference itself pins nothing for this path (SURVEY §0.4), so
this is the strongest pin available offline: parity stays "unpinned" w.r.t. a reference binary.
"""
import os

import numpy as np
import pytest

import imu_streams
from vicalib_b200 import synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _oracle_for_reproj(model, d, i):
    from oracle.binding import Oracle

    o = Oracle()
    K = synth.NUM_INTR[model]
    o.n_cams, o.n_frames, o.n_obs = 1, 1, 1
    o._obs_cam = np.zeros(1, dtype=np.int32)
    o.set_cameras([model], d["intr"][i][None], d["q_ck"][i][None], d["p_ck"][i][None])
    o.set_frames(d["T_wk"][i][None], np.zeros((1, 3)), np.zeros(1))
    import ctypes as C
    from oracle.binding import _c, _p

    o.L.vo_set_observations(o.h, C.c_int64(1), _p(_c([0], np.int32)), _p(_c([0], np.int32)), _p(_c(d["p_w"][i])), _p(_c(d["z"][i])))
    return o, K


# reproj_edge_kat.npz: each model's small-argument branches (FOV: rad^2 < 1e-5, w^2 <= 1e-5), image centre, border
@pytest.mark.parametrize("fixture", ["reproj_kat.npz", "reproj_edge_kat.npz"])
@pytest.mark.parametrize("name", ["linear", "fov", "poly2", "poly3", "kb4"])
def test_reprojection_kat(name, fixture):
    z = np.load(os.path.join(GOLD, fixture))
    model = synth.MODEL_IDS[name]
    d = {k[len(name) + 1:]: z[k] for k in z.files if k.startswith(name + "_")}
    for i in range(d["r"].shape[0]):
        o, K = _oracle_for_reproj(model, d, i)
        r, J = o.eval_reproj()
        assert np.abs(r[0] - d["r"][i]).max() <= 1e-10 * max(1.0, np.abs(d["r"][i]).max())
        Jg = d["J"][i]
        assert np.abs(J[0][:, :12 + K] - Jg).max() <= 1e-10 * np.abs(Jg).max()


# imu_edge_kat.npz (switch 0 only): ties at both ends, intervals without an interior sample, an end moved across a sample
# by ts, an interval ending past the last sample
@pytest.mark.parametrize("fixture,switch", [("imu_kat.npz", 0), ("imu_kat.npz", 1), ("imu_edge_kat.npz", 0)], ids=["0", "1", "edge"])
def test_imu_kat(fixture, switch):
    from oracle.binding import Oracle

    z = np.load(os.path.join(GOLD, fixture))
    nf = len(z["ftime"])
    p = synth.make_problem(models=("linear",), n_frames=nf, inertial=True, seed=1)
    p.T_wp, p.v_w, p.ftime = z["T_wp"].copy(), z["v_w"].copy(), z["ftime"].copy()
    p.imu_t, p.imu_w, p.imu_a = z["imu_t"].copy(), z["imu_w"].copy(), z["imu_a"].copy()
    p.g, p.b, p.sf, p.ts = z["g"].copy(), z["b"].copy(), z["sf"].copy(), float(z["ts"])
    o = Oracle(p, inertial=1, rotation_only=switch, bias_active=1, scale_active=1, optimize_ts=1)
    o.set_imu_weights(np.broadcast_to(z["W"], (nf - 1, 9, 9)).copy())
    r, J = o.eval_imu()
    assert np.abs(r - z["r"][switch]).max() <= 1e-9 * np.abs(z["r"][switch]).max()
    Jz = z["J"][switch].copy()
    kink = imu_streams.ts_kinks(z)  # column 32 (ts) of intervals with a sample on an end
    J[kink, :, 32] = Jz[kink, :, 32] = 0.0
    assert np.abs(J - Jz).max() <= 1e-9 * np.abs(Jz).max()


def test_imu_weights_kat():
    """UpdateImuWeights against an independent computation: tests/golden/make_weights_golden.py propagates the
    covariance with exact (mpmath, central-difference) Jacobians of the integrator and of the residual map — none
    of the reference's hand-derived derivative formulas — with unit scale factors, where those formulas are exact
    up to the truncated series of d exp(w)/dw.  Measured agreement 7e-11; tolerance 1e-8 relative."""
    from oracle.binding import Oracle

    z = np.load(os.path.join(GOLD, "imu_weights_kat.npz"))
    p = synth.make_problem(models=("linear",), n_frames=2, inertial=True, seed=1)
    p.T_wp, p.v_w, p.ftime = z["T_wp"].copy(), z["v_w"].copy(), z["ftime"].copy()
    p.imu_t, p.imu_w, p.imu_a = z["imu_t"].copy(), z["imu_w"].copy(), z["imu_a"].copy()
    p.g, p.b, p.sf, p.ts = z["g"].copy(), z["b"].copy(), z["sf"].copy(), float(z["ts"])
    assert synth.GYRO_SIGMA == float(z["sigma_g"]) and synth.ACCEL_SIGMA == float(z["sigma_a"])
    o = Oracle(p, inertial=1, bias_active=1, scale_active=1, optimize_ts=1)
    o.update_imu_weights()
    W = o.imu_weights()[0]
    assert np.abs(W - z["W"]).max() <= 1e-8 * np.abs(z["W"]).max()
    assert np.abs(W @ W - z["info"]).max() <= 1e-8 * np.abs(z["info"]).max()
