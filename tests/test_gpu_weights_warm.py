"""GPU: warm-started UpdateImuWeights eigen-decompositions.

Each interval's Jacobi eigen-decomposition of P starts from the eigenvectors of its last update.  W = V L^-1/2 V^T does
not depend on which orthogonal V diagonalises P, so a warm update equals a cold one (from the identity) to rounding.
Every comparison takes the weights a SOLVE left — its updates ran at a sequence of accepted states, each one started
from the vectors of the state before — and compares them with one cold update at the same state:
- solves of 1 to 200 iterations on both inertial engines (200: the vectors' drift from orthogonal over a long solve);
- a first step that is one large jump (velocities of the start perturbed by 0.5 m/s, a Gauss-Newton-sized radius);
- a stationary rig at the identity orientation, where P's eigenvalues come in nearly equal pairs and the vectors of
  the state before are arbitrary inside those pairs' planes.
The singular branch (zero IMU noise: P = 0) leaves the weights untouched, cold and warm.
Cold starts: a load alone (vcgpu_set_cameras / _frames / _imu / _imu_params), and the start of a solve without any
upload, each give the bits of a cold start.

A cold update is forced without touching the state or the weights: vcgpu_set_imu_weights marks the vectors cold.
"""
import dataclasses

import numpy as np
import pytest

from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
MULTI_LAUNCH = 4  # vcgpu_set_profiling bit 2
# relative to max |W|: about 1e3 above the largest warm-vs-cold difference measured on an H100 80GB HBM3 (700 W)
WARM_BAR = 1e-8


def _problem(n_frames=64, seed=5):
    return synth.make_problem(models=("poly3", "poly3"), n_frames=n_frames, grid=(14, 10), inertial=True, seed=seed)


def _calibrator(p, mode=0, **opts):
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.load(p)
    g.set_flags(**ALL_ON)
    o = dict(function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
    o.update(opts)
    g.set_options(**o)
    g.set_profiling(mode, False)
    return g


def _solve_vs_cold(g):
    """The weights the solve left (warm-started updates) and one cold update at the same state, relative max diff."""
    s = g.solve()
    w_solve = g.imu_weights().copy()
    g.set_imu_weights(w_solve)  # same weights, vectors marked cold
    g.update_imu_weights()
    w_cold = g.imu_weights().copy()
    assert np.all(np.isfinite(w_cold))
    return s, np.abs(w_solve - w_cold).max() / np.abs(w_cold).max()


@pytest.mark.parametrize("mode", [0, MULTI_LAUNCH], ids=["persistent", "multi_launch"])
def test_solve_weights_equal_cold(mode):
    p = _problem()
    for iters in (1, 2, 5, 30, 200):
        s, err = _solve_vs_cold(_calibrator(p, mode, max_iters=iters))
        assert s["successful_steps"] >= 1
        print(f"iters {iters} ({s['successful_steps']} accepted): max |W_solve - W_cold| / max |W| = {err:.3e}")
        assert err <= WARM_BAR


def test_large_jump():
    p = _problem()
    rng = np.random.default_rng(3)
    p = dataclasses.replace(p, v_w=p.v_w + 0.5 * rng.standard_normal(p.v_w.shape))
    g = _calibrator(p, max_iters=2, init_radius=1e16)
    before = g.state()["v_w"].copy()
    s, err = _solve_vs_cold(g)
    jump = np.abs(g.state()["v_w"] - before).max()
    print(f"large jump: max |dv| = {jump:.3f} m/s, {s['successful_steps']} accepted, rel diff {err:.3e}")
    assert s["successful_steps"] >= 1 and jump > 0.1
    assert err <= WARM_BAR


def test_nearly_repeated_eigenvalues():
    p = _problem(n_frames=32)
    nf, n_imu = p.T_wp.shape[0], p.imu_t.shape[0]
    T = np.zeros((nf, 7))
    T[:, 3] = 1.0  # identity orientation, at the origin
    acc = np.tile([0.0, 0.0, 9.80665], (n_imu, 1))
    p = dataclasses.replace(p, T_wp=T, v_w=np.zeros((nf, 3)), imu_w=np.zeros((n_imu, 3)), imu_a=acc,
                            b=np.zeros_like(p.b), sf=np.ones_like(p.sf))
    for iters in (1, 3):
        s, err = _solve_vs_cold(_calibrator(p, max_iters=iters))
        print(f"stationary rig, {iters} iterations ({s['successful_steps']} accepted): rel diff {err:.3e}")
        assert err <= WARM_BAR
    g = _calibrator(p)  # and at the symmetric state itself: cold, then warm from its own vectors
    g.update_imu_weights()
    w1 = g.imu_weights().copy()
    g.update_imu_weights()
    assert np.abs(g.imu_weights() - w1).max() <= WARM_BAR * np.abs(w1).max()


def test_singular_branch_leaves_weights():
    from vicalib_b200.synth import ACCEL_SIGMA, GYRO_SIGMA

    p = _problem(n_frames=16)
    g = _calibrator(p)
    g.set_imu(p.imu_t, p.imu_w, p.imu_a, 0.0, 0.0)  # no noise: P = 0
    w0 = np.tile(np.diag(np.arange(1.0, 10.0)), (p.n_frames - 1, 1, 1))
    g.set_imu_weights(w0)
    g.update_imu_weights()  # cold
    assert np.array_equal(g.imu_weights(), w0)
    g.update_imu_weights()  # warm
    assert np.array_equal(g.imu_weights(), w0)
    g.set_imu(p.imu_t, p.imu_w, p.imu_a, GYRO_SIGMA, ACCEL_SIGMA)
    g.update_imu_weights()
    assert not np.array_equal(g.imu_weights(), w0)


def test_load_alone_starts_cold():
    p = _problem()
    fresh = _calibrator(p)
    fresh.update_imu_weights()
    w_fresh = fresh.imu_weights().copy()
    g = _calibrator(p, max_iters=10)
    g.solve()
    g.update_imu_weights()  # leaves warm vectors of another state behind
    g.load(p)               # flags untouched: only the uploads mark the vectors cold
    g.update_imu_weights()
    assert np.array_equal(g.imu_weights(), w_fresh)


def test_solve_starts_cold_without_upload():
    p = _problem()
    g = _calibrator(p, max_iters=6)
    g.solve()
    g.update_imu_weights()  # warm vectors of the solved state; the next solve must not start from them
    st, w = g.state(), g.imu_weights().copy()
    s2 = g.solve()          # no upload in between
    p2 = dataclasses.replace(p, T_wp=st["T_wp"], v_w=st["v_w"], intr=st["intr"], q_ck=st["q_ck"], p_ck=st["p_ck"],
                             g=st["g"], b=st["b"], sf=st["sf"], ts=float(np.ravel(st["ts"])[0]))
    h = _calibrator(p2, max_iters=6)
    h.set_imu_weights(w)
    s3 = h.solve()
    assert s2["iterations"] == s3["iterations"] and s2["final_cost"] == s3["final_cost"]
    assert np.array_equal(g.imu_weights(), h.imu_weights())
    for k in ("T_wp", "v_w", "intr", "g", "b", "sf"):
        assert np.array_equal(g.state()[k], h.state()[k]), k
