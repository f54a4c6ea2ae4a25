"""GPU: the DOGLEG strategy on the device (vc_dogleg.cuh; the reference's solver setting,
vicalibrator.h:151) against the CPU oracle's DoglegStrategy restatement on identical seeded inputs.

The per-iteration trace must match: same accept/reject sequence, cost after every iteration to 1e-9
relative, trust-region radius to 1e-6 relative (the dogleg point is a ratio of small inner products);
solved parameters to 1e-6 relative (north_star's tolerance).  Rigs up to G = 104 (vision) and 127 (inertial): lanes
of arrow_matvec_frames_kernel that hold several global columns, both inertial engines.

With live IMU weights, the weights after the solve must be the oracle's, the last accepted step's update included: to
1e-7 relative per interval where a solve stops on an accepted step (the bar of
test_gpu_imu_parity.test_update_imu_weights_matches_oracle), to 1e-6 after the six-iteration inertial trace.
"""
import numpy as np
import pytest

import chain_plan
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, bias_active=1, scale_active=1, optimize_ts=1)
WEIGHTS_BAR = 1e-7


def _both(p, iters, inertial=False, **opts):
    from oracle.binding import Oracle
    from vicalib_b200.capi import Calibrator

    flags = ALL_ON if inertial else {}
    opts = dict(dict(max_iters=iters, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, strategy=1), **opts)
    o = Oracle(p, **flags)
    o.set_options(num_threads=8, **opts)
    so = o.solve()
    g = Calibrator()
    g.load(p)
    if inertial:
        g.set_flags(**flags)
    g.set_options(**opts)
    sg = g.solve()
    return o, so, g, sg


def _weights_rel(W, W_ref):
    """Largest per-interval relative difference of two sets of IMU weights."""
    return float((np.abs(W - W_ref).max((1, 2)) / np.abs(W_ref).max((1, 2))).max())


@pytest.mark.parametrize("models,intr_init,n_frames", [
    (("poly3",), "perturbed", 30), (("fov", "kb4"), "perturbed", 30), (("poly2",), "seed", 30),
    (chain_plan.rig_with_globals(51, False), "perturbed", 33), (chain_plan.rig_with_globals(104, False), "perturbed", 30),
], ids=["models0-perturbed", "models1-perturbed", "models2-seed", "G51_33f", "G104_30f"])
def test_dogleg_trace_matches_oracle(models, intr_init, n_frames):
    p = synth.make_problem(models=models, n_frames=n_frames, grid=(14, 10), seed=13, intr_init=intr_init)
    o, so, g, sg = _both(p, 6)  # converged to rounding after ~7 iterations; compare the descent
    ro, rg = so["rows"], sg["rows"]
    assert len(ro) == len(rg)
    # columns: iteration, cost, cost_change, gmax, gnorm, step_norm, rho, radius, successful
    assert np.array_equal(ro[:, 8], rg[:, 8]), "accept/reject sequence differs"
    assert np.abs(rg[:, 1] - ro[:, 1]).max() <= 1e-9 * ro[:, 1].max()
    assert np.abs(rg[:, 7] - ro[:, 7]).max() <= 1e-6 * ro[:, 7].max()
    xo, xg = o.state(), g.state()
    for k in ("intr", "q_ck", "p_ck", "T_wp"):
        assert np.abs(xg[k] - xo[k]).max() <= 1e-6 * max(np.abs(xo[k]).max(), 1.0), k


def test_dogleg_converges_like_lm():
    from vicalib_b200.capi import Calibrator

    p = synth.make_problem(models=("poly3",), n_frames=60, grid=(14, 10), seed=4)
    out = {}
    for strategy in (0, 1):
        g = Calibrator()
        g.load(p)
        g.set_options(max_iters=60, strategy=strategy)
        s = g.solve()
        out[strategy] = (s, g.state())
    (s0, x0), (s1, x1) = out[0], out[1]
    assert s1["termination"] in (1, 2, 3, 4), s1  # converged, not out of iterations
    assert abs(s1["final_cost"] - s0["final_cost"]) <= 1e-5 * s0["final_cost"]
    assert np.abs(x0["intr"] - x1["intr"]).max() <= 1e-3 * np.abs(x0["intr"]).max()


INERTIAL_RIGS = ((("poly3",), 24), (chain_plan.rig_with_globals(67), 33), (chain_plan.rig_with_globals(68), 37),
                 (chain_plan.rig_with_globals(127), 41))
INERTIAL_WEIGHTS_BAR = 1e-6  # largest measured 3.1e-8 (G = 28); a weight update left out moves them by >= 8.9e-5


def test_dogleg_inertial_matches_oracle():
    """The Gauss-Newton step of an inertial DOGLEG iteration is the chain solve's: the persistent one up to G = 67, the
    multi-launch engine's from G = 68 (rigs G = 28, 67, 68, 127).  Six iterations with live weights; state bars of
    test_gpu_imu_engines.test_deferred_weights_queue (the velocities, gravity, biases and scale factors are weakly
    observed over ~1 s of motion).  The weights follow the state, so they carry its differences along those weak
    directions: the bar is that of the full-size parity test."""
    for models, n_frames in INERTIAL_RIGS:
        p = synth.make_problem(models=models, n_frames=n_frames, grid=(14, 10), inertial=True, seed=17)
        o, so, g, sg = _both(p, 6, inertial=True)
        G = g.G
        assert G == chain_plan.rig_globals(models)
        ro, rg = so["rows"], sg["rows"]
        assert len(ro) == len(rg), G
        assert np.array_equal(ro[:, 8], rg[:, 8]), G
        assert np.abs(rg[:, 1] - ro[:, 1]).max() <= 1e-7 * ro[:, 1].max(), G
        xo, xg = o.state(), g.state()
        for k in ("T_wp", "q_ck", "p_ck", "intr"):
            assert np.abs(xg[k] - xo[k]).max() <= 1e-6 * max(np.abs(xo[k]).max(), 1.0), (G, k)
        weak = max(np.abs(xg[k] - xo[k]).max() for k in ("v_w", "g", "b", "sf"))
        rel = _weights_rel(g.imu_weights(), o.imu_weights())
        print(f"\nDOGLEG inertial G={G}: v_w / g / b / sf {weak:.1e}, weights {rel:.1e}")
        assert weak <= 2e-5, G
        assert rel <= INERTIAL_WEIGHTS_BAR, G


@pytest.mark.parametrize("stop", ["max_iters", "gradient_tol"])
def test_dogleg_last_weight_update_matches_oracle(stop):
    """A DOGLEG solve that ends on an accepted step (iteration limit, gradient tolerance) still runs the weight update
    the reference's iteration callback runs after it.  Without that update the weights stay those of the accepted
    step before, which differ from the oracle's by far more than the bar."""
    from oracle.binding import Oracle

    p = synth.make_problem(models=("poly3",), n_frames=24, grid=(14, 10), inertial=True, seed=17)
    live = dict(update_imu_weights=1)
    rows = _both(p, 8, inertial=True, **live)[1]["rows"]
    accepted = [int(r[0]) for r in rows[1:] if r[8] == 1]
    gmax = rows[:, 3]
    if stop == "max_iters":
        k, opts, term = accepted[-1], dict(max_iters=accepted[-1]), 0
    else:  # an accepted step that brings the largest gradient entry clearly below every earlier one
        k = next(it for it in accepted[1:] if gmax[it] < 0.99 * gmax[:it].min())
        opts, term = dict(max_iters=k + 4, gradient_tol=float(np.sqrt(gmax[k] * gmax[:k].min()))), 2
    o, so, g, sg = _both(p, opts.pop("max_iters"), inertial=True, **live, **opts)
    for s in (so, sg):
        assert int(s["iterations"]) == k and int(s["termination"]) == term and s["rows"][-1, 8] == 1
    W_o = o.imu_weights()
    rel = _weights_rel(g.imu_weights(), W_o)
    # the weights of the accepted step before
    j = max(it for it in accepted if it < k)
    o_j = Oracle(p, **ALL_ON)
    o_j.set_options(max_iters=j, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, strategy=1, num_threads=8, **live)
    o_j.solve()
    stale = _weights_rel(o_j.imu_weights(), W_o)
    print(f"\nDOGLEG stop on {stop} at iteration {k}: weights {rel:.1e}, one update {stale:.1e}")
    assert stale >= 1e3 * WEIGHTS_BAR
    assert rel <= WEIGHTS_BAR
