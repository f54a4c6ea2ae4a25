"""GPU: the inertial LM on the target workload (2 poly3 cameras, 2000 frames, IMU) is deterministic.

Two runs from the same start give the same state and cost bit for bit: every reduction of the persistent kernels adds in
a fixed order.  A run with the phase clocks on (vcgpu_set_profiling bit 3) gives the same bits as well: recording them
changes nothing the solve computes.

A free-running solve (no iteration callback) gives the bits of the same solve with one, on both strategies and engines.
"""
import numpy as np
import pytest

from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
PHASE_CLOCKS = 8  # vcgpu_set_profiling bit 3
MULTI_LAUNCH = 4  # vcgpu_set_profiling bit 2
STATE_KEYS = ("T_wp", "v_w", "q_ck", "p_ck", "intr", "g", "b", "sf")


def _run(p, mode):
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.load(p)
    g.set_flags(**ALL_ON)
    g.set_options(max_iters=8, function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
    g.set_profiling(mode, False)
    s = g.solve()
    assert s["kernel_launches"] <= 2 * s["iterations"] + 12, "the persistent inertial kernels did not run"
    return s, g.state()


@pytest.mark.parametrize("mode", [0, MULTI_LAUNCH], ids=["persistent", "multi_launch"])
@pytest.mark.parametrize("inertial", [False, True], ids=["vision", "inertial"])
@pytest.mark.parametrize("strategy", [0, 1], ids=["lm", "dogleg"])
def test_free_running_solve_is_bit_identical(strategy, inertial, mode):
    """Without an iteration callback the host enqueues iterations in batches (the persistent vision LM: the whole loop
    in one launch) and looks at the control block only between them, so iterations are queued after the one that ends
    the solve; they do nothing.  The same kernels run in the same order as with a callback: the same bits."""
    from vicalib_b200.capi import Calibrator

    p = synth.make_problem(models=("poly3",), n_frames=30 if inertial else 40, grid=(14, 10), inertial=inertial, seed=8)
    out = []
    for free_running in (False, True):
        g = Calibrator()
        g.load(p)
        if inertial:
            g.set_flags(**ALL_ON)
        # converges by the function tolerance within 50 iterations (live weights make the inertial cost creep at 1e-6)
        g.set_options(max_iters=50, strategy=strategy, update_imu_weights=1, function_tol=1e-5 if inertial else 1e-6)
        g.set_profiling(mode, False)
        s = g.solve(free_running=free_running)
        out.append((s, g.state(), g.imu_weights() if inertial else None))
    (s0, st0, w0), (s1, st1, w1) = out
    assert s0["termination"] in (1, 2, 3, 4) and len(s0["rows"]) == s0["iterations"] + 1 and len(s1["rows"]) == 0
    for k in ("iterations", "successful_steps", "termination", "final_cost"):
        assert s1[k] == s0[k], k
    for k in STATE_KEYS:
        assert np.array_equal(st1[k], st0[k]), k
    assert st1["ts"] == st0["ts"]
    if inertial:
        assert np.array_equal(w1, w0)


def test_target_solve_is_bit_identical():
    p = synth.make_config("target")
    s0, st0 = _run(p, 0)
    s1, st1 = _run(p, 0)
    s2, st2 = _run(p, PHASE_CLOCKS)
    assert s0["successful_steps"] > 0
    for s, st in ((s1, st1), (s2, st2)):
        assert s["successful_steps"] == s0["successful_steps"] and s["iterations"] == s0["iterations"]
        assert s["final_cost"] == s0["final_cost"]
        for k in STATE_KEYS:
            assert np.array_equal(st[k], st0[k]), k
