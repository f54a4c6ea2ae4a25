"""GPU: the inertial LM on the target workload (2 poly3 cameras, 2000 frames, IMU) is deterministic.

Two runs from the same start give the same state and cost bit for bit: every reduction of the persistent kernels adds in
a fixed order.  A run with the phase clocks on (vcgpu_set_profiling bit 3) gives the same bits as well: recording them
changes nothing the solve computes.
"""
import numpy as np
import pytest

from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
PHASE_CLOCKS = 8  # vcgpu_set_profiling bit 3
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
