"""GPU: how many CTAs stay with the inertial solve, and so which CTAs take the deferred weight tasks and the
back-substitution items, changes nothing in what the solve computes.

Rigs on each branch of the host's rule (solver_plan.solver_ctas): weight tasks in one round on a 64-frame rig (128
of 132 CTAs stay with the solve on an H100) and on the 2000-frame target shape (7 stay), the fallback to 8 on 2500
frames (157 tasks), and VCGPU_N_SOLVER set.  Each run is a subprocess (the variable is read once per process); its
weights and state after four LM iterations with live weights must be bit for bit those of the same build with
VCGPU_N_SOLVER=8.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import chain_plan
import solver_plan

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMS, _ = chain_plan.device_or_h100()
ITERS = 4
KEYS = ("T_wp", "v_w", "q_ck", "p_ck", "intr", "g", "b", "sf", "ts")
_RUN = """
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from vicalib_b200 import synth
from vicalib_b200.capi import Calibrator
p = synth.make_problem(models=("poly3",), n_frames=int(sys.argv[2]), grid=(4, 3), inertial=True, seed=31)
g = Calibrator()
g.load(p)
g.set_flags(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
g.set_options(max_iters={it}, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, update_imu_weights=1)
s = g.solve()
st = g.state()
np.savez(sys.argv[3], W=g.imu_weights(), **{{k: np.asarray(st[k]) for k in {keys!r}}})
print(s["kernel_launches"], s["iterations"], s["successful_steps"])
""".format(it=ITERS, keys=KEYS)


def _solve(tmp_path, n_frames, n_solver):
    env = dict(os.environ)
    env.pop("VCGPU_N_SOLVER", None)
    if n_solver is not None:
        env["VCGPU_N_SOLVER"] = str(n_solver)
    out_file = tmp_path / f"run_{n_frames}_{n_solver}.npz"
    out = subprocess.run([sys.executable, "-c", _RUN, ROOT, str(n_frames), str(out_file)], env=env, capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    launches, iters, accepted = (int(v) for v in out.stdout.split()[-3:])
    assert iters == ITERS and launches <= 2 * iters + 12, (launches, iters)  # the persistent inertial kernels ran
    assert accepted >= 2, accepted  # an iteration after an accepted step: the weights queue ran
    with np.load(out_file) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("n_frames,n_solver,branch", [
    (64, None, "one round"),
    (2000, None, "one round"),
    (2500, None, "fallback"),
    (2000, 3, "set"),
], ids=["64-one_round", "2000-one_round", "2500-fallback", "2000-set3"])
def test_solver_ctas_change_no_bit(tmp_path, n_frames, n_solver, branch):
    if branch == "one round":
        assert solver_plan.weight_rounds(n_frames, SMS) == 1 and solver_plan.solver_ctas(n_frames, SMS) != 8
    elif branch == "fallback":
        assert solver_plan.solver_ctas(n_frames, SMS) == chain_plan.n_solver(n_frames, SMS)
        assert solver_plan.weight_rounds(n_frames, SMS) > 1
    got = _solve(tmp_path, n_frames, n_solver)
    ref = _solve(tmp_path, n_frames, 8)
    assert np.abs(ref["W"] - 500 * np.eye(9)).max() > 1.0  # the weights did change
    for k in ("W",) + KEYS:
        assert np.array_equal(got[k], ref[k]), (k, np.abs(got[k] - ref[k]).max())
