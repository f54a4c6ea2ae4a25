"""The plain DOGLEG reference (dogleg_ref.py) against the oracle's DoglegStrategy restatement, one iteration per branch.

The oracle's first row gives the model change as cost_change / rho and the radius it leaves; the reference predicts
both from the normal equations at the start point.  Largest measured (x86-64): model change 1.7e-12 relative, radius
3.2e-11 (the Gauss-Newton branch, where the radius grows to 3 |gn|: the oracle's block Cholesky is not refined).
"""
import pytest

import dogleg_ref
from vicalib_b200 import synth

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
MODEL_BAR = 1e-9
RADIUS_BAR = 3e-8


def one_iteration(p, flags, radius):
    from oracle.binding import Oracle

    o = Oracle(p, **flags)
    o.set_options(max_iters=1, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, init_radius=radius, strategy=1,
                  update_imu_weights=0)
    return o.solve()["rows"][1]


@pytest.mark.parametrize("inertial", [False, True], ids=["vision", "inertial"])
def test_reference_matches_oracle_dogleg_iteration(inertial):
    from oracle.binding import Oracle

    p = synth.make_problem(models=("poly3",), n_frames=12, grid=(14, 10), inertial=inertial, seed=31)
    flags = ALL_ON if inertial else {}
    ne = Oracle(p, **flags).normal_equations()
    scale = dogleg_ref.jacobi_scale(ne)
    radii = dogleg_ref.branch_radii(dogleg_ref.dogleg_step(ne, scale, 1e4))
    for branch, radius in radii.items():
        ref = dogleg_ref.dogleg_step(ne, scale, radius)
        assert ref["branch"] == branch
        row = one_iteration(p, flags, radius)
        rho = row[6]
        model = row[2] / rho
        assert abs(model - ref["model_change"]) <= MODEL_BAR * abs(ref["model_change"]), branch
        expected = dogleg_ref.radius_after(radius, rho, ref["step_norm"])
        assert abs(row[7] - expected) <= RADIUS_BAR * expected, branch
