"""GPU: one DOGLEG iteration (vc_dogleg.cuh) against a plain long-double reference (dogleg_ref.py), on the shapes where
its kernels take their longer paths, once per branch of the dogleg point.

Shapes (rigs and frame counts from chain_plan.py):
- vision (fd = 6) with G = 10, 32, 33, 51 and 104: arrow_matvec_frames_kernel's lanes hold up to four global columns;
  9, 10, 15 and 20 frames give every frame count mod kMvWarps and an odd number of per-CTA partials for
  arrow_matvec_globals_kernel's pairwise sum;
- vision with 3000 frames x 1 fov (18 011 entries): dl_dots_kernel's slices take a second pass;
- inertial (fd = 9) with G = 28, 41, 67, 68 and 127: 67 is the last rig of the persistent chain solve, 68 the first
  of the multi-launch engine; 2 and 3 frames (the dense solve alone); 2113 frames (a wide level 0 in two rounds);
- one case without Jacobi scaling.

Each case runs with max_iters = 1, all tolerances 0 and fixed IMU weights (the normal equations taken before the solve
are the ones its iteration uses).  The reference picks one radius per branch: 1.5 |gn| (Gauss-Newton step),
0.5 alpha |g~| (clipped Cauchy step) and their geometric mean (dogleg segment).  Each run is checked three ways:
- the model change, cost_change / rho of the device's row, against the reference's;
- the radius the iteration leaves: max(R, 3 |step~|), R or R / 2 by rho (in the Gauss-Newton branch: 3 |gn|);
- the state, against the oracle's after its own one-iteration DOGLEG solve at the same initial radius.
Every step is accepted (rho > 1 on these problems), so a step the device finds invalid fails the test outright.
The bars sit about 1e3 above the largest errors measured on an H100 80GB HBM3 (700 W): model change 2.5e-10 (segment
branch, G = 104), radius 1.8e-9 (Gauss-Newton branch, G = 104: |gn| of a system regularised by mu = 1e-8 only), state
7.1e-8 (Gauss-Newton branch, 3 inertial frames: the oracle's step is not refined, and the IMU globals of so short a
chain are weakly observed).  The added tests take ~10 s in all.
"""
import os

import numpy as np
import pytest

import chain_plan
import dogleg_ref
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
MODEL_BAR = 3e-7    # largest measured 2.5e-10
RADIUS_BAR = 2e-6   # largest measured 1.8e-9
STATE_BAR = 1e-4    # largest measured 7.1e-8

SMS, SMEM_OPTIN = chain_plan.device_or_h100()
VISION = ((10, 9), (32, 10), (33, 15), (51, 20), (104, 9))      # (G, frames)
INERTIAL = ((28, 33), (41, 35), (67, 37), (68, 39), (127, 41))
LONG_VISION = 3000
WIDE_FRAMES = next(n for n, claims in chain_plan.chain_cases(SMS) if "wide0_rounds2" in claims)


def _case(name, models, n_frames, inertial, grid=(14, 10), jacobi=1):
    return pytest.param(models, n_frames, grid, inertial, jacobi, id=name)


CASES = (
    [_case(f"vision_G{G}_{n}f", chain_plan.rig_with_globals(G, False), n, False) for G, n in VISION]
    + [_case(f"vision_{LONG_VISION}f", ("fov",), LONG_VISION, False, grid=(4, 3))]
    + [_case(f"inertial_G{G}_{n}f", chain_plan.rig_with_globals(G), n, True) for G, n in INERTIAL]
    + [_case(f"inertial_{n}f", ("poly3",), n, True) for n in (2, 3)]
    + [_case(f"inertial_{WIDE_FRAMES}f", ("poly2",), WIDE_FRAMES, True, grid=(4, 3))]
    + [_case("vision_G33_15f_unscaled", chain_plan.rig_with_globals(33, False), 15, False, jacobi=0)]
)


def test_cases_reach_the_kernel_paths():
    frames = [n for _, n in VISION]
    assert {n % chain_plan.MV_WARPS for n in frames} == set(range(chain_plan.MV_WARPS))
    assert any(chain_plan.matvec_parts(n) % 2 for n in frames)
    assert max(G for G, _ in VISION) > 3 * 32  # a lane of arrow_matvec_frames_kernel holds four columns
    assert chain_plan.dot_passes(LONG_VISION * 6 + chain_plan.rig_globals(("fov",), False)) >= 2
    assert chain_plan.dot_passes(max(n * 9 + G for G, n in INERTIAL)) == 1
    assert chain_plan.persistent_fits(67, 37, SMEM_OPTIN) and not chain_plan.persistent_fits(68, 39, SMEM_OPTIN)
    assert {"wide0_rounds2", "levels4"} <= chain_plan.branches(WIDE_FRAMES, SMS)


def _opts(jacobi, radius=1e4):
    return dict(max_iters=1, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, strategy=1, update_imu_weights=0,
                jacobi_scaling=jacobi, init_radius=radius)


def _calibrator(p, flags, opts):
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.load(p)
    if flags:
        g.set_flags(**flags)
    g.set_options(**opts)
    return g


def _state_err(st_g, st_o, keys):
    return max(np.abs(np.asarray(st_g[k]) - st_o[k]).max() / max(np.abs(st_o[k]).max(), 1.0) for k in keys)


@pytest.mark.parametrize("models,n_frames,grid,inertial,jacobi", CASES)
def test_dogleg_iteration_matches_reference(models, n_frames, grid, inertial, jacobi):
    from oracle.binding import Oracle

    p = synth.make_problem(models=models, n_frames=n_frames, grid=grid, inertial=inertial, seed=41)
    flags = ALL_ON if inertial else {}
    g = _calibrator(p, flags, _opts(jacobi))
    ne = g.normal_equations()
    assert g.fd == (9 if inertial else 6) and g.G == chain_plan.rig_globals(models, inertial)
    n = n_frames * g.fd + g.G
    scale = dogleg_ref.jacobi_scale(ne) if jacobi else np.ones(n)
    radii = dogleg_ref.branch_radii(dogleg_ref.dogleg_step(ne, scale, 1e4))
    keys = ("intr", "q_ck", "p_ck", "T_wp") + (("v_w", "g", "b", "sf", "ts") if inertial else ())
    errs = {}
    for branch, radius in radii.items():
        ref = dogleg_ref.dogleg_step(ne, scale, radius)
        assert ref["branch"] == branch
        g = _calibrator(p, flags, _opts(jacobi, radius))
        s = g.solve()
        assert s["iterations"] == 1
        row = s["rows"][1]
        assert row[8] == 1, f"{branch} step not accepted (rho {row[6]})"
        rho = row[6]
        model = row[2] / rho
        expected = dogleg_ref.radius_after(radius, rho, ref["step_norm"])
        o = Oracle(p, **flags)
        o.set_options(num_threads=os.cpu_count() or 4, **_opts(jacobi, radius))
        o.solve()
        errs[branch] = (abs(model - ref["model_change"]) / abs(ref["model_change"]), abs(row[7] - expected) / expected,
                        _state_err(g.state(), o.state(), keys), rho)
    print(f"\nDOGLEG G={g.G} nf={n_frames}: " + ", ".join(
        f"{b} model {m:.1e} radius {r:.1e} state {x:.1e} (rho {rho:.2f})" for b, (m, r, x, rho) in errs.items()))
    for branch, (m, r, x, _) in errs.items():
        assert m <= MODEL_BAR, (branch, m)
        assert r <= RADIUS_BAR, (branch, r)
        assert x <= STATE_BAR, (branch, x)
