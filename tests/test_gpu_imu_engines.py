"""GPU: the two inertial engines on the LM path, and the rigs at the edges of what each one takes.

- The persistent kernels (chain_solve_kernel + eval_mega_kernel) against the multi-launch engine (vc_chain.cuh, selected
  with vcgpu_set_profiling bit 2) after a fixed number of iterations: the same accepted-step count, cost within 1e-10,
  state within 1e-8.  Shapes: G = 41; G = 67 with 256 frames (4 top nodes: N = 103 takes the 7-tile dense L D L^T); a
  chain that needs a wide level 0 in two rounds and four elimination levels; two cameras that miss frames, and one
  camera, with a frame no camera sees.
- The normal equations of both engines' reprojection builds on those last two rigs, against the oracle.
- The persistent engine's fit boundary: G = 67 runs persistent, G = 68 multi-launch; both against the oracle.
- The largest rigs vcgpu_set_cameras accepts (G = 127 and 122), with 4 top nodes and with 1, on the multi-launch engine.
- The deferred weights queue with more 16-interval tasks than CTAs leaving the solve, against the oracle, the
  multi-launch engine, and the same run with every CTA but one kept in the solve (bit for bit) and with the weights
  computed in the evaluation launch instead (to rounding).  The weights are compared after the solve: the update the
  last accepted step calls for must have run on every path.
- The same without an oracle, on both strategies and engines and whatever ends the solve: one more update after the
  solve leaves the weights as they are.

Which frame counts reach which branch comes from the host model of the plan (chain_plan.py).
"""
import dataclasses
import os
import subprocess
import sys

import numpy as np
import pytest

import chain_plan
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
MULTI_LAUNCH = 4  # vcgpu_set_profiling bit 2
STATE_KEYS = ("T_wp", "v_w", "q_ck", "p_ck", "intr", "g", "b", "sf")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SMS, SMEM_OPTIN = chain_plan.device_or_h100()


def _persistent_ran(s):
    """Two cooperative launches per iteration plus a fixed set-up; the multi-launch engine takes ~20 per iteration."""
    return s["kernel_launches"] <= 2 * s["iterations"] + 12


def _calibrator(p, mode=0, **opts):
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.load(p)
    g.set_flags(**ALL_ON)
    g.set_options(**opts)
    g.set_profiling(mode, False)
    return g


UNSEEN_FRAME = 50


def _missing_frames(p):
    """test_gpu_persistent.test_cameras_missing_frames' observations: camera 1 misses every third frame, camera 0 every
    seventh, and no camera sees frame UNSEEN_FRAME (on a one-camera rig, only that)"""
    keep = p.obs_frame != UNSEEN_FRAME
    if p.n_cams > 1:
        keep &= ~((p.obs_cam == 1) & (p.obs_frame % 3 == 0)) & ~((p.obs_cam == 0) & (p.obs_frame % 7 == 2))
    return dataclasses.replace(p, obs_frame=p.obs_frame[keep], obs_cam=p.obs_cam[keep], p_w=p.p_w[keep], p_c=p.p_c[keep],
                               grid_idx=p.grid_idx[keep])


MISSING_RIGS = [("poly3", "fov"), ("poly3",)]
ENGINE_CASES = [
    (("poly3", "poly3"), 200, (14, 10), False),                                              # G = 41
    (("poly3",) * 4, chain_plan.TOP * chain_plan.CHUNK ** 2, (14, 10), False),               # G = 67, 4 top nodes
    (("poly3",), chain_plan.CHUNK * SMS * chain_plan.GROUPS + 1, (4, 3), False),             # wide level 0, 2 rounds
    (MISSING_RIGS[0], 120, (14, 10), True),                                                  # cameras that miss frames
    (MISSING_RIGS[1], 120, (14, 10), True),                                                  # one camera, a frame unseen
]


@pytest.mark.parametrize("models,n_frames,grid,missing", ENGINE_CASES,
                         ids=["G41", "G67_top4", "wide0_rounds2", "missing_frames", "unseen_frame"])
def test_persistent_matches_multi_launch(models, n_frames, grid, missing):
    G = chain_plan.rig_globals(models)
    assert chain_plan.persistent_fits(G, n_frames, SMEM_OPTIN)
    if G == 67:
        assert chain_plan.top_nodes(n_frames) == chain_plan.TOP and chain_plan.dense_tiles(chain_plan.dense_n(G, n_frames)) == 7
    if grid == (4, 3):
        assert {"wide0_rounds2", "levels4"} <= chain_plan.branches(n_frames, SMS)
    p = synth.make_problem(models=models, n_frames=n_frames, grid=grid, inertial=True, seed=17)
    if missing:
        p = _missing_frames(p)
    iters = 6
    opts = dict(max_iters=iters, function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
    g0, g1 = _calibrator(p, 0, **opts), _calibrator(p, MULTI_LAUNCH, **opts)
    assert g0.G == G
    s0, s1 = g0.solve(), g1.solve()
    assert _persistent_ran(s0), s0["kernel_launches"]
    assert not _persistent_ran(s1), s1["kernel_launches"]
    assert s0["iterations"] == s1["iterations"] == iters
    assert s0["successful_steps"] == s1["successful_steps"]
    assert abs(s0["final_cost"] - s1["final_cost"]) <= 1e-10 * s1["final_cost"]
    st0, st1 = g0.state(), g1.state()
    for k in STATE_KEYS:
        assert np.abs(st0[k] - st1[k]).max() <= 1e-8 * max(np.abs(st1[k]).max(), 1.0), k
    assert abs(st0["ts"] - st1["ts"]) <= 1e-8


@pytest.mark.parametrize("mode", [0, MULTI_LAUNCH], ids=["eval_mega", "multi_launch"])
@pytest.mark.parametrize("models", MISSING_RIGS, ids=["missing_frames", "unseen_frame"])
def test_missing_frames_normal_equations(models, mode):
    """The reprojection build of each inertial engine (eval_mega_kernel, fused_build_kernel<9>) on frames that a camera
    misses or that no camera sees, against the oracle; the columns of E of a camera that misses a frame are exactly 0."""
    from oracle.binding import Oracle

    p = _missing_frames(synth.make_problem(models=models, n_frames=120, grid=(14, 10), inertial=True, seed=5))
    o, g = Oracle(p, **ALL_ON), _calibrator(p, mode)
    assert chain_plan.persistent_fits(g.G, p.n_frames, SMEM_OPTIN)
    ne_o, ne_g = o.normal_equations(), g.normal_equations()
    assert abs(ne_g["cost"] - ne_o["cost"]) <= 1e-11 * ne_o["cost"]
    for k in ("B", "U", "E", "gf", "C", "gc"):
        assert np.abs(ne_g[k] - ne_o[k]).max() <= 1e-10 * np.abs(ne_o[k]).max(), k
    seen = np.zeros((p.n_cams, p.n_frames), dtype=bool)
    seen[p.obs_cam, p.obs_frame] = True
    assert not seen[:, UNSEEN_FRAME].any()
    off = 0
    for c, m in enumerate(p.models):
        n = 6 + synth.NUM_INTR[int(m)]
        assert not ne_g["E"][~seen[c], :, off:off + n].any(), c
        off += n


def _lm_against_oracle(models, n_frames, max_iters, function_tol, **opts):
    from oracle.binding import Oracle

    p = synth.make_problem(models=models, n_frames=n_frames, grid=(14, 10), inertial=True, seed=21)
    o = Oracle(p, **ALL_ON)
    g = _calibrator(p)
    o.set_options(function_tol=function_tol, max_iters=max_iters, **opts)
    g.set_options(function_tol=function_tol, max_iters=max_iters, **opts)
    return p, o, g


@pytest.mark.parametrize("models,persistent", [(("kb4",) * 3 + ("linear",), True), (("kb4",) * 3 + ("fov",), False)],
                         ids=["G67", "G68"])
def test_persistent_fit_boundary(models, persistent):
    """Bars of test_gpu_imu_parity.test_lm_solve_with_imu_fixed_weights."""
    G = chain_plan.rig_globals(models)
    assert G == (67 if persistent else 68)
    assert chain_plan.persistent_fits(G, 40, SMEM_OPTIN) == persistent
    p, o, g = _lm_against_oracle(models, 40, 40, 1e-13, update_imu_weights=0)
    s_o, s_g = o.solve(), g.solve()
    assert _persistent_ran(s_g) == persistent, s_g["kernel_launches"]
    assert abs(s_g["final_cost"] - s_o["final_cost"]) <= 1e-8 * s_o["final_cost"]
    st_o, st_g = o.state(), g.state()
    for c, m in enumerate(p.models):
        K = synth.NUM_INTR[int(m)]
        rel = np.abs(st_g["intr"][c, :K] - st_o["intr"][c, :K]) / np.maximum(np.abs(st_o["intr"][c, :K]), 1e-3)
        assert rel.max() <= 1e-6
    for k in ("T_wp", "v_w", "q_ck", "p_ck", "g", "b", "sf"):
        assert np.abs(st_g[k] - st_o[k]).max() <= 1e-6 * max(1.0, np.abs(st_o[k]).max()), k
    assert abs(st_g["ts"] - st_o["ts"]) <= 1e-8


@pytest.mark.parametrize("n_frames", [chain_plan.TOP * chain_plan.CHUNK, chain_plan.TOP * chain_plan.CHUNK + 1],
                         ids=["top4", "top1"])
@pytest.mark.parametrize("models", [("kb4",) * 8, ("kb4",) * 3 + ("poly3",) * 5], ids=["8xkb4", "3xkb4_5xpoly3"])
def test_largest_rigs_match_oracle(models, n_frames):
    """The largest rigs the C API accepts, on the multi-launch engine: the chain elimination asks for more than 200 KB
    of shared memory at G >= 122, the dense solve of [globals | 4 top nodes] at G >= 124.  Bars of
    test_gpu_vision_parity.test_eight_cameras_match_oracle."""
    G = chain_plan.rig_globals(models)
    assert G in (127, 122) and not chain_plan.persistent_fits(G, n_frames, SMEM_OPTIN)
    req = chain_plan.multi_launch_requests(G, True, chain_plan.top_nodes(n_frames))
    assert max(req.values()) <= chain_plan.engine_smem_optin(SMEM_OPTIN)
    p, o, g = _lm_against_oracle(models, n_frames, 12, 1e-12)
    ne_o, ne_g = o.normal_equations(), g.normal_equations()
    assert o.G == g.G == G
    for k in ("B", "E", "gf", "C", "gc"):
        assert np.abs(ne_g[k] - ne_o[k]).max() <= 1e-9 * max(np.abs(ne_o[k]).max(), 1e-300), k
    s_o, s_g = o.solve(), g.solve()
    assert not _persistent_ran(s_g)
    assert abs(s_g["final_cost"] - s_o["final_cost"]) <= 1e-8 * s_o["final_cost"]
    st_o, st_g = o.state(), g.state()
    assert np.abs(st_g["T_wp"] - st_o["T_wp"]).max() <= 1e-6
    assert np.abs(st_g["p_ck"] - st_o["p_ck"]).max() <= 1e-6
    for c, m in enumerate(p.models):
        K = synth.NUM_INTR[int(m)]
        rel = np.abs(st_g["intr"][c, :K] - st_o["intr"][c, :K]) / np.maximum(np.abs(st_o["intr"][c, :K]), 1e-3)
        assert rel.max() <= 1e-5, c  # 12 iterations, not converged: rounding differences grow along weak directions


WEIGHTS_FRAMES, WEIGHTS_ITERS = 5000, 4
_WEIGHTS_RUN = """
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from vicalib_b200 import synth
from vicalib_b200.capi import Calibrator
p = synth.make_problem(models=("poly3",), n_frames={n}, grid=(4, 3), inertial=True, seed=23)
g = Calibrator()
g.load(p)
g.set_flags(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
g.set_options(max_iters={it}, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, update_imu_weights=1)
s = g.solve()
np.save(sys.argv[2], g.imu_weights())
np.save(sys.argv[3], g.state()["T_wp"])
print(s["kernel_launches"], s["iterations"], s["successful_steps"])
""".format(n=WEIGHTS_FRAMES, it=WEIGHTS_ITERS)


def _weights_subprocess(tmp_path, tag, env_var):
    env = dict(os.environ)
    env[env_var] = {"VCGPU_N_SOLVER": str(SMS - 1), "VCGPU_NO_DEFERRED_WEIGHTS": "1"}[env_var]
    w, t = tmp_path / f"w_{tag}.npy", tmp_path / f"t_{tag}.npy"
    out = subprocess.run([sys.executable, "-c", _WEIGHTS_RUN, ROOT, str(w), str(t)], env=env, capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    launches, iters, accepted = (int(v) for v in out.stdout.split()[-3:])
    return np.load(w), np.load(t), launches, iters, accepted


def test_deferred_weights_queue(tmp_path):
    """5000 frames: 313 weight tasks for the 124 CTAs that leave the solve (132 SMs), so CTAs take several tasks each."""
    from oracle.binding import Oracle

    assert chain_plan.weight_tasks(WEIGHTS_FRAMES) > chain_plan.leaving_ctas(WEIGHTS_FRAMES, SMS)
    p = synth.make_problem(models=("poly3",), n_frames=WEIGHTS_FRAMES, grid=(4, 3), inertial=True, seed=23)
    opts = dict(max_iters=WEIGHTS_ITERS, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, update_imu_weights=1)
    g = _calibrator(p, **opts)
    o = Oracle(p, **ALL_ON)
    o.set_options(**opts)
    s_g, s_o = g.solve(), o.solve()
    assert _persistent_ran(s_g), s_g["kernel_launches"]
    assert s_g["iterations"] == WEIGHTS_ITERS and s_g["successful_steps"] == s_o["successful_steps"]
    assert abs(s_g["final_cost"] - s_o["final_cost"]) <= 1e-8 * s_o["final_cost"]
    W_g, W_o = g.imu_weights(), o.imu_weights()
    assert np.abs(W_o - 500 * np.eye(9)).max() > 1.0  # the weights did change
    rel = np.abs(W_g - W_o).max((1, 2)) / np.abs(W_o).max((1, 2))
    assert rel.max() <= 1e-7, int(rel.argmax())
    st_g, st_o = g.state(), o.state()
    for k in ("T_wp", "q_ck", "p_ck", "intr"):
        assert np.abs(st_g[k] - st_o[k]).max() <= 1e-6 * max(1.0, np.abs(st_o[k]).max()), k
    for k in ("v_w", "g", "b", "sf"):
        assert np.abs(st_g[k] - st_o[k]).max() <= 2e-5, k
    # the multi-launch engine updates the weights after every accepted step too, the one of the last iteration included
    g_m = _calibrator(p, MULTI_LAUNCH, **opts)
    s_m = g_m.solve()
    assert not _persistent_ran(s_m) and s_m["successful_steps"] == s_g["successful_steps"]
    W_m = g_m.imu_weights()
    assert (np.abs(W_m - W_g).max((1, 2)) / np.abs(W_g).max((1, 2))).max() <= 1e-9
    # one team computes each interval's weight, whichever CTA takes the task: with all CTAs but one kept in the solve
    # the weights are bit for bit those of the default run
    W, T, launches, iters, accepted = _weights_subprocess(tmp_path, "n_solver", "VCGPU_N_SOLVER")
    assert iters == WEIGHTS_ITERS and accepted == s_g["successful_steps"] and launches <= 2 * iters + 12
    assert np.array_equal(W, W_g), np.abs(W - W_g).max()
    assert np.array_equal(T, st_g["T_wp"])
    # computed in the evaluation launch instead, the team's code is compiled into another kernel (imu_weights_team is
    # force-inlined per caller, and the compiler may contract its products differently there): the same weights to
    # rounding, and they must include the update of the last accepted step
    W, T, launches, iters, accepted = _weights_subprocess(tmp_path, "no_deferred", "VCGPU_NO_DEFERRED_WEIGHTS")
    assert iters == WEIGHTS_ITERS and accepted == s_g["successful_steps"] and launches <= 2 * iters + 12
    assert (np.abs(W - W_g).max((1, 2)) / np.abs(W_g).max((1, 2))).max() <= 1e-10
    assert np.abs(T - st_g["T_wp"]).max() <= 1e-12 * np.abs(st_g["T_wp"]).max()


@pytest.mark.parametrize("stop", ["max_iters", "function_tol", "gradient_tol", "param_tol"])
@pytest.mark.parametrize("mode", [0, MULTI_LAUNCH], ids=["persistent", "multi_launch"])
@pytest.mark.parametrize("strategy", [0, 1], ids=["lm", "dogleg"])
def test_weights_are_current_after_solve(strategy, mode, stop):
    """Whatever ends a solve with live weights, the weights it leaves are those of its last accepted state: updating
    them once more changes them only to rounding (the update after the solve runs in imu_weights_kernel, the one in
    the persistent solve launch in another kernel; see test_deferred_weights_queue)."""
    p = synth.make_problem(models=("poly3",), n_frames=40, grid=(14, 10), inertial=True, seed=29)
    base = dict(strategy=strategy, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, update_imu_weights=1)
    if stop == "max_iters":
        opts, term = dict(base, max_iters=4), 0
    elif stop == "function_tol":
        opts, term = dict(base, max_iters=100, function_tol=1e-6), 1
    elif stop == "param_tol":  # a parameter tolerance between a step's norm and every earlier one (over |x|: all blocks
        # are free here, and |x| moves by far less than the gap between the step norms)
        rows = _calibrator(p, mode, **dict(base, max_iters=12)).solve()["rows"]
        sn = rows[:, 5]
        k = next(it for it in range(2, len(rows)) if 0 < sn[it] < 0.5 * sn[1:it][sn[1:it] > 0].min())
        x = np.sqrt(sum(np.sum(np.square(v)) for v in (p.T_wp, p.v_w, p.q_ck, p.p_ck, p.intr, p.g, p.b, p.sf, [p.ts])))
        opts, term = dict(base, max_iters=k + 4, param_tol=float(np.sqrt(sn[k] * sn[1:k][sn[1:k] > 0].min())) / x), 3
    else:  # a gradient tolerance between an accepted step's largest gradient entry and every earlier one
        rows = _calibrator(p, mode, **dict(base, max_iters=8)).solve()["rows"]
        gmax = rows[:, 3]
        k = next(it for it in range(2, len(rows)) if rows[it, 8] == 1 and gmax[it] < 0.99 * gmax[:it].min())
        opts, term = dict(base, max_iters=k + 4, gradient_tol=float(np.sqrt(gmax[k] * gmax[:k].min()))), 2
    g = _calibrator(p, mode, **opts)
    s = g.solve()
    assert s["termination"] == term
    if strategy == 0:
        assert _persistent_ran(s) == (mode == 0), s["kernel_launches"]
    if stop == "param_tol":
        assert s["iterations"] == k
    if stop not in ("function_tol", "param_tol"):
        assert s["rows"][-1, 8] == 1  # the solve ends on an accepted step
    W = g.imu_weights()
    assert np.abs(W - 500 * np.eye(9)).max() > 1.0  # the weights did change
    g.update_imu_weights()
    rel = (np.abs(g.imu_weights() - W).max((1, 2)) / np.abs(W).max((1, 2))).max()
    assert rel <= 1e-10, rel
