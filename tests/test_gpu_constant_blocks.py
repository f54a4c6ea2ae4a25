"""GPU: constant parameter blocks on every solve engine, against the CPU oracle (or a dense numpy solve where noted).

- Normal equations with fixed intrinsics on each build path (fused, multi-launch inertial, eval_mega_kernel),
  and with residual-block multiplicities: 1e-10 relative per block family; the intrinsic columns of E and rows and
  columns of C and gc exactly 0.
- The damped arrow solve with constant columns against numpy.linalg.solve with those columns deleted, where the LM
  floor makes their pivots 1e-6 / radius (down to 1e-22): constant entries of the step exactly 0.
- LM and DOGLEG solves with constant blocks on each engine: the oracle's result, and every constant block back bit for
  bit (Ceres never moves them; so3_plus / se3_plus would renormalise a quaternion even with a zero step).
- The parameter tolerance: x_norm covers the free blocks only, so the solve stops where the oracle (and Ceres) does.
"""
import numpy as np
import pytest

import chain_plan
import constant_blocks as cb
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

MULTI_LAUNCH = 4  # vcgpu_set_profiling bit 2
STAGES = [
    dict(inertial=1, rotation_only=1, bias_active=0, scale_active=0, optimize_ts=1),
    dict(inertial=1, rotation_only=0, bias_active=1, scale_active=0, optimize_ts=1),
    dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1),
    dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=0),
]
ALL_ON = STAGES[2]
STATE_KEYS = ("T_wp", "v_w", "q_ck", "p_ck", "intr", "g", "b", "sf")


def _pair(p, flags, mode=0, **opts):
    from oracle.binding import Oracle
    from vicalib_b200.capi import Calibrator

    o = Oracle(p, **flags)
    g = Calibrator()
    g.load(p)
    g.set_flags(**flags)
    g.set_profiling(mode, False)
    if opts:
        o.set_options(**opts)
        g.set_options(**opts)
    return o, g


def _relerr(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _intr_cols(o, models):
    """global columns of the intrinsics"""
    cols, off = [], 0
    for m in models:
        K = synth.NUM_INTR[int(m)]
        cols += list(range(off + 6, off + 6 + K))
        off += 6 + K
    return np.array(cols)


def _check_ne(o, g, models, bar=1e-10):
    ne_o, ne_g = o.normal_equations(), g.normal_equations()
    assert abs(ne_g["cost"] - ne_o["cost"]) <= 1e-11 * ne_o["cost"]
    for k in ("B", "U", "E", "gf", "C", "gc"):
        if np.abs(ne_o[k]).max() > 0:
            assert _relerr(ne_g[k], ne_o[k]) <= bar, k
        else:
            assert np.abs(ne_g[k]).max() == 0.0, k
    return ne_g


# ------------------------------------------------------------------ normal equations
VISION_MODELS = [("linear",), ("fov",), ("poly2",), ("poly3",), ("kb4",), ("poly3", "fov", "kb4")]


@pytest.mark.parametrize("mode", [0], ids=["fused"])
@pytest.mark.parametrize("models", VISION_MODELS, ids=["+".join(m) for m in VISION_MODELS])
def test_vision_normal_equations_fixed_intrinsics(models, mode):
    p = synth.make_problem(models=models, n_frames=12, grid=(14, 10), seed=7 + len(models))
    o, g = _pair(p, cb.FIX, mode)
    ne = _check_ne(o, g, p.models)
    ic = _intr_cols(o, p.models)
    assert np.array_equal(ne["E"][:, :, ic], np.zeros_like(ne["E"][:, :, ic]))
    assert not ne["C"][ic].any() and not ne["C"][:, ic].any() and not ne["gc"][ic].any()


@pytest.mark.parametrize("mode", [0, MULTI_LAUNCH], ids=["eval_mega", "multi_launch"])
@pytest.mark.parametrize("flags", STAGES, ids=["stage2", "stage3", "all_on", "no_ts"])
def test_inertial_normal_equations_fixed_intrinsics(flags, mode):
    p = synth.make_problem(models=("poly3", "kb4"), n_frames=14, grid=(14, 10), inertial=True, seed=21)
    flags = dict(flags, fix_intrinsics=1)
    o, g = _pair(p, flags, mode)
    ne = _check_ne(o, g, p.models)
    ic = _intr_cols(o, p.models)
    assert not ne["E"][:, :, ic].any() and not ne["C"][ic].any() and not ne["C"][:, ic].any() and not ne["gc"][ic].any()


def test_eight_cameras_fixed_intrinsics():
    """G = 119: the multi-launch engine's build"""
    p = synth.make_problem(models=("poly3",) * 8, n_frames=40, grid=(14, 10), inertial=True, seed=88)
    o, g = _pair(p, dict(ALL_ON, fix_intrinsics=1))
    assert g.G == 119
    ne = _check_ne(o, g, p.models, bar=1e-9)
    ic = _intr_cols(o, p.models)
    assert not ne["E"][:, :, ic].any() and not ne["C"][ic].any() and not ne["gc"][ic].any()


@pytest.mark.parametrize("mode", [0, MULTI_LAUNCH], ids=["fused", "multi_launch"])
@pytest.mark.parametrize("inertial", [False, True], ids=["vision", "inertial"])
def test_multiplicities(inertial, mode):
    """visual_mult = 3, imu_mult = 2: the residual-block multiplicities of the staged flow scale every Gram build"""
    p = synth.make_problem(models=("poly3", "fov"), n_frames=16, grid=(14, 10), inertial=inertial, seed=31)
    flags = dict(ALL_ON if inertial else {}, visual_mult=3.0, imu_mult=2.0)
    o, g = _pair(p, flags, mode)
    _check_ne(o, g, p.models)
    assert g.num_residuals() == o.num_residuals() == 3 * 2 * p.n_obs + (2 * 9 * (p.n_frames - 1) if inertial else 0)
    assert abs(g.cost() - o.cost()) <= 1e-10 * o.cost()


@pytest.mark.parametrize("mode", [0, MULTI_LAUNCH], ids=["persistent", "multi_launch"])
def test_multiplicities_lm_solve(mode):
    """test_lm_solve_with_imu_fixed_weights with the multiplicities, over a fixed number of iterations (past
    convergence, rounding decides which steps are accepted, and the poses' weak directions follow)"""
    p = synth.make_problem(models=("poly3",), n_frames=40, grid=(14, 10), inertial=True, seed=21)
    o, g = _pair(p, dict(ALL_ON, visual_mult=3.0, imu_mult=2.0), mode, function_tol=0.0, gradient_tol=0.0,
                 param_tol=0.0, max_iters=8, update_imu_weights=0)
    s_o, s_g = o.solve(), g.solve()
    assert (s_g["kernel_launches"] <= 2 * s_g["iterations"] + 12) == (mode == 0), s_g["kernel_launches"]
    assert s_g["successful_steps"] == s_o["successful_steps"]
    assert np.allclose(s_g["rows"][:, 1], s_o["rows"][: len(s_g["rows"]), 1], rtol=1e-8)
    assert abs(s_g["final_cost"] - s_o["final_cost"]) <= 1e-8 * s_o["final_cost"]
    st_o, st_g = o.state(), g.state()
    rel = np.abs(st_g["intr"][0, :7] - st_o["intr"][0, :7]) / np.maximum(np.abs(st_o["intr"][0, :7]), 1e-3)
    assert rel.max() <= 1e-6
    for k in ("T_wp", "v_w", "q_ck", "p_ck", "g", "b", "sf"):
        assert np.abs(st_g[k] - st_o[k]).max() <= 1e-6 * max(1.0, np.abs(st_o[k]).max()), k
    assert abs(st_g["ts"] - st_o["ts"]) <= 1e-8


# ------------------------------------------------------------------ damped arrow solve, constant columns
def _dense(ne, scale, D2):
    """S H S + diag(D2) and -S g, dense"""
    nf, fd, G = ne["B"].shape[0], ne["B"].shape[1], ne["C"].shape[0]
    nfp = nf * fd
    H = np.zeros((nfp + G, nfp + G))
    for f in range(nf):
        s = slice(f * fd, (f + 1) * fd)
        H[s, s] = ne["B"][f]
        H[s, nfp:] = ne["E"][f]
        H[nfp:, s] = ne["E"][f].T
        if f > 0:
            sp = slice((f - 1) * fd, f * fd)
            H[sp, s] = ne["U"][f]
            H[s, sp] = ne["U"][f].T
    H[nfp:, nfp:] = ne["C"]
    H = scale[:, None] * H * scale[None, :] + np.diag(D2)
    return H, -scale * np.concatenate([ne["gf"].ravel(), ne["gc"]])


ARROW_CASES = [
    ("vision_2cam", ("poly3", "fov"), 12, False),
    ("vision_8cam", ("poly3",) * 8, 16, False),                                 # G = 104
    ("G41", ("poly3", "poly3"), 200, True),
    ("G67_top4", ("poly3",) * 4, chain_plan.TOP * chain_plan.CHUNK ** 2, True),  # 4 top nodes, 7-tile dense L D L^T
    ("G127", ("kb4",) * 8, 64, True),                                           # multi-launch engine
]


@pytest.mark.parametrize("radius", [1e4, 1e16])
@pytest.mark.parametrize("name,models,n_frames,inertial", ARROW_CASES, ids=[c[0] for c in ARROW_CASES])
def test_arrow_solve_constant_columns(name, models, n_frames, inertial, radius):
    from vicalib_b200.capi import Calibrator

    G = chain_plan.rig_globals(models, inertial)
    if name == "G67_top4":
        assert chain_plan.top_nodes(n_frames) == chain_plan.TOP and chain_plan.dense_tiles(chain_plan.dense_n(G, n_frames)) == 7
    if name == "G127":
        assert not chain_plan.persistent_fits(G, n_frames, chain_plan.device_or_h100()[1])
    p = synth.make_problem(models=models, n_frames=n_frames, grid=(14, 10), inertial=inertial, seed=13)
    flags = dict(ALL_ON, fix_intrinsics=1) if inertial else dict(cb.FIX)
    g = Calibrator()
    g.load(p)
    g.set_flags(**flags)
    assert g.G == G
    ne = g.normal_equations()
    fd, nfp = g.fd, n_frames * g.fd
    diag = np.concatenate([np.einsum("fii->fi", ne["B"]).ravel(), np.diag(ne["C"])])
    scale = 1.0 / (1.0 + np.sqrt(diag))
    D2 = np.clip(diag * scale * scale, 1e-6, 1e32) / radius
    from oracle.binding import Oracle

    mask = Oracle(p, **flags).global_mask()
    const = np.concatenate([np.zeros(nfp, bool), mask == 0])
    assert const.sum() >= 4 * len(models) and D2[const].max() == 1e-6 / radius
    x = g.solve_arrow(scale, D2)
    assert np.array_equal(x[const], np.zeros(const.sum()))
    H, rhs = _dense(ne, scale, D2)
    keep = ~const
    Hk = H[np.ix_(keep, keep)]
    x_ref = np.linalg.solve(Hk, rhs[keep])
    # both solves lose cond * eps; near radius 1e16 the damping no longer bounds the condition number
    bar = max(1e-8, 1e-15 * np.linalg.cond(Hk))
    assert _relerr(x[keep], x_ref) <= bar


# ------------------------------------------------------------------ solves: constant blocks bit for bit
def _engine(s, inertial, persistent):
    """whether the launch count is that of the persistent engine: one launch per iteration (vision), two (inertial)"""
    per = 2 if inertial else 1
    return (s["kernel_launches"] <= per * s["iterations"] + 12) == persistent


SOLVE_CASES = [
    ("vision_fix", cb.vision_problem, cb.FIX, 0, 0), ("vision_fix", cb.vision_problem, cb.FIX, 0, MULTI_LAUNCH),
    ("vision_fix", cb.vision_problem, cb.FIX, 1, 0), ("vision_fix", cb.vision_problem, cb.FIX, 1, MULTI_LAUNCH),
    ("inertial_fix", cb.inertial_problem, cb.INERTIAL_FIX, 0, 0),
    ("inertial_fix", cb.inertial_problem, cb.INERTIAL_FIX, 0, MULTI_LAUNCH),
    ("inertial_fix", cb.inertial_problem, cb.INERTIAL_FIX, 1, 0),
    ("inertial_fix", cb.inertial_problem, cb.INERTIAL_FIX, 1, MULTI_LAUNCH),
    ("rotation_only", cb.inertial_problem, cb.STAGE_ROT_ONLY, 0, 0),
    ("rotation_only", cb.inertial_problem, cb.STAGE_ROT_ONLY, 0, MULTI_LAUNCH),
    ("rotation_only", cb.inertial_problem, cb.STAGE_ROT_ONLY, 1, 0),
]
_MODE = {0: "persistent", MULTI_LAUNCH: "multi_launch"}


@pytest.mark.parametrize("name,make,flags,strategy,mode", SOLVE_CASES,
                         ids=[f"{c[0]}-{'lm' if c[3] == 0 else 'dogleg'}-{_MODE[c[4]]}" for c in SOLVE_CASES])
def test_solve_keeps_constant_blocks(name, make, flags, strategy, mode):
    p = make()
    inertial = bool(flags.get("inertial"))
    before = cb.constant_parts(cb.uploaded(p), p, flags)
    if not inertial:
        assert cb.moves_on_renormalisation(p.q_ck[0]) and cb.moves_on_renormalisation(before["T_wp_unused"][0, :4])
    o, g = _pair(p, flags, mode, max_iters=20, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, strategy=strategy)
    s_o, s_g = o.solve(), g.solve()
    if strategy == 0:
        assert _engine(s_g, inertial, mode == 0), s_g["kernel_launches"]
    assert s_g["iterations"] == s_o["iterations"] == 20
    # iteration by iteration the same algorithm, up to convergence; past it, accepting a step is decided by rounding
    assert np.allclose(s_g["rows"][:7, 1], s_o["rows"][:7, 1], rtol=1e-8)
    assert abs(s_g["final_cost"] - s_o["final_cost"]) <= 1e-9 * s_o["final_cost"]
    st_o, st_g = o.state(), g.state()
    for k in STATE_KEYS:
        assert np.abs(st_g[k] - st_o[k]).max() <= 1e-6 * max(1.0, np.abs(st_o[k]).max()), k
    after = cb.constant_parts(st_g, p, flags)
    for k, v in before.items():
        assert np.array_equal(after[k], v), k


# ------------------------------------------------------------------ parameter tolerance
PT_RUNS = [(c, s, m) for c in cb.PT_CASES for s, m in ((0, 0), (0, MULTI_LAUNCH), (1, 0))]


@pytest.mark.parametrize("case,strategy,mode", PT_RUNS,
                         ids=[f"{c[0]}-{'lm' if s == 0 else 'dogleg'}-{_MODE[m]}" for c, s, m in PT_RUNS])
def test_param_tol_stops_on_free_block_norm(case, strategy, mode):
    """The oracle's rows and states give a tolerance under which the free-block rule stops at iteration k and the
    all-block rule at j < k; the device must stop at k with the oracle's state."""
    name, make, flags = case
    p = make()
    rows, norms, win = cb.param_tol_case(p, flags, strategy)
    assert win is not None
    tol, k, j = win
    assert cb.stops_at(rows, norms, tol, 0) == k and cb.stops_at(rows, norms, tol, 1) == j < k
    o, g = _pair(p, flags, mode, max_iters=k + 5, function_tol=0.0, gradient_tol=0.0, param_tol=tol, strategy=strategy)
    s_o, s_g = o.solve(), g.solve()
    assert s_o["termination"] == 3 and s_o["iterations"] == k
    if strategy == 0:
        assert _engine(s_g, bool(flags.get("inertial")), mode == 0), s_g["kernel_launches"]
    assert (s_g["termination"], s_g["iterations"], s_g["successful_steps"]) == (3, k, s_o["successful_steps"])
    st_o, st_g = o.state(), g.state()
    for key in STATE_KEYS:
        assert np.abs(st_g[key] - st_o[key]).max() <= 1e-6 * max(1.0, np.abs(st_o[key]).max()), key
