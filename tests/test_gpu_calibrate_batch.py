"""GPU: vcgpu_calibrate_batch — ViCalibrator::SolveThread's staged flow for a batch of rigs, every solve in the batch
cluster kernels, DOGLEG inside the inertial ones.

The reference is flow_reference (test_cpu_calibrate_flow.py's restatement of the host mirror's SolveThread) run with
per-handle calls: Calibrator.solve (inertial DOGLEG on the multi-launch engine, vision stages on the persistent vision
kernel), evaluate, remove_outliers.  The batch and the per-handle calls are two summation orders of one algorithm, so
the bars are test_gpu_imu_engines.py's: the same iterations, accepted steps and termination per solve, cost within
1e-10 and state within 1e-8 (relative), ts within 1e-8, weights within 1e-9.  Between batches a rig's trajectory must
not move at all.
"""
import numpy as np
import pytest

import chain_plan
from test_cpu_calibrate_flow import flow_reference, stage_of
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
COST_BAR, STATE_BAR, TS_BAR, WEIGHTS_BAR = 1e-10, 1e-8, 1e-8, 1e-9
TOL0 = dict(function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
STATE_KEYS = ("T_wp", "v_w", "q_ck", "p_ck", "intr", "g", "b", "sf")
COUNTS = ("iterations", "successful_steps", "termination", "num_residuals")
DL = dict(strategy=1)


class Rig:
    def __init__(self, flags=None, opts=None, **kw):
        from vicalib_b200.capi import Calibrator

        self.p = synth.make_problem(inertial=True, **kw)
        self.flags = dict(ALL_ON, **(flags or {}))
        self.opts = dict(max_iters=6, **TOL0, **DL) if opts is None else opts
        self.g = Calibrator()
        self.reset()

    def reset(self):
        self.g.load(self.p)
        self.g.set_flags(**self.flags)
        self.g.set_options(**self.opts)

    def result(self, s):
        W = self.g.imu_weights() if self.g.flags.inertial else np.zeros((0, 9, 9))
        return s, self.g.state(), W


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1.0))


def _agree(got, ref, what="", cost_bar=COST_BAR, state_bar=STATE_BAR, weights_bar=WEIGHTS_BAR, ts_bar=TS_BAR):
    (s, st, W), (s0, st0, W0) = got, ref
    for k in COUNTS:
        assert s[k] == s0[k], (what, k, s[k], s0[k])
    assert abs(s["final_cost"] - s0["final_cost"]) <= cost_bar * s0["final_cost"], (what, s["final_cost"], s0["final_cost"])
    state = max(_rel(st[k], st0[k]) for k in STATE_KEYS)
    assert state <= state_bar, (what, state)
    assert abs(st["ts"] - st0["ts"]) <= ts_bar, what
    if len(W0):
        w = float((np.abs(W - W0).max((1, 2)) / np.abs(W0).max((1, 2))).max())
        assert w <= weights_bar, (what, w)


def _same_bits(a, b, what=""):
    (d, st, W), (d0, st0, W0) = a, b
    for k in ("solves", "iterations", "finished", "stage", "outliers_removed", "mse"):
        assert d[k] == d0[k], (what, k)
    for k in ("iterations", "successful_steps", "termination", "initial_cost", "final_cost"):
        assert d["last"][k] == d0["last"][k], (what, k)
    for k in STATE_KEYS:
        assert np.array_equal(st[k], st0[k]), (what, k)
    assert st["ts"] == st0["ts"] and np.array_equal(W, W0), what


def _flow(rigs, **flow):
    from vicalib_b200.capi import calibrate_batch

    out = calibrate_batch([r.g for r in rigs], **flow)
    return [(d, r.g.state(), r.g.imu_weights() if r.g.flags.inertial else np.zeros((0, 9, 9))) for (d, _), r in zip(out, rigs)]


# ------------------------------------------------------------------ 1. inertial DOGLEG alone, against vcgpu_solve
SHAPES = [
    dict(models=("poly3",), n_frames=24, grid=(14, 10), seed=1),                        # one CTA per cluster
    dict(models=("poly3", "kb4"), n_frames=200, grid=(14, 10), seed=2),                 # two
    dict(models=chain_plan.rig_with_globals(67), n_frames=256, grid=(8, 6), seed=3),   # G = 67
    dict(models=("poly3", "poly3"), n_frames=2000, grid=(4, 3), seed=4),                # eight, target-shaped
]
ONE_SOLVE = dict(calibrate_imu=True, remove_outliers=False, block_duplication=False, gravity_initialized=True, max_solves=1)


@pytest.mark.parametrize("weights", [0, 1], ids=["weights_fixed", "weights_live"])
def test_dogleg_one_solve_against_solo(weights):
    rigs = [Rig(opts=dict(max_iters=6, update_imu_weights=weights, **TOL0, **DL), **kw) for kw in SHAPES]
    rigs += [Rig(flags=f, opts=dict(max_iters=6, update_imu_weights=weights, **TOL0, **DL), **SHAPES[1])
             for f in (dict(rotation_only=1, bias_active=0, scale_active=0), dict(scale_active=0), dict(optimize_ts=0, fix_intrinsics=1))]
    ref = [r.result(r.g.solve(free_running=True)) for r in rigs]
    for r in rigs:
        r.reset()
    got = _flow(rigs, **ONE_SOLVE)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert a[0]["solves"] == 1
        # rigs 4 and 5 (rotation only; scale factors constant) with live weights: the two summation orders' costs have
        # been seen 2e-10 apart on an H100, past the 1e-10 bar, with every count agreeing
        _agree((a[0]["last"], a[1], a[2]), b, f"rig {i}", cost_bar=1e-9 if weights and i in (4, 5) else COST_BAR)


# ------------------------------------------------------------------ 2. the branches of the dogleg point, a rejected step
BRANCH_RIG = dict(models=("poly3",), n_frames=48, grid=(14, 10), seed=7)
MODEL_BAR = 3e-7  # test_gpu_dogleg_shapes.py's bar on the model change against dogleg_ref
# One iteration from a start far from the solution: the cost after it is first-order in the step, and the Gauss-Newton
# step of a system regularised by mu = 1e-8 only is as exact as its conditioning allows (test_gpu_dogleg_shapes.py
# measures 1.8e-9 in |gn| against a long-double reference).  The two summation orders' costs after the Gauss-Newton
# branch's iteration were seen 4.4e-9 apart on an H100, so these iterations are held to 1e-8 in cost and 1e-6 in state;
# every count must agree.  (After a converged solve the cost is second-order in the step: the 1e-10 bar above.)
ONE_STEP_BARS = dict(cost_bar=1e-8, state_bar=1e-6)


def _one_iteration(radius):
    return dict(max_iters=1, init_radius=radius, update_imu_weights=0, **TOL0, **DL)


def test_dogleg_branches():
    """One iteration at a radius per branch of the dogleg point, chosen as test_gpu_dogleg_shapes.py chooses them from
    dogleg_ref's step at the rig's normal equations: 1.5 |gn| (Gauss-Newton step), 0.5 alpha |g~| (truncated Cauchy
    step), their geometric mean (interpolated point).  The solo solve's row shows the branch: its model change
    (cost_change / rho) is the reference's for that branch and the radius it leaves is radius_after's for that step.
    The batch's iteration agrees with the solo one at each radius."""
    import dogleg_ref

    r = Rig(opts=_one_iteration(1e4), **BRANCH_RIG)
    ne = r.g.normal_equations()
    scale = dogleg_ref.jacobi_scale(ne)
    radii = dogleg_ref.branch_radii(dogleg_ref.dogleg_step(ne, scale, 1e4))
    assert set(radii) == {"gauss_newton", "cauchy", "segment"}
    for branch, radius in radii.items():
        ref = dogleg_ref.dogleg_step(ne, scale, radius)
        assert ref["branch"] == branch
        r.opts = _one_iteration(radius)
        r.reset()
        solo = r.g.solve()
        row = solo["rows"][1]
        assert solo["iterations"] == 1 and row[8] == 1, (branch, row)
        model = row[2] / row[6]
        assert abs(model - ref["model_change"]) <= MODEL_BAR * abs(ref["model_change"]), (branch, model, ref["model_change"])
        expected = dogleg_ref.radius_after(radius, row[6], ref["step_norm"])
        assert abs(row[7] - expected) <= 2e-6 * expected, (branch, row[7], expected)
        want = r.result(solo)
        r.reset()
        got = _flow([r], **ONE_SOLVE)[0]
        _agree((got[0]["last"], got[1], got[2]), want, branch, **ONE_STEP_BARS)


def test_dogleg_rejected_step():
    """A start far from the solution (velocities scaled up, poses shifted) at a large radius: the solo solve's rows show
    a rejected step that halves the radius; the batch follows the solo solve through it and the iterations after it."""
    r = Rig(opts=dict(max_iters=10, init_radius=1e4, update_imu_weights=0, **TOL0, **DL), **BRANCH_RIG)
    r.p.v_w = r.p.v_w * 20.0
    r.p.T_wp = r.p.T_wp.copy()
    r.p.T_wp[:, 4:] += 0.3 * np.sin(np.arange(len(r.p.T_wp)))[:, None]
    r.reset()
    solo = r.g.solve()
    rows = solo["rows"]
    rejected = [k for k in range(1, len(rows)) if not rows[k][8] and rows[k][7] == 0.5 * rows[k - 1][7]]
    assert rejected, rows[:, [6, 7, 8]]
    # up to the first rejected iteration and the one after it (which recomputes everything at the halved radius)
    r.opts = dict(r.opts, max_iters=rejected[0] + 1)
    r.reset()
    solo = r.g.solve()
    assert not solo["rows"][rejected[0]][8]
    want = r.result(solo)
    r.reset()
    got = _flow([r], **ONE_SOLVE)[0]
    _agree((got[0]["last"], got[1], got[2]), want, "rejected", cost_bar=1e-7, state_bar=1e-5)


# ------------------------------------------------------------------ 3. the whole flow against the restatement
FLOWS = [
    dict(calibrate_imu=False, remove_outliers=True, block_duplication=True),
    dict(calibrate_imu=True, remove_outliers=True, block_duplication=True),
    dict(calibrate_imu=True, remove_outliers=False, block_duplication=False),
]


@pytest.mark.parametrize("strategy", [0, 1], ids=["lm", "dogleg"])
@pytest.mark.parametrize("fi", range(len(FLOWS)))
def test_flow_against_restatement(strategy, fi):
    flow = dict(FLOWS[fi], outlier_threshold=2.0, gravity_initialized=False, max_solves=12)
    start = dict(inertial=0, rotation_only=1, bias_active=0, scale_active=0)
    kws = [dict(models=("poly3",), n_frames=40, grid=(14, 10), seed=21), dict(models=("poly3", "kb4"), n_frames=64, grid=(14, 10), seed=22)]
    opts = [dict(max_iters=k, strategy=strategy) for k in (25, 4)]  # the second rig needs more solves per stage
    rigs = [Rig(flags=start, opts=o, **kw) for o, kw in zip(opts, kws)]
    ref = []
    for r in rigs:
        trace = flow_reference(r.g, r.p, **flow)
        ref.append((trace, r.g.state(), r.g.imu_weights() if r.g.flags.inertial else np.zeros((0, 9, 9))))
        r.reset()
    got = _flow(rigs, **flow)
    for i, ((d, st, W), (trace, st0, W0)) in enumerate(zip(got, ref)):
        assert d["solves"] == len(trace["solves"]), (i, d["solves"], len(trace["solves"]))
        assert d["iterations"] == sum(s["iterations"] for s in trace["solves"]), i
        assert d["outliers_removed"] == trace["removed"], i
        assert d["finished"] == trace["finished"] and d["stage"] == trace["stage"], i
        # the last of up to 12 solves, each started where the previous one of its own way ended: the two summation
        # orders drift apart over the trajectory (seen on an H100: 7e-9 in cost, 1e-5 in state, 3e-8 in ts, 1e-7 in the
        # weights),
        # so the bars here are the drift's, and the counts of every solve above are what the flow is held to
        _agree((d["last"], st, W), (trace["solves"][-1], st0, W0), f"flow {fi} rig {i}", cost_bar=1e-7, state_bar=1e-4, weights_bar=1e-5,
               ts_bar=1e-6)
    print(f"\nflow {fi} strategy {strategy}: stages {[t['stages'] for t, _, _ in ref]}")


# ------------------------------------------------------------------ 4. independence, max_solves, the handle afterwards
def test_independence():
    flow = dict(calibrate_imu=True, remove_outliers=True, outlier_threshold=2.0, block_duplication=True, max_solves=8)
    start = dict(inertial=0, rotation_only=1, bias_active=0, scale_active=0)
    target = Rig(flags=start, opts=dict(max_iters=10, strategy=1), models=("poly3",), n_frames=200, grid=(14, 10), seed=31)
    alone = _flow([target], **flow)[0]
    others = [Rig(flags=start, opts=dict(max_iters=10, strategy=k % 2), models=("poly3",), n_frames=n, grid=(14, 10), seed=40 + k)
              for k, n in enumerate((24, 48, 96, 300, 24, 64, 128))]
    target.reset()
    among = _flow([target] + others, **flow)[0]
    _same_bits(among, alone, "among 7")
    for r in [target] + others:
        r.reset()
    rev = _flow(others[::-1] + [target], **flow)[-1]
    _same_bits(rev, alone, "reversed")


def test_max_solves_caps():
    r = Rig(flags=dict(inertial=0, rotation_only=1, bias_active=0, scale_active=0), opts=dict(max_iters=1, strategy=1),
            models=("poly3",), n_frames=24, grid=(14, 10), seed=51)
    d = _flow([r], calibrate_imu=True, remove_outliers=True, max_solves=3)[0][0]
    assert d["solves"] == 3 and not d["finished"] and d["last"]["termination"] == 0


def test_handle_afterwards():
    from vicalib_b200.capi import Calibrator

    r = Rig(opts=dict(max_iters=4, **TOL0, **DL), models=("poly3",), n_frames=48, grid=(14, 10), seed=61)
    _flow([r], **ONE_SOLVE)
    st = r.g.state()
    after = r.result(r.g.solve(free_running=True))
    fresh = Calibrator()
    fresh.load(r.p)
    fresh.set_cameras(r.p.models, st["intr"], st["q_ck"], st["p_ck"])
    fresh.set_frames(st["T_wp"], st["v_w"], r.p.ftime)
    fresh.set_imu_params(st["g"], st["b"], st["sf"], st["ts"])
    fresh.set_flags(**{k: getattr(r.g.flags, k) for k, _ in type(r.g.flags)._fields_})
    fresh.set_options(**r.opts)
    s = fresh.solve(free_running=True)
    for k in COUNTS + ("initial_cost", "final_cost"):
        assert after[0][k] == s[k], k
    st1 = fresh.state()
    for k in STATE_KEYS:
        assert np.array_equal(after[1][k], st1[k]), k


# ------------------------------------------------------------------ 5. refusals
def test_refusals():
    import ctypes as C

    from vicalib_b200.capi import Flow, VcgpuError, calibrate_batch, lib

    a = Rig(opts=dict(max_iters=3, **TOL0, **DL), models=("poly3",), n_frames=24, grid=(14, 10), seed=71)
    b = Rig(opts=dict(max_iters=3, **TOL0, **DL), models=("poly3",), n_frames=24, grid=(14, 10), seed=72)
    ref = [r.result(r.g.solve(free_running=True)) for r in (a, b)]
    for r in (a, b):
        r.reset()
    with pytest.raises(VcgpuError, match="handle 1: the same handle as 0"):
        calibrate_batch([a.g, a.g])
    with pytest.raises(VcgpuError, match="handle 0: max_solves <= 0"):
        calibrate_batch([a.g, b.g], max_solves=0)
    b.g.set_options(update_state_every_iteration=1)
    with pytest.raises(VcgpuError, match="handle 1: .*update_state_every_iteration"):
        calibrate_batch([a.g, b.g])
    b.g.set_options(update_state_every_iteration=0)
    b.g.set_profiling(True)
    with pytest.raises(VcgpuError, match="handle 1: .*a vcgpu_set_profiling bit"):
        calibrate_batch([a.g, b.g])
    b.g.set_profiling(False)
    hs = (C.c_void_p * 2)(a.g.h, b.g.h)
    assert lib().vcgpu_calibrate_batch(hs, C.c_int(2), None, None, None) == -1
    assert "handle 0: null flow" in lib().vcgpu_last_error(a.g.h).decode()
    assert lib().vcgpu_calibrate_batch(hs, C.c_int(0), C.byref(Flow()), None, None) == -1
    for r, want in zip((a, b), ref):
        got = r.result(r.g.solve(free_running=True))
        for k in COUNTS + ("initial_cost", "final_cost"):
            assert got[0][k] == want[0][k], k
        for k in STATE_KEYS:
            assert np.array_equal(got[1][k], want[1][k]), k


def test_refusals_of_later_stages():
    """A rig that starts at the vision stage with calibrate_imu on is checked against the inertial batch too, before
    anything runs: phase clocks (the vision batch takes them, the inertial one does not) and a rig whose inertial
    system is past the inertial clusters' fit (G = 68) are refused with their index; without calibrate_imu they pass.
    Every handle then solves as a fresh one does."""
    from vicalib_b200.capi import VcgpuError, calibrate_batch

    vision = dict(inertial=0, rotation_only=1, bias_active=0, scale_active=0)
    a = Rig(flags=vision, opts=dict(max_iters=3, **TOL0, **DL), models=("poly3",), n_frames=24, grid=(14, 10), seed=81)
    b = Rig(flags=vision, opts=dict(max_iters=3, **TOL0, **DL), models=("poly3",), n_frames=24, grid=(14, 10), seed=82)
    c = Rig(flags=vision, opts=dict(max_iters=3, **TOL0, **DL), models=chain_plan.rig_with_globals(68), n_frames=24, grid=(8, 6), seed=83)
    rigs = (a, b, c)
    ref = [r.result(r.g.solve(free_running=True)) for r in rigs]
    for r in rigs:
        r.reset()
    b.g.set_profiling(8)
    with pytest.raises(VcgpuError, match="handle 1: at its inertial stages: a vcgpu_set_profiling bit"):
        calibrate_batch([a.g, b.g], calibrate_imu=True)
    b.g.set_profiling(0)
    with pytest.raises(VcgpuError, match="handle 2: at its inertial stages: the rig does not fit the persistent inertial kernels"):
        calibrate_batch([a.g, b.g, c.g], calibrate_imu=True)
    for r, want in zip(rigs, ref):
        got = r.result(r.g.solve(free_running=True))
        for k in COUNTS + ("initial_cost", "final_cost"):
            assert got[0][k] == want[0][k], k
        for k in STATE_KEYS:
            assert np.array_equal(got[1][k], want[1][k]), k
    c.reset()
    d = _flow([c], calibrate_imu=False, remove_outliers=False, max_solves=1)[0][0]
    assert d["solves"] == 1 and d["stage"] in (capi_stage("VISION"), capi_stage("FINISHED"))


def capi_stage(name):
    from vicalib_b200 import capi

    return getattr(capi, "FLOW_" + name)


def test_inertial_flags_without_calibrate_imu():
    """calibrate_imu off: a rig whose flags start inertial runs vision solves only and reports the vision stage"""
    r = Rig(opts=dict(max_iters=1, strategy=1), models=("poly3",), n_frames=24, grid=(14, 10), seed=91)
    d = _flow([r], calibrate_imu=False, remove_outliers=False, max_solves=2)[0][0]
    assert d["solves"] == 2 and not d["finished"] and d["stage"] == capi_stage("VISION")
    assert d["flags"]["inertial"] == 0


def test_stage_names():
    from vicalib_b200 import capi

    assert stage_of(dict(inertial=0, rotation_only=1, bias=0, scale=0)) == capi.FLOW_VISION
    assert stage_of(dict(inertial=1, rotation_only=0, bias=1, scale=1)) == capi.FLOW_SCALE
