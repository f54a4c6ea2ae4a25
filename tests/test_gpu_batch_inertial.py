"""GPU: vcgpu_solve_batch_inertial (one thread-block cluster per rig: chain_solve_batch_kernel + eval_mega_batch_kernel)
against vcgpu_solve of the same rig alone (the cooperative grid: chain_solve_kernel + eval_mega_kernel).

Both run the same two routines (chain_solve, eval_mega) on a different number of CTAs, so the two are two summation
orders of one algorithm and the bars are the ones test_gpu_imu_engines.py states for that: the same iterations,
accepted steps and termination, cost within 1e-10 and state within 1e-8 (relative), ts within 1e-8, and the weights
after the solve within 1e-9 of each interval's largest entry.  Between batches a rig's result must not move at all:
its cluster size is a function of the rig alone, so every comparison of one rig in different batches is bit for bit.

Every case solves each handle alone first, uploads the problem again (which resets the state and the weights) and
then solves the batch.  Not covered here: handles on different devices and frame-sharded handles (both need more than
one GPU); their refusals are argument checks next to the ones tested.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import batch_imu_plan
import chain_plan
import imu_streams
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
COST_BAR, STATE_BAR, TS_BAR, WEIGHTS_BAR = 1e-10, 1e-8, 1e-8, 1e-9
TOL0 = dict(function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
STATE_KEYS = ("T_wp", "v_w", "q_ck", "p_ck", "intr", "g", "b", "sf")
COUNTS = ("iterations", "successful_steps", "termination", "num_residuals")
TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)


class Rig:
    """a problem, its flags and options, and one handle"""

    def __init__(self, problem=None, flags=None, opts=None, **kw):
        from vicalib_b200.capi import Calibrator

        self.p = problem if problem is not None else synth.make_problem(inertial=True, **kw)
        self.g = Calibrator()
        self.g.load(self.p)
        self.g.set_flags(**dict(ALL_ON, **(flags or {})))
        self.g.set_options(**(opts if opts is not None else dict(max_iters=6, **TOL0)))

    def reset(self):
        self.g.load(self.p)

    def result(self, s):
        W = self.g.imu_weights() if self.g.flags.inertial else np.zeros((0, 9, 9))
        return s, self.g.state(), W

    def solo(self):
        return self.result(self.g.solve(free_running=True))


def _batch(rigs):
    from vicalib_b200.capi import solve_batch_inertial

    sums = solve_batch_inertial([r.g for r in rigs])
    return [r.result(s) for s, r in zip(sums, rigs)]


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1.0))


def _agree(got, ref, what=""):
    (s, st, W), (s0, st0, W0) = got, ref
    for k in COUNTS:
        assert s[k] == s0[k], (what, k, s[k], s0[k])
    assert abs(s["final_cost"] - s0["final_cost"]) <= COST_BAR * s0["final_cost"], (what, s["final_cost"], s0["final_cost"])
    assert abs(s["initial_cost"] - s0["initial_cost"]) <= COST_BAR * s0["initial_cost"], what
    state = max(_rel(st[k], st0[k]) for k in STATE_KEYS)
    assert state <= STATE_BAR, (what, state)
    assert abs(st["ts"] - st0["ts"]) <= TS_BAR, what
    w = float((np.abs(W - W0).max((1, 2)) / np.abs(W0).max((1, 2))).max()) if len(W0) else 0.0
    assert w <= WEIGHTS_BAR, (what, w)
    return abs(s["final_cost"] - s0["final_cost"]) / s0["final_cost"], state


def _same_bits(got, ref, what=""):
    (s, st, W), (s0, st0, W0) = got, ref
    for k in COUNTS + ("initial_cost", "final_cost", "kernel_launches"):
        assert s[k] == s0[k], (what, k, s[k], s0[k])
    for k in STATE_KEYS:
        assert np.array_equal(st[k], st0[k]), (what, k)
    assert st["ts"] == st0["ts"] and np.array_equal(W, W0), what


def _solo_then_batch(rigs, what):
    """every rig alone, then (from the same start) all of them in one call; returns the batch's and the solo results"""
    ref = [r.solo() for r in rigs]
    for r in rigs:
        r.reset()
    got = _batch(rigs)
    worst = [0.0, 0.0]
    for i, (a, b) in enumerate(zip(got, ref)):
        c, s = _agree(a, b, f"{what} rig {i}")
        worst = [max(worst[0], c), max(worst[1], s)]
    print(f"\n{what}: {len(rigs)} rigs, batch vs solo: cost {worst[0]:.1e} state {worst[1]:.1e}")
    return got, ref


# ------------------------------------------------------------------ 1. batch against solo
SHAPES = [
    dict(models=("poly3",), n_frames=24, grid=(14, 10), seed=1),
    dict(models=("poly3", "kb4"), n_frames=200, grid=(14, 10), seed=2),
    dict(models=chain_plan.rig_with_globals(67), n_frames=256, grid=(8, 6), seed=3),  # the edge of the fit
    dict(models=("poly3", "poly3"), n_frames=2000, grid=(4, 3), seed=4),               # target-shaped
]


def check_against_solo(weights):
    """the four shapes, weights held or live; a function of its own so that a subprocess can run it with
    VCGPU_NO_DEFERRED_WEIGHTS set (read once per process)"""
    assert chain_plan.rig_globals(SHAPES[2]["models"]) == 67
    assert [batch_imu_plan.cluster_size(kw["n_frames"]) for kw in SHAPES] == [2, 8, 8, 8]
    rigs = [Rig(opts=dict(max_iters=6, update_imu_weights=weights, **TOL0), **kw) for kw in SHAPES]
    got, _ = _solo_then_batch(rigs, f"shapes, update_imu_weights={weights}")
    if weights:
        for _, _, W in got:
            assert np.abs(W - 500 * np.eye(9)).max() > 1.0  # the weights did change


@pytest.mark.parametrize("weights", [0, 1], ids=["fixed_weights", "live_weights"])
def test_batch_matches_solo(weights):
    check_against_solo(weights)


@pytest.mark.parametrize("weights", [0, 1], ids=["fixed_weights", "live_weights"])
def test_batch_matches_solo_no_deferred(weights):
    """vcgpu_solve with the weights computed in eval_mega_kernel (the batch always computes them in its evaluation)"""
    env = dict(os.environ, VCGPU_NO_DEFERRED_WEIGHTS="1")
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {TESTS!r}]; import test_gpu_batch_inertial as t; "
            f"t.check_against_solo({weights})")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]


# ------------------------------------------------------------------ 2. independence, bit for bit
def test_result_does_not_depend_on_the_batch():
    opts = dict(max_iters=5, update_imu_weights=1, **TOL0)
    target = Rig(opts=opts, models=("poly3", "kb4"), n_frames=200, grid=(14, 10), seed=10)
    like = [Rig(opts=opts, models=("poly3",), n_frames=100 + 20 * i, grid=(8, 6), seed=11 + i) for i in range(7)]
    mixed = [Rig(opts=opts, models=("fov",), n_frames=n, grid=(8, 6), seed=20 + i) for i, n in enumerate((12, 24, 50, 14, 30))]
    assert {batch_imu_plan.cluster_size(r.p.n_frames) for r in like} == {8}
    assert {batch_imu_plan.cluster_size(r.p.n_frames) for r in mixed} == {1, 2, 4}

    def run(rigs):
        for r in rigs:
            r.reset()
        return dict(zip(map(id, rigs), _batch(rigs)))

    alone = run([target])
    among = run([target] + like)
    reverse = run(([target] + like)[::-1])
    mix = run(mixed[:2] + [target] + mixed[2:])
    for name, res in (("among 7 others", among), ("reversed", reverse), ("other cluster sizes", mix)):
        _same_bits(res[id(target)], alone[id(target)], name)
    for r in like:
        _same_bits(reverse[id(r)], among[id(r)], "the others, reversed")


# ------------------------------------------------------------------ 3. each rig stops on its own
def _thresholds(p):
    """a gradient and a parameter tolerance that end the solve of p at a known iteration (test_gpu_imu_engines'
    test_weights_are_current_after_solve)"""
    r = Rig(problem=p, opts=dict(max_iters=12, update_imu_weights=1, **TOL0))
    rows = r.g.solve()["rows"]
    gmax, sn = rows[:, 3], rows[:, 5]
    k = next(it for it in range(2, len(rows)) if rows[it, 8] == 1 and gmax[it] < 0.99 * gmax[:it].min())
    gtol = float(np.sqrt(gmax[k] * gmax[:k].min()))
    j = next(it for it in range(2, len(rows)) if 0 < sn[it] < 0.5 * sn[1:it][sn[1:it] > 0].min())
    x = np.sqrt(sum(np.sum(np.square(v)) for v in (p.T_wp, p.v_w, p.q_ck, p.p_ck, p.intr, p.g, p.b, p.sf, [p.ts])))
    ptol = float(np.sqrt(sn[j] * sn[1:j][sn[1:j] > 0].min())) / x
    return gtol, ptol


def test_each_rig_stops_on_its_own():
    p = synth.make_problem(models=("poly3",), n_frames=40, grid=(14, 10), inertial=True, seed=29)
    gtol, ptol = _thresholds(p)
    base = dict(update_imu_weights=1, **TOL0)
    cases = [(dict(base, max_iters=3), 0), (dict(base, max_iters=100, function_tol=1e-4), 1),
             (dict(base, max_iters=100, gradient_tol=gtol), 2), (dict(base, max_iters=100, param_tol=ptol), 3)]
    rigs = [Rig(problem=p, opts=o) for o, _ in cases]
    rigs.append(Rig(opts=dict(base, max_iters=7), models=("poly3", "fov"), n_frames=150, grid=(8, 6), seed=30))
    got, _ = _solo_then_batch(rigs, "own stops")
    assert [s["termination"] for s, _, _ in got[:4]] == [term for _, term in cases]
    assert got[0][0]["iterations"] == 3 and got[4][0]["iterations"] == 7
    print("iterations", [s["iterations"] for s, _, _ in got])


# ------------------------------------------------------------------ 4. flags
def test_flags():
    kw = dict(models=("poly3", "fov"), n_frames=60, grid=(14, 10))
    live = dict(max_iters=6, update_imu_weights=1, **TOL0)
    cases = [dict(flags=dict(fix_intrinsics=1)), dict(flags=dict(rotation_only=1)),
             dict(flags=dict(bias_active=0, scale_active=0, optimize_ts=0)), dict(flags=dict(visual=0)),
             dict(flags={}, opts=dict(live, jacobi_scaling=0))]
    rigs = [Rig(seed=40 + i, flags=c["flags"], opts=c.get("opts", live), **kw) for i, c in enumerate(cases)]
    uploaded = [r.g.state() for r in rigs]
    got, _ = _solo_then_batch(rigs, "flags")
    assert np.array_equal(got[0][1]["intr"], uploaded[0]["intr"])  # fix_intrinsics: constant, bit for bit
    assert not np.array_equal(got[1][1]["intr"], uploaded[1]["intr"])
    off = got[2][1]
    assert np.array_equal(off["b"], uploaded[2]["b"]) and np.array_equal(off["sf"], uploaded[2]["sf"])
    assert off["ts"] == uploaded[2]["ts"]


# ------------------------------------------------------------------ 5. the IMU streams of real recordings
STREAMS = [("short_gaps", 1), ("long_gap", 0), ("partial", 1), ("imu20", 0), ("samples2", 0)]


def test_imu_streams():
    streams = [imu_streams.build(name) for name, _ in STREAMS]
    for s in streams:
        s.p = imu_streams.perturbed(s.p)
    rigs = [Rig(problem=s.p, opts=dict(max_iters=6, update_imu_weights=w, **TOL0)) for s, (_, w) in zip(streams, STREAMS)]
    got, _ = _solo_then_batch(rigs, "IMU streams")
    part = streams[2]
    f = list(part.untouched_frames)
    assert f and np.array_equal(got[2][1]["v_w"][f], part.p.v_w[f])  # velocities no IMU factor touches


# ------------------------------------------------------------------ 6. more clusters than fit at once
def test_more_clusters_than_are_resident():
    first = Rig(opts=dict(max_iters=4, **TOL0), models=("poly3",), n_frames=80, grid=(6, 5), seed=100)
    size, resident = first.g.batch_plan_inertial()
    assert size == 8 == batch_imu_plan.cluster_size(80) and resident >= 1
    rigs = [first] + [Rig(opts=dict(max_iters=4, **TOL0), models=("poly3",), n_frames=80, grid=(6, 5), seed=101 + i)
                      for i in range(resident + 3)]
    got, _ = _solo_then_batch(rigs, f"{len(rigs)} rigs, {resident} clusters resident")
    assert all(s["iterations"] == 4 for s, _, _ in got)


# ------------------------------------------------------------------ 7. launch count, device time, the handle afterwards
def test_launches_and_the_handle_afterwards():
    specs = [(dict(models=("poly3",), n_frames=50, grid=(14, 10), seed=200 + i), i % 2, 3 + i) for i in range(6)]
    rigs = [Rig(opts=dict(max_iters=it, update_imu_weights=w, **TOL0), **kw) for kw, w, it in specs]
    got, ref = _solo_then_batch(rigs, "launch counts")
    for (s, _, _), (s0, _, _), (_, w, it) in zip(got, ref, specs):
        assert s["kernel_launches"] == batch_imu_plan.launches(it, w) == s0["kernel_launches"], (s["kernel_launches"], s0["kernel_launches"])
    assert len({s["device_seconds"] for s, _, _ in got}) == 1  # the batch's loop, shared
    # a vcgpu_solve after the batch gives the bits a fresh handle gives
    for r, (kw, w, it) in zip(rigs[:3], specs):
        r.reset()
        fresh = Rig(opts=dict(max_iters=it, update_imu_weights=w, **TOL0), **kw)
        _same_bits(r.solo(), fresh.solo(), "vcgpu_solve after the batch")


# ------------------------------------------------------------------ 8. refusals
def _refused(handles, index):
    from vicalib_b200.capi import VcgpuError, solve_batch_inertial

    with pytest.raises(VcgpuError) as e:
        solve_batch_inertial(handles)
    assert "vcgpu error -1" in str(e.value)
    if index is not None:
        assert f"handle {index}:" in str(e.value), str(e.value)


def test_refusals():
    from vicalib_b200.capi import VcgpuError

    kw = dict(models=("poly3",), n_frames=30, grid=(10, 7))
    opts = dict(max_iters=4, **TOL0)
    fresh = [Rig(seed=700 + i, opts=opts, **kw).solo() for i in range(2)]
    good = [Rig(seed=700 + i, opts=opts, **kw) for i in range(2)]

    def bad(flags=None, options=None, profiling=None, flush=False, **shape):
        r = Rig(seed=702, opts=dict(opts, **(options or {})), flags=flags, **(shape or kw))
        if profiling is not None or flush:
            r.g.set_profiling(profiling or 0, flush)
        return r

    specs = [dict(flags=dict(inertial=0)), dict(options=dict(strategy=1)), dict(options=dict(update_state_every_iteration=1)),
             dict(profiling=1), dict(profiling=4), dict(profiling=8), dict(flush=True),
             dict(models=chain_plan.rig_with_globals(68), n_frames=12, grid=(14, 10))]
    assert chain_plan.rig_globals(specs[-1]["models"]) == 68
    _refused([], None)                                   # n = 0
    _refused([good[0].g, good[1].g, None], 2)            # a null handle
    _refused([None, good[0].g], 0)
    _refused([good[0].g, good[1].g, good[0].g], 2)       # a repeated handle
    bads = [bad(**s) for s in specs]
    for b in bads:
        _refused([good[0].g, good[1].g, b.g], 2)
        _refused([b.g, good[0].g, good[1].g], 0)
    with pytest.raises(VcgpuError):
        bads[0].g.batch_plan_inertial()
    with pytest.raises(VcgpuError):
        bads[-1].g.batch_plan_inertial()
    # nothing ran: every handle of the refused batches solves alone as a fresh one does, in as many launches
    for g, f in zip(good, fresh):
        _same_bits(g.solo(), f, "after the refusals")
    for b, s in zip(bads, specs):
        _same_bits(b.solo(), bad(**s).solo(), f"refused {s}")
