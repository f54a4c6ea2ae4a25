"""GPU: vcgpu_solve_batch (one thread-block cluster per rig, lm_mega_batch_kernel) against vcgpu_solve of the same rig
alone (the cooperative grid, lm_mega_kernel).

Both run the same loop (mega_solve, vc_mega.cuh) on a different number of CTAs, so the two are two summation orders of
one algorithm and the bars are the ones test_gpu_persistent.py states for that: the same iteration count, accepted-step
count and termination, cost to 1e-10 and state to 1e-8 (relative).  Between batches a rig's result must not move at
all: its cluster size is a function of the rig alone, so every comparison of one rig in different batches is bit for
bit.

Every case solves each handle alone first, uploads the problem again (which resets the state) and then solves the
batch, so that a handle is also seen to work through both entry points.  Not covered here: handles on different
devices and frame-sharded handles (both need more than one GPU); their refusals are argument checks next to the ones
tested.
"""
import numpy as np
import pytest

import batch_plan
import chain_plan
import constant_blocks
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

COST_BAR, STATE_BAR = 1e-10, 1e-8
TOL0 = dict(function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
VISION_KEYS = ("intr", "q_ck", "p_ck", "T_wp")
COUNTS = ("iterations", "successful_steps", "termination", "num_residuals")
MULTI_LAUNCH = 4
REJECTING = dict(models=("poly3", "fov"), n_frames=60, grid=(14, 10), seed=11, pose_noise=(0.1, 0.2))  # DOGLEG rejects two steps


class Rig:
    """a problem, its options, and one handle"""

    def __init__(self, problem=None, strategy=0, flags=None, opts=None, **kw):
        from vicalib_b200.capi import Calibrator

        self.p = problem if problem is not None else synth.make_problem(**kw)
        self.g = Calibrator()
        self.g.load(self.p)
        if flags:
            self.g.set_flags(**flags)
        self.g.set_options(strategy=strategy, **(opts if opts is not None else dict(max_iters=6, **TOL0)))

    def reset(self):
        self.g.load(self.p)

    def solo(self):
        s = self.g.solve(free_running=True)
        return s, self.g.state()


def _batch(rigs):
    from vicalib_b200.capi import solve_batch

    sums = solve_batch([r.g for r in rigs])
    return [(s, r.g.state()) for s, r in zip(sums, rigs)]


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1.0))


def _agree(got, ref, what=""):
    (s, st), (s0, st0) = got, ref
    for k in COUNTS:
        assert s[k] == s0[k], (what, k, s[k], s0[k])
    assert abs(s["final_cost"] - s0["final_cost"]) <= COST_BAR * s0["final_cost"], (what, s["final_cost"], s0["final_cost"])
    assert abs(s["initial_cost"] - s0["initial_cost"]) <= COST_BAR * s0["initial_cost"], what
    state = max(_rel(st[k], st0[k]) for k in VISION_KEYS)
    assert state <= STATE_BAR, (what, state)
    return abs(s["final_cost"] - s0["final_cost"]) / s0["final_cost"], state


def _same_bits(got, ref, what=""):
    (s, st), (s0, st0) = got, ref
    for k in COUNTS + ("initial_cost", "final_cost", "kernel_launches"):
        assert s[k] == s0[k], (what, k, s[k], s0[k])
    for k in VISION_KEYS:
        assert np.array_equal(st[k], st0[k]), (what, k)


def _solo_then_batch(rigs, what):
    """every rig alone, then (from the same start) all of them in one call; returns the batch's results"""
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
DOZEN = [
    dict(models=("poly3",), n_frames=12, grid=(14, 10), seed=1),
    dict(models=("linear",), n_frames=25, grid=(8, 6), seed=2),
    dict(models=("fov",), n_frames=50, grid=(14, 10), seed=3),
    dict(models=("poly2",), n_frames=90, grid=(10, 7), seed=4),
    dict(models=("kb4",), n_frames=130, grid=(14, 10), seed=5),
    dict(models=("fov", "kb4"), n_frames=40, grid=(14, 10), seed=6),
    dict(models=("poly3", "fov"), n_frames=200, grid=(8, 6), seed=7),
    dict(models=("poly3", "poly2", "linear"), n_frames=64, grid=(14, 10), seed=8),
    dict(models=("poly3", "poly2", "fov"), n_frames=33, grid=(14, 10), seed=9),  # DOGLEG: one warp fewer (static share)
    dict(models=("poly3", "poly3", "kb4", "fov"), n_frames=80, grid=(14, 10), seed=10),  # G = 51
    dict(models=("poly3",), n_frames=400, grid=(6, 5), seed=11),
    REJECTING,
]


@pytest.mark.parametrize("strategy", [0, 1], ids=["lm", "dogleg"])
def test_batch_matches_solo(strategy):
    rigs = [Rig(strategy=strategy, **kw) for kw in DOZEN]
    assert len({r.g.G for r in rigs}) >= 6
    got, _ = _solo_then_batch(rigs, "dozen " + ("DOGLEG" if strategy else "LM"))
    if strategy == 1:
        assert got[-1][0]["successful_steps"] < got[-1][0]["iterations"], "no rejected step in the trace"


# ------------------------------------------------------------------ 2. independence, bit for bit
def test_result_does_not_depend_on_the_batch():
    target = Rig(strategy=1, **REJECTING)
    others = [Rig(strategy=i % 2, models=(("poly3",), ("fov",), ("kb4", "linear"))[i % 3], n_frames=20 + 3 * i, grid=(8, 6),
                  seed=100 + i) for i in range(39)]

    def run(rigs):
        for r in rigs:
            r.reset()
        return dict(zip(map(id, rigs), _batch(rigs)))

    alone = run([target])
    first = run([target] + others)
    last = run(others + [target])
    reverse = run(([target] + others)[::-1])
    again = run(others + [target])
    for name, res in (("first of 40", first), ("last of 40", last), ("reversed", reverse), ("second call", again)):
        _same_bits(res[id(target)], alone[id(target)], name)
    for r in others:  # and every other rig: same bits first, last, reversed
        for res in (last, reverse, again):
            _same_bits(res[id(r)], first[id(r)], "others")


# ------------------------------------------------------------------ 3. more clusters than fit at once
def test_more_clusters_than_are_resident():
    w = batch_plan.batch_warps(chain_plan.rig_globals(("poly3",), False), 1)
    assert batch_plan.cluster_size(40, w) == 4 and batch_plan.cluster_size(70, w) == 8
    rigs = [Rig(models=("poly3",), n_frames=40, grid=(6, 5), seed=200 + i, opts=dict(max_iters=4, **TOL0)) for i in range(80)]
    rigs += [Rig(models=("poly3",), n_frames=70, grid=(6, 5), seed=300 + i, opts=dict(max_iters=4, **TOL0)) for i in range(20)]
    assert 80 * 4 > chain_plan.device_or_h100()[0] and 20 * 8 > chain_plan.device_or_h100()[0]
    got, _ = _solo_then_batch(rigs, "queued clusters")
    assert all(s["iterations"] == 4 for s, _ in got)


# ------------------------------------------------------------------ 4. every cluster size, both strategies, one call
def test_every_cluster_size_in_one_call():
    frames = [10, 30, 60, 120, 3000]
    w = batch_plan.batch_warps(chain_plan.rig_globals(("fov",), False), 1)
    assert [batch_plan.cluster_size(n, w) for n in frames] == [1, 2, 4, 8, 8]
    assert -(-3000 // 8) > chain_plan.K["kGtabMax"]  # more (frame, camera) pairs per CTA than the group table holds
    rigs = [Rig(strategy=i % 2, models=("fov",), n_frames=n, grid=(4, 3) if n > 1000 else (10, 7), seed=400 + i,
                opts=dict(max_iters=4, **TOL0)) for i, n in enumerate(frames)]
    rigs += [Rig(strategy=1 - i % 2, models=("fov",), n_frames=n, grid=(10, 7), seed=410 + i, opts=dict(max_iters=4, **TOL0))
             for i, n in enumerate(frames[:4])]
    plan = batch_plan.groups([(r.g.opts.strategy, r.p.n_frames, w) for r in rigs])
    assert len(plan) == 8  # cluster sizes 1, 2, 4 and 8 in both strategies; LM's group of 8 holds three rigs
    _solo_then_batch(rigs, "all cluster sizes")


# ------------------------------------------------------------------ 5. each rig stops on its own
def test_each_rig_stops_on_its_own():
    noises = [(2e-3, 5e-3), (0.02, 0.05), (0.1, 0.2), (1e-4, 1e-4), (0.05, 0.1), (0.02, 0.05)]
    rigs = [Rig(strategy=i % 2, models=("poly3", "fov"), n_frames=50, grid=(14, 10), seed=500 + i, pose_noise=pn,
                opts=dict(max_iters=2 if i == 5 else 50)) for i, pn in enumerate(noises)]
    got, ref = _solo_then_batch(rigs, "own stops")
    iters = [s["iterations"] for s, _ in got]
    terms = [s["termination"] for s, _ in got]
    print("iterations", iters, "terminations", terms)
    assert got[5][0]["iterations"] == 2 and got[5][0]["termination"] == 0  # the iteration limit
    assert len(set(iters)) >= 3 and len(set(terms)) >= 2, (iters, terms)


# ------------------------------------------------------------------ 6. constant blocks and unused frames
def test_constant_blocks_come_back_as_uploaded():
    cases = [(constant_blocks.vision_problem(seed=3), constant_blocks.FIX), (constant_blocks.vision_problem(seed=4), {}),
             (constant_blocks.vision_problem(seed=5, n_frames=40), constant_blocks.FIX),
             (synth.make_problem(models=("kb4",), n_frames=30, grid=(14, 10), seed=6), constant_blocks.FIX)]
    rigs = [Rig(problem=p, strategy=i % 2, flags=dict(f)) for i, (p, f) in enumerate(cases)]
    got, _ = _solo_then_batch(rigs, "constant blocks")
    for (p, f), (_, st) in zip(cases, got):
        up = constant_blocks.constant_parts(constant_blocks.uploaded(p), p, f)
        back = constant_blocks.constant_parts(st, p, f)
        assert up.keys() == back.keys() and ("intr" in up) == bool(f)
        for k in up:
            assert np.array_equal(np.asarray(back[k]).ravel(), np.asarray(up[k]).ravel()), k


# ------------------------------------------------------------------ 7. the handle afterwards
def test_handle_after_a_batch():
    kws = [dict(models=("poly3", "fov"), n_frames=50, grid=(14, 10), seed=600), dict(models=("kb4",), n_frames=20, grid=(14, 10), seed=601)]
    opts = dict(max_iters=3, **TOL0)
    solo = [Rig(opts=opts, **kw) for kw in kws]
    bat = [Rig(opts=opts, **kw) for kw in kws]
    ref = [r.solo() for r in solo]
    got = _batch(bat)
    for a, b, rs, rb in zip(got, ref, solo, bat):
        _agree(a, b, "first three iterations")
        ne_s, ne_b = rs.g.normal_equations(), rb.g.normal_equations()
        for k in ("B", "E", "gf", "C", "gc"):
            assert _rel(ne_b[k], ne_s[k]) <= STATE_BAR, k
        assert abs(ne_b["cost"] - ne_s["cost"]) <= COST_BAR * ne_s["cost"]
        assert _rel(rb.g.covariance(), rs.g.covariance()) <= 1e-6  # an inverse: the state's 1e-8 times its conditioning
    for a, rs, rb in zip(got, solo, bat):  # a solo solve continues from the batch's state
        s2, b2 = rs.solo(), rb.solo()
        assert abs(b2[0]["initial_cost"] - a[0]["final_cost"]) <= COST_BAR * a[0]["final_cost"]
        assert b2[0]["final_cost"] < a[0]["final_cost"]
        _agree(b2, s2, "three more iterations, alone")


# ------------------------------------------------------------------ 8. refusals
def _refused(handles, index):
    from vicalib_b200.capi import VcgpuError, solve_batch

    with pytest.raises(VcgpuError) as e:
        solve_batch(handles)
    assert "vcgpu error -1" in str(e.value)
    if index is not None:
        assert f"handle {index}:" in str(e.value), str(e.value)


def test_refusals():
    from vicalib_b200.capi import VcgpuError

    kw = dict(models=("poly3",), n_frames=30, grid=(10, 7))
    opts = dict(max_iters=4, **TOL0)
    fresh = Rig(seed=700, opts=opts, **kw).solo()
    good = [Rig(seed=700, opts=opts, **kw), Rig(seed=701, opts=opts, **kw)]
    ref1 = Rig(seed=701, opts=opts, **kw).solo()

    def bad_with(**changes):
        r = Rig(seed=702, opts=opts, **kw)
        if "flags" in changes:
            r.g.set_flags(**changes["flags"])
        if "options" in changes:
            r.g.set_options(**changes["options"])
        if "profiling" in changes or "flush" in changes:
            r.g.set_profiling(changes.get("profiling", 0), changes.get("flush", False))
        return r

    _refused([], None)                                   # n = 0
    _refused([good[0].g, None, good[1].g], 1)            # a null handle
    _refused([good[0].g, good[1].g, good[0].g], 2)       # a repeated handle
    bads = [bad_with(flags=dict(visual=0)),              # no active observation
            bad_with(options=dict(update_state_every_iteration=1)),
            bad_with(profiling=1), bad_with(profiling=MULTI_LAUNCH),
            Rig(models=("poly3",), n_frames=12, grid=(14, 10), inertial=True, seed=703, flags=dict(inertial=1), opts=opts),
            Rig(models=chain_plan.rig_with_globals(104, False), n_frames=12, grid=(14, 10), seed=704, opts=opts),  # beyond the fit
            bad_with(flush=True)]                        # L2 flushing
    for bad in bads:
        _refused([good[0].g, good[1].g, bad.g], 2)
        _refused([bad.g, good[0].g], 0)
        with pytest.raises(VcgpuError):                  # the plan query refuses what the batch refuses
            bad.g.batch_plan()
    # nothing ran: every handle of the refused batches solves alone as a fresh one does, in as many launches
    _same_bits(good[0].solo(), fresh, "after the refusals")
    _same_bits(good[1].solo(), ref1, "after the refusals")
    s = bads[1].g.solve()  # update_state_every_iteration: vcgpu_solve takes it
    assert s["iterations"] == 4
    # bit 2 is no profiling bit: set_profiling refuses it and leaves the handle solving as a fresh twin does
    two = Rig(seed=702, opts=opts, **kw)
    with pytest.raises(VcgpuError):
        two.g.set_profiling(2, False)
    _same_bits(two.solo(), Rig(seed=702, opts=opts, **kw).solo(), "set_profiling(2) refused")
    for bad in bads[2:4]:
        bad.g.set_profiling(0, False)
    after = _batch(bads[2:4] + [Rig(seed=702, opts=opts, **kw)])  # and, the bit cleared, the batch does
    for a in after[1:]:
        _same_bits(a, after[0], "the same rig three times")


# ------------------------------------------------------------------ 9. one launch per group
def test_one_launch_per_group():
    rigs = [Rig(models=("poly3",), n_frames=50, grid=(14, 10), seed=800 + i) for i in range(12)]
    got, ref = _solo_then_batch(rigs, "like rigs")
    for (s, _), (s0, _) in zip(got, ref):
        # the start point's build and reduction and the Jacobi scale, then the one launch the twelve share (a solo
        # solve: the same prelude and its own cooperative launch)
        assert s["kernel_launches"] == 3 + 1 == s0["kernel_launches"], (s["kernel_launches"], s0["kernel_launches"])
    assert len({s["device_seconds"] for s, _ in got}) == 1  # the time of the launch they all ran in
