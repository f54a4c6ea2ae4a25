"""GPU: every device consumer of the IMU stream against the oracle, on the streams of imu_streams.py (jittered, gapped,
slow, partial coverage, frame-tied, dropped frames, 0-2 samples).

- eval_imu (imu_raw_residual in the multi-launch imu_eval): r and J to 1e-9; intervals without measurements exactly 0.
- The normal equations of both inertial engines (eval_mega_kernel, the multi-launch build), 1e-10 per block family.
- update_imu_weights (imu_weights_kernel) from a non-default weight pattern: intervals with >= 2 RK4 steps equal to the
  oracle at 1e-7, intervals without measurements unchanged bit for bit, single- and zero-step intervals (no interior
  sample: the weight is decided by rounding, DESIGN.md UpdateImuWeights) finite and symmetric.
- LM solves with live weights on the streams where every covered interval has >= 2 steps: the persistent engine with
  the deferred weights queue (chain_solve_kernel), the same with the weights in the evaluation launch
  (VCGPU_NO_DEFERRED_WEIGHTS, eval_mega_kernel), the multi-launch engine (imu_weights_kernel); one DOGLEG solve.  Bars
  of test_gpu_imu_parity.test_lm_solve_with_weight_updates and test_gpu_imu_engines.test_deferred_weights_queue.
- Fixed-weight LM solves on the 20 Hz and long-gap streams (single-step intervals), bars of
  test_lm_solve_with_imu_fixed_weights.
- Partial coverage: the velocity of a frame no IMU factor touches comes back bit for bit; time offsets either side of
  the ones where HasElement flips at the two coverage edges.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import imu_streams
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
MULTI_LAUNCH = 4  # vcgpu_set_profiling bit 2
ENGINES = [0, MULTI_LAUNCH]
ENGINE_IDS = ["persistent", "multi_launch"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LM_ITERS = 6
LM_OPTS = dict(max_iters=LM_ITERS, function_tol=0.0, gradient_tol=0.0, param_tol=0.0)


def _persistent_ran(s):
    """test_gpu_imu_engines._persistent_ran: two cooperative launches per iteration plus a fixed set-up"""
    return s["kernel_launches"] <= 2 * s["iterations"] + 12


def _relerr(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _stream(name):
    s = imu_streams.build(name)
    s.p = imu_streams.perturbed(s.p)
    return s


def _pair(p, mode=0, **opts):
    from oracle.binding import Oracle
    from vicalib_b200.capi import Calibrator

    o = Oracle(p, **ALL_ON)
    g = Calibrator()
    g.load(p)
    g.set_flags(**ALL_ON)
    g.set_profiling(mode, False)
    if opts:
        o.set_options(**opts)
        g.set_options(**opts)
    return o, g


def _weights0(ni):
    """a non-default weight pattern: symmetric, positive definite, distinct per interval"""
    rng = np.random.default_rng(11)
    W = 3.0 * rng.standard_normal((ni, 9, 9))
    return 0.5 * (W + W.transpose(0, 2, 1)) + np.arange(400.0, 409.0) * np.eye(9)


@pytest.mark.parametrize("name", imu_streams.NAMES)
def test_eval_imu(name):
    s = _stream(name)
    o, g = _pair(s.p)
    W = _weights0(s.p.n_frames - 1)
    o.set_imu_weights(W)
    g.set_imu_weights(W)
    r_o, J_o = o.eval_imu()
    r_g, J_g = g.eval_imu()
    off = ~s.cls["covered"]
    assert not r_o[off].any() and not J_o[off].any()
    assert not r_g[off].any() and not J_g[off].any()  # no measurements: exactly 0 on the device
    if s.cls["covered"].any():
        assert np.abs(r_g - r_o).max() <= 1e-9 * max(np.abs(r_o).max(), 1.0)
        assert np.abs(J_g - J_o).max() <= 1e-9 * np.abs(J_o).max()


@pytest.mark.parametrize("mode", ENGINES, ids=ENGINE_IDS)
@pytest.mark.parametrize("name", imu_streams.NAMES)
def test_normal_equations(name, mode):
    s = _stream(name)
    o, g = _pair(s.p, mode)
    W = _weights0(s.p.n_frames - 1)
    o.set_imu_weights(W)
    g.set_imu_weights(W)
    ne_o, ne_g = o.normal_equations(), g.normal_equations()
    assert abs(ne_g["cost"] - ne_o["cost"]) <= 1e-11 * ne_o["cost"]
    for k in ("B", "U", "E", "gf", "C", "gc"):
        assert _relerr(ne_g[k], ne_o[k]) <= 1e-10, k


@pytest.mark.parametrize("name", imu_streams.NAMES)
def test_update_imu_weights(name):
    s = _stream(name)
    c = s.cls
    o, g = _pair(s.p)
    W0 = _weights0(s.p.n_frames - 1)
    o.set_imu_weights(W0)
    g.set_imu_weights(W0)
    o.update_imu_weights()
    g.update_imu_weights()
    W_o, W_g = o.imu_weights(), g.imu_weights()
    for k in range(s.p.n_frames - 1):
        if not c["covered"][k]:
            assert np.array_equal(W_g[k], W0[k]), k
        elif c["comparable"][k]:
            assert np.abs(W_g[k] - W_o[k]).max() <= 1e-7 * np.abs(W_o[k]).max(), k
        else:  # single- or zero-step: decided by rounding, not compared
            assert np.isfinite(W_g[k]).all(), (k, W_g[k])
            assert np.abs(W_g[k] - W_g[k].T).max() <= 1e-12 * np.abs(W_g[k]).max(), k


def _compare_live(p, s_o, s_g, st_o, st_g, W_o, W_g, cls):
    """bars of test_lm_solve_with_weight_updates (state) and test_deferred_weights_queue (weights)"""
    assert s_g["successful_steps"] == s_o["successful_steps"]
    assert abs(s_g["final_cost"] - s_o["final_cost"]) <= 1e-6 * s_o["final_cost"]
    for k in ("T_wp", "q_ck", "p_ck", "intr"):
        assert np.abs(st_g[k] - st_o[k]).max() <= 1e-6 * max(1.0, np.abs(st_o[k]).max()), k
    for k in ("v_w", "g", "b", "sf"):
        assert np.abs(st_g[k] - st_o[k]).max() <= 2e-5, k
    on = cls["covered"]
    assert np.abs(W_o[on] - 500 * np.eye(9)).max() > 1.0  # the weights did change
    rel = np.abs(W_g[on] - W_o[on]).max((1, 2)) / np.abs(W_o[on]).max((1, 2))
    assert rel.max() <= 1e-7, int(np.flatnonzero(on)[rel.argmax()])
    assert np.array_equal(W_g[~on], W_o[~on])  # 500 I where there are no measurements


def _oracle_solve(p, strategy=0, update_imu_weights=1):
    from oracle.binding import Oracle

    o = Oracle(p, **ALL_ON)
    o.set_options(strategy=strategy, update_imu_weights=update_imu_weights, **LM_OPTS)
    return o.solve(), o.state(), o.imu_weights()


@pytest.mark.parametrize("mode", ENGINES, ids=ENGINE_IDS)
@pytest.mark.parametrize("name", imu_streams.COMPARABLE)
def test_lm_live_weights(name, mode):
    s = _stream(name)
    _o, g = _pair(s.p, mode, update_imu_weights=1, **LM_OPTS)
    s_g = g.solve()
    assert _persistent_ran(s_g) == (mode == 0), s_g["kernel_launches"]
    s_o, st_o, W_o = _oracle_solve(s.p)
    _compare_live(s.p, s_o, s_g, st_o, g.state(), W_o, g.imu_weights(), s.cls)


_NO_DEFERRED_RUN = """
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests")
import imu_streams
from vicalib_b200.capi import Calibrator
s = imu_streams.build(sys.argv[2])
p = imu_streams.perturbed(s.p)
g = Calibrator()
g.load(p)
g.set_flags(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
g.set_options(max_iters={it}, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, update_imu_weights=1)
r = g.solve()
st = g.state()
np.savez(sys.argv[3], W=g.imu_weights(), launches=r["kernel_launches"], iterations=r["iterations"],
         successful_steps=r["successful_steps"], final_cost=r["final_cost"], **st)
""".format(it=LM_ITERS)


@pytest.mark.parametrize("name", imu_streams.COMPARABLE)
def test_lm_live_weights_no_deferred(name, tmp_path):
    """The persistent engine with the weights computed in eval_mega_kernel instead of chain_solve_kernel's deferred
    queue (VCGPU_NO_DEFERRED_WEIGHTS is read once per process: a subprocess, as test_deferred_weights_queue does)."""
    out = tmp_path / "run.npz"
    env = dict(os.environ, VCGPU_NO_DEFERRED_WEIGHTS="1")
    run = subprocess.run([sys.executable, "-c", _NO_DEFERRED_RUN, ROOT, name, str(out)], env=env, capture_output=True,
                         text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-2000:]
    z = np.load(out)
    s_g = {k: float(z[k]) for k in ("iterations", "successful_steps", "final_cost")}
    assert int(z["launches"]) <= 2 * s_g["iterations"] + 12  # the persistent engine ran
    s = _stream(name)
    s_o, st_o, W_o = _oracle_solve(s.p)
    st_g = {k: z[k] for k in ("T_wp", "q_ck", "p_ck", "intr", "v_w", "g", "b", "sf")}
    _compare_live(s.p, s_o, s_g, st_o, st_g, W_o, z["W"], s.cls)


def test_dogleg_live_weights():
    """Inertial DOGLEG runs on the multi-launch engine."""
    s = _stream("jittered")
    _o, g = _pair(s.p, MULTI_LAUNCH, strategy=1, update_imu_weights=1, **LM_OPTS)
    s_g = g.solve()
    assert not _persistent_ran(s_g)
    s_o, st_o, W_o = _oracle_solve(s.p, strategy=1)
    _compare_live(s.p, s_o, s_g, st_o, g.state(), W_o, g.imu_weights(), s.cls)


@pytest.mark.parametrize("mode", ENGINES, ids=ENGINE_IDS)
@pytest.mark.parametrize("name", ["imu20", "long_gap"])
def test_lm_fixed_weights_single_step(name, mode):
    """Streams with single-step intervals, weights held (bars of test_lm_solve_with_imu_fixed_weights)."""
    s = _stream(name)
    assert s.cls["single"].any()
    _o, g = _pair(s.p, mode, update_imu_weights=0, **LM_OPTS)
    s_g = g.solve()
    assert _persistent_ran(s_g) == (mode == 0), s_g["kernel_launches"]
    s_o, st_o, _W = _oracle_solve(s.p, update_imu_weights=0)
    st_g = g.state()
    assert s_g["successful_steps"] == s_o["successful_steps"]
    assert abs(s_g["final_cost"] - s_o["final_cost"]) <= 1e-8 * s_o["final_cost"]
    for c, m in enumerate(s.p.models):
        K = synth.NUM_INTR[int(m)]
        rel = np.abs(st_g["intr"][c, :K] - st_o["intr"][c, :K]) / np.maximum(np.abs(st_o["intr"][c, :K]), 1e-3)
        assert rel.max() <= 1e-6
    for k in ("T_wp", "v_w", "q_ck", "p_ck", "g", "b", "sf"):
        assert np.abs(st_g[k] - st_o[k]).max() <= 1e-6 * max(1.0, np.abs(st_o[k]).max()), k
    assert abs(st_g["ts"] - st_o["ts"]) <= 1e-8


@pytest.mark.parametrize("mode", ENGINES, ids=ENGINE_IDS)
def test_partial_untouched_velocities(mode):
    """A frame no IMU factor touches has a zero velocity gradient, so a zero velocity step: its velocity comes back
    bit for bit, while its pose moves with the vision terms."""
    s = _stream("partial")
    _o, g = _pair(s.p, mode, update_imu_weights=1, **LM_OPTS)
    s_g = g.solve()
    assert s_g["successful_steps"] > 0
    st = g.state()
    f = list(s.untouched_frames)
    assert np.array_equal(st["v_w"][f], s.p.v_w[f])
    assert np.abs(st["T_wp"][f] - s.p.T_wp[f]).max(1).min() > 1e-9  # every one of those poses moved
    touched = np.setdiff1d(np.arange(s.p.n_frames), f)
    assert (np.abs(st["v_w"][touched] - s.p.v_w[touched]).max(1) > 0).all()


def test_time_offset_across_coverage_edges():
    """Time offsets either side of the two where HasElement flips on the partial stream: interval 2 gains its
    measurements when ftime[2] >= t_0 + ts, interval n-3 when ftime[n-3] <= t_last + ts (bars of
    test_imu_time_offset_boundary_crossing)."""
    s = _stream("partial")
    p = s.p
    nf = p.n_frames
    edges = [(p.ftime[2] - p.imu_t[0], 2), (p.ftime[nf - 3] - p.imu_t[-1], nf - 3)]
    o, g = _pair(p)
    for edge, k in edges:
        seen = set()
        for ts in (edge - 2e-7, edge + 2e-7):
            cls = imu_streams.classify(p, ts)
            seen.add(bool(cls["covered"][k]))
            o.set_imu_params(p.g, p.b, p.sf, ts)
            g.set_imu_params(p.g, p.b, p.sf, ts)
            r_o, J_o = o.eval_imu()
            r_g, J_g = g.eval_imu()
            assert not r_g[~cls["covered"]].any() and not J_g[~cls["covered"]].any()
            assert np.abs(r_g - r_o).max() <= 1e-9 * max(np.abs(r_o).max(), 1.0), ts
            assert np.abs(J_g - J_o).max() <= 1e-9 * np.abs(J_o).max(), ts
            assert np.abs(J_g[:, :, 32] - J_o[:, :, 32]).max() <= 1e-9 * np.abs(J_o).max(), ts
            ne_o, ne_g = o.normal_equations(), g.normal_equations()  # eval_mega_kernel
            assert abs(ne_g["cost"] - ne_o["cost"]) <= 1e-11 * ne_o["cost"]
            for key in ("B", "U", "gf", "C", "gc"):
                assert _relerr(ne_g[key], ne_o[key]) <= 1e-10, key
        assert seen == {False, True}, (edge, k)  # the offsets do straddle the flip
