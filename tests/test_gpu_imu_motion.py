"""GPU: the inertial path under vigorous motion (imu_motion.py: 200 Hz / 400 Hz / 1 kHz IMUs, |w| up to 7 rad/s, 9-51 RK4
steps per interval, the rig's attitude across pi) and across the quaternion double cover.

Against references, at the bars the suite already uses for the same comparison:
- eval_imu (imu_eval_kernel) against tests/golden/imu_vigorous_kat.npz, switch 0 and 1 (test_gpu_golden.py, 1e-9);
- eval_imu and the normal equations of both inertial engines on each builder against the oracle (test_gpu_imu_streams.py);
- a cold update_imu_weights against the oracle, 1e-7 relative per interval;
- LM solves with live weights on both engines against the oracle (test_gpu_imu_streams._compare_live);
- the weights a solve leaves against one cold update at the same state (test_gpu_weights_warm.py);
- solve_batch_inertial with a vigorous rig next to a gentle one against each rig's own solve (test_gpu_batch_inertial.py);
- covariance() and frame_covariance() against a dense inverse (test_gpu_covariance.py, test_gpu_frame_covariance.py).

Sign invariance: a scattered third of the frame quaternions and one camera's q_ck negated, on an inertial rig and a
vision-only rig, against the same handle unflipped: residuals, tangent Jacobians, normal equations (both engines) and
weights to 1e-12 of the largest entry; LM solves on the persistent and multi-launch engines and through
vcgpu_solve_batch / vcgpu_solve_batch_inertial take the same accept / reject sequence and reach the same state up to
each block's sign (oracle-parity bars), and every negated quaternion comes back with the sign it went in with;
covariance() and frame_covariance() at the solved state.
"""
import dataclasses
import os

import numpy as np
import pytest

import imu_motion
import test_gpu_batch_inertial as tbi
import test_gpu_covariance as tcov
import test_gpu_frame_covariance as tfc
import test_gpu_imu_streams as tis
import test_gpu_weights_warm as tww
from test_cpu_imu_motion import kat_problem
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ALL_ON = tis.ALL_ON
ENGINES, ENGINE_IDS, MULTI_LAUNCH = tis.ENGINES, tis.ENGINE_IDS, tis.MULTI_LAUNCH
SIGN_BAR = 1e-12


def _motion(name):
    return imu_motion.build(name)


@pytest.mark.parametrize("switch", [0, 1])
def test_imu_kernel_vs_vigorous_kat(switch):
    from vicalib_b200.capi import Calibrator

    z = np.load(os.path.join(GOLD, "imu_vigorous_kat.npz"))
    p = kat_problem(z)
    g = Calibrator()
    g.set_cameras([0], np.array([[300, 300, 320, 240, 0, 0, 0, 0, 0, 0.0]]), np.array([[0, 0, 0, 1.0]]), np.zeros((1, 3)))
    g.set_frames(p.T_wp, p.v_w, p.ftime)
    g.set_observations(np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros((0, 3)), np.zeros((0, 2)))
    g.set_imu(p.imu_t, p.imu_w, p.imu_a, synth.GYRO_SIGMA, synth.ACCEL_SIGMA)
    g.set_imu_params(p.g, p.b, p.sf, p.ts)
    g.set_flags(inertial=1, rotation_only=switch, bias_active=1, scale_active=1, optimize_ts=1)
    g.set_imu_weights(np.broadcast_to(z["W"], (p.n_frames - 1, 9, 9)).copy())
    r, J = g.eval_imu()
    err_r = np.abs(r - z["r"][switch]).max() / np.abs(z["r"][switch]).max()
    err_J = np.abs(J - z["J"][switch]).max() / np.abs(z["J"][switch]).max()
    print(f"\nimu_eval_kernel vs vigorous KAT, switch {switch}: r {err_r:.1e}, J {err_J:.1e}")
    assert err_r <= 1e-9 and err_J <= 1e-9


@pytest.mark.parametrize("name", imu_motion.NAMES)
def test_eval_imu(name):
    m = _motion(name)
    o, g = tis._pair(m.p)
    W = tis._weights0(m.p.n_frames - 1)
    o.set_imu_weights(W)
    g.set_imu_weights(W)
    r_o, J_o = o.eval_imu()
    r_g, J_g = g.eval_imu()
    assert np.abs(r_g - r_o).max() <= 1e-9 * max(np.abs(r_o).max(), 1.0)
    assert np.abs(J_g - J_o).max() <= 1e-9 * np.abs(J_o).max()


@pytest.mark.parametrize("mode", ENGINES, ids=ENGINE_IDS)
@pytest.mark.parametrize("name", imu_motion.NAMES)
def test_normal_equations(name, mode):
    m = _motion(name)
    o, g = tis._pair(m.p, mode)
    W = tis._weights0(m.p.n_frames - 1)
    o.set_imu_weights(W)
    g.set_imu_weights(W)
    ne_o, ne_g = o.normal_equations(), g.normal_equations()
    assert abs(ne_g["cost"] - ne_o["cost"]) <= 1e-11 * ne_o["cost"]
    for k in ("B", "U", "E", "gf", "C", "gc"):
        assert tis._relerr(ne_g[k], ne_o[k]) <= 1e-10, k


@pytest.mark.parametrize("name", imu_motion.NAMES)
def test_update_imu_weights(name):
    m = _motion(name)
    o, g = tis._pair(m.p)
    W0 = tis._weights0(m.p.n_frames - 1)
    o.set_imu_weights(W0)
    g.set_imu_weights(W0)
    o.update_imu_weights()
    g.update_imu_weights()
    W_o, W_g = o.imu_weights(), g.imu_weights()
    assert m.cls["comparable"].all()
    rel = np.abs(W_g - W_o).max((1, 2)) / np.abs(W_o).max((1, 2))
    print(f"\n{name}: weights vs oracle {rel.max():.1e}")
    assert rel.max() <= 1e-7, int(rel.argmax())


@pytest.mark.parametrize("mode", ENGINES, ids=ENGINE_IDS)
@pytest.mark.parametrize("name", imu_motion.NAMES)
def test_lm_live_weights(name, mode):
    m = _motion(name)
    _o, g = tis._pair(m.p, mode, update_imu_weights=1, **tis.LM_OPTS)
    s_g = g.solve()
    assert tis._persistent_ran(s_g) == (mode == 0), s_g["kernel_launches"]
    s_o, st_o, W_o = tis._oracle_solve(m.p)
    tis._compare_live(m.p, s_o, s_g, st_o, g.state(), W_o, g.imu_weights(), m.cls)


@pytest.mark.parametrize("mode", ENGINES, ids=ENGINE_IDS)
def test_solve_weights_equal_cold(mode):
    m = _motion("imu400")
    s, err = tww._solve_vs_cold(tww._calibrator(m.p, mode, max_iters=10))
    print(f"\nimu400: {s['successful_steps']} accepted, max |W_solve - W_cold| / max |W| = {err:.3e}")
    assert s["successful_steps"] >= 1 and err <= tww.WARM_BAR


def test_batch_vigorous_next_to_gentle():
    rigs = [tbi.Rig(_motion("imu400").p), tbi.Rig(models=("poly3", "kb4"), n_frames=40, grid=(10, 7), seed=2),
            tbi.Rig(_motion("imu1000").p)]
    tbi._solo_then_batch(rigs, "vigorous and gentle")


def _cov_problem():
    """90 frames (3 s) of vigorous motion at 30 Hz / 200 Hz, two cameras"""
    p = synth.make_problem(models=("poly3", "poly2"), n_frames=90, inertial=True, seed=15, motion="vigorous")
    assert len(imu_motion.regime(p)["sign_flips"]) >= 1
    return p


def test_covariances():
    g, o = tfc._solved(_cov_problem(), dict(ALL_ON))
    tcov._check(g, o, True)
    tfc._check(g, o, True)


# ------------------------------------------------------------------ sign invariance on the device
def _rig(kind):
    """(problem, flags, flipped problem, flipped frames, flipped camera)"""
    if kind == "inertial":
        p, flags = _motion("imu400").p, dict(ALL_ON)
    else:
        p, flags = imu_motion.vision(), {}
    frames, cams = imu_motion.scattered(p.n_frames), [p.n_cams - 1]
    return p, flags, imu_motion.flipped(p, frames, cams), frames, cams


def _handle(p, flags, mode=0, **opts):
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.load(p)
    g.set_flags(**flags)
    g.set_profiling(mode, False)
    if opts:
        g.set_options(**opts)
    return g


def _same(a, b, what, bits):
    err = np.abs(a - b).max() / max(np.abs(a).max(), 1e-300)
    assert err <= SIGN_BAR, (what, err)
    if np.array_equal(a, b):
        bits.append(what)


@pytest.mark.parametrize("kind", ["inertial", "vision"])
def test_sign_invariance_evaluations(kind):
    p, flags, q, _frames, _cams = _rig(kind)
    inertial = kind == "inertial"
    bits = []
    for mode, mid in zip(ENGINES, ENGINE_IDS):
        a, b = _handle(p, flags, mode), _handle(q, flags, mode)
        if inertial:
            W = tis._weights0(p.n_frames - 1)
            a.set_imu_weights(W)
            b.set_imu_weights(W)
        if mode == 0:
            for (x, y), k in zip(zip(a.eval_reproj(), b.eval_reproj()), ("r_reproj", "J_reproj")):
                _same(x, y, k, bits)
            if inertial:
                for (x, y), k in zip(zip(a.eval_imu(), b.eval_imu()), ("r_imu", "J_imu")):
                    _same(x, y, k, bits)
        na, nb = a.normal_equations(), b.normal_equations()
        for k in ("B", "U", "E", "gf", "C", "gc"):
            _same(na[k], nb[k], f"{mid}:{k}", bits)
        assert abs(na["cost"] - nb["cost"]) <= SIGN_BAR * na["cost"]
        if inertial and mode == 0:
            a.update_imu_weights()
            b.update_imu_weights()
            _same(a.imu_weights(), b.imu_weights(), "W", bits)
    print(f"\n{kind}: bit-identical under q -> -q: {bits}")


def _unflip(st, frames, cams):
    st = dict(st)
    st["T_wp"], st["q_ck"] = st["T_wp"].copy(), st["q_ck"].copy()
    st["T_wp"][frames, :4] *= -1.0
    st["q_ck"][cams] *= -1.0
    return st


def _same_solve(s_a, s_b, st_a, st_b, q, frames, cams, rows=True):
    for k in ("iterations", "successful_steps", "termination"):
        assert s_a[k] == s_b[k], (k, s_a[k], s_b[k])
    if rows:
        assert np.array_equal(s_a["rows"][:, 8], s_b["rows"][:, 8])  # the accept / reject sequence
    assert abs(s_a["final_cost"] - s_b["final_cost"]) <= 1e-6 * s_a["final_cost"]
    # every negated quaternion comes back with its sign: it stays on the side of the one it started from
    assert (np.einsum("ij,ij->i", st_b["T_wp"][:, :4], q.T_wp[:, :4]) > 0).all()
    assert (np.einsum("ij,ij->i", st_b["q_ck"], q.q_ck) > 0).all()
    u = _unflip(st_b, frames, cams)
    for k in ("T_wp", "q_ck", "p_ck", "intr"):
        assert np.abs(u[k] - st_a[k]).max() <= 1e-6 * max(1.0, np.abs(st_a[k]).max()), k
    for k in ("v_w", "g", "b", "sf"):
        assert np.abs(u[k] - st_a[k]).max() <= 2e-5, k
    return all(np.array_equal(u[k], st_a[k]) for k in u)


@pytest.mark.parametrize("engine", ["persistent", "multi_launch", "batch"])
@pytest.mark.parametrize("kind", ["inertial", "vision"])
def test_sign_invariance_solve(kind, engine):
    from vicalib_b200.capi import solve_batch, solve_batch_inertial

    p, flags, q, frames, cams = _rig(kind)
    opts = dict(tis.LM_OPTS, update_imu_weights=1) if kind == "inertial" else dict(tis.LM_OPTS)
    mode = MULTI_LAUNCH if engine == "multi_launch" else 0
    a, b = _handle(p, flags, mode, **opts), _handle(q, flags, mode, **opts)
    if engine == "batch":
        call = solve_batch_inertial if kind == "inertial" else solve_batch
        s_a, s_b = call([a, b])
    else:
        s_a, s_b = a.solve(), b.solve()
    assert s_a["successful_steps"] >= 1
    bits = _same_solve(s_a, s_b, a.state(), b.state(), q, frames, cams, rows=engine != "batch")
    if kind == "inertial":
        W_a, W_b = a.imu_weights(), b.imu_weights()
        assert (np.abs(W_a - W_b).max((1, 2)) / np.abs(W_a).max((1, 2))).max() <= 1e-7
    print(f"\n{kind} {engine}: states bit-identical up to sign: {bits}")


@pytest.mark.parametrize("kind", ["inertial", "vision"])
def test_sign_invariance_covariances(kind):
    """covariance() and frame_covariance() of a solved state and of the same state with the quaternions negated"""
    if kind == "inertial":
        p, flags = _cov_problem(), dict(ALL_ON)
    else:
        p, flags = imu_motion.vision(), {}
    g = _handle(p, flags, 0, function_tol=1e-12, max_iters=15)
    g.solve()
    st = g.state()
    p = dataclasses.replace(p, intr=st["intr"], q_ck=st["q_ck"], p_ck=st["p_ck"], T_wp=st["T_wp"], v_w=st["v_w"],
                            g=st["g"], b=st["b"], sf=st["sf"], ts=st["ts"])
    q = imu_motion.flipped(p, imu_motion.scattered(p.n_frames), [p.n_cams - 1])
    a, b = _handle(p, flags), _handle(q, flags)
    if kind == "inertial":
        a.set_imu_weights(g.imu_weights())
        b.set_imu_weights(g.imu_weights())
    bits = []
    _same(a.covariance(), b.covariance(), "covariance", bits)
    _same(a.frame_covariance(), b.frame_covariance(), "frame_covariance", bits)
    print(f"\n{kind}: bit-identical under q -> -q: {bits}")
