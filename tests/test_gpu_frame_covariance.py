"""GPU: vcgpu_get_frame_covariance (the [frame, frame] blocks of (J^T J)^-1 by a selected inversion of the frame
elimination, vc_frame_cov.cuh) against the frame blocks of a dense numpy inverse of the oracle's J^T J at the state the
device converged to, with test_gpu_covariance.py's correlation-scaled bars: 1e-6 vision, 1e-4 inertial.  Covers the
camera models, the inertial flags, fixed intrinsics, frames no camera sees, the chain's level shapes up to 600 frames,
G = 67 and 68 (the persistent inertial kernels' last fitting G and the first one beyond), exact symmetry, the handle left
as it was, and the refusal of a singular system."""
import dataclasses

import numpy as np
import pytest

import chain_plan
import target_views as tv
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
BAR = {False: 1e-6, True: 1e-4}
NUMERIC = -3


def _dense_frame_cov(o, used, live):
    """[frame, frame] blocks of inv(J^T J) from the oracle's block normal equations, with the rows and columns of the
    constant globals, the unused frames (used[f] == False) and a frame's tangents from `live` on removed; those blocks,
    rows and columns are 0"""
    ne = o.normal_equations()
    nf, fd, G = ne["B"].shape[0], o.fd, o.G
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
    keep = np.concatenate([(used[:, None] & (np.arange(fd) < live)[None, :]).ravel(), o.global_mask() != 0])
    # inverted after a symmetric diagonal scaling to unit diagonal: an unscaled LU of these systems (conditioned ~1e11
    # after scaling, far more before) loses digits the scaled one keeps
    Hk = H[np.ix_(keep, keep)]
    d = 1.0 / np.sqrt(np.diag(Hk))
    Hi = np.zeros_like(H)
    Hi[np.ix_(keep, keep)] = np.linalg.inv(Hk * d[:, None] * d[None, :]) * d[:, None] * d[None, :]
    return np.stack([Hi[f * fd:(f + 1) * fd, f * fd:(f + 1) * fd] for f in range(nf)])


def _solved(p, flags, max_iters=15):
    """a handle solved from p, and the oracle at the state it converged to"""
    from oracle.binding import Oracle
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.load(p)
    g.set_flags(**flags)
    g.set_options(function_tol=1e-12, max_iters=max_iters)
    g.solve()
    st = g.state()
    p2 = dataclasses.replace(p, intr=st["intr"], q_ck=st["q_ck"], p_ck=st["p_ck"], T_wp=st["T_wp"], v_w=st["v_w"],
                             g=st["g"], b=st["b"], sf=st["sf"], ts=st["ts"])
    o = Oracle(p2, **flags)
    if flags.get("inertial", 0):
        o.set_imu_weights(g.imu_weights())
    return g, o


def _check(g, o, inertial, used=None):
    nf = g.n_frames
    used = np.ones(nf, bool) if used is None else used
    cov = g.frame_covariance()
    fd = 9 if inertial else 6
    # a rotation-only run reads no velocity: those rows and columns are 0, as a constant block's are
    live = 6 if inertial and g.flags.rotation_only else fd
    assert cov.shape == (nf, fd, fd)
    assert np.array_equal(cov, cov.transpose(0, 2, 1))  # exactly symmetric
    assert not cov[~used].any() and not cov[:, live:].any()  # exactly 0.0
    ref = _dense_frame_cov(o, used, live)
    sd = np.sqrt(np.einsum("fii->fi", ref[used][:, :live, :live]))
    assert np.all(sd > 0)
    err = (np.abs(cov[used][:, :live, :live] - ref[used][:, :live, :live]) / (sd[:, :, None] * sd[:, None, :])).max()
    print(f"\n{nf} frames, fd {fd}, G {g.G}: frame covariance vs dense inverse {err:.1e}")
    assert err <= BAR[inertial], err
    return cov


@pytest.mark.parametrize("models,inertial,flags", [
    (("poly3",), False, {}),
    (("fov", "kb4"), False, {}),
    (("poly3", "poly2"), True, dict(ALL_ON)),
    (("poly3",), True, dict(inertial=1, rotation_only=1, bias_active=0, scale_active=0, optimize_ts=1)),
    (("poly3", "fov"), False, dict(fix_intrinsics=1)),
    (("kb4",), True, dict(ALL_ON, fix_intrinsics=1)),
], ids=["poly3", "fov_kb4", "inertial_all", "rotation_only", "fixed_intrinsics", "inertial_fixed_intrinsics"])
def test_matches_dense_inverse(models, inertial, flags):
    nf = 90 if inertial else 18
    p = synth.make_problem(models=models, n_frames=nf, inertial=inertial, seed=15)
    g, o = _solved(p, flags)
    _check(g, o, inertial)


def test_vision_frames_no_camera_sees():
    """runs of frames no camera sees, at both ends and inside: exactly 0, and the others as if those frames were not
    in the problem"""
    v = tv.build("unseen_runs")
    g, o = _solved(v.p, v.flags)
    _check(g, o, False, used=tv.counts(v.p).sum(0) > 0)


def test_inertial_camera_no_frame_sees():
    """a rig with a camera no frame sees: the frames keep full blocks"""
    v = tv.build("unseen_camera_inertial")
    g, o = _solved(v.p, v.flags)
    _check(g, o, True)


def test_inertial_frames_missing_cameras():
    """a chunk of frames inside the chain that no camera sees (their blocks come from the IMU terms alone) and a run
    seen by one camera of two.  (The target_views rigs of this kind are 24 frames long, or have two-chunk runs at both
    ends; they converge to systems too close to singular, ~1e15 after scaling, for any two inverses to agree to the
    bar.)"""
    p = synth.make_problem(models=("poly3", "poly3"), n_frames=90, grid=(10, 7), inertial=True, seed=45)
    c = chain_plan.CHUNK
    gone = ((p.obs_frame >= 40) & (p.obs_frame < 40 + c)) | ((p.obs_frame >= 60) & (p.obs_frame < 76) & (p.obs_cam == 1))
    p = tv.keep(p, ~gone)
    n = tv.counts(p)
    assert not n[:, 40:40 + c].any() and not n[1, 60:76].any() and n[0, 60:76].all()
    g, o = _solved(p, dict(ALL_ON))
    _check(g, o, True)


# every level shape of the chain's level table up to 600 frames: ragged chunks, a lone separator (on one and on two
# levels), one, two and kCsTop nodes at the top, one to three elimination levels
LEVEL_CASES = [9, 17, 32, 33, 65, 257, 513, 600]


def test_level_cases_cover_the_level_shapes():
    shapes = set()
    for nf in LEVEL_CASES:
        sizes = chain_plan.level_sizes(nf)
        shapes |= {("levels", len(sizes) - 1), ("top", sizes[-1])}
        if chain_plan.lone_separator_levels(nf):
            shapes.add("lone_last")
        if len(chain_plan.lone_separator_levels(nf)) >= 2:
            shapes.add("lone_last_twice")
    assert {("levels", 1), ("levels", 2), ("levels", 3), ("top", 1), ("top", 2), ("top", chain_plan.TOP), "lone_last",
            "lone_last_twice"} <= shapes


@pytest.mark.parametrize("nf", LEVEL_CASES)
def test_level_shapes(nf):
    # a few seconds of motion whatever the frame count, so that gravity and the biases are observable
    p = synth.make_problem(models=("poly3",), n_frames=nf, grid=(8, 6), inertial=True, seed=100 + nf,
                           frame_rate=min(30.0, nf / 3.0))
    g, o = _solved(p, dict(ALL_ON))
    _check(g, o, True)


@pytest.mark.parametrize("G", [67, 68])
def test_many_globals(G):
    """G = 67, the largest rig the persistent inertial kernels take, and G = 68, which only the multi-launch engine
    serves; the selected inversion runs on the multi-launch chain kernels for both"""
    models = chain_plan.rig_with_globals(G)
    p = synth.make_problem(models=models, n_frames=90, grid=(8, 6), inertial=True, seed=G)
    g, o = _solved(p, dict(ALL_ON))
    assert g.G == G
    _check(g, o, True)


def _snapshot(g):
    st = g.state()
    W = g.imu_weights() if g.flags.inertial else np.zeros(0)
    return {k: np.asarray(v).tobytes() for k, v in st.items()}, W.tobytes()


@pytest.mark.parametrize("inertial", [False, True], ids=["vision", "inertial"])
def test_no_side_effects(inertial):
    """state and IMU weights are left bit for bit, and a following solve gives the bits a fresh handle gives"""
    from vicalib_b200.capi import Calibrator

    def make():
        p = synth.make_problem(models=("poly3", "kb4"), n_frames=60 if inertial else 20, inertial=inertial, seed=7)
        g = Calibrator()
        g.load(p)
        g.set_flags(**(ALL_ON if inertial else {}))
        g.set_options(max_iters=4)
        return g

    g, fresh = make(), make()
    g.solve()
    fresh.solve()
    before = _snapshot(g)
    g.frame_covariance()
    assert _snapshot(g) == before
    s, s0 = g.solve(free_running=True), fresh.solve(free_running=True)
    for k in ("iterations", "successful_steps", "termination", "initial_cost", "final_cost"):
        assert s[k] == s0[k], k
    assert _snapshot(g) == _snapshot(fresh)


def test_singular_system_is_refused():
    """every reprojection residual weighted 0: the frames' columns are empty, so J^T J is singular; nothing is written"""
    from vicalib_b200.capi import Calibrator, _p

    p = synth.make_problem(models=("poly3", "poly3"), n_frames=18, seed=90)
    g = Calibrator()
    g.load(p)
    g.set_flags(visual_mult=0.0)
    out = np.full((18, 6, 6), np.nan)
    assert g.L.vcgpu_get_frame_covariance(g.h, _p(out)) == NUMERIC
    assert np.isnan(out).all()
