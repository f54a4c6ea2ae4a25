"""GPU: vcgpu_get_frame_cross_covariance (the [frame f, globals] and [frame f, frame f+1] blocks of (J^T J)^-1: vision
-X_f Σ_gg and X_f Σ_gg X_f+1^T, inertial level 0 of the selected inversion's level walk, vc_frame_cov.cuh) against the
dense inverse of the oracle's J^T J at the state the device converged to, with the frame call's correlation-scaled bars
|ΔΣ_ij| / sqrt(Σ_ii Σ_jj): 1e-6 vision, 1e-4 inertial.  Covers test_gpu_frame_covariance.py's cases (camera models,
inertial flags, fixed intrinsics, the chain's level shapes, G = 67 and 68, frames no camera sees, a camera no frame sees,
inertial frames missing cameras), the exact zeros, the handle left as it was, a singular system and null arguments."""
import numpy as np
import pytest

import chain_plan
import target_views as tv
from dense_cov import corr_errors, cross_blocks, dense_inverse, exact_zeros
from test_gpu_frame_covariance import ALL_ON, BAR, LEVEL_CASES, NUMERIC, _solved
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

INVALID = -1


def _keep(g, o, inertial, used):
    nf, fd = g.n_frames, 9 if inertial else 6
    used = np.ones(nf, bool) if used is None else used
    # a rotation-only run reads no velocity: those rows and columns are 0, as a constant block's are
    live = 6 if inertial and g.flags.rotation_only else fd
    return used, live, used[:, None] & (np.arange(fd) < live)[None, :], o.global_mask() != 0


def check(g, o, inertial, fg, fn, used=None):
    """fg, fn of rig g: the shapes, the exact zeros and the dense inverse's blocks within the bar; returns the errors and
    the dense inverse's standard deviations of the globals"""
    nf, fd, G = g.n_frames, 9 if inertial else 6, g.G
    assert fg.shape == (nf, fd, G) and fn.shape == (nf - 1, fd, fd)
    used, live, keep_f, keep_g = _keep(g, o, inertial, used)
    assert exact_zeros(fg, fn, keep_f, keep_g)
    Hi, _ = dense_inverse(o, used, live)
    ref_fg, ref_fn = cross_blocks(Hi, nf, fd)
    sd = np.sqrt(np.diag(Hi))
    sd_f, sd_g = sd[:nf * fd].reshape(nf, fd), sd[nf * fd:]
    assert np.all(sd_f[keep_f] > 0) and np.all(sd_g[keep_g] > 0)
    eg, en = corr_errors(fg, fn, ref_fg, ref_fn, sd_f, sd_g, keep_f, keep_g)
    print(f"\n{nf} frames, fd {fd}, G {G}: vs dense inverse, frame x globals {eg:.1e}, frame x next frame {en:.1e}")
    assert eg <= BAR[inertial] and en <= BAR[inertial], (eg, en)
    return eg, en, sd_g


def _check(g, o, inertial, used=None):
    fg, fn = g.frame_cross_covariance()
    return check(g, o, inertial, fg, fn, used)


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


@pytest.mark.parametrize("nf", LEVEL_CASES)
def test_level_shapes(nf):
    """interior nodes, separators, a last chunk without a right separator, and the top nodes' blocks straight from the
    dense inverse, on every level shape of test_gpu_frame_covariance.py"""
    p = synth.make_problem(models=("poly3",), n_frames=nf, grid=(8, 6), inertial=True, seed=100 + nf,
                           frame_rate=min(30.0, nf / 3.0))
    g, o = _solved(p, dict(ALL_ON))
    _check(g, o, True)


@pytest.mark.parametrize("G", [67, 68])
def test_many_globals(G):
    p = synth.make_problem(models=chain_plan.rig_with_globals(G), n_frames=90, grid=(8, 6), inertial=True, seed=G)
    g, o = _solved(p, dict(ALL_ON))
    assert g.G == G
    _check(g, o, True)


def test_vision_frames_no_camera_sees():
    """runs of frames no camera sees, at both ends and inside: their rows, and their columns of the previous frame's
    Σ_f,f+1, exactly 0"""
    v = tv.build("unseen_runs")
    g, o = _solved(v.p, v.flags)
    used = tv.counts(v.p).sum(0) > 0
    assert not used.all()
    _check(g, o, False, used=used)


def test_vision_camera_no_frame_sees():
    """a camera no active observation sees: its globals' columns of Σ_fg exactly 0"""
    v = tv.build("unseen_camera")
    g, o = _solved(v.p, v.flags)
    fg, fn = g.frame_cross_covariance()
    check(g, o, False, fg, fn)
    assert (o.global_mask() == 0).sum() > 6  # the camera's globals, beside camera 0's constant extrinsics
    assert not fg[:, :, o.global_mask() == 0].any()


def test_inertial_camera_no_frame_sees():
    v = tv.build("unseen_camera_inertial")
    g, o = _solved(v.p, v.flags)
    _check(g, o, True)


def test_inertial_frames_missing_cameras():
    """test_gpu_frame_covariance.py's rig: a chunk of frames inside the chain no camera sees and a run seen by one
    camera of two"""
    p = synth.make_problem(models=("poly3", "poly3"), n_frames=90, grid=(10, 7), inertial=True, seed=45)
    c = chain_plan.CHUNK
    gone = ((p.obs_frame >= 40) & (p.obs_frame < 40 + c)) | ((p.obs_frame >= 60) & (p.obs_frame < 76) & (p.obs_cam == 1))
    p = tv.keep(p, ~gone)
    g, o = _solved(p, dict(ALL_ON))
    _check(g, o, True)


def test_relative_motion_covariance():
    """Σ_ff + Σ_f+1,f+1 - Σ_f,f+1 - Σ_f,f+1^T from the calls against the dense inverse's: positive definite, and within
    four times the bar (one per term) relative to the two frames' own standard deviations.  (Consecutive frames are
    strongly correlated, so the relative motion's deviations are far smaller than either frame's, and the terms cancel.)"""
    p = synth.make_problem(models=("poly3", "poly2"), n_frames=90, inertial=True, seed=15)
    g, o = _solved(p, dict(ALL_ON))
    S = g.frame_covariance()
    _, fn = g.frame_cross_covariance()
    rel = S[:-1] + S[1:] - fn - fn.transpose(0, 2, 1)
    Hi, _ = dense_inverse(o, np.ones(g.n_frames, bool), 9)
    D = np.stack([Hi[f * 9:(f + 1) * 9, f * 9:(f + 1) * 9] for f in range(g.n_frames)])
    _, rfn = cross_blocks(Hi, g.n_frames, 9)
    ref = D[:-1] + D[1:] - rfn - rfn.transpose(0, 2, 1)
    sd = np.sqrt(np.einsum("fii->fi", D))
    sd = np.maximum(sd[:-1], sd[1:])
    err = (np.abs(rel - ref) / (sd[:, :, None] * sd[:, None, :])).max()
    print(f"\nrelative motion covariance vs dense inverse {err:.1e} (of the frames' deviations)")
    assert np.all(np.linalg.eigvalsh(0.5 * (rel + rel.transpose(0, 2, 1))) > 0)
    assert err <= 4 * BAR[True], err


def _snapshot(g):
    st = g.state()
    W = g.imu_weights() if g.flags.inertial else np.zeros(0)
    return {k: np.asarray(v).tobytes() for k, v in st.items()}, W.tobytes()


@pytest.mark.parametrize("inertial", [False, True], ids=["vision", "inertial"])
def test_no_side_effects(inertial):
    """the state and IMU weights are left bit for bit, and frame_covariance() and covariance() then return the bits an
    untouched handle returns"""
    from vicalib_b200.capi import Calibrator

    def make():
        p = synth.make_problem(models=("poly3", "kb4"), n_frames=60 if inertial else 20, inertial=inertial, seed=7)
        g = Calibrator()
        g.load(p)
        g.set_flags(**(ALL_ON if inertial else {}))
        g.set_options(max_iters=4)
        g.solve()
        return g

    g, fresh = make(), make()
    assert _snapshot(g) == _snapshot(fresh)
    g.frame_cross_covariance()
    assert _snapshot(g) == _snapshot(fresh)
    assert g.frame_covariance().tobytes() == fresh.frame_covariance().tobytes()
    assert g.covariance().tobytes() == fresh.covariance().tobytes()
    assert _snapshot(g) == _snapshot(fresh)


def test_singular_system_is_refused():
    """every reprojection residual weighted 0: J^T J is singular; nothing is written"""
    from vicalib_b200.capi import Calibrator, _p

    p = synth.make_problem(models=("poly3", "poly3"), n_frames=18, seed=90)
    g = Calibrator()
    g.load(p)
    g.set_flags(visual_mult=0.0)
    fg, fn = np.full((18, 6, g.G), np.nan), np.full((17, 6, 6), np.nan)
    assert g.L.vcgpu_get_frame_cross_covariance(g.h, _p(fg), _p(fn)) == NUMERIC
    assert np.isnan(fg).all() and np.isnan(fn).all()


def test_null_arguments():
    """both outputs null, or a null handle: refused; one output null: the other is written, the same bits"""
    from vicalib_b200.capi import Calibrator, _p

    g = Calibrator()
    g.load(synth.make_problem(models=("poly3",), n_frames=18, seed=91))
    assert g.L.vcgpu_get_frame_cross_covariance(g.h, None, None) == INVALID
    assert "both null" in g.L.vcgpu_last_error(g.h).decode()
    fg, fn = np.zeros((18, 6, g.G)), np.zeros((17, 6, 6))
    assert g.L.vcgpu_get_frame_cross_covariance(None, _p(fg), _p(fn)) == INVALID
    both = g.frame_cross_covariance()
    assert g.L.vcgpu_get_frame_cross_covariance(g.h, _p(fg), None) == 0
    assert g.L.vcgpu_get_frame_cross_covariance(g.h, None, _p(fn)) == 0
    assert fg.tobytes() == both[0].tobytes() and fn.tobytes() == both[1].tobytes()
