"""Target views without a GPU: every builder's edges (target_views.py), the long-double reference of the reprojection
blocks against the oracle's normal equations, per frame and per (frame, camera) block, and the oracle's rule for a
camera no active observation sees: Ceres removes its blocks (Program::RemoveFixedBlocks), so a solve leaves them as
they were, the parameter tolerance's x_norm leaves them out, and the global mask is 0 on their columns.
"""
import numpy as np
import pytest

import constant_blocks as cb
import target_views as tv
from vicalib_b200 import synth


def _oracle(v, **opts):
    from oracle.binding import Oracle

    o = Oracle(v.p, **v.flags)
    if opts:
        o.set_options(**opts)
    return o


def _cam_cols(p, c):
    o = tv.cam_offsets(p.models)[c]
    return np.arange(o, o + 6 + synth.NUM_INTR[int(p.models[c])])


@pytest.mark.parametrize("name", tv.NAMES)
def test_builder_edges(name):
    v = tv.build(name)  # each builder asserts its own edges
    p = v.p
    assert p.n_obs == len(p.obs_cam) == len(p.p_w) == len(p.p_c) == len(p.grid_idx)
    key = p.obs_cam.astype(np.int64) * p.n_frames + p.obs_frame
    assert np.all(np.diff(key) >= 0)  # still sorted by (camera, frame)
    # the kept observations are make_problem's: within a pixel of the truth's projection
    assert np.abs(p.p_c - tv.true_pixels(p)).max() < 1.0


@pytest.mark.parametrize("name", tv.NAMES)
def test_reference_matches_oracle(name):
    """The long-double sums against the oracle's float64 ones: 1e-12 of the sum over absolute values, entry by entry."""
    v = tv.build(name)
    o = _oracle(v)
    if v.inertial:
        o.set_flags(**v.flags, imu_mult=0.0)  # the reprojection blocks alone
    ne = o.normal_equations()
    r, J = o.eval_reproj()
    ref, ab = tv.reproj_blocks(v.p, r, J, o.global_mask(), o.fd, o.G)
    assert abs(ne["cost"] - float(ref["cost"])) <= 1e-12 * float(ref["cost"])
    bad = tv.block_errors(ne, ref, ab, v.p.models, 1e-12)
    assert not bad, bad[:8]
    assert not ne["U"].any()


def test_reference_sees_one_corner():
    """One corner dropped from one 33-corner view moves that view's blocks far beyond the bar"""
    v = tv.build("counts")
    p = v.p
    n = tv.counts(p)
    f = int(np.flatnonzero(n[0] == 33)[0])
    drop = int(np.flatnonzero((p.obs_cam == 0) & (p.obs_frame == f))[17])
    o = _oracle(v)
    r, J = o.eval_reproj()
    ref, ab = tv.reproj_blocks(p, r, J, o.global_mask(), o.fd, o.G)
    act = np.ones(p.n_obs, np.uint8)
    act[drop] = 0
    ref2, _ = tv.reproj_blocks(p, r, J, o.global_mask(), o.fd, o.G, active=act)
    bad = tv.block_errors({k: np.asarray(ref2[k], np.float64) for k in ("B", "E", "gf", "C", "gc")}, ref, ab, p.models,
                          1e-11)
    assert ("B", f, -1) in [b[:3] for b in bad] and ("E", f, 0) in [b[:3] for b in bad]
    assert min(b[3] for b in bad if b[1] == f) > 1e6


UNSEEN = ["unseen_camera", "unseen_camera_inertial"]


@pytest.mark.parametrize("name", UNSEEN)
def test_oracle_global_mask_drops_unseen_camera(name):
    v = tv.build(name)
    m = _oracle(v).global_mask()
    c = v.unseen_cam
    assert not m[_cam_cols(v.p, c)].any()
    for k in range(v.p.n_cams):
        if k != c:
            assert m[_cam_cols(v.p, k)][6:].all()  # the seen cameras' intrinsics stay free
    assert not cb.cams_used(v.p)[c] and cb.cams_used(v.p).sum() == v.p.n_cams - 1


@pytest.mark.parametrize("strategy", [0, 1], ids=["lm", "dogleg"])
@pytest.mark.parametrize("name", UNSEEN)
def test_oracle_keeps_unseen_camera(name, strategy):
    v = tv.build(name)
    p, c = v.p, v.unseen_cam
    before = cb.constant_parts(cb.uploaded(p), p, v.flags)
    assert f"q_ck{c}" in before and cb.moves_on_renormalisation(before[f"q_ck{c}"])
    o = _oracle(v, max_iters=10, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, strategy=strategy)
    free, whole = cb.state_norms(cb.uploaded(p), p, v.flags)
    assert abs(o.state_norm() - free) <= 1e-14 * free and whole > free
    s = o.solve()
    assert s["iterations"] == 10 and s["successful_steps"] >= 4
    st = o.state()
    after = cb.constant_parts(st, p, v.flags)
    for k, val in before.items():
        assert np.array_equal(after[k], val), k
    assert abs(o.state_norm() - cb.state_norms(st, p, v.flags)[0]) <= 1e-14 * free


def test_oracle_camera_emptied_by_outliers():
    """rmse 0 for one camera: remove_outliers takes all its corners, and the camera leaves the solve"""
    v = tv.build("one_camera2")
    o = _oracle(v)
    assert o.global_mask()[_cam_cols(v.p, 1)].all()
    n = o.remove_outliers(np.array([np.inf, 0.0]), 1.0)
    assert n == int((v.p.obs_cam == 1).sum())
    assert not o.global_mask()[_cam_cols(v.p, 1)].any()
    assert cb.cams_used(v.p, o.obs_active()).tolist() == [True, False]
