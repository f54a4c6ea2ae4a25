"""CPU: the reference of vcgpu_get_view_information (tests/view_info_ref.py) against the dense normal equations.
  schur       appending the candidate as a frame at its predicted pixels and inverting the oracle's J^T J gives the
              posterior (Sigma^-1 + S)^-1 and the gain: five models, 1, 2 and 4 cameras
  visibility  KB4 corners beyond 90 degrees, poly folds, FOV's domain, corners behind the camera, the facing test and
              the image edges
  properties  gain >= 0, more corners never lower it, chaining two views through post equals appending both
  behaviour   after fronto-parallel views, a tilted view lowers var(fu) more than a fronto-parallel one (Zhang)"""
import dataclasses

import numpy as np
import pytest

import dense_cov
import projection_ref as P
import view_info_ref as V
import wide_lenses as W
from oracle.binding import Oracle
from vicalib_b200 import synth


def _target(p):
    return np.unique(p.p_w, axis=0)


def _facing(p):
    """the grid's normal pointing at the cameras"""
    return np.array([0.0, 0.0, np.sign(np.mean(p.T_wp[:, 6]))])


def _sigma(o, p):
    Hi, keep = dense_cov.dense_inverse(o, np.ones(p.n_frames, bool), o.fd)
    nfp = p.n_frames * o.fd
    return Hi[nfp:, nfp:]


def _used(p):
    return np.array([(p.obs_cam == c).any() for c in range(p.n_cams)])


def _append(p, T, p_w, seen, pix, used):
    """p with the candidate as one more frame observing its seen corners (of used cameras) at their predicted pixels"""
    cams = [c for c in range(p.n_cams) if used[c]]
    sel = [(c, j) for c in cams for j in np.flatnonzero(seen[c])]
    return dataclasses.replace(
        p, T_wp=np.vstack([p.T_wp, T]), v_w=np.vstack([p.v_w, np.zeros(3)]), ftime=np.r_[p.ftime, p.ftime[-1] + 1.0],
        obs_frame=np.r_[p.obs_frame, np.full(len(sel), p.n_frames)].astype(np.int32),
        obs_cam=np.r_[p.obs_cam, [c for c, _ in sel]].astype(np.int32), p_w=np.vstack([p.p_w, [p_w[j] for _, j in sel]]),
        p_c=np.vstack([p.p_c, [pix[c, j] for c, j in sel]]))


def _candidate(p, k, dw=0.05, dt=0.02, seed=0):
    """frame k's pose, turned by dw and moved by dt"""
    rng = np.random.default_rng(seed)
    T = p.T_wp[k].copy()
    R = synth.quat_to_mat(T[:4]) @ P._so3_exp(rng.normal(0, dw, 3))
    return np.r_[synth.mat_to_quat(R), T[4:] + rng.normal(0, dt, 3)]


def _info(p, o, Sigma, T, **kw):
    st = o.state()
    return V.information(Sigma, p.models, st["intr"], st["q_ck"], st["p_ck"], _used(p), o.global_mask(), T, _target(p),
                         kw.pop("width", 640), kw.pop("height", 480), **kw)


SCHUR = [("linear",), ("fov",), ("poly2",), ("poly3",), ("kb4",), ("poly3", "kb4"), ("linear", "fov", "poly2", "kb4")]


@pytest.mark.parametrize("models", SCHUR, ids=["_".join(m) for m in SCHUR])
def test_schur_identity(models):
    p = synth.make_problem(models=models, n_frames=8, grid=(8, 6), seed=31)
    o = Oracle(p)
    Sigma = _sigma(o, p)
    st = o.state()
    T = _candidate(p, 3)
    r = _info(p, o, Sigma, T[None, :])
    assert r["n_seen"][0].sum() >= 4
    seen, pix = V.visibility(p.models, st["intr"], st["q_ck"], st["p_ck"], T, _target(p), 640, 480)
    q = _append(p, T, _target(p), seen, pix, _used(p))
    oq = Oracle(q)
    Sq = _sigma(oq, q)
    F = np.diag(Sigma) != 0
    scale = np.sqrt(np.outer(np.diag(Sigma), np.diag(Sigma)))
    err = np.abs(r["post"][0] - Sq)[np.ix_(F, F)] / scale[np.ix_(F, F)]
    assert err.max() < 1e-8, err.max()
    ld = np.linalg.slogdet(Sigma[np.ix_(F, F)])[1] - np.linalg.slogdet(Sq[np.ix_(F, F)])[1]
    assert abs(0.5 * ld - r["gain"][0]) < 1e-8 * max(1.0, abs(ld)), (ld, r["gain"][0])
    assert r["gain"][0] > 0


def test_visibility_wide_lenses():
    # KB4 beyond 90 degrees: the fisheye sees corners behind its image plane, up to theta_max
    lens = W.build("kb4_fisheye")
    p = lens.p
    st = dict(intr=p.intr, q_ck=p.q_ck, p_ck=p.p_ck)
    pw = _target(p)
    n90 = 0
    for k in range(p.n_frames):
        seen, pix = V.visibility(p.models, st["intr"], st["q_ck"], st["p_ck"], p.T_wp[k], pw, 1e6, 1e6)
        Rwp = synth.quat_to_mat(p.T_wp[k, :4])
        pc = (pw - p.T_wp[k, 4:]) @ Rwp @ synth.quat_to_mat(p.q_ck[0]).T + p.p_ck[0]
        th = np.arctan2(np.hypot(pc[:, 0], pc[:, 1]), pc[:, 2])
        inside = (pix[0] >= 0).all(1) & (pix[0] < 1e6).all(1)
        assert np.array_equal(seen[0], (th < P.limit(synth.KB4, p.intr[0])) & inside)
        n90 += int((seen[0] & (pc[:, 2] < 0)).sum())
    assert n90 > 0
    # poly: nothing at or past the fold, nothing behind the camera
    for name in ("poly2_barrel", "poly3_barrel"):
        p = W.build(name).p
        lim = P.limit(int(p.models[0]), p.intr[0])
        for k in range(0, p.n_frames, 3):
            T = _candidate(p, k, dw=0.6, seed=k)
            seen, _ = V.visibility(p.models, p.intr, p.q_ck, p.p_ck, T, _target(p), 1e6, 1e6)
            pc = (_target(p) - T[4:]) @ synth.quat_to_mat(T[:4]) @ synth.quat_to_mat(p.q_ck[0]).T + p.p_ck[0]
            with np.errstate(all="ignore"):
                r = np.hypot(pc[:, 0], pc[:, 1]) / pc[:, 2]
            assert not (seen[0] & ((pc[:, 2] <= 0) | ~(r < lim))).any()
    # FOV near its domain edge: every seen corner's distorted radius keeps r_d |w| < pi / 2
    p = W.build("fov_w12").p
    w = p.intr[0, 4]
    for k in range(0, p.n_frames, 3):
        seen, pix = V.visibility(p.models, p.intr, p.q_ck, p.p_ck, p.T_wp[k], _target(p), 1e6, 1e6)
        rd = np.hypot((pix[0, :, 0] - p.intr[0, 2]) / p.intr[0, 0], (pix[0, :, 1] - p.intr[0, 3]) / p.intr[0, 1])
        assert (rd[seen[0]] * w < np.pi / 2).all()


def test_facing_and_image_edges():
    p = synth.make_problem(models=("linear",), n_frames=4, grid=(8, 6), seed=3)
    pw = _target(p)
    T = p.T_wp[1]
    n = _facing(p)
    a, pix = V.visibility(p.models, p.intr, p.q_ck, p.p_ck, T, pw, 640, 480, n)
    b, _ = V.visibility(p.models, p.intr, p.q_ck, p.p_ck, T, pw, 640, 480, -n)
    c, _ = V.visibility(p.models, p.intr, p.q_ck, p.p_ck, T, pw, 640, 480)
    assert a.sum() > 0 and b.sum() == 0 and np.array_equal(a, c)
    # the image is [0, width) x [0, height): a corner exactly on the right edge is out, one exactly on 0 is in
    u = pix[0, a[0], 0]
    j = np.flatnonzero(a[0])[np.argmax(u)]
    w_edge = pix[0, j, 0]
    on, _ = V.visibility(p.models, p.intr, p.q_ck, p.p_ck, T, pw, w_edge, 480)
    assert not on[0, j]
    intr = p.intr.copy()
    intr[0, 2] -= pix[0, j, 0]  # move u0 so that corner j lands on u = 0 exactly
    on, pix0 = V.visibility(p.models, intr, p.q_ck, p.p_ck, T, pw, 640, 480)
    if pix0[0, j, 0] == 0.0:
        assert on[0, j]


def test_properties_and_chaining():
    p = synth.make_problem(models=("poly3", "kb4"), n_frames=8, grid=(8, 6), seed=32)
    o = Oracle(p)
    Sigma = _sigma(o, p)
    st = o.state()
    pw = _target(p)
    Ts = np.stack([_candidate(p, k, seed=k) for k in range(p.n_frames)])
    r = _info(p, o, Sigma, Ts)
    assert (r["gain"] >= 0).all()
    # more corners never lower the gain
    args = (Sigma, p.models, st["intr"], st["q_ck"], st["p_ck"], _used(p), o.global_mask())
    g_half = V.information(*args, Ts[:2], pw[: len(pw) // 2], 640, 480)["gain"]
    assert (g_half <= r["gain"][:2] + 1e-12).all()
    # chaining: post of view 0 as the prior of view 1 equals appending both frames
    r0 = V.information(*args, Ts[:1], pw, 640, 480)
    r1 = V.information(r0["post"][0], *args[1:], Ts[1:2], pw, 640, 480)
    q = p
    for T in Ts[:2]:
        seen, pix = V.visibility(p.models, st["intr"], st["q_ck"], st["p_ck"], T, pw, 640, 480)
        q = _append(q, T, pw, seen, pix, _used(p))
    Sq = _sigma(Oracle(q), q)
    F = np.diag(Sigma) != 0
    scale = np.sqrt(np.outer(np.diag(Sigma), np.diag(Sigma)))
    assert (np.abs(r1["post"][0] - Sq)[np.ix_(F, F)] / scale[np.ix_(F, F)]).max() < 1e-8
    assert abs(r0["gain"][0] + r1["gain"][0] - 0.5 * (np.linalg.slogdet(Sigma[np.ix_(F, F)])[1] - np.linalg.slogdet(Sq[np.ix_(F, F)])[1])) < 1e-7


def test_tilted_view_constrains_focal_length():
    """Zhang: views of a plane fronto-parallel to the camera leave the focal length coupled to the distance; a view
    turned about an axis in the plane separates them.  On a rig seen only fronto-parallel, a ~45 degree view lowers
    var(fu) more than another fronto-parallel view at the same distance."""
    p = synth.make_problem(models=("linear",), n_frames=10, grid=(10, 8), seed=33, tilt=(0.0, 0.0))
    pw = _target(p)
    centre = pw.mean(0)
    side = np.sign(np.mean(p.T_wp[:, 6]))
    # replace the frames by near fronto-parallel views at 0.45 m (exactly fronto-parallel views leave J^T J singular),
    # shifted sideways and looking at the grid's centre (a turn of at most 6 degrees), observed without noise
    Ts = [V.rig_pose(V.look_at(centre + np.array([dx, dy, side * 0.45]), centre), p.q_ck[0], p.p_ck[0])
          for dx, dy in [(-0.04, -0.03), (0.04, -0.03), (-0.04, 0.03), (0.04, 0.03), (0.0, 0.0), (0.02, -0.01)]]
    obs = [V.visibility(p.models, p.intr, p.q_ck, p.p_ck, T, pw, 640, 480) for T in Ts]
    sel = [(f, j) for f, (s, _) in enumerate(obs) for j in np.flatnonzero(s[0])]
    q = dataclasses.replace(p, T_wp=np.stack(Ts), v_w=np.zeros((len(Ts), 3)), ftime=np.arange(len(Ts), dtype=float),
                            obs_frame=np.array([f for f, _ in sel], np.int32), obs_cam=np.zeros(len(sel), np.int32),
                            p_w=pw[[j for _, j in sel]], p_c=np.array([obs[f][1][0, j] for f, j in sel]))
    o = Oracle(q)
    Sigma = _sigma(o, q)
    fronto = V.rig_pose(V.look_at(centre + np.array([0.01, 0.02, side * 0.45]), centre), p.q_ck[0], p.p_ck[0])
    tilt = V.rig_pose(V.look_at(centre + np.array([side * 0.32, 0.0, side * 0.32]), centre), p.q_ck[0], p.p_ck[0])
    r = V.information(Sigma, q.models, q.intr, q.q_ck, q.p_ck, np.array([True]), o.global_mask(), np.stack([fronto, tilt]), pw, 640, 480)
    assert (r["n_seen"] > 20).all(), r["n_seen"]
    fu = 6  # camera 0's first intrinsic
    assert r["var"][1, fu] < r["var"][0, fu] < Sigma[fu, fu], (r["var"][:, fu], Sigma[fu, fu])
    assert r["gain"][1] > r["gain"][0]
