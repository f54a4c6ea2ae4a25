"""Target views of the kinds real recordings produce, cut from synthetic problems, with per-(camera, frame) corner counts
that each builder checks against the edge it claims.

synth.make_problem has every camera see the whole grid in every frame.  Recordings do not: the target leaves the image
partway, a camera sees a corner of it, some frames see it from one camera only, the target is out of view for a while,
and one camera of a rig may never track it.  The reprojection builds work on corner slabs (build_frame_warp: 32-corner
slabs with a prefetch of the next, padded to the MMA depth; fused_build_kernel: 144-corner passes), so the count of a
(camera, frame) group decides which code runs.  Each builder starts from make_problem and keeps a subset of its
observations (so the data stays consistent with the trajectory), then asserts that its edge is really present: a later
change to synth cannot quietly remove the edge from a test.

Views of 1-3 corners leave a frame pose underdetermined: builders put them only in frames another camera constrains.
"""
import dataclasses

import numpy as np

import chain_plan
import constant_blocks as cb
from vicalib_b200 import synth

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
# the group counts at the edges of the build kernels' slabs (32) and passes (144), and a view of more than two passes
BOUNDARY_COUNTS = (1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65, 143, 144, 145, 287, 288, 289, 600)


@dataclasses.dataclass
class View:
    name: str
    p: synth.Problem
    flags: dict
    unseen_cam: int = -1  # a camera no observation sees (-1: none)

    @property
    def inertial(self):
        return bool(self.flags.get("inertial", 0))


def counts(p):
    """[n_cams, n_frames] corners per (camera, frame) group"""
    n = np.zeros((p.n_cams, p.n_frames), dtype=np.int64)
    np.add.at(n, (np.asarray(p.obs_cam), np.asarray(p.obs_frame)), 1)
    return n


def keep(p, sel):
    """p with the observations sel selects (a boolean mask or indices), in their order"""
    sel = np.asarray(sel)
    return dataclasses.replace(p, obs_frame=p.obs_frame[sel].copy(), obs_cam=p.obs_cam[sel].copy(),
                               p_w=p.p_w[sel].copy(), p_c=p.p_c[sel].copy(), grid_idx=p.grid_idx[sel].copy())


def true_pixels(p):
    """the noise-free projection of every observation at the truth"""
    out = np.zeros((p.n_obs, 2))
    T, tr = p.truth["T_wp"], p.truth
    for c in range(p.n_cams):
        s = p.obs_cam == c
        f = p.obs_frame[s]
        Rwk = synth.quat_to_mat(T[f, :4])
        pk = np.einsum("nji,nj->ni", Rwk, p.p_w[s] - T[f, 4:])
        pc = pk @ synth.quat_to_mat(tr["q_ck"][c]).T + tr["p_ck"][c]
        out[s] = synth.project(int(p.models[c]), pc, tr["intr"][c])
    return out


def _constrained(n, min_corners=20):
    """every frame some camera sees has a camera with at least min_corners corners"""
    seen = n.sum(0) > 0
    return bool(np.all(n.max(0)[seen] >= min_corners))


def cropped(models=("poly3", "fov", "kb4"), n_frames=24, grid=(14, 10), seed=41, inertial=False):
    """A crop window moves across each camera's image: it keeps the corners whose true projection lies on the near side
    of a line that sweeps across the target's image from its first corner to its last, so view sizes grow from one
    corner (a corner of the target) to the full grid.  Each camera's sweep starts at another frame, so the cameras
    of a frame see very different parts of the target."""
    p = synth.make_problem(models=models, n_frames=n_frames, grid=grid, seed=seed, inertial=inertial)
    uv = true_pixels(p)
    sel = np.zeros(p.n_obs, dtype=bool)
    nc = p.n_cams
    for c in range(nc):
        for f in range(n_frames):
            s = np.flatnonzero((p.obs_cam == c) & (p.obs_frame == f))
            d = uv[s] @ np.array([1.0, 1.3])  # distance along the sweep direction
            t = ((f + c * n_frames // nc) % n_frames) / (n_frames - 1)  # 0 .. 1 along the sweep
            sel[s] = d <= d.min() + t * (d.max() - d.min())
    p = keep(p, sel)
    n = counts(p)
    assert n.min() == 1                                     # a single corner
    assert n.max() == grid[0] * grid[1]                     # the whole grid
    assert len(np.unique(n)) >= n_frames                    # sizes change smoothly, not in a few steps
    assert np.all(n.max(0) > 2 * n.min(0))                  # cameras of a frame see very different parts
    assert _constrained(n)
    return View("cropped", p, dict(ALL_ON) if inertial else {})


def boundary_counts(models=("poly3", "kb4"), grid=(30, 20), seed=42, inertial=False):
    """A 30 x 20 grid (600 corners).  Camera 0 sees BOUNDARY_COUNTS[f] corners of frame f, camera 1
    BOUNDARY_COUNTS[f + 9]: every slab and pass boundary of both build kernels, one view of more than two passes, and
    the two cameras of a frame always at different counts (a frame with a 1-3 corner view has >= 63 in the other)."""
    nf = len(BOUNDARY_COUNTS)
    p = synth.make_problem(models=models, n_frames=nf, grid=grid, seed=seed, inertial=inertial)
    rng = np.random.default_rng(seed)
    sel = np.zeros(p.n_obs, dtype=bool)
    for c in range(p.n_cams):
        for f in range(nf):
            s = np.flatnonzero((p.obs_cam == c) & (p.obs_frame == f))
            k = BOUNDARY_COUNTS[(f + 9 * c) % nf]
            sel[np.sort(rng.permutation(s)[:k])] = True
    p = keep(p, sel)
    n = counts(p)
    for c in range(p.n_cams):
        assert set(n[c].tolist()) == set(BOUNDARY_COUNTS), c
    assert np.all(n[0] != n[1])
    assert _constrained(n, 63)
    return View("counts", p, dict(ALL_ON) if inertial else {})


def one_camera(n_cams, n_frames=24, grid=(14, 10), seed=43, inertial=False):
    """Every other frame is seen by one camera only, each camera in turn: the frame's E columns of the others are 0."""
    models = ("poly3", "fov", "kb4", "poly2")[:n_cams]
    p = synth.make_problem(models=models, n_frames=n_frames, grid=grid, seed=seed + n_cams, inertial=inertial)
    only = np.where(np.arange(n_frames) % 2 == 1, (np.arange(n_frames) // 2) % n_cams, -1)
    p = keep(p, (only[p.obs_frame] < 0) | (only[p.obs_frame] == p.obs_cam))
    n = counts(p)
    single = (n > 0).sum(0) == 1
    assert np.array_equal(single, only >= 0)
    assert set(np.argmax(n[:, single], axis=0).tolist()) == set(range(n_cams))  # each camera in turn
    assert np.all((n > 0).sum(0)[~single] == n_cams)
    return View(f"one_camera{n_cams}", p, dict(ALL_ON) if inertial else {})


VISION_UNSEEN = ((0, 3), (11, 15), (27, 30))  # [start, end) runs no camera sees, the first and last frames among them


def unseen_runs_vision(n_frames=30, grid=(14, 10), seed=44):
    """Runs of frames no camera sees, at both ends and inside: those frames are in no residual (unused)."""
    p = synth.make_problem(models=("poly3", "fov"), n_frames=n_frames, grid=grid, seed=seed)
    gone = np.zeros(n_frames, dtype=bool)
    for a, b in VISION_UNSEEN:
        gone[a:b] = True
    for f in np.flatnonzero(gone)[:2]:
        cb.unfix(p.T_wp[f, :4])  # an unused pose that renormalisation would move
    p = keep(p, ~gone[p.obs_frame])
    n = counts(p)
    assert np.array_equal(n.sum(0) == 0, gone) and gone[0] and gone[-1]
    return View("unseen_runs", p, {})


def inertial_unseen(n_frames=80):
    """[start, end) runs of the inertial case: two elimination chunks each, at both ends and inside"""
    w = 2 * chain_plan.CHUNK
    return ((0, w), (n_frames // 2 - w // 2, n_frames // 2 + w // 2), (n_frames - w, n_frames))


def unseen_runs_inertial(n_frames=80, grid=(10, 7), seed=45):
    """Runs of two elimination chunks (chain_plan.CHUNK frames each) no camera sees, at both ends and inside: the chain
    solve eliminates chunks built from IMU blocks alone."""
    p = synth.make_problem(models=("poly3", "poly3"), n_frames=n_frames, grid=grid, seed=seed, inertial=True)
    gone = np.zeros(n_frames, dtype=bool)
    for a, b in inertial_unseen(n_frames):
        gone[a:b] = True
    p = keep(p, ~gone[p.obs_frame])
    n = counts(p)
    assert np.array_equal(n.sum(0) == 0, gone)
    for a, b in inertial_unseen(n_frames):
        assert b - a >= 2 * chain_plan.CHUNK and a % chain_plan.CHUNK == 0 and not n[:, a:b].any()
    assert gone[0] and gone[-1]
    return View("unseen_runs_inertial", p, dict(ALL_ON))


def unseen_camera_rig(inertial):
    """(problem, camera, flags) of unseen_camera before the camera's observations go: camera 1 of a 3-camera vision rig
    (camera 0 fixes the gauge of a vision solve), camera 0 of a 2-camera inertial rig (its rotation is free there).
    The camera's quaternion is off unit length, so a renormalising update would move it."""
    if inertial:
        p = synth.make_problem(models=("poly3", "fov"), n_frames=90, grid=(14, 10), seed=46, inertial=True)
        c, flags = 0, dict(ALL_ON)
    else:
        p = synth.make_problem(models=("poly3", "kb4", "fov"), n_frames=24, grid=(14, 10), seed=47)
        c, flags = 1, {}
    cb.unfix(p.q_ck[c])
    assert cb.moves_on_renormalisation(p.q_ck[c])
    return p, c, flags


def unseen_camera(inertial):
    """One camera of the rig has no observation (unseen_camera_rig)."""
    p, c, flags = unseen_camera_rig(inertial)
    p = keep(p, p.obs_cam != c)
    n = counts(p)
    assert not n[c].any() and np.all(np.delete(n, c, axis=0) > 0)
    return View("unseen_camera_inertial" if inertial else "unseen_camera", p, flags, unseen_cam=c)


BUILDERS = {
    "cropped": cropped,
    "counts": boundary_counts,
    "one_camera2": lambda: one_camera(2),
    "one_camera4": lambda: one_camera(4),
    "unseen_runs": unseen_runs_vision,
    "unseen_camera": lambda: unseen_camera(False),
    "cropped_inertial": lambda: cropped(models=("poly3", "fov"), n_frames=32, inertial=True),
    "counts_inertial": lambda: boundary_counts(inertial=True),
    "one_camera2_inertial": lambda: one_camera(2, inertial=True),
    "unseen_runs_inertial": unseen_runs_inertial,
    "unseen_camera_inertial": lambda: unseen_camera(True),
}
NAMES = tuple(BUILDERS)
VISION = tuple(n for n in NAMES if not n.endswith("_inertial"))
INERTIAL = tuple(n for n in NAMES if n.endswith("_inertial"))


def build(name):
    return BUILDERS[name]()


# ------------------------------------------------------------------ long-double reference of the reprojection blocks
def cam_offsets(models):
    off, out = 0, []
    for m in models:
        out.append(off)
        off += 6 + synth.NUM_INTR[int(m)]
    return out


def reproj_blocks(p, r, J, mask, fd, G, active=None):
    """B_f, E_f, g_f, C, g_c and the cost of the reprojection residuals, summed in np.longdouble from the per-observation
    loss-free residuals r [n, 2] and tangent Jacobians J [n, 2, 22] (pose 6 | w_ck 3 | p_ck 3 | intrinsics K): the
    SoftLOne(0.5) corrector scales both by sqrt(rho') (rho'' < 0, so Ceres' alpha is 0), the global mask zeroes the
    constant columns.  Also returns the same sums over absolute values (the scale of each entry's rounding error)."""
    ld = np.longdouble
    nf = p.n_frames
    out = {k: np.zeros(s, dtype=ld) for k, s in (("B", (nf, fd, fd)), ("E", (nf, fd, G)), ("gf", (nf, fd)),
                                                 ("C", (G, G)), ("gc", (G,)))}
    ab = {k: np.zeros_like(v) for k, v in out.items()}
    offs = cam_offsets(p.models)
    r = r.astype(ld)
    J = J.astype(ld)
    s = np.sum(r * r, axis=1)
    tmp = np.sqrt(1 + s / ld(0.25))
    cost = np.sum(ld(0.25) * (tmp - 1)) if active is None else np.sum((ld(0.25) * (tmp - 1))[active > 0])
    sc = np.sqrt(1 / tmp)
    for c in range(p.n_cams):
        K = synth.NUM_INTR[int(p.models[c])]
        o, NG = offs[c], 6 + K
        idx = np.flatnonzero((p.obs_cam == c) & (np.ones(p.n_obs, bool) if active is None else active > 0))
        if len(idx) == 0:
            continue
        m = mask[o:o + NG].astype(ld)
        Jf = J[idx, :, :6] * sc[idx, None, None]                       # [n, 2, 6]
        Jc = J[idx, :, 6:6 + NG] * sc[idx, None, None] * m              # [n, 2, NG]
        rr = r[idx] * sc[idx, None]                                      # [n, 2]
        fr = p.obs_frame[idx]
        t = np.einsum("nra,nrb->nab", Jf, Jf)
        np.add.at(out["B"][:, :6, :6], fr, t)
        np.add.at(ab["B"][:, :6, :6], fr, np.abs(t))
        t = np.einsum("nra,nrb->nab", Jf, Jc)
        np.add.at(out["E"][:, :6, o:o + NG], fr, t)
        np.add.at(ab["E"][:, :6, o:o + NG], fr, np.abs(t))
        t = np.einsum("nra,nr->na", Jf, rr)
        np.add.at(out["gf"][:, :6], fr, t)
        np.add.at(ab["gf"][:, :6], fr, np.abs(t))
        t = np.einsum("nra,nrb->nab", Jc, Jc)
        out["C"][o:o + NG, o:o + NG] += t.sum(0)
        ab["C"][o:o + NG, o:o + NG] += np.abs(t).sum(0)
        t = np.einsum("nra,nr->na", Jc, rr)
        out["gc"][o:o + NG] += t.sum(0)
        ab["gc"][o:o + NG] += np.abs(t).sum(0)
    out["cost"] = cost
    return out, ab


def block_errors(ne, ref, ab, models, bar, extra=None):
    """Entry by entry, |ne - ref| <= bar * (sum over absolute values) [+ extra, a per-key allowance], reported per frame
    and per (frame, camera) block: [(block, frame or -1, camera or -1, worst ratio)] of the blocks that fail.  An entry
    whose sum over absolute values is 0 (a camera that does not see the frame, a constant column) must be exactly 0."""
    G = ne["C"].shape[0]
    offs = cam_offsets(models)
    cols = [slice(o, o + 6 + synth.NUM_INTR[int(m)]) for o, m in zip(offs, models)]
    if G > cols[-1].stop:
        cols.append(slice(cols[-1].stop, G))  # the IMU globals (camera -1 below)
    bad = []

    def check(key, idx, f, c):
        d = np.abs(ne[key][idx].astype(np.longdouble) - ref[key][idx])
        lim = bar * ab[key][idx] + (0 if extra is None else extra.get(key, 0))
        if np.any(d > lim):
            bad.append((key, f, c, float(np.max(d / np.maximum(lim, 1e-300)))))

    for f in range(ne["B"].shape[0]):
        check("B", (f,), f, -1)
        check("gf", (f,), f, -1)
        for c, s in enumerate(cols):
            check("E", (f, slice(None), s), f, c if c < len(models) else -1)
    for c, s in enumerate(cols):
        check("C", (s,), -1, c if c < len(models) else -1)
        check("gc", (s,), -1, c if c < len(models) else -1)
    return bad
