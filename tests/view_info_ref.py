"""Reference of vcgpu_get_view_information (include/vcgpu.h) in numpy, with the candidate's Jacobians from the oracle.

visibility() applies the header's rule to every (camera, corner) of a candidate on its own: the domain limits come from
projection_ref.limit (numpy's polynomial roots, not the device's bisection), the pixel from synth.project.  blocks()
places the seen corners of the used cameras as one frame's observations at their predicted pixels and takes the
oracle's eval_reproj Jacobians; B, E and C are formed densely, weighted by visual_mult and masked by the global mask.
information() forms S = C - E^T B^-1 E and the gain, variances and posterior on F (the rows of Sigma whose diagonal is
not 0.0) in float64.
"""
import types

import numpy as np

import projection_ref as P
from oracle.binding import Oracle
from vicalib_b200 import synth


def camera_offsets(models):
    off = np.cumsum([0] + [6 + synth.NUM_INTR[int(m)] for m in models])
    return off[:-1], off[1:]


def visibility(models, intr, q_ck, p_ck, T, p_w, width, height, facing=None):
    """(seen [n_cams, n_pts] bool, pixels [n_cams, n_pts, 2]) of the candidate pose T (q | t)"""
    T = np.asarray(T, float)
    p_w = np.asarray(p_w, float).reshape(-1, 3)
    Rwp = synth.quat_to_mat(T[:4])
    pk = (p_w - T[4:]) @ Rwp  # R_wp^T (p_w - t)
    nc = len(models)
    seen = np.zeros((nc, len(p_w)), bool)
    pix = np.zeros((nc, len(p_w), 2))
    width = np.broadcast_to(np.asarray(width), (nc,))
    height = np.broadcast_to(np.asarray(height), (nc,))
    for c in range(nc):
        m, ins = int(models[c]), np.asarray(intr[c], float)
        Rck = synth.quat_to_mat(np.asarray(q_ck[c], float))
        pc = pk @ Rck.T + np.asarray(p_ck[c], float)
        with np.errstate(all="ignore"):
            z = synth.project(m, pc, ins)
            lim = P.limit(m, ins)
            if m == synth.KB4:
                ok = np.arctan2(np.hypot(pc[:, 0], pc[:, 1]), pc[:, 2]) < lim
            else:
                ok = pc[:, 2] > 0
                if m in (synth.POLY2, synth.POLY3):
                    ok &= (pc[:, 0] / pc[:, 2]) ** 2 + (pc[:, 1] / pc[:, 2]) ** 2 < lim * lim
                elif m == synth.FOV and ins[4] ** 2 > 1e-5:
                    w = ins[4]
                    rd = np.hypot((z[:, 0] - ins[2]) / ins[0], (z[:, 1] - ins[3]) / ins[1])
                    rs = rd / (2 * np.tan(w / 2) / w)
                    ok &= (rs * rs < 1e-5) | (rd * abs(w) < np.pi / 2)
            ok &= (z[:, 0] >= 0) & (z[:, 0] < width[c]) & (z[:, 1] >= 0) & (z[:, 1] < height[c])
            if facing is not None:
                ck = -Rck.T @ np.asarray(p_ck[c], float)
                cw = Rwp @ ck + T[4:]
                ok &= (cw[None, :] - p_w) @ np.asarray(facing, float) > 0
        seen[c] = ok
        pix[c] = z
    return seen, pix


def _problem(models, intr, q_ck, p_ck, T, pw, cam, pix):
    n = len(pw)
    e = np.zeros((0, 3))
    nc = len(models)
    return types.SimpleNamespace(
        models=np.asarray(models, np.int32), intr=np.asarray(intr, float).reshape(nc, 10), q_ck=np.asarray(q_ck, float).reshape(nc, 4),
        p_ck=np.asarray(p_ck, float).reshape(nc, 3), T_wp=np.asarray(T, float).reshape(1, 7), v_w=np.zeros((1, 3)),
        ftime=np.zeros(1), obs_frame=np.zeros(n, np.int32), obs_cam=np.asarray(cam, np.int32), p_w=np.asarray(pw, float).reshape(-1, 3),
        p_c=np.asarray(pix, float).reshape(-1, 2), imu_t=np.zeros(0), imu_w=e, imu_a=e, g=np.zeros(2), b=np.zeros(6), sf=np.ones(6),
        ts=0.0, n_cams=nc, n_frames=1, n_obs=n)


def blocks(models, intr, q_ck, p_ck, T, p_w, seen, pix, used, mask, G, visual_mult=1.0):
    """(B [6, 6], E [6, G], C [G, G], n_contributing) of the seen corners of the used cameras"""
    cams = [c for c in range(len(models)) if used[c]]
    sel = [(c, j) for c in cams for j in np.flatnonzero(seen[c])]
    B, E, Cm = np.zeros((6, 6)), np.zeros((6, G)), np.zeros((G, G))
    if not sel:
        return B, E, Cm, 0
    cam = np.array([c for c, _ in sel])
    pw = np.array([p_w[j] for _, j in sel])
    px = np.array([pix[c, j] for c, j in sel])
    o = Oracle(_problem(models, intr, q_ck, p_ck, T, pw, cam, px))
    _, J = o.eval_reproj()
    lo, _ = camera_offsets(models)
    Jg = np.zeros((len(sel), 2, G))
    for k, c in enumerate(cam):
        K = synth.NUM_INTR[int(models[c])]
        Jg[k, :, lo[c]:lo[c] + 6 + K] = J[k, :, 6:12 + K]
    Jg *= np.asarray(mask, float)[None, None, :]
    Jp = J[:, :, :6].reshape(-1, 6)
    Jg = Jg.reshape(-1, G)
    return visual_mult * Jp.T @ Jp, visual_mult * Jp.T @ Jg, visual_mult * Jg.T @ Jg, len(sel)


def schur(B, E, Cm):
    return Cm - E.T @ np.linalg.solve(B, E)


def posterior(Sigma, S):
    """(gain, post [G, G]) of the prior Sigma and the added information S on F"""
    F = np.diag(Sigma) != 0.0
    SF = Sigma[np.ix_(F, F)]
    d = np.sqrt(np.diag(SF))
    L = np.linalg.cholesky(SF / d[:, None] / d[None, :])
    W = L.T @ (d[:, None] * S[np.ix_(F, F)] * d[None, :]) @ L
    M = np.eye(len(d)) + W
    gain = 0.5 * np.linalg.slogdet(M)[1]
    postF = d[:, None] * (L @ np.linalg.solve(M, L.T)) * d[None, :]
    post = np.zeros_like(Sigma)
    post[np.ix_(F, F)] = 0.5 * (postF + postF.T)
    return gain, post


def information(Sigma, models, intr, q_ck, p_ck, used, mask, T_wp, p_w, width, height, facing=None, visual_mult=1.0):
    """per candidate: dict(n_seen [n, n_cams], gain [n], var [n, G], post [n, G, G]), the header's exact cases included"""
    Sigma = np.asarray(Sigma, float)
    G = len(Sigma)
    T_wp = np.asarray(T_wp, float).reshape(-1, 7)
    out = dict(n_seen=np.zeros((len(T_wp), len(models)), np.int32), gain=np.zeros(len(T_wp)), var=np.zeros((len(T_wp), G)),
               post=np.zeros((len(T_wp), G, G)))
    for i, T in enumerate(T_wp):
        seen, pix = visibility(models, intr, q_ck, p_ck, T, p_w, width, height, facing)
        out["n_seen"][i] = seen.sum(1)
        B, E, Cm, n = blocks(models, intr, q_ck, p_ck, T, p_w, seen, pix, used, mask, G, visual_mult)
        if n == 0:
            gain, post = 0.0, Sigma.copy()
        elif n < 4:
            gain, post = np.nan, np.full((G, G), np.nan)
        else:
            gain, post = posterior(Sigma, schur(B, E, Cm))
        out["gain"][i], out["post"][i], out["var"][i] = gain, post, np.diag(post)
    return out


def look_at(cam_pos, target, up=(0.0, -1.0, 0.0)):
    """the rig pose (q | t) whose camera 0 (q_ck = identity, p_ck = 0) sits at cam_pos looking at target"""
    z = np.asarray(target, float) - np.asarray(cam_pos, float)
    z /= np.linalg.norm(z)
    x = np.cross(up, z)
    if np.linalg.norm(x) < 1e-9:
        x = np.cross((1.0, 0.0, 0.0), z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z], 1)  # camera axes in the world
    return np.r_[synth.mat_to_quat(R), cam_pos]


def rig_pose(cam_pose, q_ck, p_ck):
    """the rig pose T_wp that puts camera 0 (q_ck, p_ck) at the camera pose cam_pose (q | t, camera to world)"""
    Rwc = synth.quat_to_mat(np.asarray(cam_pose[:4], float))
    Rck = synth.quat_to_mat(np.asarray(q_ck, float))
    Rwp = Rwc @ Rck  # p_c = R_ck p_k + p_ck: R_wp = R_wc R_ck, t = c_w - R_wp (-R_ck^T p_ck)
    t = np.asarray(cam_pose[4:], float) + Rwp @ (Rck.T @ np.asarray(p_ck, float))
    return np.r_[synth.mat_to_quat(Rwp), t]
