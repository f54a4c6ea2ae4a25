"""Reference of vcgpu_get_projection_covariance (include/vcgpu.h) in numpy, with the Jacobian taken from the oracle.

unproject() follows the header's rules one pixel at a time: the closed forms of linear and FOV, and Newton from r_d for
poly and KB4 inside [0, limit).  The limits (the folds) come from numpy's polynomial roots here, not from the device's
bisection.  jacobian() places an observation at the point, p_w = T_wk T_ck^-1 P_c with T_wk the identity, and takes
the camera's columns of the oracle's eval_reproj.  At infinity the point is its direction with p_ck = 0 and the p_ck
columns are zeroed.  projection_covariance() forms J Sigma_c J^T from those.
"""
import types

import numpy as np

from oracle.binding import Oracle
from vicalib_b200 import synth

NEWTON_ITERS = 50
NEWTON_TOL = 1e-14
IMAGE_TOL = 1e-15


def _first_positive_root(c, smax):
    """the smallest real root in (0, smax) of sum c[i] s^i, or smax"""
    r = np.roots(np.asarray(c, dtype=np.float64)[::-1])
    r = r[(np.abs(r.imag) <= 1e-12 * np.maximum(1.0, np.abs(r.real))) & (r.real > 0) & (r.real < smax)].real
    return float(r.min()) if len(r) else smax


def limit(model, intr):
    """poly: r_fold (inf without a fold); KB4: theta_max; other models: inf"""
    if model in (synth.POLY2, synth.POLY3):
        k = list(intr[4:synth.NUM_INTR[model]])
        s = _first_positive_root([1.0] + [(2 * i + 3) * kk for i, kk in enumerate(k)], np.inf)
        return float(np.sqrt(s))
    if model == synth.KB4:
        s = _first_positive_root([1.0] + [(2 * i + 3) * kk for i, kk in enumerate(intr[4:8])], np.pi ** 2)
        return float(min(np.pi, np.sqrt(s)))
    return np.inf


def _radius(model, intr, rd, lim):
    k = list(intr[4:synth.NUM_INTR[model]])

    def img(r):
        s = r * r
        return r * (1 + sum(kk * s ** (i + 1) for i, kk in enumerate(k))), 1 + sum((2 * i + 3) * kk * s ** (i + 1) for i, kk in enumerate(k))

    if np.isfinite(lim) and not rd < img(lim)[0]:
        return None
    r = rd
    for _ in range(NEWTON_ITERS):
        g, d = img(r)
        if not d > 0:
            return None
        if abs(g - rd) <= IMAGE_TOL * rd:
            return r
        step = (g - rd) / d
        r -= step
        if not (0 <= r < lim):
            return None
        if abs(step) <= NEWTON_TOL * r:
            return r
    return None


def unproject(model, intr, pix):
    """the unit ray whose projection is pix, or NaN outside the model's domain"""
    fu, fv, u0, v0 = intr[:4]
    xd, yd = (pix[0] - u0) / fu, (pix[1] - v0) / fv
    rd = np.hypot(xd, yd)
    nan = np.full(3, np.nan)
    p = np.array([xd, yd, 1.0])
    if model == synth.FOV:
        w = intr[4]
        if w * w > 1e-5:
            m = 2 * np.tan(w / 2)
            f = m / w
            if not (rd / f) ** 2 < 1e-5:
                if not rd * abs(w) < np.pi / 2:
                    return nan
                f = rd / (np.tan(rd * w) / m)
            p = np.array([xd / f, yd / f, 1.0])
    elif model in (synth.POLY2, synth.POLY3):
        r = _radius(model, intr, rd, limit(model, intr))
        if r is None:
            return nan
        k = intr[4:synth.NUM_INTR[model]]
        f = 1 + sum(kk * r ** (2 * i + 2) for i, kk in enumerate(k))
        p = np.array([xd / f, yd / f, 1.0])
    elif model == synth.KB4:
        th = _radius(model, intr, rd, limit(model, intr))
        if th is None:
            return nan
        if rd == 0:
            return np.array([0.0, 0.0, 1.0])
        return np.array([np.sin(th) * xd / rd, np.sin(th) * yd / rd, np.cos(th)])
    return p / np.linalg.norm(p)


def unproject_all(models, intr, cam_id, pix):
    return np.array([unproject(int(models[c]), intr[c], z) for c, z in zip(cam_id, pix)]).reshape(-1, 3)


def _problem(model, intr, q_ck, p_ck, p_w):
    n = len(p_w)
    e = np.zeros((0, 3))
    return types.SimpleNamespace(
        models=np.array([model], np.int32), intr=np.asarray(intr, float).reshape(1, 10), q_ck=np.asarray(q_ck, float).reshape(1, 4),
        p_ck=np.asarray(p_ck, float).reshape(1, 3), T_wp=np.array([[0, 0, 0, 1, 0, 0, 0.0]]), v_w=np.zeros((1, 3)),
        ftime=np.zeros(1), obs_frame=np.zeros(n, np.int32), obs_cam=np.zeros(n, np.int32), p_w=np.asarray(p_w, float),
        p_c=np.zeros((n, 2)), imu_t=np.zeros(0), imu_w=e, imu_a=e, g=np.zeros(2), b=np.zeros(6), sf=np.ones(6), ts=0.0,
        n_cams=1, n_frames=1, n_obs=n)


def jacobian(model, intr, q_ck, p_ck, rays, depth, rig):
    """[n, 2, 6 + K]: the oracle's eval_reproj columns (w_ck | p_ck | intrinsics) of one camera at the points d * ray
    (d == 0: at infinity); camera frame: the intrinsics' columns only"""
    K = synth.NUM_INTR[model]
    rays = np.asarray(rays, float).reshape(-1, 3)
    d = np.zeros(len(rays)) if depth is None else np.broadcast_to(np.asarray(depth, float), (len(rays),))
    inf = ~(d > 0)
    pc = np.where(inf[:, None], rays, rays * d[:, None])
    pck = np.where(inf[:, None], 0.0, np.asarray(p_ck, float)[None, :])
    R = synth.quat_to_mat(np.asarray(q_ck, float))
    pk = (pc - pck) @ R  # R^T (P_c - p_ck)
    J = np.zeros((len(rays), 2, 6 + K))
    for fin in (False, True):  # one oracle problem for the points at infinity (p_ck = 0), one for the others
        s = inf != fin
        if not s.any():
            continue
        o = Oracle(_problem(model, intr, q_ck, p_ck if fin else np.zeros(3), pk[s]))
        _, Jo = o.eval_reproj()
        J[s] = Jo[:, :, 6:12 + K]
    J[inf, :, 3:6] = 0.0
    if not rig:
        J[:, :, :6] = 0.0
    return J


def jacobian_fd(model, intr, q_ck, p_ck, ray, depth, rig, h=1e-6):
    """central differences of the projection of the fixed point, through oracle.binding.project, in the tangent
    (w_ck | p_ck | intrinsics): q_ck moves as q_ck * exp(dw), p_ck and the intrinsics additively"""
    from oracle.binding import project

    K = synth.NUM_INTR[model]
    R = synth.quat_to_mat(np.asarray(q_ck, float))
    inf = not depth > 0
    pc = np.asarray(ray, float) * (1.0 if inf else depth)
    pk = R.T @ (pc - (0.0 if inf else np.asarray(p_ck, float)))

    def proj(x):
        dw, dp, di = x[:3], x[3:6], x[6:]
        Rx = R @ _so3_exp(dw) if rig else R
        p = Rx @ pk + ((0.0 if inf else np.asarray(p_ck, float)) + (dp if rig else 0.0))
        return synth.project(model, p[None, :], np.asarray(intr, float) + np.r_[di, np.zeros(10 - K)])[0]

    J = np.zeros((2, 6 + K))
    for j in range(6 + K):
        if not rig and j < 6:
            continue
        e = np.zeros(6 + K)
        step = h * max(1.0, abs(intr[j - 6])) if j >= 6 else h
        e[j] = step
        J[:, j] = (proj(e) - proj(-e)) / (2 * step)
    if inf:
        J[:, 3:6] = 0.0
    return J


def _so3_exp(w):
    th = np.linalg.norm(w)
    W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    if th < 1e-12:
        return np.eye(3) + W
    return np.eye(3) + np.sin(th) / th * W + (1 - np.cos(th)) / th ** 2 * W @ W


def camera_block(S, models, c):
    """camera c's (6 + K)^2 block of the G x G matrix"""
    off = sum(6 + synth.NUM_INTR[int(m)] for m in models[:c])
    N = 6 + synth.NUM_INTR[int(models[c])]
    return S[off:off + N, off:off + N]


def projection_covariance(S, models, intr, q_ck, p_ck, cam_id, pix, depth=None, rig=False):
    """(cov [n, 3], rays [n, 3]) of every point from the G x G matrix S and the cameras' state"""
    cam_id = np.asarray(cam_id)
    pix = np.asarray(pix, float).reshape(-1, 2)
    rays = unproject_all(models, intr, cam_id, pix)
    d = np.zeros(len(cam_id)) if depth is None else np.broadcast_to(np.asarray(depth, float), (len(cam_id),))
    cov = np.full((len(cam_id), 3), np.nan)
    for c in np.unique(cam_id):
        s = (cam_id == c) & np.isfinite(rays[:, 0])
        if not s.any():
            continue
        J = jacobian(int(models[c]), intr[c], q_ck[c], p_ck[c], rays[s], d[s], rig)
        Sz = np.einsum("nai,ij,nbj->nab", J, camera_block(S, models, c), J)
        cov[s] = np.stack([Sz[:, 0, 0], Sz[:, 0, 1], Sz[:, 1, 1]], 1)
    return cov, rays
