"""Reference of vcgpu_get_imu_influence (include/vcgpu.h) in numpy, on the oracle's IMU rows and dense inverse.

influence() takes the oracle at the handle's state and IMU weights: Sigma is dense_cov's dense inverse of the oracle's
J^T J, J_w and r_w are the oracle's eval_imu (W-weighted, loss-free) in P's order (frame k: pose 6, v 3 | frame k+1 |
IMU globals 15) with constant IMU globals' columns masked; the CauchyLoss(100) weight w = imu_mult rho'(|r_w|^2) is
applied here.  refit() is the independent check: one Gauss-Newton step of the dense system with interval k taken out."""
import numpy as np

from vicalib_b200 import synth

# vcgpu_eval_imu's columns (pose2 6 | pose1 6 | v2 3 | v1 3 | globals 15) in P's order
LOCAL = np.r_[np.arange(6, 12), np.arange(15, 18), np.arange(0, 6), np.arange(12, 15), np.arange(18, 33)]


def weights(r, imu_mult):
    """imu_mult rho'(|r|^2) of CauchyLoss(100), as the solve weights an interval"""
    s = (r ** 2).sum(1)
    return imu_mult / (1.0 + s / 1e4)


def imu_offset(models):
    """the IMU globals' offset in the globals: after every camera's 6 + K"""
    return int(sum(6 + synth.NUM_INTR[int(m)] for m in models))


def rows(o, models, imu_mult):
    """per interval: (P's indices into the dense system [33], J~ [9, 33], r~ [9], has measurements)"""
    r, J = o.eval_imu()
    nf, fd = o.n_frames, o.fd
    nfp = nf * fd
    io = imu_offset(models)
    mask = o.global_mask()[io:io + 15]
    sw = np.sqrt(weights(r, imu_mult))
    out = []
    for k in range(nf - 1):
        P = np.r_[k * fd + np.arange(9), (k + 1) * fd + np.arange(9), nfp + io + np.arange(15)]
        Jk = J[k][:, LOCAL].copy()
        Jk[:, 18:] *= mask[None, :]
        out.append((P, sw[k] * Jk, sw[k] * r[k], bool(J[k].any())))  # no measurements: zero rows (the solve's)
    return out


def influence(o, Hi, models, imu_mult=1.0):
    """dict(h [n, 9, 9], stud [n], infl [n]) with the header's exact cases; Hi the dense inverse, and correlation
    scales sc_* as influence_ref.influence gives them"""
    nfp = o.n_frames * o.fd
    Sg = Hi[nfp:, nfp:]
    F = np.flatnonzero(np.diag(Sg) != 0.0)
    SF = Sg[np.ix_(F, F)]
    n = o.n_frames - 1
    h, stud, infl = np.full((n, 9, 9), np.nan), np.full(n, np.nan), np.full(n, np.nan)
    sc_h, sc_stud, sc_infl = np.full((n, 9, 9), np.nan), np.full(n, np.nan), np.full(n, np.nan)
    for k, (P, Jt, rt, ok) in enumerate(rows(o, models, imu_mult)):
        if not ok:
            continue
        SPP = Hi[np.ix_(P, P)]
        H = Jt @ SPP @ Jt.T
        h[k] = 0.5 * (H + H.T)
        s = np.abs(Jt) @ np.sqrt(np.abs(np.diag(SPP)))
        sc_h[k] = np.outer(s, s)
        D = np.eye(9) - h[k]
        try:
            np.linalg.cholesky(D)
        except np.linalg.LinAlgError:
            continue
        u = np.linalg.solve(D, rt)
        stud[k] = rt @ u
        a = Jt.T @ u
        dg = Hi[np.ix_(nfp + F, P)] @ a
        infl[k] = dg @ np.linalg.solve(SF, dg)
        M = Hi[np.ix_(P, nfp + F)] @ np.linalg.solve(SF, Hi[np.ix_(nfp + F, P)])
        sc_stud[k] = (np.abs(u) @ s) ** 2
        sc_infl[k] = (np.abs(a) @ np.sqrt(np.abs(np.diag(M)))) ** 2 + 2 * abs(infl[k]) * sc_stud[k] / max(abs(stud[k]), 1e-300)
    return dict(h=h, stud=stud, infl=infl, sc_h=sc_h, sc_stud=sc_stud, sc_infl=sc_infl)


def assemble(nf, fd, Sgg, Sff, Sfg, Sfn):
    """a dense [nf fd + G]^2 matrix holding only the blocks influence() reads: Sigma_ff, Sigma_f,f+1, Sigma_fg and
    Sigma_gg, as vcgpu_get_frame_covariance, vcgpu_get_frame_cross_covariance and vcgpu_get_covariance return them"""
    nfp, G = nf * fd, len(Sgg)
    Hi = np.zeros((nfp + G, nfp + G))
    for f in range(nf):
        s = slice(f * fd, (f + 1) * fd)
        Hi[s, s] = Sff[f]
        Hi[s, nfp:] = Sfg[f]
        Hi[nfp:, s] = Sfg[f].T
        if f + 1 < nf:
            t = slice((f + 1) * fd, (f + 2) * fd)
            Hi[s, t] = Sfn[f]
            Hi[t, s] = Sfn[f].T
    Hi[nfp:, nfp:] = Sgg
    return Hi


def refit(H, g, keep, P, Jt, rt, nfp, F):
    """(shift of the globals on F, r~ after the step) of one Gauss-Newton step with the interval's rows taken out, less
    the step of the system as it is (influence_ref.refit for a block of rows)"""
    n = len(g)
    A = np.zeros((len(rt), n))
    A[:, P] = Jt
    H2 = H - A.T @ A
    g2 = g - A.T @ rt
    k = np.flatnonzero(keep)
    s = 1.0 / np.sqrt(np.diag(H)[k])  # Jacobi-scaled solves: the inertial systems are conditioned ~1e11 unscaled

    def step(M, b):
        return -s * np.linalg.solve(M[np.ix_(k, k)] * s[:, None] * s[None, :], b[k] * s)

    d0, d1 = np.zeros(n), np.zeros(n)
    d0[k] = step(H, g)
    d1[k] = step(H2, g2)
    d = d1 - d0
    return d[nfp + F], rt + A @ d
