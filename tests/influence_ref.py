"""Reference of vcgpu_get_observation_influence (include/vcgpu.h) in numpy, on the oracle's Jacobians and dense inverse.

influence() takes the oracle at the handle's state, with the handle's active observations: Sigma is dense_cov's
dense inverse of the oracle's J^T J (which sums the active observations only), J and r are the oracle's eval_reproj of
every observation, removed ones included, restricted to P = (frame pose 6 | camera globals 6 + K) with constant
globals' columns masked; the SoftLOne weight w = visual_mult rho'(|r|^2) is applied here.  refit() is the independent
check: one Gauss-Newton step of the dense system with observation i taken out (or, removed, put back in)."""
import numpy as np

from vicalib_b200 import synth


def camera_offsets(models):
    return np.cumsum([0] + [6 + synth.NUM_INTR[int(m)] for m in models])[:-1]


def weights(r, visual_mult):
    """visual_mult rho'(|r|^2) of SoftLOne with b = 0.25, as the solve weights a corner"""
    s = (r ** 2).sum(1)
    return visual_mult / np.sqrt(1.0 + s / 0.25)


def rows(o, models, obs_frame, obs_cam, visual_mult):
    """per observation: (P's indices into the dense system [12 + K], J~ [2, 12 + K], r~ [2]) as lists"""
    r, J = o.eval_reproj()
    nf, fd = o.n_frames, o.fd
    nfp = nf * fd
    goff = camera_offsets(models)
    mask = o.global_mask()
    sw = np.sqrt(weights(r, visual_mult))
    out = []
    for i in range(len(r)):
        c, f = int(obs_cam[i]), int(obs_frame[i])
        NG = 6 + synth.NUM_INTR[int(models[c])]
        P = np.r_[f * fd + np.arange(6), nfp + goff[c] + np.arange(NG)]
        Ji = J[i, :, :6 + NG].copy()
        Ji[:, 6:] *= mask[goff[c]:goff[c] + NG][None, :]
        out.append((P, sw[i] * Ji, sw[i] * r[i]))
    return out


def influence(o, Hi, models, obs_frame, obs_cam, active, frame_used, visual_mult=1.0):
    """dict(h [n, 3], stud [n], infl [n]) with the header's exact cases; Hi the dense inverse (dense_cov.dense_inverse)"""
    nfp = o.n_frames * o.fd
    Sg = Hi[nfp:, nfp:]
    F = np.flatnonzero(np.diag(Sg) != 0.0)
    SF = Sg[np.ix_(F, F)]
    cam_used = np.array([((np.asarray(obs_cam) == c) & (active > 0)).any() for c in range(len(models))])
    n = len(obs_frame)
    h, stud, infl = np.full((n, 3), np.nan), np.full(n, np.nan), np.full(n, np.nan)
    # correlation scales: what each output moves by when every entry of Sigma moves by its own sqrt(Sigma_ii Sigma_jj),
    # to first order with every product's sign its worst (as dense_cov.corr_errors scales Sigma's entries)
    sc_h, sc_stud, sc_infl = np.full((n, 3), np.nan), np.full(n, np.nan), np.full(n, np.nan)
    for i, (P, Jt, rt) in enumerate(rows(o, models, obs_frame, obs_cam, visual_mult)):
        if not cam_used[obs_cam[i]] or not frame_used[obs_frame[i]]:
            continue
        SPP = Hi[np.ix_(P, P)]
        H = Jt @ SPP @ Jt.T
        h[i] = H[0, 0], 0.5 * (H[0, 1] + H[1, 0]), H[1, 1]
        s = np.abs(Jt) @ np.sqrt(np.abs(np.diag(SPP)))
        sc_h[i] = s[0] * s[0], s[0] * s[1], s[1] * s[1]
        D = np.eye(2) + (-H if active[i] else H)
        if not (D[0, 0] > 0 and np.linalg.det(D) > 0):
            continue
        u = np.linalg.solve(D, rt)
        stud[i] = rt @ u
        dg = Hi[np.ix_(nfp + F, P)] @ Jt.T @ u
        infl[i] = dg @ np.linalg.solve(SF, dg)
        a = Jt.T @ u
        M = Hi[np.ix_(P, nfp + F)] @ np.linalg.solve(SF, Hi[np.ix_(nfp + F, P)])
        sc_stud[i] = (np.abs(u) @ s) ** 2
        sc_infl[i] = (np.abs(a) @ np.sqrt(np.abs(np.diag(M)))) ** 2 + 2 * abs(infl[i]) * sc_stud[i] / max(abs(stud[i]), 1e-300)
    return dict(h=h, stud=stud, infl=infl, sc_h=sc_h, sc_stud=sc_stud, sc_infl=sc_infl)


def assemble(nf, fd, Sgg, Sff, Sfg):
    """a dense [nf fd + G]^2 matrix holding only the blocks influence() reads: Sigma_ff, Sigma_fg and Sigma_gg, e.g. as
    vcgpu_get_frame_covariance, vcgpu_get_frame_cross_covariance and vcgpu_get_covariance return them"""
    nfp, G = nf * fd, len(Sgg)
    Hi = np.zeros((nfp + G, nfp + G))
    for f in range(nf):
        s = slice(f * fd, (f + 1) * fd)
        Hi[s, s] = Sff[f]
        Hi[s, nfp:] = Sfg[f]
        Hi[nfp:, s] = Sfg[f].T
    Hi[nfp:, nfp:] = Sgg
    return Hi


def dense_system(o, used, live):
    """(H, g, keep) of the oracle's normal equations in dense form, kept rows as dense_cov.dense_inverse keeps them"""
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
    g = np.r_[ne["gf"].ravel(), ne["gc"]]
    keep = np.concatenate([(used[:, None] & (np.arange(fd) < live)[None, :]).ravel(), o.global_mask() != 0])
    return H, g, keep


def refit(H, g, keep, P, Jt, rt, active, nfp, F):
    """(shift of the globals on F, r~ after the step) of one Gauss-Newton step with the observation's rows taken out
    (active) or put in (removed), less the step of the system as it is.  g = 0 takes the state as the stationary point
    the definition assumes; at a tightly converged state the step from the oracle's own g agrees to its convergence."""
    n = len(g)
    A = np.zeros((2, n))
    A[:, P] = Jt
    sg = -1.0 if active else 1.0
    H2 = H + sg * A.T @ A
    g2 = g + sg * A.T @ rt
    k = np.flatnonzero(keep)
    d0, d1 = np.zeros(n), np.zeros(n)
    d0[k] = -np.linalg.solve(H[np.ix_(k, k)], g[k])
    d1[k] = -np.linalg.solve(H2[np.ix_(k, k)], g2[k])
    d = d1 - d0
    return d[nfp + F], rt + A @ d
