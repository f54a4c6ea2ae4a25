"""The dense inverse of the oracle's J^T J, every block kept: the reference of the frame covariance calls' blocks off the
block diagonal (Σ[frame f, globals], Σ[frame f, frame f+1]).  Built as test_gpu_frame_covariance._dense_frame_cov
builds its [frame, frame] blocks."""
import numpy as np


def dense_inverse(o, used, live):
    """inv(J^T J) [nf fd + G]^2 from the oracle's block normal equations, with the rows and columns of the constant
    globals, the unused frames (used[f] == False) and a frame's tangents from `live` on removed (those rows and columns
    are 0).  Returns (inverse, kept: the boolean mask of the rows kept)."""
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
    # inverted after a symmetric diagonal scaling to unit diagonal, as _dense_frame_cov does
    Hk = H[np.ix_(keep, keep)]
    d = 1.0 / np.sqrt(np.diag(Hk))
    Hi = np.zeros_like(H)
    Hi[np.ix_(keep, keep)] = np.linalg.inv(Hk * d[:, None] * d[None, :]) * d[:, None] * d[None, :]
    return Hi, keep


def cross_blocks(Hi, nf, fd):
    """(Σ_fg [nf, fd, G], Σ_f,f+1 [nf - 1, fd, fd]) of a dense inverse"""
    nfp = nf * fd
    fg = Hi[:nfp, nfp:].reshape(nf, fd, -1)
    fn = np.stack([Hi[f * fd:(f + 1) * fd, (f + 1) * fd:(f + 2) * fd] for f in range(nf - 1)]) if nf > 1 else np.zeros((0, fd, fd))
    return fg, fn


def corr_errors(fg, fn, ref_fg, ref_fn, sd_f, sd_g, keep_f, keep_g):
    """the correlation-scaled errors |ΔΣ_ij| / sqrt(Σ_ii Σ_jj) of the kept entries of fg and fn; sd_f [nf, fd] and
    sd_g [G] the reference's standard deviations, keep_f [nf, fd] and keep_g [G] the kept tangents"""
    mg = keep_f[:, :, None] & keep_g[None, None, :]
    mn = keep_f[:-1, :, None] & keep_f[1:, None, :]
    with np.errstate(divide="ignore", invalid="ignore"):  # the dropped tangents' deviations are 0; masked out below
        eg = (np.abs(fg - ref_fg) / (sd_f[:, :, None] * sd_g[None, None, :]))[mg].max(initial=0.0)
        en = (np.abs(fn - ref_fn) / (sd_f[:-1, :, None] * sd_f[1:, None, :]))[mn].max(initial=0.0)
    return float(eg), float(en)


def exact_zeros(fg, fn, keep_f, keep_g):
    """True where every entry the calls leave out is exactly 0.0: the rows of dropped frame tangents, the columns of
    constant or unused globals, and in fn the columns of frame f+1's dropped tangents"""
    zg = ~(keep_f[:, :, None] & keep_g[None, None, :])
    zn = ~(keep_f[:-1, :, None] & keep_f[1:, None, :])
    return bool(np.all(fg[zg] == 0.0) and np.all(fn[zn] == 0.0) and not np.signbit(fg[zg]).any() and not np.signbit(fn[zn]).any())
