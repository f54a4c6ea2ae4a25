"""CPU model of vcgpu_get_frame_covariance's recurrences (vc_frame_cov.cuh), checked against np.linalg.inv.

Inertial: the chain elimination over chain_plan's level table keeps, per eliminated node p, M_p = T^-1 H_Iy restricted
to p (the device's Z_p[:, 0:2FD+G]); the dense [globals | top nodes] system is inverted; then every level, top-down,
gets Σ_py = -M_p Σ_yy and Σ_pq = K_pq + M_p Σ_yy M_q^T, K = T^-1, and keeps Σ_kk, Σ_k,k+1 and Σ_kg of every node as
the boundary of the level below.  Vision: Σ_ff = B_f^-1 + W_f Σ_gg W_f^T, W_f = B_f^-1 E_f.

The systems are the block normal equations of random least-squares problems with the solver's structure (frame blocks
B, couplings U[f] = H[f-1, f], E, C)."""
import numpy as np
import pytest

import chain_plan

C_ = chain_plan.CHUNK


def random_system(nf, G, fd, rng, chain=True):
    B, U, E = np.zeros((nf, fd, fd)), np.zeros((nf, fd, fd)), np.zeros((nf, fd, G))
    C = np.eye(G)
    for f in range(nf):
        Jf, Jg = rng.standard_normal((12, fd)), 0.3 * rng.standard_normal((12, G))
        B[f] += Jf.T @ Jf
        E[f] += Jf.T @ Jg
        C += Jg.T @ Jg
    for f in range(1, nf if chain else 1):
        J1, J2, Jg = rng.standard_normal((fd, fd)), rng.standard_normal((fd, fd)), 0.3 * rng.standard_normal((fd, G))
        B[f - 1] += J1.T @ J1
        B[f] += J2.T @ J2
        U[f] = J1.T @ J2
        E[f - 1] += J1.T @ Jg
        E[f] += J2.T @ Jg
        C += Jg.T @ Jg
    return B, U, E, C


def dense(B, U, E, C):
    nf, fd, G = B.shape[0], B.shape[1], C.shape[0]
    nfp = nf * fd
    H = np.zeros((nfp + G, nfp + G))
    for f in range(nf):
        s = slice(f * fd, (f + 1) * fd)
        H[s, s] = B[f]
        H[s, nfp:] = E[f]
        H[nfp:, s] = E[f].T
        if f > 0:
            sp = slice((f - 1) * fd, f * fd)
            H[sp, s] = U[f]
            H[s, sp] = U[f].T
    H[nfp:, nfp:] = C
    return H


def tridiag(A, U, first, m):
    """the block-tridiagonal matrix of nodes first .. first+m-1 (U[k] = H[k-1, k])"""
    fd = A.shape[1]
    T = np.zeros((m * fd, m * fd))
    for i in range(m):
        T[i * fd:(i + 1) * fd, i * fd:(i + 1) * fd] = A[first + i]
        if i > 0:
            T[(i - 1) * fd:i * fd, i * fd:(i + 1) * fd] = U[first + i]
            T[i * fd:(i + 1) * fd, (i - 1) * fd:i * fd] = U[first + i].T
    return T


def chain_frame_cov(B, U, E, C, sizes):
    """Σ_kk, Σ_k,k+1, Σ_kg of level 0 (every frame) by elimination over `sizes`, then the selected inversion."""
    nf, fd, G = B.shape[0], B.shape[1], C.shape[0]
    assert sizes[0] == nf
    levels = [dict(A=B.copy(), U=U.copy(), E=E.copy())]
    S = C.copy()
    # ---- eliminate (chain_eliminate_kernel)
    for l in range(len(sizes) - 1):
        L, n, ns = levels[l], sizes[l], sizes[l + 1]
        nxt = dict(A=L["A"][::C_].copy(), U=np.zeros((ns, fd, fd)), E=L["E"][::C_].copy())
        assert nxt["A"].shape[0] == ns
        L["M"] = {}
        for j in range(ns):
            s = j * C_
            m, hasR = min(C_ - 1, n - 1 - s), s + C_ < n
            if m == 0:
                assert not hasR  # one GPU: a lone separator is the level's last node
                continue
            T = tridiag(L["A"], L["U"], s + 1, m)
            Hy = np.zeros((m * fd, 2 * fd + G))
            Hy[:fd, :fd] = L["U"][s + 1].T
            if hasR:
                Hy[-fd:, fd:2 * fd] = L["U"][s + m + 1]
            Hy[:, 2 * fd:] = L["E"][s + 1:s + m + 1].reshape(m * fd, G)
            M = np.linalg.solve(T, Hy)
            for i in range(m):
                L["M"][s + 1 + i] = M[i * fd:(i + 1) * fd]
            Sch = Hy.T @ M
            nxt["A"][j] -= Sch[:fd, :fd]
            nxt["E"][j] -= Sch[:fd, 2 * fd:]
            if hasR:
                nxt["A"][j + 1] -= Sch[fd:2 * fd, fd:2 * fd]
                nxt["E"][j + 1] -= Sch[fd:2 * fd, 2 * fd:]
                nxt["U"][j + 1] = -Sch[:fd, fd:2 * fd]
            S -= Sch[2 * fd:, 2 * fd:]
        levels.append(nxt)
    # ---- the dense phase: the inverse of [globals | top nodes] (dense_solve_kernel's inversion)
    top, nt = levels[-1], sizes[-1]
    N = G + nt * fd
    D = np.zeros((N, N))
    D[:G, :G] = S
    for t in range(nt):
        o = G + t * fd
        D[o:o + fd, o:o + fd] = top["A"][t]
        D[o:o + fd, :G] = top["E"][t]
        D[:G, o:o + fd] = top["E"][t].T
        if t > 0:
            D[o - fd:o, o:o + fd] = top["U"][t]
            D[o:o + fd, o - fd:o] = top["U"][t].T
    X = np.linalg.inv(D)
    Sgg = X[:G, :G]
    sig = dict(kk=np.zeros((nt, fd, fd)), kn=np.zeros((nt, fd, fd)), kg=np.zeros((nt, fd, G)))
    for t in range(nt):
        o = G + t * fd
        sig["kk"][t] = X[o:o + fd, o:o + fd]
        sig["kg"][t] = X[o:o + fd, :G]
        if t + 1 < nt:
            sig["kn"][t] = X[o:o + fd, o + fd:o + 2 * fd]
    # ---- the levels, top-down (chain_selinv_kernel)
    for l in range(len(sizes) - 2, -1, -1):
        L, n, up = levels[l], sizes[l], sig
        sig = dict(kk=np.zeros((n, fd, fd)), kn=np.zeros((n, fd, fd)), kg=np.zeros((n, fd, G)))
        for j in range(sizes[l + 1]):
            s = j * C_
            m, hasR = min(C_ - 1, n - 1 - s), s + C_ < n
            Syy = np.zeros((2 * fd + G, 2 * fd + G))
            Syy[:fd, :fd] = up["kk"][j]
            Syy[:fd, 2 * fd:] = up["kg"][j]
            Syy[2 * fd:, :fd] = up["kg"][j].T
            Syy[2 * fd:, 2 * fd:] = Sgg
            if hasR:
                Syy[fd:2 * fd, fd:2 * fd] = up["kk"][j + 1]
                Syy[:fd, fd:2 * fd] = up["kn"][j]
                Syy[fd:2 * fd, :fd] = up["kn"][j].T
                Syy[fd:2 * fd, 2 * fd:] = up["kg"][j + 1]
                Syy[2 * fd:, fd:2 * fd] = up["kg"][j + 1].T
            sig["kk"][s] = up["kk"][j]
            sig["kg"][s] = up["kg"][j]
            if m == 0:
                continue
            K = np.linalg.inv(tridiag(L["A"], L["U"], s + 1, m))
            P = {p: L["M"][p] @ Syy for p in range(s + 1, s + m + 1)}  # -Σ_py
            sig["kn"][s] = -P[s + 1][:, :fd].T
            for i in range(m):
                p = s + 1 + i
                sig["kk"][p] = K[i * fd:(i + 1) * fd, i * fd:(i + 1) * fd] + P[p] @ L["M"][p].T
                sig["kg"][p] = -P[p][:, 2 * fd:]
                if i + 1 < m:
                    sig["kn"][p] = K[i * fd:(i + 1) * fd, (i + 1) * fd:(i + 2) * fd] + P[p] @ L["M"][p + 1].T
                elif hasR:
                    sig["kn"][p] = -P[p][:, fd:2 * fd]
    return sig


def vision_frame_cov(B, E, C):
    Binv = np.linalg.inv(B)
    W = Binv @ E
    Sgg = np.linalg.inv(C - np.einsum("fki,fkj->ij", E, W))
    return Binv + np.einsum("fig,gh,fjh->fij", W, Sgg, W)


def _check_chain(nf, G, sizes=None, seed=0):
    fd = chain_plan.FD
    B, U, E, C = random_system(nf, G, fd, np.random.default_rng(seed))
    sig = chain_frame_cov(B, U, E, C, sizes or chain_plan.level_sizes(nf))
    Hi = np.linalg.inv(dense(B, U, E, C))
    nfp = nf * fd
    ref_kk = np.stack([Hi[f * fd:(f + 1) * fd, f * fd:(f + 1) * fd] for f in range(nf)])
    ref_kn = np.stack([Hi[f * fd:(f + 1) * fd, (f + 1) * fd:(f + 2) * fd] if f + 1 < nf else np.zeros((fd, fd))
                       for f in range(nf)])
    ref_kg = Hi[:nfp, nfp:].reshape(nf, fd, G)
    scale = np.abs(Hi).max()
    for k, ref in (("kk", ref_kk), ("kn", ref_kn), ("kg", ref_kg)):
        err = np.abs(sig[k] - ref).max() / scale
        assert err <= 1e-10, (k, err)


@pytest.mark.parametrize("nf", [2, 3, 8, 9, 64, 65, 72, 513])
def test_chain_frame_counts(nf):
    _check_chain(nf, 13)


@pytest.mark.parametrize("G", [13, 41, 67])
def test_chain_globals(G):
    _check_chain(72, G, seed=G)


def _branch_frames(branch):
    """The fewest frames whose level table takes `branch`.  The wide branches are where a level has more chunks than
    SMs; the level table itself does not depend on the SM count, so they are looked up on a 2-SM device, where they come
    at CPU-invertible sizes.  Four elimination levels need 2049 frames with the device's top of kCsTop nodes; the model
    takes them at 513 frames with a top of one node (the same recurrences, one more level)."""
    if branch == "levels4":
        return 513, chain_plan.level_sizes(513, top=1)
    for n in range(2, 1000):
        if branch in chain_plan.branches(n, sms=2):
            return n, None
    raise AssertionError(branch)


@pytest.mark.parametrize("branch", chain_plan.BRANCHES)
def test_chain_branches(branch):
    nf, sizes = _branch_frames(branch)
    if sizes is not None:
        assert len(sizes) - 1 >= 4
    _check_chain(nf, 13, sizes)


def test_lone_separator_and_top4_shapes():
    assert 0 in chain_plan.lone_separator_levels(9) and chain_plan.top_nodes(32) == chain_plan.TOP
    for nf in (9, 17, 32, 33, 257):
        _check_chain(nf, 13, seed=nf)


@pytest.mark.parametrize("G", [13, 41, 67])
def test_vision_closed_form(G):
    fd, nf = 6, 40
    B, U, E, C = random_system(nf, G, fd, np.random.default_rng(G), chain=False)
    assert not U.any()
    Hi = np.linalg.inv(dense(B, U, E, C))
    ref = np.stack([Hi[f * fd:(f + 1) * fd, f * fd:(f + 1) * fd] for f in range(nf)])
    assert np.abs(vision_frame_cov(B, E, C) - ref).max() <= 1e-10 * np.abs(Hi).max()
