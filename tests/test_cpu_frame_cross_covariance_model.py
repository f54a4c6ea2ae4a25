"""CPU model of vcgpu_get_frame_cross_covariance's blocks, checked against np.linalg.inv.

Inertial: level 0 of test_cpu_frame_covariance_model.py's level walk keeps Σ_k,k+1 and Σ_kg of every frame, the blocks
the call unscales; they are checked on every branch of the chain's level table.  Vision: Σ_fg = -X_f Σ_gg and
Σ_f,f+1 = X_f Σ_gg X_f+1^T with X_f = B_f^-1 E_f (frame_cross_cov_block).  And the relative-motion covariance of two
consecutive frames assembled from the three calls' blocks."""
import numpy as np
import pytest

import chain_plan
from test_cpu_frame_covariance_model import _branch_frames, chain_frame_cov, dense, random_system, vision_frame_cov


def _ref(Hi, nf, fd, G):
    nfp = nf * fd
    kn = np.stack([Hi[f * fd:(f + 1) * fd, (f + 1) * fd:(f + 2) * fd] for f in range(nf - 1)])
    return kn, Hi[:nfp, nfp:].reshape(nf, fd, G)


def vision_cross_cov(B, E, C):
    X = np.linalg.solve(B, E)
    Sgg = np.linalg.inv(C - np.einsum("fki,fkj->ij", E, X))
    P = X @ Sgg
    return np.einsum("fig,fjg->fij", P[:-1], X[1:]), -P


@pytest.mark.parametrize("branch", chain_plan.BRANCHES)
def test_chain_cross_blocks_on_every_branch(branch):
    nf, sizes = _branch_frames(branch)
    fd, G = chain_plan.FD, 13
    B, U, E, C = random_system(nf, G, fd, np.random.default_rng(7))
    sig = chain_frame_cov(B, U, E, C, sizes or chain_plan.level_sizes(nf))
    Hi = np.linalg.inv(dense(B, U, E, C))
    kn, kg = _ref(Hi, nf, fd, G)
    scale = np.abs(Hi).max()
    assert np.abs(sig["kn"][:-1] - kn).max() <= 1e-10 * scale
    assert not sig["kn"][-1].any()  # the last frame has no next one
    assert np.abs(sig["kg"] - kg).max() <= 1e-10 * scale


@pytest.mark.parametrize("G", [13, 67, 68])
def test_vision_cross_closed_form(G):
    fd, nf = 6, 40
    B, U, E, C = random_system(nf, G, fd, np.random.default_rng(G), chain=False)
    Hi = np.linalg.inv(dense(B, U, E, C))
    kn, kg = _ref(Hi, nf, fd, G)
    fn, fg = vision_cross_cov(B, E, C)
    scale = np.abs(Hi).max()
    assert np.abs(fn - kn).max() <= 1e-10 * scale
    assert np.abs(fg - kg).max() <= 1e-10 * scale


@pytest.mark.parametrize("inertial", [False, True], ids=["vision", "inertial"])
def test_relative_motion_covariance(inertial):
    """Σ_ff + Σ_f+1,f+1 - Σ_f,f+1 - Σ_f,f+1^T is the covariance of x_f+1 - x_f: D Σ D^T with D = [-I I]"""
    fd = chain_plan.FD if inertial else 6
    nf, G = 33, 13
    B, U, E, C = random_system(nf, G, fd, np.random.default_rng(3), chain=inertial)
    if inertial:
        sig = chain_frame_cov(B, U, E, C, chain_plan.level_sizes(nf))
        kk, kn = sig["kk"], sig["kn"][:-1]
    else:
        kk, (kn, _) = vision_frame_cov(B, E, C), vision_cross_cov(B, E, C)
    rel = kk[:-1] + kk[1:] - kn - kn.transpose(0, 2, 1)
    Hi = np.linalg.inv(dense(B, U, E, C))
    for f in range(nf - 1):
        D = np.zeros((fd, Hi.shape[0]))
        D[:, f * fd:(f + 1) * fd] = -np.eye(fd)
        D[:, (f + 1) * fd:(f + 2) * fd] = np.eye(fd)
        assert np.abs(rel[f] - D @ Hi @ D.T).max() <= 1e-10 * np.abs(Hi).max()
