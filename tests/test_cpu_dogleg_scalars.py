"""The DOGLEG step from its six scalars, as the persistent kernel forms it (vc_mega.cuh, U1), against the plain reference.

The persistent kernel never forms H step: it takes the dogleg point and the model change from |g~|^2, u.Hu, |gn|^2,
g~.gn, u.Hx and x.Hx (u = g~ / D, x the Gauss-Newton step, gn = D x), each summed from per-frame shares:
  step.g      = cg |g~|^2 + cn g~.gn
  step.H.step = cg^2 u.Hu + 2 cg cn u.Hx + cn^2 x.Hx
`dogleg_from_scalars` restates that arithmetic (with dogleg_point's branch rule, vc_dogleg.cuh); on random arrow systems
its model change and |step~| must equal dogleg_ref.dogleg_step's, which forms the step vector and H step explicitly, for
each of the three branches.  Largest measured (x86-64): 2.6e-16 relative; the bar sits about 4e3 above it.
"""
import numpy as np
import pytest

import dogleg_ref
from chain_plan import arrow_matvec

BAR = 1e-12  # largest measured 2.6e-16 (float64 scalars against long-double vectors)


def dogleg_point(radius, alpha, g2, gn2, b):
    """(cg, cn, |step~|): step~ = cg g~ + cn gn (Ceres DoglegStrategy::ComputeTraditionalDoglegStep)"""
    gn_norm, g_norm = np.sqrt(gn2), np.sqrt(g2)
    if gn_norm <= radius:
        return 0.0, 1.0, gn_norm
    if g_norm * alpha >= radius:
        return -(radius / g_norm), 0.0, radius
    b_dot_a = -alpha * b
    a_sq = (alpha * g_norm) ** 2
    bma_sq = a_sq - 2.0 * b_dot_a + gn_norm * gn_norm
    c = b_dot_a - a_sq
    d = np.sqrt(c * c + bma_sq * (radius * radius - a_sq))
    beta = (d - c) / bma_sq if c <= 0.0 else (radius * radius - a_sq) / (d + c)
    cg, cn = -alpha * (1.0 - beta), beta
    return cg, cn, np.sqrt(max(0.0, cg * cg * g2 + 2.0 * cg * cn * b + cn * cn * gn2))


def dogleg_from_scalars(radius, g2, uHu, gn2, b, uHx, xHx):
    """model change and |step~| of the DOGLEG step from the six scalars"""
    alpha = g2 / uHu
    cg, cn, step_norm = dogleg_point(radius, alpha, g2, gn2, b)
    model_change = -(cg * g2 + cn * b) - 0.5 * (cg * cg * uHu + 2.0 * cg * cn * uHx + cn * cn * xHx)
    return dict(model_change=model_change, step_norm=step_norm)


def scalars(ne, scale, mu=dogleg_ref.MU):
    """the six scalars of a DOGLEG step on (ne, scale), in long double"""
    ld = np.longdouble
    s = np.asarray(scale, dtype=np.float64)
    D = np.sqrt(np.clip(dogleg_ref._diag(ne) * s * s, 1e-6, 1e32))
    g = np.concatenate([ne["gf"].ravel(), ne["gc"]]) * s
    gt = (g / D).astype(ld)
    u = gt / D
    x = dogleg_ref.gauss_newton(ne, s, D * D * mu).astype(ld)
    gn = x * D
    Hu, Hx = arrow_matvec(ne, s, u.astype(np.float64)), arrow_matvec(ne, s, x.astype(np.float64))
    return (np.sum(gt * gt), np.sum(u * Hu), np.sum(gn * gn), np.sum(gt * gn), np.sum(u * Hx), np.sum(x * Hx))


def random_arrow(rng, nf=7, fd=6, G=9, rows=24):
    """normal equations J^T J, J^T r of a random least-squares problem with the block-arrow structure (frames couple to
    the globals only)"""
    B = np.zeros((nf, fd, fd))
    E = np.zeros((nf, fd, G))
    gf = np.zeros((nf, fd))
    C = np.zeros((G, G))
    gc = np.zeros(G)
    for f in range(nf):
        J = rng.standard_normal((rows, fd + G)) * np.exp(rng.uniform(-2, 2, fd + G))
        r = rng.standard_normal(rows)
        H, g = J.T @ J, J.T @ r
        B[f], E[f], C = H[:fd, :fd], H[:fd, fd:], C + H[fd:, fd:]
        gf[f], gc = g[:fd], gc + g[fd:]
    return dict(B=B, U=np.zeros_like(B), E=E, gf=gf, C=C, gc=gc)


@pytest.mark.parametrize("seed", range(4))
def test_step_from_scalars_matches_reference(seed):
    rng = np.random.default_rng(seed)
    ne = random_arrow(rng)
    scale = dogleg_ref.jacobi_scale(ne)
    t = [float(v) for v in scalars(ne, scale)]
    radii = dogleg_ref.branch_radii(dogleg_ref.dogleg_step(ne, scale, 1e4))
    for branch, radius in radii.items():
        ref = dogleg_ref.dogleg_step(ne, scale, radius)
        assert ref["branch"] == branch
        got = dogleg_from_scalars(radius, *t)
        assert abs(got["model_change"] - ref["model_change"]) <= BAR * abs(ref["model_change"]), branch
        assert abs(got["step_norm"] - ref["step_norm"]) <= BAR * ref["step_norm"], branch
