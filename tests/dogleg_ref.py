"""Plain reference of one DOGLEG step, in numpy, as the header of vc_dogleg.cuh states it.

On the Jacobi-scaled block-arrow system H = S J^T J S, g = S J^T r (the blocks of `normal_equations()`):
  D      = sqrt(clamp(diag H, 1e-6, 1e32))
  g~     = g / D,   alpha = |g~|^2 / (u . H u),  u = g~ / D           Cauchy step = -alpha g~
  gn     = D * [(H + mu D^2)^-1 (-g)]                                  Gauss-Newton step
  step~  = gn                              if |gn| <= radius           branch "gauss_newton"
         = -(radius / |g~|) g~             if alpha |g~| >= radius     branch "cauchy"
         = the dogleg point on the segment otherwise                   branch "segment"
  step   = step~ / D,  model change = -step.g - step.H.step / 2

Sums are taken in np.longdouble.  The Gauss-Newton system is factored in float64 (scipy.sparse) and the solution
refined once with a residual computed in long double.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from chain_plan import arrow_matvec

MU = 1e-8  # DoglegStrategy's initial (and smallest) Gauss-Newton regularisation


def jacobi_scale(ne):
    """1 / (1 + sqrt(diag H)) of the unscaled system."""
    return 1.0 / (1.0 + np.sqrt(_diag(ne)))


def _diag(ne):
    return np.concatenate([np.einsum("fii->fi", ne["B"]).ravel(), np.diag(ne["C"])])


def _sparse(ne, scale, D2):
    """S H S + diag(D2) as a float64 CSC matrix."""
    nf, fd, _ = ne["B"].shape
    G = ne["C"].shape[0]
    nfp = nf * fd
    rows, cols, vals = [], [], []

    def put(r0, c0, blk):
        r, c = np.meshgrid(np.arange(blk.shape[-2]), np.arange(blk.shape[-1]), indexing="ij")
        rows.append((r0[:, None, None] + r[None]).ravel())
        cols.append((c0[:, None, None] + c[None]).ravel())
        vals.append(blk.ravel())

    f0 = np.arange(nf) * fd
    put(f0, f0, ne["B"])
    put(f0[:-1], f0[1:], ne["U"][1:])
    put(f0[1:], f0[:-1], np.swapaxes(ne["U"][1:], 1, 2))
    put(f0, np.full(nf, nfp), ne["E"])
    put(np.full(nf, nfp), f0, np.swapaxes(ne["E"], 1, 2))
    put(np.array([nfp]), np.array([nfp]), ne["C"][None])
    n = nfp + G
    H = sp.csc_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))
    S = sp.diags(scale)
    return (S @ H @ S + sp.diags(D2)).tocsc()


def gauss_newton(ne, scale, D2):
    """x = (S H S + diag(D2))^-1 (-S g): float64 sparse LU, one refinement step with a long-double residual."""
    ld = np.longdouble
    g = np.concatenate([ne["gf"].ravel(), ne["gc"]]) * scale
    lu = spla.splu(_sparse(ne, scale, D2))
    x = lu.solve(-g)

    def residual(x):
        return -g.astype(ld) - arrow_matvec(ne, scale, x) - D2.astype(ld) * x.astype(ld)

    return x + lu.solve(residual(x).astype(np.float64))


def dogleg_step(ne, scale, radius, mu=MU):
    """One DOGLEG step at `radius`.  Returns alpha, |g~|, |gn|, the branch, |step~| and the model change."""
    ld = np.longdouble
    s = np.asarray(scale, dtype=np.float64)
    D = np.sqrt(np.clip(_diag(ne) * s * s, 1e-6, 1e32))
    g = np.concatenate([ne["gf"].ravel(), ne["gc"]]) * s
    gt = (g / D).astype(ld)
    u = gt / D
    g2 = np.sum(gt * gt)
    alpha = g2 / np.sum(u * arrow_matvec(ne, s, u.astype(np.float64)))
    gn = gauss_newton(ne, s, D * D * mu).astype(ld) * D
    gn2 = np.sum(gn * gn)
    g_norm, gn_norm = np.sqrt(g2), np.sqrt(gn2)
    if gn_norm <= radius:
        branch, st = "gauss_newton", gn
    elif alpha * g_norm >= radius:
        branch, st = "cauchy", -(radius / g_norm) * gt
    else:  # Ceres DoglegStrategy::ComputeTraditionalDoglegStep
        branch = "segment"
        b_dot_a = -alpha * np.sum(gt * gn)
        a_sq = (alpha * g_norm) ** 2
        bma_sq = a_sq - 2 * b_dot_a + gn2
        c = b_dot_a - a_sq
        d = np.sqrt(c * c + bma_sq * (ld(radius) ** 2 - a_sq))
        beta = (d - c) / bma_sq if c <= 0 else (ld(radius) ** 2 - a_sq) / (d + c)
        st = -alpha * (1 - beta) * gt + beta * gn
    step = st / D
    model_change = -np.sum(step * g) - 0.5 * np.sum(step * arrow_matvec(ne, s, step.astype(np.float64)))
    return dict(alpha=float(alpha), g_norm=float(g_norm), gn_norm=float(gn_norm), branch=branch,
                step_norm=float(np.sqrt(np.sum(st * st))), model_change=float(model_change))


def branch_radii(ref):
    """One radius per branch from a step's alpha |g~| and |gn| (any radius's step gives them): 1.5 |gn| takes the
    Gauss-Newton step, 0.5 alpha |g~| the clipped Cauchy step, their geometric mean the dogleg segment."""
    cauchy, gn = ref["alpha"] * ref["g_norm"], ref["gn_norm"]
    assert cauchy < gn, "the Cauchy point lies outside the Gauss-Newton step: no segment branch"
    return {"gauss_newton": 1.5 * gn, "cauchy": 0.5 * cauchy, "segment": float(np.sqrt(cauchy * gn))}


def radius_after(radius, rho, step_norm):
    """The radius a DOGLEG iteration leaves: accepted (rho > 1e-3) with rho > 0.75 grows it to 3 |step~|, with
    rho < 0.25 halves it; a rejected step halves it."""
    if rho > 1e-3:
        return max(radius, 3.0 * step_norm) if rho > 0.75 else (0.5 * radius if rho < 0.25 else radius)
    return 0.5 * radius
