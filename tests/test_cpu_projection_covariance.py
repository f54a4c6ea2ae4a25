"""CPU: the reference of vcgpu_get_projection_covariance (tests/projection_ref.py) against the oracle.
  unprojection  the round trip through oracle.binding.project to 1e-12 px for all five models, on the wide-lens rigs'
                lenses (KB4 to 100 degrees, FOV at w = 0.9 and 1.2, poly lenses up to their folds), FOV's small-rad and
                w^2 <= 1e-5 branches and the image centre
  domain        a pixel just inside the poly fold, the FOV limit or the KB4 limit is finite, one just outside is NaN
  Jacobian      the oracle's eval_reproj columns against central differences of the projection
  infinity      RIG at d = 0 is RIG with Sigma_c's p_ck rows and columns zeroed, and the limit of large d
  Monte Carlo   the covariance of projections with intrinsics drawn from N(x, Sigma_c) against J Sigma_c J^T"""
import numpy as np
import pytest

import projection_ref as P
import wide_lenses as W
from oracle.binding import project
from vicalib_b200 import synth

# (model, intrinsics without padding, largest angle off the axis in degrees) of every lens model as the wide rigs use it
LENSES = {
    "linear_wide": (synth.LINEAR, [100.0, 101.0, 320.0, 240.0], 71.0),
    "fov_w09": (synth.FOV, [190.0, 191.0, 320.0, 240.0, W.FOV_W[0]], 81.0),
    "fov_w12": (synth.FOV, [190.0, 191.0, 320.0, 240.0, W.FOV_W[1]], 81.0),
    "poly2_barrel": (synth.POLY2, [320.0, 321.0, 320.0, 240.0] + W.POLY2_BARREL, None),
    "poly3_barrel": (synth.POLY3, [320.0, 321.0, 320.0, 240.0] + W.POLY3_BARREL, None),
    "kb4_fisheye": (synth.KB4, [190.0, 191.0, 320.0, 240.0] + W.KB4_FISHEYE, 100.0),
    "poly3_mild": (synth.POLY3, [320.0, 321.0, 320.0, 240.0, -0.05, 0.01, -0.001], 50.0),
}


def _intr(v):
    return np.r_[np.asarray(v, float), np.zeros(10 - len(v))]


def _rays(model, intr, max_deg, n=400, seed=0):
    """rays out to max_deg off the axis (poly: to 0.999 of the fold), at every azimuth"""
    rng = np.random.default_rng(seed)
    if max_deg is None:
        th_max = np.arctan(0.999 * P.limit(model, intr))
    else:
        th_max = np.radians(max_deg)
    th = np.r_[0.0, 1e-4, rng.uniform(0, th_max, n - 3), th_max]
    ph = rng.uniform(-np.pi, np.pi, n)
    return np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], 1)


@pytest.mark.parametrize("name", list(LENSES))
def test_round_trip(name):
    model, v, deg = LENSES[name]
    intr = _intr(v)
    worst, worst_ray = 0.0, 0.0
    for x in _rays(model, intr, deg):
        z = project(model, x, intr)
        r = P.unproject(model, intr, z)
        assert np.isfinite(r).all(), (name, x, z)
        worst = max(worst, np.abs(project(model, r, intr) - z).max())
        worst_ray = max(worst_ray, np.abs(r - x).max())
    print(f"{name}: round trip {worst:.1e} px, ray {worst_ray:.1e}")
    assert worst <= 1e-12 and worst_ray <= 1e-9, (worst, worst_ray)


@pytest.mark.parametrize("w,rad", [(0.9, 1e-4), (1.2, 2e-3), (0.9, 3.2e-3), (1e-3, 0.5), (-0.9, 0.7), (0.9, 0.0)],
                         ids=["small_rad", "small_rad_2", "branch_edge", "small_w", "negative_w", "centre"])
def test_fov_branches(w, rad):
    intr = _intr([190.0, 191.0, 320.0, 240.0, w])
    for ph in np.linspace(-np.pi, np.pi, 7):
        x = np.array([rad * np.cos(ph), rad * np.sin(ph), 1.0])
        x /= np.linalg.norm(x)
        z = project(synth.FOV, x, intr)
        r = P.unproject(synth.FOV, intr, z)
        assert np.abs(project(synth.FOV, r, intr) - z).max() <= 1e-12
        assert np.abs(r - x).max() <= 1e-9


@pytest.mark.parametrize("model", [synth.LINEAR, synth.POLY2, synth.POLY3, synth.KB4])
def test_image_centre(model):
    v = {synth.LINEAR: [300.0, 310.0, 321.5, 239.5], synth.POLY2: [300.0, 310.0, 321.5, 239.5] + W.POLY2_BARREL,
         synth.POLY3: [300.0, 310.0, 321.5, 239.5] + W.POLY3_BARREL, synth.KB4: [300.0, 310.0, 321.5, 239.5] + W.KB4_FISHEYE}[model]
    assert np.array_equal(P.unproject(model, _intr(v), np.array([321.5, 239.5])), [0.0, 0.0, 1.0])


def _edge_pixels(model, intr):
    """the image radius r_d of the domain's limit, and the pixels at r_d (1 -+ 1e-9) along a diagonal"""
    if model == synth.FOV:
        rd = np.pi / 2 / abs(intr[4])
    else:
        lim = P.limit(model, intr)
        k = intr[4:synth.NUM_INTR[model]]
        s = lim * lim
        rd = lim * (1 + sum(kk * s ** (i + 1) for i, kk in enumerate(k)))
    d = np.array([np.cos(0.3), np.sin(0.3)])
    return rd, [intr[2:4] + intr[:2] * d * rd * f for f in (1 - 1e-9, 1 + 1e-9)]


@pytest.mark.parametrize("name", ["poly2_barrel", "poly3_barrel", "fov_w09", "fov_w12", "kb4_fisheye", "kb4_fold"])
def test_domain_edges(name):
    if name == "kb4_fold":  # a KB4 lens whose d(theta) folds before pi
        model, intr = synth.KB4, _intr([190.0, 191.0, 320.0, 240.0, -0.08, 0.0, 0.0, 0.0])
    else:
        model, intr = LENSES[name][0], _intr(LENSES[name][1])
    rd, (inside, outside) = _edge_pixels(model, intr)
    r_in, r_out = P.unproject(model, intr, inside), P.unproject(model, intr, outside)
    print(f"{name}: limit at r_d = {rd:.6f}")
    assert np.isfinite(r_in).all() and np.isnan(r_out).all(), (r_in, r_out)
    assert np.abs(project(model, r_in, intr) - inside).max() <= 1e-9


def test_folds_agree_with_the_wide_rigs():
    assert abs(P.limit(synth.POLY2, _intr(LENSES["poly2_barrel"][1])) - W.poly_fold(W.POLY2_BARREL)) < 1e-4
    assert abs(P.limit(synth.POLY3, _intr(LENSES["poly3_barrel"][1])) - W.poly_fold(W.POLY3_BARREL)) < 1e-4
    assert abs(P.limit(synth.KB4, _intr(LENSES["kb4_fisheye"][1])) - W.kb4_monotone_to(W.KB4_FISHEYE)) < 1e-4
    assert P.limit(synth.KB4, _intr([190.0, 191.0, 320.0, 240.0, 0.01, 0.0, 0.0, 0.0])) == np.pi


def _pose(seed):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=4)
    return q / np.linalg.norm(q), rng.normal(scale=0.1, size=3)


@pytest.mark.parametrize("name", list(LENSES))
@pytest.mark.parametrize("depth", [0.0, 0.7, 3.0], ids=["inf", "d07", "d3"])
@pytest.mark.parametrize("rig", [False, True], ids=["camera", "rig"])
def test_jacobian_against_differences(name, depth, rig):
    model, v, deg = LENSES[name]
    intr = _intr(v)
    q, t = _pose(len(name))
    rays = _rays(model, intr, deg, n=12, seed=3)
    J = P.jacobian(model, intr, q, t, rays, depth, rig)
    for k, x in enumerate(rays):
        Jd = P.jacobian_fd(model, intr, q, t, x, depth, rig)
        scale = np.abs(Jd).max(axis=1, keepdims=True)
        assert np.abs(J[k] - Jd).max() <= 1e-7 * scale.max(), (name, k, J[k], Jd)
    if not rig:
        assert not J[:, :, :6].any()
    if depth == 0.0:
        assert not J[:, :, 3:6].any()


def _spd(N, seed, scale=1e-4):
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(N, N))
    return scale * (A @ A.T + N * np.eye(N)) / N


@pytest.mark.parametrize("name", ["kb4_fisheye", "poly3_barrel", "fov_w09"])
def test_infinity(name):
    model, v, deg = LENSES[name]
    intr = _intr(v)
    N = 6 + synth.NUM_INTR[model]
    S = _spd(N, 1)
    S0 = S.copy()
    S0[3:6, :] = 0.0
    S0[:, 3:6] = 0.0
    q, t = _pose(5)
    models, cams = np.array([model]), dict(intr=intr[None], q_ck=q[None], p_ck=t[None])
    x = _rays(model, intr, deg, n=20, seed=4)
    pix = np.array([project(model, r, intr) for r in x])
    cam = np.zeros(len(pix), int)
    c_inf, _ = P.projection_covariance(S, models, cams["intr"], cams["q_ck"], cams["p_ck"], cam, pix, None, rig=True)
    c_zero, _ = P.projection_covariance(S0, models, cams["intr"], cams["q_ck"], cams["p_ck"], cam, pix, None, rig=True)
    c_far, _ = P.projection_covariance(S, models, cams["intr"], cams["q_ck"], cams["p_ck"], cam, pix, 1e7, rig=True)
    assert np.array_equal(c_inf, c_zero)
    assert np.abs(c_far - c_inf).max() <= 1e-6 * np.abs(c_inf).max()


@pytest.mark.parametrize("name", ["kb4_fisheye", "poly3_barrel", "fov_w12", "linear_wide"])
def test_monte_carlo(name):
    """intrinsics drawn from N(x, Sigma_c), a fixed ray: the projections' sample covariance matches J Sigma_c J^T
    within its sampling error (the covariance is small enough that the projection is linear to well below that)"""
    model, v, deg = LENSES[name]
    intr = _intr(v)
    K = synth.NUM_INTR[model]
    S = np.zeros((6 + K, 6 + K))
    Si = _spd(K, 7, scale=1e-8) * np.outer(np.maximum(1, np.abs(intr[:K])), np.maximum(1, np.abs(intr[:K])))
    S[6:, 6:] = Si
    x = _rays(model, intr, deg, n=8, seed=9)[5]
    pix = project(model, x, intr)
    cov, _ = P.projection_covariance(S, np.array([model]), intr[None], np.array([[0, 0, 0, 1.0]]), np.zeros((1, 3)), [0], pix[None])
    rng = np.random.default_rng(11)
    n = 4000
    samples = rng.multivariate_normal(intr[:K], Si, size=n)
    z = np.array([synth.project(model, x[None], np.r_[s, np.zeros(10 - K)])[0] for s in samples])
    C = np.cov(z.T)
    ref = np.array([[cov[0, 0], cov[0, 1]], [cov[0, 1], cov[0, 2]]])
    # the standard error of a sample covariance entry: sqrt((S_aa S_bb + S_ab^2) / n)
    se = np.sqrt((np.outer(np.diag(ref), np.diag(ref)) + ref ** 2) / n)
    print(f"{name}: sample {C.ravel()}, J S J^T {ref.ravel()}, |diff| / se {np.abs(C - ref).max() / se.max():.2f}")
    assert (np.abs(C - ref) <= 5 * se).all(), (C, ref, se)
