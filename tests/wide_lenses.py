"""Rigs with wide-angle and fisheye lenses, cut from synth.make_problem's lens regimes, each of which asserts the regime it
claims, so that a later change to synth cannot quietly remove the edge a test relies on.

synth's default lens is narrow: a focal length of ~320 px on 640 x 480, mild distortion (TRUTH_DIST), the camera
0.36-0.58 m from the grid and looking at it, so no corner is much more than 40 degrees off the axis.  The cameras vicalib
offers FOV and KB4 for see far more: here every lens works near the edge of its model.
- kb4_fisheye: a KB4 fisheye (f ~ 190 px) whose k4 theta^9 term moves a rim corner by several pixels; the camera turns
  up to 1.3 rad away from the grid, so some views put corners behind the image plane (theta > 90 degrees, Z < 0), where
  only atan2 gives theta and dtheta/dZ keeps its sign.
- fov_w09 / fov_w12: FOV lenses (f ~ 190 px) seeing rays out to ~80 degrees (rad ~ 5.7), at w = 0.9 and w = 1.2.
- poly2_barrel / poly3_barrel: strong barrel distortion, the factor f(r^2) well below 1 at the rim, the image radius
  r f(r^2) monotone over every view (past its first maximum, the fold, the model maps two rays to one pixel).
- linear_wide: a pinhole (f ~ 100 px) seeing rays out to rad ~ 3.
- kb4_poly3, fov_kb4 and their _inertial variants: rigs mixing a fisheye with a barrel or FOV lens.
Corners outside the image, and (every model but KB4) corners not in front of the camera, are culled.

Each builder reports, per camera, the largest angle off the axis, the share of corners beyond 60 degrees and the count
beyond 90, and the rim displacement of the model's highest-order term (the largest pixel shift over the corners when
that coefficient is set to 0; for FOV, w -> 0 is the pinhole); and for the rig, whether the LM damping clamp
clamp(diag, 1e-6, 1e32) of the Jacobi-scaled system engages on a free column at the starting point.
"""
import dataclasses

import numpy as np

import target_views as tv
from vicalib_b200 import synth

ALL_ON = tv.ALL_ON
# fisheye KB4 coefficients: d(theta) = theta + k1 theta^3 + ... + k4 theta^9 rises monotonically to beyond 120 degrees
KB4_FISHEYE = [0.04, -0.02, 0.005, -0.0005]
POLY2_BARREL = [-0.32, 0.04]          # fold at r = 1.236 (51 degrees)
POLY3_BARREL = [-0.3, 0.06, -0.005]   # fold at r = 1.932 (62.6 degrees)
FOV_W = (0.9, 1.2)


@dataclasses.dataclass
class Lens(tv.View):
    regime: dict = dataclasses.field(default_factory=dict)


def camera_points(p):
    """[n_obs, 3] camera-frame coordinates of every observation at the truth"""
    out = np.zeros((p.n_obs, 3))
    T, tr = p.truth["T_wp"], p.truth
    for c in range(p.n_cams):
        s = p.obs_cam == c
        f = p.obs_frame[s]
        pk = np.einsum("nji,nj->ni", synth.quat_to_mat(T[f, :4]), p.p_w[s] - T[f, 4:])
        out[s] = pk @ synth.quat_to_mat(tr["q_ck"][c]).T + tr["p_ck"][c]
    return out


def poly_fold(k):
    """the smallest r > 0 at which d(r f(r^2))/dr = 0 (inf if none below 10)"""
    x = np.linspace(1e-6, 100.0, 2_000_001)
    d = 1 + sum((2 * i + 3) * kk * x ** (i + 1) for i, kk in enumerate(k))
    bad = np.flatnonzero(d <= 0)
    return float(np.sqrt(x[bad[0]])) if len(bad) else np.inf


def kb4_monotone_to(k):
    """the smallest theta > 0 at which d'(theta) = 0 (inf if none below pi)"""
    th = np.linspace(0.0, np.pi, 200_001)
    d = 1 + sum((2 * i + 3) * kk * th ** (2 * i + 2) for i, kk in enumerate(k))
    bad = np.flatnonzero(d <= 0)
    return float(th[bad[0]]) if len(bad) else np.inf


def _without_last(model, intr):
    """the model with its highest-order coefficient at 0: (model, intrinsics)"""
    K = synth.NUM_INTR[model]
    q = np.array(intr, dtype=np.float64)
    if model == synth.FOV:
        return synth.LINEAR, q  # w -> 0: the factor is 1 (Calibu's w^2 <= 1e-5 branch)
    q[K - 1] = 0.0
    return model, q


def camera_regime(p, c, pc=None):
    pc = camera_points(p) if pc is None else pc
    s = p.obs_cam == c
    x = pc[s]
    model, intr = int(p.models[c]), p.truth["intr"][c]
    th = np.degrees(np.arctan2(np.hypot(x[:, 0], x[:, 1]), x[:, 2]))
    out = dict(model=model, n=int(s.sum()), theta_max=float(th.max()), share60=float(np.mean(th > 60)),
               n90=int(np.sum(th > 90)), views90=int(len(np.unique(p.obs_frame[s][th > 90]))), rim=0.0)
    if model != synth.LINEAR:
        m0, i0 = _without_last(model, intr)
        out["rim"] = float(np.linalg.norm(synth.project(model, x, intr) - synth.project(m0, x, i0), axis=1).max())
    if model != synth.KB4:
        r = np.hypot(x[:, 0], x[:, 1]) / x[:, 2]
        out["rad_max"] = float(r.max())
        if model in (synth.POLY2, synth.POLY3):
            k = intr[4:synth.NUM_INTR[model]]
            out["fold"] = poly_fold(k)
            out["factor_rim"] = float((1 + sum(kk * r ** (2 * i + 2) for i, kk in enumerate(k))).min())
    else:
        out["monotone_to"] = np.degrees(kb4_monotone_to(intr[4:8]))
    return out


def clamp_regime(p, flags):
    """the smallest and largest diagonal entry of the Jacobi-scaled system over the free columns at the start, and
    whether clamp(diag, 1e-6, 1e32) changes one of them"""
    from oracle.binding import Oracle

    o = Oracle(p, **flags)
    ne = o.normal_equations()
    d = np.concatenate([np.einsum("fii->fi", ne["B"]).ravel(), np.diag(ne["C"])])
    live = np.concatenate([np.ones(ne["B"].shape[0] * ne["B"].shape[1], bool), o.global_mask() != 0])
    sd = (d / (1 + np.sqrt(d)) ** 2)[live]
    return dict(diag_min=float(sd.min()), diag_max=float(sd.max()), clamp=bool(sd.min() < 1e-6 or sd.max() > 1e32))


def regime(p, flags):
    pc = camera_points(p)
    return dict(cams=[camera_regime(p, c, pc) for c in range(p.n_cams)], **clamp_regime(p, flags))


def _short_of_folds(p, margin=0.97):
    """p without the corners a barrel camera sees beyond margin x its fold (a detector finds no grid there: the image
    folds back on itself)"""
    x = camera_points(p)
    sel = np.ones(p.n_obs, bool)
    for c, m in enumerate(p.models):
        if int(m) in (synth.POLY2, synth.POLY3):
            s = p.obs_cam == c
            fold = poly_fold(p.truth["intr"][c, 4:synth.NUM_INTR[int(m)]])
            sel[s] = np.hypot(x[s, 0], x[s, 1]) / x[s, 2] < margin * fold
    return tv.keep(p, sel)


def _lens(name, models, focal, dist, standoff, tilt, n_frames, seed, inertial=False, fold_cut=False):
    p = synth.make_problem(models=models, n_frames=n_frames, grid=(14, 10), seed=seed, inertial=inertial, focal=focal,
                           dist=dist, standoff=standoff, tilt=tilt, cull=True)
    if fold_cut:
        p = _short_of_folds(p)
    flags = dict(ALL_ON) if inertial else {}
    lens = Lens(name, p, flags, regime=regime(p, flags))
    n = tv.counts(p)
    assert n.max(0).min() >= 40 and n.sum(1).min() >= 1000, n  # every frame well constrained, every camera well seen
    assert not lens.regime["clamp"], lens.regime  # the damping clamp does not engage: a lens that made it would be news
    return lens


def _check_fisheye(r, views90=3):
    assert r["model"] == synth.KB4
    assert r["theta_max"] > 95 and r["n90"] >= 20 and r["views90"] >= views90, r
    assert r["share60"] > 0.25 and r["rim"] > 1.0, r
    assert r["monotone_to"] > r["theta_max"] + 10, r


def _check_fov(r):
    assert r["model"] == synth.FOV and 78 < r["theta_max"] < 86 and r["rad_max"] > 4.7, r
    assert r["share60"] > 0.05, r


def _check_poly(r, factor):
    assert r["model"] in (synth.POLY2, synth.POLY3)
    assert r["rad_max"] < r["fold"] and r["rad_max"] > 0.85 * r["fold"], r  # monotone over every view, near its limit
    assert r["factor_rim"] < factor and r["rim"] > 1.0, r


def kb4_fisheye(inertial=False):
    lens = _lens("kb4_fisheye", ("kb4",), 190.0, [KB4_FISHEYE], (0.3, 0.08), (1.0, 0.3), 30, 51)
    _check_fisheye(lens.regime["cams"][0])
    return lens


def fov(w):
    lens = _lens(f"fov_w{int(round(10 * w)):02d}", ("fov",), 190.0, [[w]], (0.3, 0.08), (0.8, 0.3), 30, 52)
    _check_fov(lens.regime["cams"][0])
    assert lens.p.truth["intr"][0, 4] == w
    return lens


def poly2_barrel():
    lens = _lens("poly2_barrel", ("poly2",), 320.0, [POLY2_BARREL], (0.33, 0.05), (0.15, 0.1), 30, 53)
    _check_poly(lens.regime["cams"][0], 0.7)
    return lens


def poly3_barrel():
    lens = _lens("poly3_barrel", ("poly3",), 320.0, [POLY3_BARREL], (0.3, 0.05), (0.3, 0.15), 30, 54)
    _check_poly(lens.regime["cams"][0], 0.55)
    return lens


def linear_wide():
    lens = _lens("linear_wide", ("linear",), 100.0, [[]], (0.3, 0.08), (0.7, 0.3), 30, 55)
    r = lens.regime["cams"][0]
    assert r["rad_max"] > 2.8 and r["share60"] > 0.03, r
    return lens


def kb4_poly3(inertial=False):
    """the rig turns far enough for the fisheye to see past 80 degrees; the barrel camera's corners beyond 0.97 of its
    fold are dropped (_short_of_folds)"""
    nf = 60 if inertial else 30
    lens = _lens("kb4_poly3" + ("_inertial" if inertial else ""), ("kb4", "poly3"), (190.0, 320.0),
                 [KB4_FISHEYE, POLY3_BARREL], (0.3, 0.05), (0.8, 0.3), nf, 56, inertial, fold_cut=True)
    k, q = lens.regime["cams"]
    assert k["theta_max"] > 80 and k["rim"] > 1.0, k
    _check_poly(q, 0.6)
    return lens


def fov_kb4(inertial=False):
    nf = 60 if inertial else 30
    lens = _lens("fov_kb4" + ("_inertial" if inertial else ""), ("fov", "kb4"), 190.0, [[FOV_W[0]], KB4_FISHEYE],
                 (0.3, 0.08), (0.95, 0.3), nf, 57, inertial)
    f, k = lens.regime["cams"]
    assert f["model"] == synth.FOV and 80 < f["theta_max"] < 90 and f["rad_max"] > 5.7, f  # FOV sees up to 90 degrees
    _check_fisheye(k)
    return lens


BUILDERS = {
    "kb4_fisheye": kb4_fisheye,
    "fov_w09": lambda: fov(FOV_W[0]),
    "fov_w12": lambda: fov(FOV_W[1]),
    "poly2_barrel": poly2_barrel,
    "poly3_barrel": poly3_barrel,
    "linear_wide": linear_wide,
    "kb4_poly3": kb4_poly3,
    "fov_kb4": fov_kb4,
    "kb4_poly3_inertial": lambda: kb4_poly3(True),
    "fov_kb4_inertial": lambda: fov_kb4(True),
}
NAMES = tuple(BUILDERS)
VISION = tuple(n for n in NAMES if not n.endswith("_inertial"))
INERTIAL = tuple(n for n in NAMES if n.endswith("_inertial"))


def build(name):
    return BUILDERS[name]()


def describe(lens):
    """one line per camera, and the clamp"""
    names = {v: k for k, v in synth.MODEL_IDS.items()}
    out = []
    for c, r in enumerate(lens.regime["cams"]):
        s = (f"{lens.name} cam {c} ({names[r['model']]}): theta max {r['theta_max']:.1f} deg, "
             f">60 deg {100 * r['share60']:.1f} %, >90 deg {r['n90']} corners in {r['views90']} views, "
             f"rim shift of the top term {r['rim']:.2f} px")
        if "rad_max" in r:
            s += f", rad max {r['rad_max']:.2f}"
        if "fold" in r:
            s += f" (fold {r['fold']:.3f}), factor at rim {r['factor_rim']:.3f}"
        out.append(s)
    g = lens.regime
    out.append(f"{lens.name}: scaled diag {g['diag_min']:.1e} .. {g['diag_max']:.2f}, clamp engages: {g['clamp']}")
    return "\n".join(out)
