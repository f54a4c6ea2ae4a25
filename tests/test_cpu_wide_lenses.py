"""CPU: the camera models far from the axis, and the wide-angle and fisheye rigs of wide_lenses.py.

- The oracle's dual-number Project against tests/golden/reproj_wide_kat.npz (60-digit mpmath, exact central
  differences; make_golden.py --wide): residuals and all 12 + K Jacobian columns at test_cpu_oracle_golden's 1e-10, on
  KB4 rows out to 100 degrees (one exactly at Z = 0, two behind the image plane), FOV rows to rad = tan 80 degrees at
  two w, strong barrel poly2 / poly3 rows up to their folds and linear rows to rad = 3.
- The fixture has the regime it is for, uses the lenses the rigs use, and make_golden.py --wide regenerates it.
- synth.project, which makes the rigs' observations, against the fixture's residuals.
- The builders' regimes (each builder asserts its own), and synth.make_problem's lens keywords: at their defaults they
  are the default problem bit for bit, and culling drops exactly the corners it claims to.
"""
import dataclasses
import os
import sys

import numpy as np
import pytest

import target_views as tv
import wide_lenses as wl
from test_cpu_imu_motion import DEFAULT_DIGESTS, _digest
from test_cpu_oracle_golden import _oracle_for_reproj
from vicalib_b200 import synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODELS = ("linear", "fov", "poly2", "poly3", "kb4")


def _rows(name):
    z = np.load(os.path.join(GOLD, "reproj_wide_kat.npz"))
    return {k[len(name) + 1:]: z[k] for k in z.files if k.startswith(name + "_")}


def _camera_point(d, i):
    """the row's camera-frame point, in binary64 as the kernels form it"""
    Rwk, Rck = synth.quat_to_mat(d["T_wk"][i, :4]), synth.quat_to_mat(d["q_ck"][i])
    return Rck @ (Rwk.T @ (d["p_w"][i] - d["T_wk"][i, 4:])) + d["p_ck"][i]


# ------------------------------------------------------------------ the oracle against the wide KAT
@pytest.mark.parametrize("name", MODELS)
def test_oracle_vs_wide_kat(name):
    d = _rows(name)
    model = synth.MODEL_IDS[name]
    worst = [0.0, 0.0]
    for i in range(d["r"].shape[0]):
        o, K = _oracle_for_reproj(model, d, i)
        r, J = o.eval_reproj()
        e_r = np.abs(r[0] - d["r"][i]).max() / max(1.0, np.abs(d["r"][i]).max())
        e_J = np.abs(J[0][:, :12 + K] - d["J"][i]).max() / np.abs(d["J"][i]).max()
        worst = [max(worst[0], e_r), max(worst[1], e_J)]
        assert e_r <= 1e-10 and e_J <= 1e-10, (i, e_r, e_J)
    print(f"\n{name}: oracle vs wide KAT, {d['r'].shape[0]} rows: r {worst[0]:.1e}, J {worst[1]:.1e}")


def test_synth_project_vs_wide_kat():
    """synth.project (atan2 for KB4) gives the fixture's residuals at its camera-frame points"""
    for name in MODELS:
        d = _rows(name)
        model = synth.MODEL_IDS[name]
        for i in range(d["r"].shape[0]):
            z = synth.project(model, _camera_point(d, i), d["intr"][i])
            assert np.abs(z - d["z"][i] - d["r"][i]).max() <= 1e-9 * max(1.0, np.abs(d["r"][i]).max()), (name, i)


def test_wide_kat_regime():
    """the rows sit where they claim: KB4 at 10-100 degrees with Z exactly 0 in one row and Z < 0 in two, the k4 term
    worth more than a pixel at the rim; FOV from its small-argument branch to tan 80 degrees at w = 0.9 and 1.2; the
    polynomials up to 0.97 of their folds with the factor well below 1; linear to rad = 3"""
    d = _rows("kb4")
    pc = np.array([_camera_point(d, i) for i in range(d["r"].shape[0])])
    th = np.degrees(np.arctan2(np.hypot(pc[:, 0], pc[:, 1]), pc[:, 2]))
    assert np.allclose(th, [10, 45, 80, 89.9, 90, 95, 100], atol=1e-9)
    assert np.sum(pc[:, 2] == 0.0) == 1 and np.sum(pc[:, 2] < 0) == 2
    assert np.all(d["intr"][:, 4:8] == wl.KB4_FISHEYE)
    t = np.radians(th.max())
    assert np.abs(d["intr"][:, 0] * wl.KB4_FISHEYE[3] * t ** 9).max() > 1.0
    assert wl.kb4_monotone_to(wl.KB4_FISHEYE) > t
    d = _rows("fov")
    pc = np.array([_camera_point(d, i) for i in range(d["r"].shape[0])])
    rad = np.hypot(pc[:, 0], pc[:, 1]) / pc[:, 2]
    assert sorted(set(d["intr"][:, 4].tolist())) == list(wl.FOV_W)
    assert rad.min() ** 2 < 1e-5 and rad.max() > np.tan(np.radians(79.99))
    for name, k in (("poly2", wl.POLY2_BARREL), ("poly3", wl.POLY3_BARREL)):
        d = _rows(name)
        assert np.all(d["intr"][:, 4:4 + len(k)] == k)
        pc = np.array([_camera_point(d, i) for i in range(d["r"].shape[0])])
        r = np.hypot(pc[:, 0], pc[:, 1]) / pc[:, 2]
        fold = wl.poly_fold(k)
        assert r.max() < fold and r.max() > 0.95 * fold, (name, r.max(), fold)
        assert 1 + sum(kk * r.max() ** (2 * i + 2) for i, kk in enumerate(k)) < 0.65
    d = _rows("linear")
    pc = np.array([_camera_point(d, i) for i in range(d["r"].shape[0])])
    assert (np.hypot(pc[:, 0], pc[:, 1]) / pc[:, 2]).max() > 2.95


def test_wide_kat_regenerates():
    """make_golden.py --wide reproduces the committed fixture bit for bit"""
    sys.path.insert(0, GOLD)
    try:
        import make_golden
    finally:
        sys.path.remove(GOLD)
    assert make_golden.KB4_FISHEYE == wl.KB4_FISHEYE and make_golden.POLY2_BARREL == wl.POLY2_BARREL
    assert make_golden.POLY3_BARREL == wl.POLY3_BARREL and tuple(make_golden.WIDE_FOV_W) == wl.FOV_W
    new = make_golden.wide_kat()
    z = np.load(os.path.join(GOLD, "reproj_wide_kat.npz"))
    assert sorted(new) == sorted(z.files)
    for k in z.files:
        assert np.array_equal(new[k], z[k]), k
    # the keys of reproj_kat.npz
    assert sorted(z.files) == sorted(np.load(os.path.join(GOLD, "reproj_kat.npz")).files)


# ------------------------------------------------------------------ the builders
@pytest.mark.parametrize("name", wl.NAMES)
def test_builder_regime(name):
    lens = wl.build(name)  # asserts its own regime
    print("\n" + wl.describe(lens))
    assert lens.inertial == name.endswith("_inertial")
    r = lens.regime
    assert not r["clamp"] and r["diag_min"] > 1e-3
    # the default lens, for contrast: no corner beyond 45 degrees
    if name == "kb4_fisheye":
        p = synth.make_problem(models=("kb4",), n_frames=30, seed=51)
        assert wl.camera_regime(p, 0)["theta_max"] < 45


def test_lens_keywords_at_their_defaults():
    """focal=320, TRUTH_DIST, standoff (0.47, 0.11), no tilt and no cull give the default problems bit for bit"""
    for kw, want in DEFAULT_DIGESTS:
        models = [synth.MODEL_IDS[m] for m in kw.get("models", ("poly3",))]
        p = synth.make_problem(focal=320.0, dist=[synth.TRUTH_DIST[m] for m in models], standoff=(0.47, 0.11), **kw)
        assert _digest(p) == want, kw
    with pytest.raises(ValueError):
        synth.make_problem(models=("kb4",), dist=[[0.1, 0.2]])
    with pytest.raises(ValueError):
        synth.make_problem(motion="vigorous", tilt=(0.5, 0.1))


def test_cull():
    """cull=True keeps exactly the corners inside the image, and (pinhole-type models) in front of the camera; the
    truth and the random draws are those of the same problem without culling"""
    kw = dict(models=("kb4", "poly3"), n_frames=12, seed=58, focal=(190.0, 320.0), dist=[wl.KB4_FISHEYE, wl.POLY3_BARREL],
              standoff=(0.3, 0.08), tilt=(1.0, 0.3))
    a, b = synth.make_problem(**kw), synth.make_problem(cull=True, **kw)
    for f in ("intr", "T_wp", "q_ck", "p_ck"):
        assert np.array_equal(getattr(a, f), getattr(b, f)) and np.array_equal(a.truth[f], b.truth[f]), f
    pc = wl.camera_points(a)
    with np.errstate(invalid="ignore"):
        inside = np.isfinite(a.p_c).all(1) & (a.p_c[:, 0] >= 0) & (a.p_c[:, 0] < 640) & (a.p_c[:, 1] >= 0) & \
            (a.p_c[:, 1] < 480)
    keep = inside & ((a.obs_cam == 0) | (pc[:, 2] > 0))
    assert np.array_equal(dataclasses.asdict(tv.keep(a, keep))["p_c"], b.p_c)
    assert np.array_equal(a.obs_frame[keep], b.obs_frame) and np.array_equal(a.obs_cam[keep], b.obs_cam)
    assert (pc[keep & (a.obs_cam == 0), 2] < 0).any()  # the fisheye keeps corners behind its image plane
    assert not keep[a.obs_cam == 1].all() and not keep[a.obs_cam == 0].all()
