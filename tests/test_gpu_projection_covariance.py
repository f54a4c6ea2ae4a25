"""GPU: vcgpu_get_projection_covariance, the pixel covariance the calibration leaves at projected points (proj_cov_kernel).
  parity     cov and rays against tests/projection_ref.py on the matrix vcgpu_get_covariance returns: all five models,
             both frames, finite depth and infinity, vision and inertial, a wide-lens rig, G = 67 and a rig of G = 112
             (past the cluster kernels)
  zeros      exact zeros for fix_intrinsics in the camera frame and for a camera no observation sees
  domain     NaN outside the model's domain, where the reference has NaN
  matrix     a passed-in matrix gives the bits of the internal one
  no effect  state, weights and the next solve's bits
  refusals   each names the point and writes nothing"""
import ctypes as C

import numpy as np
import pytest

import chain_plan
import projection_ref as P
import target_views as tv
import wide_lenses as W
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
# Bars: cov relative to the point's largest |S_uu|, |S_vv|; rays absolute.  Measured on an H100 80GB HBM3 (700 W): cov
# 3.7e-11 (G = 112, 8 x KB4), 1.1e-12 elsewhere; rays 2.5e-15.
COV_BAR, RAY_BAR = 1e-10, 1e-12


def _solved(p, flags, iters=15):
    """a handle solved on p; models: its camera models, for the reference"""
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.models = np.asarray(p.models)
    g.load(p)
    g.set_flags(**flags)
    g.set_options(function_tol=1e-12, max_iters=iters)
    g.solve()
    return g


def _grid(n_cams, nu=24, nv=18, extra=()):
    """every camera's pixels on an nu x nv grid over 640 x 480 (corners included), plus extra pixels"""
    u, v = np.meshgrid(np.linspace(0, 639, nu), np.linspace(0, 479, nv))
    px = np.r_[np.stack([u.ravel(), v.ravel()], 1), np.asarray(extra, float).reshape(-1, 2)]
    cam = np.repeat(np.arange(n_cams), len(px)).astype(np.int32)
    return cam, np.tile(px, (n_cams, 1))


def _depths(n, seed):
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.3, 3.0, n)
    d[::5] = 0.0
    return d


def _compare(g, cam, pix, depth, frame, S=None):
    st = g.state()
    S = g.covariance() if S is None else S
    cov, ray = g.projection_covariance(cam, pix, depth, frame, rays=True)
    ref, rref = P.projection_covariance(S, g.models, st["intr"], st["q_ck"], st["p_ck"], cam, pix, depth, frame == "rig")
    nan = np.isnan(rref[:, 0])
    assert np.array_equal(np.isnan(ray[:, 0]), nan) and np.isnan(cov[nan]).all() and np.isnan(ray[nan]).all()
    ok = ~nan
    scale = np.maximum(np.abs(ref[ok, 0]), np.abs(ref[ok, 2]))
    e_cov = (np.abs(cov[ok] - ref[ok]).max(1) / np.where(scale > 0, scale, 1.0)).max() if ok.any() else 0.0
    e_ray = np.abs(ray[ok] - rref[ok]).max() if ok.any() else 0.0
    assert np.array_equal(cov[ok][scale == 0], np.zeros_like(cov[ok][scale == 0]))
    return e_cov, e_ray, int(nan.sum())


CASES = {
    "linear": (("linear",), False),
    "fov": (("fov",), False),
    "poly2": (("poly2",), False),
    "poly3": (("poly3",), False),
    "kb4": (("kb4",), False),
    "poly3_kb4_inertial": (("poly3", "kb4"), True),
}


@pytest.mark.parametrize("name", list(CASES))
def test_parity(name):
    models, inertial = CASES[name]
    p = synth.make_problem(models=models, n_frames=90 if inertial else 18, inertial=inertial, seed=15)
    g = _solved(p, ALL_ON if inertial else {})
    # pixels far outside the image too: every model but linear has a domain they leave
    cam, pix = _grid(g.n_cams, extra=[(-4000.0, 240.0), (320.0, 9000.0), (320.0, 240.0)])
    for frame in ("camera", "rig"):
        for depth in (None, _depths(len(cam), 1)):
            e_cov, e_ray, n_nan = _compare(g, cam, pix, depth, frame)
            print(f"{name} {frame} {'inf' if depth is None else 'depth'}: cov {e_cov:.1e}, ray {e_ray:.1e}, {n_nan} NaN")
            assert e_cov <= COV_BAR and e_ray <= RAY_BAR, (frame, e_cov, e_ray)


@pytest.mark.parametrize("name", ["fov_kb4", "kb4_poly3_inertial"])
def test_wide_lens_rig(name):
    lens = W.build(name)
    g = _solved(lens.p, lens.flags, iters=10)
    cam, pix = _grid(g.n_cams, 32, 24)
    for frame in ("camera", "rig"):
        e_cov, e_ray, n_nan = _compare(g, cam, pix, _depths(len(cam), 2), frame)
        print(f"{name} {frame}: cov {e_cov:.1e}, ray {e_ray:.1e}, {n_nan} NaN of {len(cam)}")
        assert e_cov <= COV_BAR and e_ray <= RAY_BAR


@pytest.mark.parametrize("G,inertial,kw", [(67, True, dict(n_frames=48, grid=(14, 10))),
                                           (112, False, dict(n_frames=40))], ids=["inertial_G67", "vision_G112"])
def test_large_rigs(G, inertial, kw):
    models = chain_plan.rig_with_globals(67) if inertial else ("kb4",) * 8
    p = synth.make_problem(models=models, inertial=inertial, seed=G, **kw)
    g = _solved(p, ALL_ON if inertial else {})
    assert g.G == G
    cam, pix = _grid(g.n_cams, 40, 30)  # > 256 points per camera: several tiles
    e_cov, e_ray, _ = _compare(g, cam, pix, _depths(len(cam), 3), "rig")
    print(f"G = {G}: {len(cam)} points, cov {e_cov:.1e}, ray {e_ray:.1e}")
    assert e_cov <= COV_BAR and e_ray <= RAY_BAR


def test_fixed_intrinsics_are_exact_zeros():
    p = synth.make_problem(models=("poly3", "fov"), n_frames=18, seed=15)
    g = _solved(p, dict(fix_intrinsics=1))
    cam, pix = _grid(2)
    cov = g.projection_covariance(cam, pix, _depths(len(cam), 4), "camera")
    assert np.array_equal(cov, np.zeros_like(cov))
    assert (g.projection_covariance(cam, pix, None, "rig")[:, 0] > 0).any()


def test_unseen_camera_is_exact_zeros():
    v = tv.build("unseen_camera")
    g = _solved(v.p, v.flags)
    c = v.unseen_cam
    cam, pix = _grid(g.n_cams)
    for frame in ("camera", "rig"):
        cov = g.projection_covariance(cam, pix, _depths(len(cam), 5), frame)
        assert np.array_equal(cov[cam == c], np.zeros_like(cov[cam == c]))
        assert (cov[cam != c][:, 0] > 0).all()


def test_passed_matrix_same_bits():
    p = synth.make_problem(models=("kb4", "poly2"), n_frames=18, seed=16)
    g = _solved(p, {})
    cam, pix = _grid(2)
    d = _depths(len(cam), 6)
    for frame in ("camera", "rig"):
        a, ra = g.projection_covariance(cam, pix, d, frame, rays=True)
        b, rb = g.projection_covariance(cam, pix, d, frame, cov=g.covariance(), rays=True)
        assert a.tobytes() == b.tobytes() and ra.tobytes() == rb.tobytes()


def _snapshot(g, inertial):
    W_ = g.imu_weights() if inertial else np.zeros(0)
    return {k: np.asarray(v).tobytes() for k, v in g.state().items()}, W_.tobytes()


@pytest.mark.parametrize("inertial", [False, True], ids=["vision", "inertial"])
def test_no_side_effects(inertial):
    from vicalib_b200.capi import Calibrator

    def make():
        g = Calibrator()
        g.load(synth.make_problem(models=("poly3", "kb4"), n_frames=60 if inertial else 20, inertial=inertial, seed=8))
        g.set_flags(**(ALL_ON if inertial else {}))
        g.set_options(max_iters=4)
        return g

    g, fresh = make(), make()
    g.solve()
    fresh.solve()
    before = _snapshot(g, inertial)
    cam, pix = _grid(2)
    g.projection_covariance(cam, pix, _depths(len(cam), 7), "rig", rays=True)
    g.projection_covariance(cam, pix, None, "camera", cov=np.eye(g.G))
    assert _snapshot(g, inertial) == before
    s, s0 = g.solve(free_running=True), fresh.solve(free_running=True)
    for k in ("iterations", "successful_steps", "termination", "initial_cost", "final_cost"):
        assert s[k] == s0[k], k
    assert _snapshot(g, inertial) == _snapshot(fresh, inertial)


def test_refusals():
    from vicalib_b200.capi import ProjPoints, VcgpuError, _proj_points, lib

    g = _solved(synth.make_problem(models=("poly3", "fov"), n_frames=18, seed=15), {}, iters=2)
    cam, pix = _grid(2, 4, 3)
    d = _depths(len(cam), 8)

    def refused(cam_id, depth=None, frame="camera", match=""):
        with pytest.raises(VcgpuError, match=match):
            g.projection_covariance(cam_id, pix, depth, frame)

    refused(np.where(np.arange(len(cam)) == 3, 2, cam), match="point 3: camera 2 outside")
    refused(np.where(np.arange(len(cam)) == 5, -1, cam), match="point 5: camera -1 outside")
    refused(cam, np.where(np.arange(len(cam)) == 7, -1e-3, d), match="point 7: depth")
    refused(cam, np.where(np.arange(len(cam)) == 2, np.nan, d), match="point 2: depth")
    refused(cam, np.where(np.arange(len(cam)) == 4, np.inf, d), match="point 4: depth")
    L = lib()
    keep, pts = _proj_points(cam, pix, d, "camera", False)
    for field, value, match in (("frame", 2, "unknown frame 2"), ("n", -1, "n < 0"), ("cov", None, "null cov")):
        bad = ProjPoints.from_buffer_copy(pts)
        setattr(bad, field, value)
        assert L.vcgpu_get_projection_covariance(g.h, None, C.byref(bad)) == -1
        assert match in L.vcgpu_last_error(g.h).decode()
        assert not keep[3].any()  # nothing written
    assert L.vcgpu_get_projection_covariance(g.h, None, None) == -1
    assert "null points" in L.vcgpu_last_error(g.h).decode()
    # an empty call writes nothing and succeeds
    assert g.projection_covariance(np.zeros(0, np.int32), np.zeros((0, 2))).shape == (0, 3)
