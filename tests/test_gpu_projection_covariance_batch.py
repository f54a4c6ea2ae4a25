"""GPU: vcgpu_get_projection_covariance_batch, the pixel covariance of projected points of many rigs in one call.
  parity     a mixed vision and inertial batch against each rig's single call, to the rounding of the matrices
  bits       a rig's outputs are the same bits under reordering and when the rest of the batch changes
  status     a rig whose J^T J is singular gets VCGPU_ERR_NUMERIC, the others are written
  refusals   each names its index and writes nothing"""
import numpy as np
import pytest

import target_views as tv
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
# relative to the point's largest |S_uu|, |S_vv|: the batch's matrices equal the single call's to rounding, which the
# covariance batch tests bound by 1e-6 (vision) and 1e-4 (inertial) of the standard deviations.  Measured on an H100
# 80GB HBM3 (700 W): 4.5e-12 (vision), 1.3e-9 (inertial)
BAR = {False: 1e-6, True: 1e-4}
NUMERIC = -3


def _rig(models, inertial, seed, nf=None, p=None, flags=None):
    from vicalib_b200.capi import Calibrator

    p = p or synth.make_problem(models=models, n_frames=nf or (90 if inertial else 18), inertial=inertial, seed=seed)
    g = Calibrator()
    g.load(p)
    g.set_flags(**(flags if flags is not None else (ALL_ON if inertial else {})))
    g.set_options(function_tol=1e-12, max_iters=10)
    g.solve()
    return g


def _points(g, seed, n=700, frame="rig"):
    rng = np.random.default_rng(seed)
    cam = rng.integers(0, g.n_cams, n).astype(np.int32)
    pix = np.stack([rng.uniform(-50, 690, n), rng.uniform(-50, 530, n)], 1)
    d = rng.uniform(0.3, 3.0, n)
    d[::4] = 0.0
    return dict(cam_id=cam, pix=pix, depth=d, frame=frame, rays=True)


def _err(a, b):
    ok = ~np.isnan(b[:, 0])
    assert np.array_equal(np.isnan(a[:, 0]), ~ok)
    scale = np.maximum(np.abs(b[ok, 0]), np.abs(b[ok, 2])).clip(1e-300)
    return (np.abs(a[ok] - b[ok]).max(1) / scale).max()


@pytest.fixture(scope="module")
def rigs():
    return [_rig(("poly3",), False, 21), _rig(("poly3", "poly2"), True, 22), _rig(("fov", "kb4"), False, 23),
            _rig(("kb4",), True, 24), _rig(("linear", "poly2"), False, 25)]


def test_parity_mixed_batch(rigs):
    from vicalib_b200.capi import projection_covariance_batch

    pts = [_points(g, i, frame="rig" if i % 2 else "camera") for i, g in enumerate(rigs)]
    out = projection_covariance_batch(rigs, pts)
    for i, (g, p) in enumerate(zip(rigs, pts)):
        cov, ray = g.projection_covariance(p["cam_id"], p["pix"], p["depth"], p["frame"], rays=True)
        e = _err(out[i][0], cov)
        inertial = bool(g.flags.inertial)
        print(f"rig {i} ({'inertial' if inertial else 'vision'}, {p['frame']}): batch vs single {e:.1e}, "
              f"{int(np.isnan(cov[:, 0]).sum())} NaN")
        assert e <= BAR[inertial]
        assert out[i][1].tobytes() == ray.tobytes()  # the rays depend on the state alone


def test_bits_under_reordering_and_composition(rigs):
    from vicalib_b200.capi import projection_covariance_batch

    pts = [_points(g, 10 + i) for i, g in enumerate(rigs)]
    ref = projection_covariance_batch(rigs, pts)
    for order in ([4, 3, 2, 1, 0], [2, 0, 4], [1], [3, 1]):
        out = projection_covariance_batch([rigs[i] for i in order], [pts[i] for i in order])
        for k, i in enumerate(order):
            assert out[k][0].tobytes() == ref[i][0].tobytes() and out[k][1].tobytes() == ref[i][1].tobytes(), (order, i)


def test_singular_rig_among_healthy(rigs):
    from vicalib_b200.capi import VcgpuError, projection_covariance_batch

    v = tv.build("unseen_runs")
    bad = _rig(None, False, 0, p=v.p, flags=v.flags)
    gs = [rigs[0], bad, rigs[1]]
    pts = [_points(g, 30 + i) for i, g in enumerate(gs)]
    with pytest.raises(VcgpuError, match="handle") as e:
        projection_covariance_batch(gs, pts)
    assert e.value.status == [0, NUMERIC, 0]
    assert e.value.covariances[1] is None
    ref = projection_covariance_batch([gs[0], gs[2]], [pts[0], pts[2]])
    for k, i in enumerate((0, 2)):
        assert e.value.covariances[i][0].tobytes() == ref[k][0].tobytes()


def test_refusals(rigs):
    from vicalib_b200.capi import VcgpuError, projection_covariance_batch

    def refused(pts, match, gs=None):
        gs = gs or rigs[:3]
        with pytest.raises(VcgpuError, match=match):
            projection_covariance_batch(gs, pts)

    pts = [_points(g, 40 + i, n=50) for i, g in enumerate(rigs[:3])]
    p = dict(pts[1], cam_id=np.where(np.arange(50) == 9, 7, pts[1]["cam_id"]).astype(np.int32))
    refused([pts[0], p, pts[2]], "handle 1: point 9: camera 7 outside")
    p = dict(pts[2], depth=np.where(np.arange(50) == 3, -1.0, pts[2]["depth"]))
    refused([pts[0], pts[1], p], "handle 2: point 3: depth")
    refused([pts[0], pts[0], pts[2]], "handle 1: the same handle as 0", gs=[rigs[0], rigs[0], rigs[2]])
    g = rigs[0]
    g.set_profiling(profile=4)
    try:
        refused(pts, "handle 0: .*profiling")
    finally:
        g.set_profiling(profile=0)
