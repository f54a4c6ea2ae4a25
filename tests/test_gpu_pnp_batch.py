"""GPU: vcgpu_pose_pnp_ransac_batch (pose_pnp_batch_kernel, one warp per view of every rig) against
vcgpu_pose_pnp_ransac on the same handle and views, which is a batch of one: what the comparisons check is the packing
of many rigs and the seeding (test_gpu_pnp.py checks the poses against the oracle).  T_cw, rmse and n_used must be the
same bits, whatever else is in the batch and in whatever order: the batch seeds a view's RANSAC draws with its index
within its rig.  Not covered:
handles on different devices (that needs more than one GPU); its refusal is an argument check next to the ones tested
here.
"""
import ctypes as C

import numpy as np
import pytest

import target_views as tv
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

RANSAC = dict(robust_its=40, robust_tol=3.0 / 300)


def _groups(p):
    """(cam, start, count) of every (camera, frame) group; observations are sorted by (camera, frame)"""
    key = p.obs_cam.astype(np.int64) * p.n_frames + p.obs_frame
    start = np.flatnonzero(np.r_[True, key[1:] != key[:-1]])
    count = np.diff(np.r_[start, len(key)])
    return p.obs_cam[start].astype(np.int32), start.astype(np.int64), count.astype(np.int32)


def _rig(p, pix=None):
    """a handle with p's cameras at their true intrinsics, and every (camera, frame) view of p"""
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.set_cameras(p.models, p.truth["intr"], p.q_ck, p.p_ck)
    cam, start, count = _groups(p)
    return g, (cam, start, count, p.p_c if pix is None else pix, p.p_w)


def _bits(out):
    return tuple(np.ascontiguousarray(a).tobytes() for a in out)


def _check(entries, **kw):
    """the batch, against each rig's own call on the same handle"""
    from vicalib_b200.capi import pose_pnp_batch

    got = pose_pnp_batch(entries, **kw)
    assert len(got) == len(entries)
    for k, ((g, views), out) in enumerate(zip(entries, got)):
        assert _bits(out) == _bits(g.pose_pnp_ransac(*views, **kw)), k
    return got


def _mixed_rigs():
    """A dozen rigs: all five models, 1 to 4 cameras per rig; views of 4, 5, 32, 33 and 600 corners, cropped views and
    views of 1-3 corners (identity pose, n_used 0), an empty view (count 0); and a rig with no views."""
    problems = [synth.make_problem(models=m, n_frames=6 + k, seed=300 + k, pixel_sigma=0.05)
                for k, m in enumerate((("linear",), ("fov",), ("poly2", "kb4"), ("poly3", "fov", "kb4"),
                                       ("kb4", "poly2", "linear", "fov"), ("linear", "poly3")))]
    problems += [tv.build(name).p for name in ("counts", "cropped", "one_camera4")]
    problems += [synth.make_problem(models=m, n_frames=f, seed=s) for m, f, s in
                 ((("poly3", "poly2"), 8, 310), (("fov",), 3, 311), (("kb4", "poly3", "fov"), 5, 312))]
    assert {int(m) for p in problems for m in p.models} == set(range(5))
    assert sorted({p.n_cams for p in problems}) == [1, 2, 3, 4]
    rigs = [_rig(p) for p in problems]
    cam, start, count, pix, pw = rigs[9][1]
    count = count.copy()
    count[[2, 5, 9]] = (3, 0, 1)
    rigs[9] = (rigs[9][0], (cam, start, count, pix, pw))
    rigs[10] = (rigs[10][0], tuple(a[:0] for a in rigs[10][1][:3]) + rigs[10][1][3:])
    return rigs


# ------------------------------------------------------------------ 1. the same bits as the single call
def test_same_bits_as_single_call():
    rigs = _mixed_rigs()
    counts = np.concatenate([v[2] for _, v in rigs])
    assert {0, 1, 2, 3, 4, 5, 32, 33, 600} <= set(counts.tolist()) and len(rigs) == 12
    assert len(rigs[10][1][0]) == 0
    got = _check(rigs)
    used = np.concatenate([u for _, _, u in got])
    T = np.concatenate([t for t, _, _ in got])
    assert np.all(used[counts < 4] == 0) and np.all(T[counts < 4] == [0, 0, 0, 1, 0, 0, 0])
    assert np.array_equal(used[counts >= 4], counts[counts >= 4])
    rev = _check(rigs[::-1])
    for a, b in zip(got, rev[::-1]):
        assert _bits(a) == _bits(b)
    sub = _check(rigs[1::3])
    for a, b in zip(got[1::3], sub):
        assert _bits(a) == _bits(b)


# ------------------------------------------------------------------ 2. RANSAC
def _outlier_rig(models, seed, every, shift=25.0, n_frames=6):
    p = synth.make_problem(models=models, n_frames=n_frames, seed=seed, pixel_sigma=0.05)
    pix = p.p_c.copy()
    pix[::every] += shift  # wrong associations
    return _rig(p, pix), p


def test_ransac_same_bits_and_oracle():
    """Gross outliers, RANSAC on: every rig the bits of its own call.  With few draws and many outliers a view's result
    depends on its draws (checked: shifting the views' indices by one changes some result), so a batch that seeded by
    the view's place in the batch would fail here.  The fourth rig also matches oracle/pnp.py called with view = its
    rig-local index (40 draws, 1 in 9 corners off)."""
    from oracle import pnp

    few = dict(robust_its=3, robust_tol=3.0 / 300)
    rigs = [_outlier_rig(m, 400 + k, 3)[0] for k, m in enumerate((("poly3",), ("kb4", "fov"), ("poly2", "linear", "poly3")))]
    g, (cam, start, count, pix, pw) = rigs[1]
    shifted = g.pose_pnp_ransac(np.r_[0, cam], np.r_[0, start], np.r_[0, count], pix, pw, **few)
    base = g.pose_pnp_ransac(cam, start, count, pix, pw, **few)
    assert _bits([a[1:] for a in shifted]) != _bits(base)
    _check(rigs, **few)
    _check(rigs[::-1], **few)

    (og, oviews), op = _outlier_rig(("poly3", "kb4"), 420, 9)
    entries = [_outlier_rig(("fov",), 421, 9)[0], _outlier_rig(("poly3",), 422, 9)[0], rigs[0], (og, oviews)]
    got = _check(entries, **RANSAC)
    T, rmse, used = got[3]
    cam, start, count, pix, pw = oviews
    for v in range(len(cam)):
        sl = slice(start[v], start[v] + count[v])
        To, ro, no = pnp.pnp_planar(int(op.models[cam[v]]), op.truth["intr"][cam[v]], pix[sl], pw[sl], view=v, **RANSAC)
        assert used[v] == no and used[v] < count[v], v
        assert np.abs(T[v] - To).max() <= 1e-8, (v, np.abs(T[v] - To).max())
        assert abs(rmse[v] - ro) <= 1e-10, v


# ------------------------------------------------------------------ 3. the workspace held by handle 0
def test_workspace_reuse():
    small = [_rig(synth.make_problem(models=("poly3",), n_frames=3, seed=500))]
    small.append(_rig(synth.make_problem(models=("kb4", "fov"), n_frames=2, seed=501)))
    large = small + [_rig(tv.build("counts").p), _rig(tv.build("cropped").p)]
    large += [_rig(synth.make_problem(models=("poly2", "poly3"), n_frames=40, seed=502 + k)) for k in range(4)]
    for kw in ({}, RANSAC):
        first = _check(small, **kw)
        _check(large, **kw)
        again = _check(small, **kw)
        for a, b in zip(first, again):
            assert _bits(a) == _bits(b)


# ------------------------------------------------------------------ 4. refusals
SENTINEL = (7.25, -3.5, -7)


class _Raw:
    """one rig's vcgpu_pnp_views with outputs pre-filled with a sentinel; any field may be overridden (None: NULL)"""

    def __init__(self, views, **over):
        from vicalib_b200.capi import PnpViews

        cam, start, count, pix, pw = views
        self.ins = dict(cam_id=np.array(cam, np.int32), start=np.array(start, np.int64), count=np.array(count, np.int32),
                        pix=np.ascontiguousarray(pix, np.float64), pw=np.ascontiguousarray(pw, np.float64))
        m = max(len(cam), 1)
        self.outs = dict(T_cw=np.full((m, 7), SENTINEL[0]), rmse_or_null=np.full(m, SENTINEL[1]),
                         n_used_or_null=np.full(m, SENTINEL[2], np.int32))
        ptr = {k: a.ctypes.data for k, a in {**self.ins, **self.outs}.items()}
        n_views = over.pop("n_views", len(cam))
        ptr.update(over)
        self.s = PnpViews(n_views, *[ptr[f] for f, _ in PnpViews._fields_[1:]])

    def untouched(self):
        return all(np.all(self.outs[k] == s) for k, s in zip(("T_cw", "rmse_or_null", "n_used_or_null"), SENTINEL))


def _call(handles, raws, n=None, views=True, **kw):
    from vicalib_b200.capi import PnpViews, lib

    n = len(handles) if n is None else n
    hs = (C.c_void_p * max(len(handles), 1))(*[None if g is None else g.h for g in handles])
    arr = (PnpViews * max(len(raws), 1))(*[r.s for r in raws]) if views else None
    kw = {**dict(robust_its=0, robust_tol=0.0), **kw}
    return lib().vcgpu_pose_pnp_ransac_batch(hs, C.c_int(n), arr, C.c_int(kw["robust_its"]), C.c_double(kw["robust_tol"]))


def _err(g):
    return g.L.vcgpu_last_error(g.h).decode()


def test_refusals():
    from vicalib_b200.capi import Calibrator

    rigs = [_rig(synth.make_problem(models=m, n_frames=4, seed=600 + k)) for k, m in enumerate((("poly3",), ("fov", "kb4"), ("linear",)))]
    hs = [g for g, _ in rigs]

    def refused(handles, raws, expect, **kw):
        rc = _call(handles, raws, **kw)
        assert rc == -1, (expect, rc)
        for r in raws:
            assert r.untouched(), expect
        live = [g for g in handles if g is not None]
        for g in live:
            msg = _err(g)
            assert msg.startswith("vcgpu_pose_pnp_ransac_batch: "), msg
            for part in expect:
                assert part in msg, (part, msg)

    good = lambda: [_Raw(v) for _, v in rigs]  # noqa: E731
    # n <= 0: refused with nothing to name
    for n in (0, -1):
        raws = good()
        assert _call(hs, raws, n=n) == -1 and all(r.untouched() for r in raws)
    refused(hs, good(), ("handle 0", "null views array"), views=False)
    refused([hs[0], None, hs[2]], good(), ("handle 1", "null handle"))
    refused([hs[0], hs[1], hs[0]], good(), ("handle 2", "the same handle as 0"))
    bare = Calibrator()
    refused([hs[0], bare, hs[2]], good(), ("handle 1", "cameras must be set first"))
    # a view vcgpu_pose_pnp_ransac refuses: the rig and the view are named
    for field, value in (("cam_id", 2), ("cam_id", -1), ("start", -1), ("count", -1)):
        raws = good()
        raws[1].ins[field][5] = value
        refused(hs, raws, ("handle 1", "view 5", "bad view description"))
    for k in ("cam_id", "start", "count", "pix", "pw"):
        raws = good()
        raws[2] = _Raw(rigs[2][1], **{k: None})
        refused(hs, raws, ("handle 2", "null view array"))
    raws = good()
    raws[1] = _Raw(rigs[1][1], T_cw=None)
    refused(hs, raws, ("handle 1", "null T_cw"))
    raws = good()
    raws[0] = _Raw(rigs[0][1], n_views=-1)
    refused(hs, raws, ("handle 0", "n_views < 0"))
    # a rig without views may have null arrays and gets nothing written; the batch still runs
    raws = good()
    raws[1] = _Raw(rigs[1][1], n_views=0, cam_id=None, start=None, count=None, pix=None, pw=None, T_cw=None)
    assert _call(hs, raws) == 0
    assert raws[1].untouched()
    for i in (0, 2):
        T, rmse, used = rigs[i][0].pose_pnp_ransac(*rigs[i][1])
        assert _bits((raws[i].outs["T_cw"], raws[i].outs["rmse_or_null"], raws[i].outs["n_used_or_null"])) == _bits((T, rmse, used))
    # and a valid batch after all of these
    _check(rigs)
    _check(rigs, **RANSAC)
