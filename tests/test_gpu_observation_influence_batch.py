"""GPU: vcgpu_get_observation_influence_batch (Sigma_gg, Sigma_ff and Sigma_fg from one elimination per rig by the
covariance cluster kernels' diagonal-and-cross mode): a mixed vision and inertial batch against the single calls, the
same bits under reordering and in sub-batches, refusals naming the index (a rig with no active observation, inertial
G = 68, which the cluster kernels do not fit), a singular rig's status."""
import numpy as np
import pytest

import chain_plan
from test_gpu_frame_covariance import ALL_ON, NUMERIC, _solved
from vicalib_b200 import capi, synth

pytestmark = pytest.mark.gpu
# the batch's covariance blocks come from the cluster kernels, the single call's from the per-handle path: equal to
# rounding, as the covariance batches are
BAR = {False: 1e-7, True: 1e-4}


def _rigs():
    out = []
    for k, (models, inertial, flags) in enumerate([(("poly3",), False, {}), (("kb4", "fov"), True, dict(ALL_ON)),
                                                    (("poly2", "linear"), False, dict(visual_mult=2.0))]):
        p = synth.make_problem(models=models, n_frames=40 if inertial else 16, inertial=inertial, seed=50 + k)
        g, _ = _solved(p, flags, max_iters=6)
        out.append((g, inertial))
    return out


def _rel(a, b):
    ok = np.isfinite(b)
    return (np.abs(a[ok] - b[ok]) / np.maximum(np.abs(b[ok]), 1e-12)).max(initial=0.0)


def test_batch_matches_single_and_is_order_free():
    rigs = _rigs()
    gs = [g for g, _ in rigs]
    single = [g.observation_influence() for g in gs]
    batch = capi.observation_influence_batch(gs)
    for (g, inertial), s, b in zip(rigs, single, batch):
        for k in s:
            assert np.array_equal(np.isnan(s[k]), np.isnan(b[k]))
        e = max(np.nanmax(np.abs(s["h"] - b["h"])), _rel(b["stud"], s["stud"]), _rel(b["infl"], s["infl"]))
        print(f"\nbatch vs single: {e:.1e}")
        assert e <= BAR[inertial], e
    rev = capi.observation_influence_batch(gs[::-1])[::-1]
    sub = [capi.observation_influence_batch([g])[0] for g in gs]
    for b, r, s in zip(batch, rev, sub):
        assert all(b[k].tobytes() == r[k].tobytes() == s[k].tobytes() for k in b)


def test_refusals_and_status():
    p = synth.make_problem(models=("poly3",), n_frames=16, seed=60)
    g, _ = _solved(p, {}, max_iters=4)
    empty = capi.Calibrator()
    empty.load(p)
    empty.remove_outliers(np.array([1e-12]), 1.0)  # no active observation left
    with pytest.raises(capi.VcgpuError, match="handle 1"):
        capi.observation_influence_batch([g, empty])
    sing = capi.Calibrator()
    sing.load(p)
    sing.set_flags(visual_mult=0.0)
    with pytest.raises(capi.VcgpuError) as e:
        capi.observation_influence_batch([g, sing])
    assert e.value.status == [0, NUMERIC] and e.value.results[1] is None
    ok = e.value.results[0]
    ref = capi.observation_influence_batch([g])[0]
    assert all(ok[k].tobytes() == ref[k].tobytes() for k in ok)


def test_batch_refuses_g68():
    """inertial G = 68 goes through the single call only: the batch refuses it by index, as the frame cross-covariance
    batch does, and writes nothing"""
    p = synth.make_problem(models=chain_plan.rig_with_globals(68), n_frames=40, grid=(8, 6), inertial=True, seed=68)
    big, _ = _solved(p, dict(ALL_ON), max_iters=2)
    assert big.G == 68
    q = synth.make_problem(models=("poly3",), n_frames=16, seed=61)
    g, _ = _solved(q, {}, max_iters=2)
    with pytest.raises(capi.VcgpuError, match="handle 1") as e:
        capi.observation_influence_batch([g, big])
    assert "observation_influence_batch" in str(e.value)
    with pytest.raises(capi.VcgpuError, match="handle 1"):
        capi.frame_cross_covariance_batch([g, big])
    assert np.isfinite(big.observation_influence(stud=False, infl=False)["h"]).all()
