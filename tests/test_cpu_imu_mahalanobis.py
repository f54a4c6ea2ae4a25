"""CPU: each IMU interval's Mahalanobis distance as UpdateImuWeights logs it (vicalibrator.h:786-794),
  dist = r^T (Jt C Jt^T)^-1 r,  r = [SE3::log(T_end * T_2w); v_end - v_w[k+1]],
the oracle's (UpdateOneImuWeight's `mahalanobis`) against the reference's own `dist` (oracle/_ref's ref_update_weight), on
a base problem, the IMU streams of imu_streams.py, the vigorous rigs of imu_motion.py with negated quaternions, and at
Unix time (imu_epoch.restamp); then a numpy model of the device formula, sum_k (V[:,k] . r)^2 / lambda_k from the
eigen-decomposition of sym(P), against r^T inv(P) r on those intervals' P.

Single-step intervals (no interior sample) are not compared: their P has rank <= 6, so the distance is decided by
rounding, in the reference too (test_cpu_imu_streams.py's note on W).  NaN in both marks an interval with no
measurements, which the reference skips."""
import dataclasses

import numpy as np
import pytest

import imu_epoch
import imu_mahalanobis_ref as M
import imu_motion
import imu_streams
from vicalib_b200 import synth

# oracle vs ref_update_weight, relative to the reference's dist: largest measured 5.7e-13 (imu_motion imu1000); the bar
# leaves a factor of about 17
REF_BAR = 1e-11
# ... at the true state, where r is ~1e-4 of the poses it is the difference of and d is of order ten: largest measured
# 7.2e-10; the bar leaves a factor of about 14
TRUTH_BAR = 1e-8


def _base():
    p = synth.make_problem(models=("poly3",), n_frames=12, grid=(14, 10), inertial=True, seed=77, ts_truth=0.003)
    return imu_streams.perturbed(p)


def _truth(p):
    """p at its true state: distances of order ten, where a perturbed state gives 1e8 .. 1e10"""
    return dataclasses.replace(p, **{k: np.array(v, copy=True) if np.ndim(v) else v for k, v in p.truth.items()})


def _cases():
    out = [("base", _base()), ("base_truth", _truth(_base()))]
    out += [(f"stream_{n}", imu_streams.perturbed(imu_streams.build(n).p)) for n in imu_streams.NAMES]
    for n in imu_motion.NAMES:
        m = imu_motion.build(n)
        out.append((f"motion_{n}", m.p))
        out.append((f"motion_{n}_flipped", imu_motion.flipped(m.p, frames=imu_motion.scattered(m.p.n_frames))))
    out += [(f"epoch_{n}", imu_epoch.realistic(n).p) for n in ("jittered", "dropped", "samples2", "imu1000")]
    return out


CASES = dict(_cases())


def _comparable(p):
    c = imu_streams.classify(p)
    return c["covered"] & (c["steps"] >= 2), c["covered"]


@pytest.fixture(scope="module")
def ref():
    L = M.ref_lib()
    if L is None:
        pytest.skip("oracle/_ref is built only where the reference tree exists")
    return L


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_ref(ref, name):
    p = CASES[name]
    d_o, d_r = M.oracle_dist(p), M.ref_dist(ref, p)
    cmp, covered = _comparable(p)
    assert np.isnan(d_r[~covered]).all(), name  # the reference logs nothing where nothing is measured
    assert np.array_equal(np.isnan(d_o), np.isnan(d_r)), name  # and NaN from a one-sample interval's zero P
    if cmp.any():
        rel = np.abs(d_o[cmp] - d_r[cmp]) / np.abs(d_r[cmp])
        assert rel.max() <= (TRUTH_BAR if name.endswith("_truth") else REF_BAR), (name, rel.max())


def test_negated_quaternions_leave_the_distance():
    """The double cover: negating frame quaternions describes the same rig, and the distance stays to rounding"""
    for n in imu_motion.NAMES:
        p = imu_motion.build(n).p
        d0 = M.oracle_dist(p)
        d1 = M.oracle_dist(imu_motion.flipped(p, frames=imu_motion.scattered(p.n_frames)))
        assert np.abs(d1 - d0).max() <= 1e-7 * np.abs(d0).max(), n


# the eigen form against the explicit inverse and the oracle, relative: largest measured 8.9e-11 (stream imu20, cond(P)
# up to 4.3e5; the other cases 1e-12 .. 2e-11 at cond(P) 1.4e3 .. 6.7e4); the bar leaves a factor of about 11
EIG_BAR = 1e-9


@pytest.mark.parametrize("name", list(CASES))
def test_eigen_form_matches_inverse(name):
    """sum (V^T r)^2 / lambda (eigh of sym P) against r^T inv(P) r and against the oracle's LU-inverse distance; prints
    the conditioning the intervals have"""
    p = CASES[name]
    cmp, _covered = _comparable(p)
    d_o = M.oracle_dist(p)
    worst, conds = 0.0, []
    for k in np.flatnonzero(cmp):
        P, r, m = M.oracle_interval(p, k)
        assert m >= 3
        d_eig = M.eig_dist(P, r)
        d_inv = float(r @ np.linalg.solve(P, r))
        conds.append(np.linalg.cond(P))
        worst = max(worst, abs(d_eig - d_inv) / abs(d_inv), abs(d_eig - d_o[k]) / abs(d_o[k]))
    if conds:
        print(f"{name}: cond(P) {min(conds):.2e} .. {max(conds):.2e}, eigen vs inverse {worst:.2e}")
    assert worst <= EIG_BAR, (name, worst)


def test_eigen_form_is_nan_where_p_is_not_positive_definite():
    P = np.diag([1.0, 2, 3, 4, 5, 6, 7, 8, 0.0])
    assert np.isnan(M.eig_dist(P, np.ones(9)))
    assert M.eig_dist(np.diag(np.arange(1.0, 10.0)), np.ones(9)) == pytest.approx(np.sum(1.0 / np.arange(1.0, 10.0)))
