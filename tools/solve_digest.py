"""What the vision solve engines compute, in a form two builds of the library can be compared by.

    python tools/solve_digest.py [workload] [out.npz]

Solves the workload (default config2) with LM and DOGLEG on the persistent kernel and on the multi-launch engine
(vcgpu_set_profiling's multi-launch bit), and 8 rigs of config 1's shape with one vcgpu_solve_batch per strategy; then
the inertial LM solve on the persistent inertial kernels: the target workload (weights held) and config3 with live
weights; then one vcgpu_solve_batch_inertial of four rigs of cluster sizes 1, 2, 4 and 8 (live weights on one), one
vcgpu_get_covariance_batch and one vcgpu_get_frame_covariance_batch of two vision rigs and those four, and
vcgpu_get_covariance and vcgpu_get_frame_covariance of one vision rig and one inertial rig of them.  Prints, per case,
the iterations, the final cost and last trust-region radius as hex floats and a SHA-256 of the final state (inertial:
with velocities, IMU parameters and the weights), per covariance its status and a SHA-256 of the matrix or blocks; with
out.npz also stores the states, costs, radii and matrices.  Equal lines mean bit-for-bit equal results.
"""
import hashlib
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vicalib_b200 import synth
from vicalib_b200.capi import (Calibrator, VcgpuError, covariance_batch, frame_covariance_batch, solve_batch,
                               solve_batch_inertial)

wl = sys.argv[1] if len(sys.argv) > 1 else "config2"
KEYS = ("intr", "q_ck", "p_ck", "T_wp")
out = {}


def report(name, g, s, radius, keys=KEYS, extra=()):
    st = g.state()
    x = np.concatenate([np.ravel(st[k]) for k in keys] + [np.ravel(e) for e in extra])
    out[name] = np.concatenate([x, [s["final_cost"], radius]])
    print(f"{name:24s} {s['iterations']:3d} it  cost {float(s['final_cost']).hex():24s} radius {float(radius).hex():24s} "
          f"state {hashlib.sha256(x.tobytes()).hexdigest()[:16]}")


p = synth.make_config(wl)
for strategy, sname in ((0, "LM"), (1, "DOGLEG")):
    for mode, mname in ((0, "persistent"), (4, "multi-launch")):
        g = Calibrator()
        g.load(p)
        g.set_options(strategy=strategy, max_iters=20, function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
        g.set_profiling(mode, False)
        s = g.solve()
        report(f"{sname} {mname}", g, s, s["rows"][-1][7])
        g.close()
    rigs = []
    for i in range(8):
        g = Calibrator()
        g.load(synth.make_problem(models=("poly3",), n_frames=50, grid=(14, 10), seed=1000 + i))
        g.set_options(strategy=strategy, max_iters=20, function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
        rigs.append(g)
    for i, (g, s) in enumerate(zip(rigs, solve_batch(rigs))):
        report(f"{sname} batch rig {i}", g, s, float("nan"))  # a batch solve reports no radius
        g.close()
IMU_KEYS = KEYS + ("v_w", "g", "b", "sf", "ts")
for wl_imu, weights in (("target", 0), ("config3", 1)):
    g = Calibrator()
    g.load(synth.make_config(wl_imu))
    g.set_flags(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
    g.set_options(max_iters=10, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, update_imu_weights=weights)
    s = g.solve()
    report(f"inertial LM {wl_imu}" + (" live weights" if weights else ""), g, s, s["rows"][-1][7], IMU_KEYS,
           (g.imu_weights(),) if weights else ())
    g.close()
imu_rigs = []
for i, n_frames in enumerate((12, 24, 50, 90)):  # cluster sizes 1, 2, 4, 8
    g = Calibrator()
    g.load(synth.make_problem(models=("poly3",), n_frames=n_frames, grid=(10, 7), inertial=True, seed=1100 + i))
    g.set_flags(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
    g.set_options(max_iters=8, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, update_imu_weights=int(i == 2))
    imu_rigs.append(g)
for i, (g, s) in enumerate(zip(imu_rigs, solve_batch_inertial(imu_rigs))):
    report(f"inertial batch rig {i}" + (" live weights" if i == 2 else ""), g, s, float("nan"), IMU_KEYS,
           (g.imu_weights(),) if i == 2 else ())
vis_rigs = []
for i, models in enumerate((("poly3",), ("fov", "kb4"))):
    g = Calibrator()
    g.load(synth.make_problem(models=models, n_frames=20 + 20 * i, grid=(10, 7), seed=1200 + i))
    vis_rigs.append(g)
cov_rigs = [vis_rigs[0], imu_rigs[0], imu_rigs[3], vis_rigs[1], imu_rigs[1], imu_rigs[2]]


def report_cov(name, c, st):
    if c is not None:
        out[name] = c
    print(f"{name:24s} status {st:2d}  cov {hashlib.sha256(c.tobytes()).hexdigest()[:16] if c is not None else '-'}")


for what, batch in (("covariance", covariance_batch), ("frame covariance", frame_covariance_batch)):
    try:
        covs, status = batch(cov_rigs), [0] * len(cov_rigs)
    except VcgpuError as e:
        if getattr(e, "status", None) is None:
            raise
        covs, status = e.covariances, e.status
    for i, (c, st) in enumerate(zip(covs, status)):
        report_cov(f"{what} batch rig {i}", c, st)
for i in (0, 4):  # a vision rig and an inertial one
    for what, call in (("covariance", Calibrator.covariance), ("frame covariance", Calibrator.frame_covariance)):
        try:
            c, st = call(cov_rigs[i]), 0
        except VcgpuError as e:
            c, st = None, int(str(e).split()[2].rstrip(":"))
        report_cov(f"{what} rig {i}", c, st)
for g in imu_rigs + vis_rigs:
    g.close()
if len(sys.argv) > 2:
    np.savez(sys.argv[2], **out)
