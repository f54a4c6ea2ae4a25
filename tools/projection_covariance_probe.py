"""Pixel covariance of a 640 x 480 grid on every camera (vcgpu_get_projection_covariance(_batch)) on the target workload
and on a batch of rigs.

    python tools/projection_covariance_probe.py [n_rigs]

Prints the card, its power limit and SM clocks, then on the target workload (2 x poly3 + IMU, 2000 frames, at its start
state): the wall time of Calibrator.projection_covariance() over every pixel of a 640 x 480 grid of each camera, rig
frame, half the points at a finite depth, with the matrix computed inside the call and with covariance()'s matrix
passed in; of capi.projection_covariance_batch() on n_rigs (default 8) vision rigs (2 x poly3, 200 frames), per rig;
each the best of five runs after a warm-up; and the device time of proj_cov_kernel alone (torch.profiler, a run of its
own) with its rate in points per second.  Reads device settings, changes none.
"""
import os
import subprocess
import sys
import time

import numpy as np
import torch  # noqa: F401  (before libvcgpu.so: torch's CUDA library needs its own NCCL symbols first)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vicalib_b200 import synth  # noqa: E402
from vicalib_b200.capi import Calibrator, projection_covariance_batch  # noqa: E402

NR = int(sys.argv[1]) if len(sys.argv) > 1 else 8
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
try:  # read-only query: a number is only meaningful next to the card, its power limit and clocks
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown (nvidia-smi not available)"
print(f"card (name, power limit, SM clock now, SM clock max): {card}")


def best(fn, reps=5):
    fn()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.append(time.perf_counter() - t0)
    return min(out)


def kernel_us(fn, name="proj_cov_kernel"):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0)
               for e in prof.key_averages() if name in e.key)


def grid(n_cams):
    u, v = np.meshgrid(np.arange(640.0), np.arange(480.0))
    px = np.stack([u.ravel(), v.ravel()], 1)
    cam = np.repeat(np.arange(n_cams), len(px)).astype(np.int32)
    d = np.where(np.arange(len(cam)) % 2 == 0, 0.0, 1.5)
    return cam, np.tile(px, (n_cams, 1)), d


p = synth.make_config("target")
g = Calibrator()
g.load(p)
g.set_flags(**ALL_ON)
cam, pix, d = grid(g.n_cams)
S = g.covariance()
cov = g.projection_covariance(cam, pix, d, "rig")
print(f"target: {p.n_frames} frames, G = {g.G}, {len(cam)} points ({g.n_cams} cameras x 640 x 480), "
      f"{int(np.isnan(cov[:, 0]).sum())} NaN, sqrt(S_uu) median {np.nanmedian(np.sqrt(cov[:, 0])):.3e} px (unit variance)")
t_own = best(lambda: g.projection_covariance(cam, pix, d, "rig"))
t_given = best(lambda: g.projection_covariance(cam, pix, d, "rig", cov=S))
k_us = kernel_us(lambda: g.projection_covariance(cam, pix, d, "rig", cov=S))
print(f"wall, best of 5: matrix computed in the call {1e3 * t_own:.3f} ms | matrix passed in {1e3 * t_given:.3f} ms")
print(f"proj_cov_kernel: {k_us:.1f} us, {len(cam) / (k_us * 1e-6) / 1e9:.2f} G points/s")

rigs, pts = [], []
for i in range(NR):
    q = synth.make_problem(models=("poly3", "poly3"), n_frames=200, seed=100 + i)
    h = Calibrator()
    h.load(q)
    rigs.append(h)
    c, x, dd = grid(h.n_cams)
    pts.append(dict(cam_id=c, pix=x, depth=dd, frame="rig"))
projection_covariance_batch(rigs, pts)
t_batch = best(lambda: projection_covariance_batch(rigs, pts)) / NR
k_b = kernel_us(lambda: projection_covariance_batch(rigs, pts))
n_pts = sum(len(x["cam_id"]) for x in pts)
print(f"batch of {NR} vision rigs (2 x poly3, 200 frames): wall per rig {1e3 * t_batch:.3f} ms; "
      f"proj_cov_kernel {k_b:.1f} us for {n_pts} points, {n_pts / (k_b * 1e-6) / 1e9:.2f} G points/s")
for h in rigs + [g]:
    h.close()
