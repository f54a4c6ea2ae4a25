"""Pose seeding of many rigs: one vcgpu_pose_pnp_ransac_batch call against vcgpu_pose_pnp_ransac per handle.

    python tools/pnp_batch_probe.py [max_n]

Prints the card, its power limit and SM clocks, then for n = 1, 8, 64 rigs (up to max_n) of 2 x poly3 cameras, 200
frames and 140 corners per view (400 views, 56 000 correspondences per rig): wall time per rig of n
vcgpu_pose_pnp_ransac calls (one per handle) against one vcgpu_pose_pnp_ransac_batch, best of three alternating runs
after a warm-up, without RANSAC (the reference's 0, 0) and with 40 draws on views whose every ninth corner is 25 px off;
beside each, the device time per rig of the arm's kernels and copies (torch.profiler, a run of its own).  The last
column says whether both arms returned the same bits.  Reads device settings, changes none.
"""
import os
import subprocess
import sys
import time

import torch  # noqa: F401  (before libvcgpu.so: torch's CUDA library needs its own NCCL symbols first)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from vicalib_b200 import synth
from vicalib_b200.capi import Calibrator, pose_pnp_batch

RUNS = 3
NS = [n for n in (1, 8, 64) if n <= (int(sys.argv[1]) if len(sys.argv) > 1 else 64)]
try:  # read-only query: a number is only meaningful next to the card, its power limit and clocks
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown (nvidia-smi not available)"
print(f"card (name, power limit, SM clock now, SM clock max): {card}\nbest of {RUNS} alternating runs after a warm-up")


def rig(seed, outliers):
    p = synth.make_problem(models=("poly3", "poly3"), n_frames=200, grid=(14, 10), seed=seed, pixel_sigma=0.05)
    g = Calibrator()
    g.set_cameras(p.models, p.truth["intr"], p.q_ck, p.p_ck)
    key = p.obs_cam.astype(np.int64) * p.n_frames + p.obs_frame
    start = np.flatnonzero(np.r_[True, key[1:] != key[:-1]])
    count = np.diff(np.r_[start, len(key)])
    pix = p.p_c.copy()
    if outliers:
        pix[::9] += 25.0
    return g, (p.obs_cam[start].astype(np.int32), start.astype(np.int64), count.astype(np.int32), pix, p.p_w)


def device_us(fn):
    """summed device time (us) of the kernels and copies fn issues"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0) for e in prof.key_averages())


def bits(outs):
    return [tuple(a.tobytes() for a in o) for o in outs]


print(f"{'case':>8s} {'n':>4s} {'views':>6s} | {'per handle':>10s} {'dev':>8s} | {'batch':>10s} {'dev':>8s} | {'wall x':>6s} | same bits   (us per rig)")
for name, kw in (("plain", {}), ("ransac", dict(robust_its=40, robust_tol=3.0 / 300))):
    rigs = [rig(2000 + i, bool(kw)) for i in range(max(NS))]
    for n in NS:
        sub = rigs[:n]
        arms = {"seq": lambda: [g.pose_pnp_ransac(*v, **kw) for g, v in sub], "batch": lambda: pose_pnp_batch(sub, **kw)}
        best = {k: 1e9 for k in arms}
        out = {}
        for run in range(RUNS + 1):  # run 0 warms both arms up
            for arm, fn in arms.items():
                t0 = time.perf_counter()
                out[arm] = fn()
                wall = time.perf_counter() - t0
                if run > 0:
                    best[arm] = min(best[arm], wall)
        us = {k: 1e6 * v / n for k, v in best.items()}
        dev = {k: device_us(fn) / n for k, fn in arms.items()}
        same = bits(out["seq"]) == bits(out["batch"])
        print(f"{name:>8s} {n:4d} {len(sub[0][1][0]):6d} | {us['seq']:10.1f} {dev['seq']:8.1f} | {us['batch']:10.1f} {dev['batch']:8.1f} "
              f"| {best['seq'] / best['batch']:6.2f} | {same}", flush=True)
    for g, _ in rigs:
        g.close()
