"""IMU Mahalanobis distances of many rigs: one vcgpu_get_imu_mahalanobis_batch call against vcgpu_get_imu_mahalanobis
called per handle.

    python tools/imu_mahalanobis_probe.py [n_frames]

Prints the card, its power limit and SM clocks, then, on 1 x poly3 + IMU rigs (n_frames frames, default 100, 200 Hz IMU,
8 x 6 corners per frame, every IMU flag on, distinct seeds) for n = 1, 8, 64 handles: the wall time per rig of n
per-handle calls and of one batch call (one timed run each, after one warm-up run of both); the device time per rig of
each arm and of the imu_mahalanobis_kernel launches alone, from one torch.profiler run of its own; and whether the two
arms' outputs are the same bits.  Reads device settings, changes none.
"""
import os
import subprocess
import sys
import time

import numpy as np
import torch  # noqa: F401  (before libvcgpu.so: torch's CUDA library needs its own NCCL symbols first)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vicalib_b200 import synth
from vicalib_b200.capi import Calibrator, imu_mahalanobis_batch

NF = int(sys.argv[1]) if len(sys.argv) > 1 else 100
NS = (1, 8, 64)
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
try:  # read-only query: a number is only meaningful next to the card, its power limit and clocks
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown (nvidia-smi not available)"
print(f"card (name, power limit, SM clock now, SM clock max): {card}\n{NF} frames per rig, one timed run per arm")


def per_handle(rigs):
    return [g.imu_mahalanobis(residuals=True) for g in rigs]


def device_us(fn, names=None):
    """summed device time (us) of the kernels fn launches (names: only those whose name contains one of them)"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    total = 0.0
    for e in prof.key_averages():
        if names is None or any(k in e.key for k in names):
            total += getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0)
    return total


rigs = []
for i in range(max(NS)):
    g = Calibrator()
    g.load(synth.make_problem(models=("poly3",), n_frames=NF, grid=(8, 6), inertial=True, seed=2000 + i))
    g.set_flags(**ALL_ON)
    rigs.append(g)
print(f"{'n':>4s} | {'per-handle us/rig':>17s} {'dev us/rig':>10s} | {'batch us/rig':>12s} {'dev us/rig':>10s} {'kernel us/rig':>13s} | wall x | same bits")
for n in NS:
    sub = rigs[:n]
    wall = {}
    for run in range(2):  # run 0 warms both arms up
        for arm, fn in (("seq", lambda: per_handle(sub)), ("batch", lambda: imu_mahalanobis_batch(sub, residuals=True))):
            t0 = time.perf_counter()
            fn()
            wall[arm] = time.perf_counter() - t0
    same = all(a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
               for a, b in zip(imu_mahalanobis_batch(sub, residuals=True), per_handle(sub)))
    d_seq = device_us(lambda: per_handle(sub)) / n
    d_batch = device_us(lambda: imu_mahalanobis_batch(sub, residuals=True)) / n
    d_kernel = device_us(lambda: imu_mahalanobis_batch(sub, residuals=True), ("imu_mahalanobis_kernel",)) / n
    print(f"{n:4d} | {1e6 * wall['seq'] / n:17.1f} {d_seq:10.1f} | {1e6 * wall['batch'] / n:12.1f} {d_batch:10.1f} "
          f"{d_kernel:13.1f} | {wall['seq'] / wall['batch']:6.2f} | {same}", flush=True)
d = imu_mahalanobis_batch(rigs[:8])
print(f"median distance over 8 rigs at their start state: {np.median(np.concatenate(d)):.3g}")
for g in rigs:
    g.close()
