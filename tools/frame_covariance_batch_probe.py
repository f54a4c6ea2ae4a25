"""Frame covariance of many rigs: one vcgpu_get_frame_covariance_batch call against vcgpu_get_frame_covariance called
per handle.

    python tools/frame_covariance_batch_probe.py [max_n]

Prints the card, its power limit and SM clocks, then, on covariance_batch_probe.py's rigs (50-frame 1 x poly3 vision
rigs and 100- and 400-frame 1 x poly3 + IMU rigs, 8 x 6 corners per frame, every IMU flag on), for n = 1, 8, 33, 132 (up
to max_n) handles with distinct seeds, solved first (K LM iterations): the wall time per rig of n per-handle calls and of
one batch call, best of three alternating runs after a warm-up; the device time per rig of each arm and of the batch's
frame covariance launches alone, from one torch.profiler run of its own; and the largest difference between the two
arms' blocks, relative to the standard deviations.
Reads device settings, changes none.
"""
import os
import subprocess
import sys
import time

import numpy as np
import torch  # noqa: F401  (before libvcgpu.so: torch's CUDA library needs its own NCCL symbols first)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vicalib_b200 import synth
from vicalib_b200.capi import Calibrator, frame_covariance_batch, solve_batch, solve_batch_inertial

K, RUNS = 10, 3
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
OPTS = dict(max_iters=K, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, update_imu_weights=0)
NS = [n for n in (1, 8, 33, 132) if n <= (int(sys.argv[1]) if len(sys.argv) > 1 else 132)]
RIGS = (("1 x poly3", False, 50), ("1 x poly3 + IMU", True, 100), ("1 x poly3 + IMU", True, 400))
FCOV_KERNELS = ("cov_frame_mega_batch_kernel", "chain_frame_cov_batch_kernel")
try:  # read-only query: a number is only meaningful next to the card, its power limit and clocks
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown (nvidia-smi not available)"
print(f"card (name, power limit, SM clock now, SM clock max): {card}\n{K} LM iterations per solve, best of {RUNS} alternating runs")


def calibrator(p, inertial):
    g = Calibrator()
    g.load(p)
    if inertial:
        g.set_flags(**ALL_ON)
    g.set_options(**OPTS)
    return g


def per_handle(rigs):
    return [g.frame_covariance() for g in rigs]


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


def corr_diff(a, b):
    sd = np.sqrt(np.maximum(np.einsum("fii->fi", b), 1e-300))
    return float((np.abs(a - b) / (sd[:, :, None] * sd[:, None, :])).max())


print(f"{'rig':>16s} {'frames':>6s} {'n':>4s} | {'per-handle us/rig':>17s} {'dev us/rig':>10s} | {'batch us/rig':>12s} "
      f"{'dev us/rig':>10s} {'launch us/rig':>13s} | wall x | max diff")
for name, inertial, nf in RIGS:
    problems = [synth.make_problem(models=("poly3",), n_frames=nf, grid=(8, 6), inertial=inertial, seed=1000 + i) for i in range(max(NS))]
    rigs = [calibrator(p, inertial) for p in problems]
    (solve_batch_inertial if inertial else solve_batch)(rigs)
    G = rigs[0].G
    for n in NS:
        sub = rigs[:n]
        best = {"seq": 1e9, "batch": 1e9}
        for run in range(RUNS + 1):  # run 0 warms both arms up
            for arm, fn in (("seq", lambda: per_handle(sub)), ("batch", lambda: frame_covariance_batch(sub))):
                t0 = time.perf_counter()
                fn()
                wall = time.perf_counter() - t0
                if run > 0:
                    best[arm] = min(best[arm], wall)
        diff = max(corr_diff(a, b) for a, b in zip(frame_covariance_batch(sub), per_handle(sub)))
        d_seq = device_us(lambda: per_handle(sub)) / n
        d_batch = device_us(lambda: frame_covariance_batch(sub)) / n
        d_launch = device_us(lambda: frame_covariance_batch(sub), FCOV_KERNELS) / n
        print(f"{name:>16s} {nf:6d} {n:4d} | {1e6 * best['seq'] / n:17.1f} {d_seq:10.1f} | {1e6 * best['batch'] / n:12.1f} {d_batch:10.1f} "
              f"{d_launch:13.1f} | {best['seq'] / best['batch']:6.2f} | {diff:.1e}   (G = {G})", flush=True)
    for g in rigs:
        g.close()
