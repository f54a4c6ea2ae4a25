"""Per-camera evaluation and outlier removal of many rigs: one vcgpu_evaluate_batch / vcgpu_remove_outliers_batch call
against vcgpu_evaluate per handle and camera / vcgpu_remove_outliers per handle.

    python tools/evaluate_batch_probe.py [max_n]

Prints the card, its power limit and SM clocks, then, on covariance_batch_probe.py's rigs (50-frame 1 x poly3 vision
rigs, 100- and 400-frame 1 x poly3 + IMU rigs, 8 x 6 corners per frame, solved first with K LM iterations) for
n = 1, 8, 33, 132 (up to max_n) handles, and on the north-star rig (2 x poly3 + IMU, 2000 frames, 560 000
observations) for n = 1:
  - evaluate: wall time per rig of n_cams vcgpu_evaluate(h, c) calls per handle against one vcgpu_evaluate_batch, best
    of three alternating runs after a warm-up, and the device time per rig of each arm from one torch.profiler run of
    its own (all kernels of the arm);
  - outliers: the same for vcgpu_remove_outliers per handle against vcgpu_remove_outliers_batch, at a threshold that
    removes nothing (so every run sees the same problem).
Reads device settings, changes none.
"""
import os
import subprocess
import sys
import time

import torch  # noqa: F401  (before libvcgpu.so: torch's CUDA library needs its own NCCL symbols first)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from vicalib_b200 import synth
from vicalib_b200.capi import Calibrator, evaluate_batch, remove_outliers_batch, solve_batch, solve_batch_inertial

K, RUNS, THRESHOLD = 10, 3, 1e6
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
OPTS = dict(max_iters=K, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, update_imu_weights=0)
NS = [n for n in (1, 8, 33, 132) if n <= (int(sys.argv[1]) if len(sys.argv) > 1 else 132)]
try:  # read-only query: a number is only meaningful next to the card, its power limit and clocks
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown (nvidia-smi not available)"
print(f"card (name, power limit, SM clock now, SM clock max): {card}\n{K} LM iterations per solve first, best of {RUNS} alternating runs")


def calibrator(p, inertial):
    g = Calibrator()
    g.load(p)
    if inertial:
        g.set_flags(**ALL_ON)
    g.set_options(**OPTS)
    return g


def per_camera(rigs):
    return [[g.evaluate(c) for c in range(g.n_cams)] for g in rigs]


def device_us(fn):
    """summed device time (us) of the kernels fn launches"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0) for e in prof.key_averages())


def measure(name, nf, sub, rmses):
    n = len(sub)
    arms = {"eval_seq": lambda: per_camera(sub), "eval_batch": lambda: evaluate_batch(sub),
            "out_seq": lambda: [g.remove_outliers(r, THRESHOLD) for g, r in zip(sub, rmses)],
            "out_batch": lambda: remove_outliers_batch(sub, rmses, THRESHOLD)}
    best = {k: 1e9 for k in arms}
    for run in range(RUNS + 1):  # run 0 warms every arm up
        for arm, fn in arms.items():
            t0 = time.perf_counter()
            fn()
            wall = time.perf_counter() - t0
            if run > 0:
                best[arm] = min(best[arm], wall)
    dev = {k: device_us(fn) / n for k, fn in arms.items()}
    # the two arms' costs, as a check that they computed the same thing
    seq = per_camera(sub)
    diff = max(abs(c - s[0]) / max(s[0], 1e-300) for (cs, _), ss in zip(evaluate_batch(sub), seq) for c, s in zip(cs, ss))
    us = {k: 1e6 * v / n for k, v in best.items()}
    print(f"{name:>16s} {nf:6d} {n:4d} | {us['eval_seq']:10.1f} {dev['eval_seq']:8.1f} | {us['eval_batch']:10.1f} {dev['eval_batch']:8.1f} "
          f"| {best['eval_seq'] / best['eval_batch']:6.2f} | {us['out_seq']:10.1f} {dev['out_seq']:8.1f} | {us['out_batch']:10.1f} "
          f"{dev['out_batch']:8.1f} | {best['out_seq'] / best['out_batch']:6.2f} | {diff:.1e}", flush=True)


print(f"{'rig':>16s} {'frames':>6s} {'n':>4s} | {'eval seq':>10s} {'dev':>8s} | {'eval batch':>10s} {'dev':>8s} | wall x "
      f"| {'out seq':>10s} {'dev':>8s} | {'out batch':>10s} {'dev':>8s} | wall x | cost rel diff   (us per rig)")
for name, inertial, nf in (("1 x poly3", False, 50), ("1 x poly3 + IMU", True, 100), ("1 x poly3 + IMU", True, 400)):
    problems = [synth.make_problem(models=("poly3",), n_frames=nf, grid=(8, 6), inertial=inertial, seed=1000 + i) for i in range(max(NS))]
    rigs = [calibrator(p, inertial) for p in problems]
    (solve_batch_inertial if inertial else solve_batch)(rigs)
    rmses = [np.array([np.sqrt(2.0 * c / b) for c, b in zip(cs, bs)]) for cs, bs in evaluate_batch(rigs)]
    for n in NS:
        measure(name, nf, rigs[:n], rmses[:n])
    for g in rigs:
        g.close()
g = calibrator(synth.make_config("target"), True)
g.solve(free_running=True)
cs, bs = evaluate_batch([g])[0]
measure("north star", g.n_frames, [g], [np.sqrt(2.0 * cs / bs)])
g.close()
