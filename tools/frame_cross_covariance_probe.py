"""The frame blocks off the diagonal next to the frame blocks on it, on the benchmark's target workload and on config 2.

    python tools/frame_cross_covariance_probe.py [out_dir]

Prints the card, its power limit and SM clocks, then per workload (target: 2 x poly3 + IMU, 2000 frames, every IMU
flag on; config2: 1 x poly3, 2000 frames), after K LM iterations: the wall time of vcgpu_get_frame_cross_covariance and
of vcgpu_get_frame_covariance, each the best of RUNS alternating calls after a warm-up, and the device time of each
call's kernels from one torch.profiler run of its own.  With out_dir, also writes the lines there as
frame_cross_covariance_probe.txt.  Reads device settings, changes none.
"""
import os
import subprocess
import sys
import time

import torch  # noqa: F401  (before libvcgpu.so: torch's CUDA library needs its own NCCL symbols first)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vicalib_b200 import synth
from vicalib_b200.capi import Calibrator

K, RUNS = 10, 5
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
lines = []


def say(s):
    print(s, flush=True)
    lines.append(s)


try:  # read-only query: a number is only meaningful next to the card, its power limit and clocks
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown (nvidia-smi not available)"
say(f"card (name, power limit, SM clock now, SM clock max): {card}\n{K} LM iterations before the calls, best of {RUNS}")


def wall(fn):
    t = time.perf_counter()
    fn()  # every call ends in a device synchronise (its copy back)
    return time.perf_counter() - t


def device_ms(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if e.device_time_total > 0
             and not e.key.startswith("Memcpy") and not e.key.startswith("Memset"))
    return us / 1e3


for name in ("target", "config2"):
    p = synth.make_config(name)
    g = Calibrator(device=0)
    g.load(p)
    g.set_flags(**(ALL_ON if p.inertial else {}))
    g.set_options(max_iters=K, function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
    g.solve()
    calls = {"frame_cross_covariance": g.frame_cross_covariance, "frame_covariance": g.frame_covariance}
    for fn in calls.values():
        fn()
    best = {k: float("inf") for k in calls}
    for _ in range(RUNS):
        for k, fn in calls.items():
            best[k] = min(best[k], wall(fn))
    dev = {k: device_ms(fn) for k, fn in calls.items()}
    fg, fn = g.frame_cross_covariance()
    say(f"{name}: {p.n_frames} frames, fd {g.fd}, G {g.G}; blocks {fg.shape} and {fn.shape}, all finite "
        f"{bool((fg == fg).all() and (fn == fn).all())}")
    for k in calls:
        say(f"  {k:22s} wall {best[k] * 1e3:9.2f} ms   kernels {dev[k]:9.2f} ms")
    g.close()

if len(sys.argv) > 1:
    os.makedirs(sys.argv[1], exist_ok=True)
    with open(os.path.join(sys.argv[1], "frame_cross_covariance_probe.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
