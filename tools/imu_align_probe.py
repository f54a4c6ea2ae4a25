"""Time of the hand-eye alignment of the gyro stream (vcgpu_align_imu, vcgpu_align_imu_batch).

    python tools/imu_align_probe.py [out_dir]

Prints the card, its power limit and SM clocks, then:
  target  the benchmark's target workload (2 x poly3 + IMU, 2000 frames), re-expressed with camera 0 as the rig frame,
          ts in [-0.1, 0.1] s at 0.5 ms (401 candidates): wall time of Calibrator.align_imu(), best of RUNS after a
          warm-up, and the device time of its kernels (torch.profiler, a run of its own) split into the grid, the
          refinement and the rest;
  batch   64 config1-size inertial rigs (1 x poly3 + IMU, 50 frames), the same grid: wall time of one
          capi.align_imu_batch() per rig against 64 Calibrator.align_imu() calls, best of RUNS, and whether both returned
          the same bits.
Wall times are CUDA-event timed between two events on the current stream around a call that ends in a device
synchronise.  With out_dir, also writes the lines there as imu_align_probe.txt.  Reads device settings, changes none.
"""
import os
import subprocess
import sys

import numpy as np
import torch  # noqa: F401  (before libvcgpu.so: torch's CUDA library needs its own NCCL symbols first)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import imu_align_ref  # noqa: E402
from vicalib_b200 import synth  # noqa: E402
from vicalib_b200.capi import Calibrator, align_imu_batch  # noqa: E402

RUNS = 5
GRID = dict(ts_lo=-0.1, ts_hi=0.1, n_ts=401)
lines = []


def say(s):
    print(s, flush=True)
    lines.append(s)


try:  # read-only query: a number is only meaningful next to the card, its power limit and clocks
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown (nvidia-smi not available)"
say(f"card (name, power limit, SM clock now, SM clock max): {card}; best of {RUNS}; grid {GRID}")


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def best(fn):
    fn()
    return min(event_ms(fn)[0] for _ in range(RUNS))


def device_split(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    torch.cuda.synchronize()
    split = {"grid": 0.0, "refine": 0.0, "other": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
        k = "grid" if "align_grid" in e.key else "refine" if "align_refine" in e.key else "other"
        split[k] += us / 1000.0
    return split


def load(p):
    g = Calibrator(device=0)
    g.load(p)
    return g


torch.cuda.init()
p = imu_align_ref.camera0_start(synth.make_config("target"))
g = load(p)
r = g.align_imu(**GRID)
ms = best(lambda: g.align_imu(**GRID))
sp = device_split(lambda: g.align_imu(**GRID))
say(f"target: {r['n_intervals']} intervals, {r['iterations']} iterations, rotation error "
    f"{imu_align_ref.angle(r['Q'], p.truth['q_ck'][0]):.2e} rad, ts {r['ts']:.6f} s: {ms:.2f} ms per call; device ms "
    + ", ".join(f"{k} {v:.2f}" for k, v in sp.items()))

rigs = [imu_align_ref.camera0_start(synth.make_problem(models=("poly3",), n_frames=50, grid=(14, 10), inertial=True,
                                                       seed=100 + i, ts_truth=0.01)) for i in range(64)]
gs = [load(q) for q in rigs]
ms_batch = best(lambda: align_imu_batch(gs, **GRID))
ms_each = best(lambda: [c.align_imu(**GRID) for c in gs])
a = align_imu_batch(gs, **GRID)
b = [c.align_imu(**GRID) for c in gs]
bits = all(np.array_equal(x["Q"], y["Q"]) and x["ts"] == y["ts"] and np.array_equal(x["b_g"], y["b_g"]) for x, y in zip(a, b))
say(f"batch of 64 config1-size inertial rigs: {ms_batch / 64:.3f} ms per rig in one call, {ms_each / 64:.3f} ms per rig "
    f"in 64 calls; same bits: {bits}")
if len(sys.argv) > 1:
    os.makedirs(sys.argv[1], exist_ok=True)
    with open(os.path.join(sys.argv[1], "imu_align_probe.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
