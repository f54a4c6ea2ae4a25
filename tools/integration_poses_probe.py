"""IMU integration poses of every interval (GetIntegrationPoses, vicalibrator.h:508-533) on the target workload: the
device's vcgpu_get_integration_poses per handle and vcgpu_get_integration_poses_batch against the host mirror's
GetIntegrationPoses(k) looped over all intervals, which is what a GUI redraw asks for.

    python tools/integration_poses_probe.py [n_rigs]

Prints the card, its power limit and SM clocks, then on the target workload (2 x poly3 + IMU, 2000 frames, 200 Hz IMU,
at its start state): the poses per rig; the wall time of Calibrator.integration_poses() (a sizes call and a fill call),
of capi.integration_poses_batch() on n_rigs (default 8) copies of the rig, per rig, and of the mirror's host loop
(C++, compiled from tests/cpp/integration_poses_oracle.cc; its loop alone, without copying the samples in), each the
best of five runs after a warm-up; the device time of the per-handle call's kernels (torch.profiler, a run of its own);
and whether the device's counts and times are the mirror's.  Reads device settings, changes none.
"""
import os
import subprocess
import sys
import time

import numpy as np
import torch  # noqa: F401  (before libvcgpu.so: torch's CUDA library needs its own NCCL symbols first)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import integration_poses_ref as R  # noqa: E402
from vicalib_b200 import synth  # noqa: E402
from vicalib_b200.capi import Calibrator, integration_poses_batch  # noqa: E402

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


def device_us(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ks = {}
    for e in prof.key_averages():
        ks[e.key] = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0)
    return ks


p = synth.make_config("target")
rigs = []
for _ in range(NR):
    g = Calibrator()
    g.load(p)
    g.set_flags(**ALL_ON)
    rigs.append(g)
poses = rigs[0].integration_poses()
total = sum(len(x) for x in poses)
print(f"target: {p.n_frames} frames, {len(p.imu_t)} IMU samples, {total} poses over {len(poses)} intervals")
t_one = best(rigs[0].integration_poses)
t_batch = best(lambda: integration_poses_batch(rigs)) / NR
mirror = []
for _ in range(6):
    n_m, sec = R.mirror_all_timed(p)
    mirror.append(sec)
t_mirror = min(mirror[1:])
print(f"wall, best of 5: per-handle call {1e3 * t_one:.3f} ms | batch of {NR}, per rig {1e3 * t_batch:.3f} ms | "
      f"mirror host loop {1e3 * t_mirror:.3f} ms")
ks = device_us(rigs[0].integration_poses)
for k, v in sorted(ks.items(), key=lambda kv: -kv[1]):
    if v > 0:
        print(f"  device {v:9.1f} us  {k[:90]}")
print(f"mirror poses {n_m}, device poses {total}; counts and times equal to the mirror's: ", end="")
want = R.mirror_poses(p)
print(all(len(a) == len(b) and a[:, 13].tobytes() == b[:, 13].tobytes() for a, b in zip(poses, want)))
print(f"largest pose difference to the mirror (q, t, v, w, relative): "
      f"{np.max([R.worst(a, b) for a, b in zip(poses, want) if len(b)], axis=0)}")
for g in rigs:
    g.close()
