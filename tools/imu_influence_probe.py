"""Time of the IMU interval diagnostics (vcgpu_get_imu_influence) next to vcgpu_get_observation_influence, on the
benchmark's target workload and on a smaller inertial rig.

    python tools/imu_influence_probe.py [out_dir]

Prints the card, its power limit and SM clocks, then per workload (target: 2 x poly3 + IMU, 2000 frames; small:
1 x poly3 + IMU, 200 frames; every IMU flag on), after K LM iterations: the wall time of Calibrator.imu_influence(),
of the same call with the observation outputs, of capi.imu_influence_batch() of that rig alone and of
Calibrator.observation_influence(), each the best of RUNS alternating calls after a warm-up; then, from one
torch.profiler run of each, the device time of the kernels split into the interval pass (imu_eval_kernel,
imu_infl_kernel), the shared and observation kernels (infl_sgg_kernel, view_prior_kernel, infl_q_kernel,
infl_obs_kernel), the covariance they need (every other kernel), the copies' device time, and the rest of the wall
time, the host's.  With out_dir, also writes the lines there as imu_influence_probe.txt.  Reads device settings,
changes none.
"""
import os
import subprocess
import sys
import time

import numpy as np
import torch  # noqa: F401  (before libvcgpu.so: torch's CUDA library needs its own NCCL symbols first)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vicalib_b200 import synth  # noqa: E402
from vicalib_b200.capi import Calibrator, imu_influence_batch  # noqa: E402

K, RUNS = 10, 5
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
IMU_PASS = ("imu_eval_kernel", "imu_infl_kernel")
SHARED = ("infl_sgg_kernel", "view_prior_kernel", "infl_q_kernel", "infl_obs_kernel")
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
    """(interval pass, shared and observation kernels, other kernels, copies and sets) device time of one call, ms"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if e.device_time_total > 0]
    copy = sum(e.device_time_total for e in ev if e.key.startswith("Memcpy") or e.key.startswith("Memset"))
    imu = sum(e.device_time_total for e in ev if any(n in e.key for n in IMU_PASS))
    shared = sum(e.device_time_total for e in ev if any(n in e.key for n in SHARED))
    return imu / 1e3, shared / 1e3, (sum(e.device_time_total for e in ev) - imu - shared - copy) / 1e3, copy / 1e3


for name in ("target", "small"):
    p = synth.make_config("target") if name == "target" else \
        synth.make_problem(models=("poly3",), n_frames=200, inertial=True, seed=7)
    g = Calibrator(device=0)
    g.load(p)
    g.set_flags(**ALL_ON)
    g.set_options(max_iters=K, function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
    g.solve()
    calls = {"imu_influence": g.imu_influence, "imu_influence(observations)": lambda: g.imu_influence(observations=True),
             "imu_influence_batch": lambda: imu_influence_batch([g]), "observation_influence": g.observation_influence}
    for fn in calls.values():
        fn()
    best = {k: float("inf") for k in calls}
    for _ in range(RUNS):
        for k, fn in calls.items():
            best[k] = min(best[k], wall(fn))
    dev = {k: device_ms(fn) for k, fn in calls.items()}
    r = g.imu_influence()
    say(f"{name}: {p.n_frames} frames, {g.n_obs} observations, G {g.G}; finite stud {int(np.isfinite(r['stud']).sum())} of "
        f"{len(r['stud'])}, sum tr(H_imu) {float(np.nansum(np.trace(r['h'], axis1=1, axis2=2))):.3f}")
    for k in calls:
        i, s, c, m = dev[k]
        say(f"  {k:28s} wall {best[k] * 1e3:8.2f} ms = interval pass {i:7.3f} + shared/observation pass {s:7.3f}"
            f" + covariance kernels {c:7.3f} + copies {m:7.3f} + host {best[k] * 1e3 - i - s - c - m:7.3f} ms")
    g.close()

if len(sys.argv) > 1:
    os.makedirs(sys.argv[1], exist_ok=True)
    with open(os.path.join(sys.argv[1], "imu_influence_probe.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
