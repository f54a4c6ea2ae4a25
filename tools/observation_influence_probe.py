"""Time of the observation diagnostics (vcgpu_get_observation_influence) next to vcgpu_get_frame_cross_covariance, on
the benchmark's target workload and on config 2.

    python tools/observation_influence_probe.py [out_dir]

Prints the card, its power limit and SM clocks, then per workload (target: 2 x poly3 + IMU, 2000 frames, every IMU
flag on; config2: 1 x poly3, 2000 frames), after K LM iterations: the wall time of Calibrator.observation_influence(),
of capi.observation_influence_batch() of that rig alone and of Calibrator.frame_cross_covariance(), each the best of
RUNS alternating calls after a warm-up (the first influence call, which sorts and uploads the observations, is timed
apart); then, from one torch.profiler run of each, the device time of the kernels split into the observation pass
(infl_sgg_kernel, view_prior_kernel, infl_q_kernel, infl_obs_kernel) and the covariance it needs (every other kernel),
the copies' device time, and the rest of the wall time, the host's.  With out_dir, also
writes the lines there as observation_influence_probe.txt.  Reads device settings, changes none.
"""
import os
import subprocess
import sys
import time

import numpy as np
import torch  # noqa: F401  (before libvcgpu.so: torch's CUDA library needs its own NCCL symbols first)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vicalib_b200 import synth  # noqa: E402
from vicalib_b200.capi import Calibrator, observation_influence_batch  # noqa: E402

K, RUNS = 10, 5
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
PASS = ("infl_sgg_kernel", "view_prior_kernel", "infl_q_kernel", "infl_obs_kernel")
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
    """(observation pass, other kernels, copies and sets) device time of one call, ms"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if e.device_time_total > 0]
    copy = sum(e.device_time_total for e in ev if e.key.startswith("Memcpy") or e.key.startswith("Memset"))
    obs = sum(e.device_time_total for e in ev if any(n in e.key for n in PASS))
    return obs / 1e3, (sum(e.device_time_total for e in ev) - obs - copy) / 1e3, copy / 1e3


for name in ("target", "config2"):
    p = synth.make_config(name)
    g = Calibrator(device=0)
    g.load(p)
    g.set_flags(**(ALL_ON if p.inertial else {}))
    g.set_options(max_iters=K, function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
    g.solve()
    first = wall(g.observation_influence)
    calls = {"observation_influence": g.observation_influence, "observation_influence_batch": lambda: observation_influence_batch([g]),
             "frame_cross_covariance": g.frame_cross_covariance}
    for fn in calls.values():
        fn()
    best = {k: float("inf") for k in calls}
    for _ in range(RUNS):
        for k, fn in calls.items():
            best[k] = min(best[k], wall(fn))
    dev = {k: device_ms(fn) for k, fn in calls.items()}
    r = g.observation_influence()
    act = g.obs_active() > 0
    tr = float((r["h"][act, 0] + r["h"][act, 2]).sum())
    say(f"{name}: {p.n_frames} frames, {g.n_obs} observations, G {g.G}; finite {bool(np.isfinite(r['infl']).all())}, "
        f"sum tr(H) {tr:.3f}")
    say(f"  first observation_influence (sorts and uploads the observations) wall {first * 1e3:9.2f} ms")
    for k in calls:
        o, c, m = dev[k]
        say(f"  {k:27s} wall {best[k] * 1e3:8.2f} ms = observation pass {o:7.3f} + covariance kernels {c:7.3f} + copies {m:7.3f}"
            f" + host {best[k] * 1e3 - o - c - m:7.3f} ms")
    g.close()

if len(sys.argv) > 1:
    os.makedirs(sys.argv[1], exist_ok=True)
    with open(os.path.join(sys.argv[1], "observation_influence_probe.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
