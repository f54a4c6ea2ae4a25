"""Time of scoring candidate views (vcgpu_get_view_information) on the north-star rig and on a rig of G = 127.

    python tools/view_information_probe.py [n_cand]

Prints the card, its power limit and SM clocks, then for each rig, the target workload (2 x poly3 + IMU, 2000 frames, G
= 41, at its start state) and 8 x KB4 + IMU (G = 127, 40 frames): n_cand (default 10^4) candidate poses, the rig's
frames turned by ~0.1 rad and moved by ~3 cm, scored against the target's corners with the prior passed in.  Reported:
the wall time of Calibrator.view_information() with variances (best of three after a warm-up) and the device time of
view_prior_kernel and view_info_kernel (torch.profiler, a run of their own), in microseconds per candidate; then the
same with the full posterior for n_cand / 10 candidates.  Reads device settings, changes none.
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
from vicalib_b200.capi import Calibrator  # noqa: E402

NC = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
try:  # read-only query: a number is only meaningful next to the card, its power limit and clocks
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown (nvidia-smi not available)"
print(f"card (name, power limit, SM clock now, SM clock max): {card}")


def best(fn, reps=3):
    fn()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.append(time.perf_counter() - t0)
    return min(out)


def kernel_us(fn, names=("view_prior_kernel", "view_info_kernel")):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [sum(getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0)
                for e in prof.key_averages() if n in e.key) for n in names]


def candidates(p, n, seed=0):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, p.n_frames, n)
    T = p.T_wp[k].copy()
    w = rng.normal(0, 0.1, (n, 3))
    th = np.linalg.norm(w, axis=1, keepdims=True)
    dq = np.concatenate([np.sin(th / 2) * w / th, np.cos(th / 2)], 1)
    q = synth.quat_mul(T[:, :4], dq)
    T[:, :4] = q / np.linalg.norm(q, axis=1, keepdims=True)
    T[:, 4:] += rng.normal(0, 0.03, (n, 3))
    return T


def run(name, p, flags):
    g = Calibrator()
    g.load(p)
    g.set_flags(**flags)
    S = g.covariance()
    pw = np.unique(p.p_w, axis=0)[:400]
    T = candidates(p, NC)
    r = g.view_information(T, pw, 640, 480, cov=S, var=True)
    fin = np.isfinite(r["gain"])
    print(f"{name}: G = {g.G}, {g.n_cams} cameras, {len(pw)} target points, {NC} candidates, {int(fin.sum())} finite gains "
          f"(median {np.median(r['gain'][fin]):.3f} nats), {r['n_seen'].sum(1).mean():.1f} corners seen per candidate")
    t = best(lambda: g.view_information(T, pw, 640, 480, cov=S, var=True))
    kp, kv = kernel_us(lambda: g.view_information(T, pw, 640, 480, cov=S, var=True))
    print(f"  var:  wall {1e6 * t / NC:.2f} us per candidate; view_prior_kernel {kp:.1f} us, view_info_kernel {kv / NC:.2f} us "
          f"per candidate ({kv / 1e3:.2f} ms)")
    m = max(NC // 10, 1)
    t = best(lambda: g.view_information(T[:m], pw, 640, 480, cov=S, post=True))
    kp, kv = kernel_us(lambda: g.view_information(T[:m], pw, 640, 480, cov=S, post=True))
    print(f"  post: {m} candidates, wall {1e6 * t / m:.2f} us per candidate; view_info_kernel {kv / m:.2f} us per candidate")
    g.close()


run("target", synth.make_config("target"), ALL_ON)
run("8 x KB4 + IMU", synth.make_problem(models=("kb4",) * 8, n_frames=40, inertial=True, seed=127), ALL_ON)
