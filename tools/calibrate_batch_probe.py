"""Time N copies of a small inertial rig (default 1 x poly3 + IMU, 200 frames) through the default staged flow
(calibrate_imu, remove_outliers, block duplication, DOGLEG) two ways: the host mirror's sequence of per-handle calls
(vcgpu_solve per stage: DOGLEG inertial stages on the multi-launch engine; vcgpu_evaluate per camera;
vcgpu_remove_outliers), and one vcgpu_calibrate_batch.

Both ways synchronise with the host throughout, so what is timed is wall time of the whole flow (perf_counter around
it, after a device synchronise), not device time.  Kernel launches are not reported: the library counts them per
solve only, which leaves out the per-handle way's evaluations and outlier removals and cannot be split per rig for
the batch.  After one warm-up pass, --reps alternating timed passes of each way; prints one JSON line per way with
the passes' wall times (min, median, max) and solves per rig.  Report the GPU's clock and power state under load
(nvidia-smi --query-gpu=clocks.sm,power.draw,power.limit, read only, sampled during the run) beside the numbers.

    python tools/calibrate_batch_probe.py --rigs 8 --frames 200
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from test_cpu_calibrate_flow import flow_reference  # noqa: E402
from vicalib_b200 import synth  # noqa: E402
from vicalib_b200.capi import Calibrator, calibrate_batch  # noqa: E402

FLOW = dict(calibrate_imu=True, remove_outliers=True, outlier_threshold=2.0, block_duplication=True, gravity_initialized=False,
            max_solves=20)
START = dict(inertial=0, rotation_only=1, bias_active=0, scale_active=0, optimize_ts=1)


def make(problems, max_iters):
    gs = []
    for p in problems:
        g = Calibrator()
        g.load(p)
        g.set_flags(**START)
        g.set_options(strategy=1, max_iters=max_iters)
        gs.append(g)
    return gs


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rigs", type=int, default=8)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--max-iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    torch.cuda.init()
    problems = [synth.make_problem(models=("poly3",), n_frames=a.frames, grid=(14, 10), inertial=True, seed=100 + k) for k in range(a.rigs)]
    walls = {"per-handle": [], "calibrate_batch": []}
    solves = {}
    for rep in range(a.reps + 1):  # a warm-up pass, then the timed ones, the two ways alternating
        gs = make(problems, a.max_iters)
        traces, wall = timed(lambda: [flow_reference(g, p, **FLOW) for g, p in zip(gs, problems)])
        solves["per-handle"] = [len(t["solves"]) for t in traces]
        if rep:
            walls["per-handle"].append(wall)
        gs = make(problems, a.max_iters)
        out, wall = timed(lambda: calibrate_batch(gs, **FLOW))
        solves["calibrate_batch"] = [d["solves"] for d, _ in out]
        if rep:
            walls["calibrate_batch"].append(wall)
    for way, w in walls.items():
        print(json.dumps(dict(way=way, rigs=a.rigs, frames=a.frames, reps=a.reps, wall_s_min=min(w), wall_s_median=float(np.median(w)),
                              wall_s_max=max(w), solves=solves[way])))
    assert solves["per-handle"] == solves["calibrate_batch"], "the two ways took different numbers of solves"


if __name__ == "__main__":
    main()
