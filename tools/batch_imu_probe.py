"""Rigs per second of vcgpu_solve_batch_inertial (one thread-block cluster per rig) against sequential vcgpu_solve calls.

    python tools/batch_imu_probe.py [max_n]

Prints the card, its power limit and SM clocks, the cluster size and how many such clusters the device holds at once
per rig, then for 1 x poly3 + IMU and 2 x poly3 + IMU rigs (8 x 6 corners per camera and frame) of 100, 400 and 2000
frames, every flag on, weights held, exactly K LM iterations (tolerances at zero), n = 1 .. max_n (default 132) handles
with distinct seeds: rigs/s and us per rig-iteration of n sequential solves and of one batch, by the wall clock of the
calls and by the device time they report (sequential: the sum of the solves' device_seconds; batch: the time of its
iteration loop).  The two arms alternate, three runs each after a warm-up run, best of three.  n = 1 is one cluster
against the cooperative grid on the same rig.  Reads device settings, changes none.
"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vicalib_b200 import synth
from vicalib_b200.capi import Calibrator, solve_batch_inertial

K, RUNS = 10, 3
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
OPTS = dict(max_iters=K, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, update_imu_weights=0)
NS = [n for n in (1, 8, 16, 33, 132) if n <= (int(sys.argv[1]) if len(sys.argv) > 1 else 132)]
RIGS = (("1 x poly3", ("poly3",)), ("2 x poly3", ("poly3", "poly3")))
FRAMES = (100, 400, 2000)
try:  # read-only query: a number is only meaningful next to the card, its power limit and clocks
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown (nvidia-smi not available)"
print(f"card (name, power limit, SM clock now, SM clock max): {card}\n{K} LM iterations per solve, best of {RUNS} alternating runs")


def problem(models, nf, seed):
    return synth.make_problem(models=models, n_frames=nf, grid=(8, 6), inertial=True, seed=seed)


def calibrator(p):
    g = Calibrator()
    g.load(p)
    g.set_flags(**ALL_ON)
    g.set_options(**OPTS)
    return g


print("clusters (cudaOccupancyMaxActiveClusters of the solve and the evaluation kernel, the smaller):")
for name, models in RIGS:
    for nf in FRAMES:
        g = calibrator(problem(models, nf, 1))
        size, resident = g.batch_plan_inertial()
        print(f"    {name} + IMU, {nf:4d} frames: cluster of {size} CTAs, {resident} resident")
        g.close()

print(f"{'rig':>16s} {'frames':>6s} {'n':>4s} | {'seq rigs/s':>10s} {'us/rig-it':>9s} {'dev us/rig-it':>13s} | "
      f"{'batch rigs/s':>12s} {'us/rig-it':>9s} {'dev us/rig-it':>13s} | wall x  device x")
for name, models in RIGS:
    for nf in FRAMES:
        problems = [problem(models, nf, 1000 + i) for i in range(max(NS))]
        rigs = [calibrator(p) for p in problems]
        for n in NS:
            best = {"seq": (1e9, 1e9), "batch": (1e9, 1e9)}
            for run in range(RUNS + 1):  # run 0 warms both arms up
                for arm in ("seq", "batch"):
                    for g, p in zip(rigs[:n], problems):
                        g.load(p)
                        g.cost()  # uploads and buffers outside the timed window, in both arms
                    t0 = time.perf_counter()
                    if arm == "seq":
                        sums = [g.solve(free_running=True) for g in rigs[:n]]
                        dev = sum(s["device_seconds"] for s in sums)
                    else:
                        sums = solve_batch_inertial(rigs[:n])
                        dev = sums[0]["device_seconds"]  # the batch's loop, shared
                    wall = time.perf_counter() - t0
                    its = sum(s["iterations"] for s in sums)
                    assert its == n * K, its
                    if run > 0:
                        best[arm] = (min(best[arm][0], wall), min(best[arm][1], dev))
            (ws, ds), (wb, db) = best["seq"], best["batch"]
            print(f"{name + ' + IMU':>16s} {nf:6d} {n:4d} | {n / ws:10.1f} {1e6 * ws / its:9.2f} {1e6 * ds / its:13.2f} | "
                  f"{n / wb:12.1f} {1e6 * wb / its:9.2f} {1e6 * db / its:13.2f} | {ws / wb:6.2f} {ds / db:9.2f}", flush=True)
        for g in rigs:
            g.close()
