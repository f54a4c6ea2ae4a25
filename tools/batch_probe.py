"""Rigs per second of vcgpu_solve_batch (one thread-block cluster per rig) against sequential vcgpu_solve calls.

    python tools/batch_probe.py [max_n]

Prints the card, its power limit and SM clocks, how many clusters of each size the device holds at once, then for
rigs of config 1's shape (1 x poly3, 50 frames x 140 corners) and of 200 frames, LM and DOGLEG, up to 20 iterations
with the tolerances at zero (a rig whose gradient vanishes stops earlier; times are divided by the iterations that
ran), n = 1 .. max_n (default 264) handles with distinct seeds: rigs/s and us per rig-iteration of n
sequential solves and of one batch, by the wall clock of the calls and by the device time they report (sequential: the
sum of the solves' device_seconds; batch: the launch's).  The two arms alternate, three runs each, best of three.
n = 1 is the cluster kernel against the 132-CTA cooperative kernel on the same rig.  Reads device settings, changes none.
"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vicalib_b200 import synth
from vicalib_b200.capi import Calibrator, solve_batch

K, RUNS = 20, 3
NS = [n for n in (1, 8, 33, 66, 132, 264) if n <= (int(sys.argv[1]) if len(sys.argv) > 1 else 264)]
try:  # read-only query: a number is only meaningful next to the card, its power limit and clocks
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown (nvidia-smi not available)"
print(f"card (name, power limit, SM clock now, SM clock max): {card}\nup to {K} iterations per solve, best of {RUNS} alternating runs")

print("clusters resident at once (cudaOccupancyMaxActiveClusters), 1 x poly3:")
for strategy in (0, 1):
    for nf in (10, 30, 60, 120):
        g = Calibrator()
        g.load(synth.make_problem(models=("poly3",), n_frames=nf, grid=(14, 10), seed=1))
        g.set_options(strategy=strategy)
        size, warps, resident = g.batch_plan()
        print(f"    {'DOGLEG' if strategy else 'LM':6s} {nf:4d} frames: cluster of {size} CTAs x {warps} warps, {resident} resident")
        g.close()

print(f"{'rig':>10s} {'strategy':>8s} {'n':>4s} | {'seq rigs/s':>10s} {'us/rig-it':>9s} {'dev us/rig-it':>13s} | "
      f"{'batch rigs/s':>12s} {'us/rig-it':>9s} {'dev us/rig-it':>13s} | wall x  device x")
for nf in (50, 200):
    problems = [synth.make_problem(models=("poly3",), n_frames=nf, grid=(14, 10), seed=1000 + i) for i in range(max(NS))]
    rigs = []
    for p in problems:
        g = Calibrator()
        g.load(p)
        rigs.append(g)
    for strategy in (0, 1):
        for g in rigs:
            g.set_options(strategy=strategy, max_iters=K, function_tol=0.0, gradient_tol=0.0, param_tol=0.0)
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
                        sums = solve_batch(rigs[:n])
                        dev = sums[0]["device_seconds"]  # like rigs: one launch
                    wall = time.perf_counter() - t0
                    its = sum(s["iterations"] for s in sums)
                    if run > 0:
                        best[arm] = (min(best[arm][0], wall), min(best[arm][1], dev))
            (ws, ds), (wb, db) = best["seq"], best["batch"]
            print(f"{nf:4d} x 140 {'DOGLEG' if strategy else 'LM':>8s} {n:4d} | {n / ws:10.0f} {1e6 * ws / its:9.2f} {1e6 * ds / its:13.2f} | "
                  f"{n / wb:12.0f} {1e6 * wb / its:9.2f} {1e6 * db / its:13.2f} | {ws / wb:6.2f} {ds / db:9.2f}", flush=True)
    for g in rigs:
        g.close()
