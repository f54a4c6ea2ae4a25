"""Per-phase device clocks of the persistent vision kernel (profile bit 8) and A/B against the multi-launch engine.

    python tools/mega_probe.py [workload] [strategy]

strategy 0 (LM, default) or 1 (DOGLEG).  Prints the card and its power limit, then us per iteration of LM persistent,
DOGLEG persistent and DOGLEG multi-launch, back to back (one launch for all iterations where the persistent kernel runs)
and with the L2 flushed before every iteration (one launch per iteration), then the phase clocks of the chosen strategy.
"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vicalib_b200 import synth
from vicalib_b200.capi import Calibrator

wl = sys.argv[1] if len(sys.argv) > 1 else "config2"
strategy = int(sys.argv[2]) if len(sys.argv) > 2 else 0
K = 20
try:  # read-only query: the number is only meaningful next to the card and its power limit
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown (nvidia-smi not available)"
print(f"card: {card}   workload {wl}, {K} iterations, best of 5")
p = synth.make_config(wl)
g = Calibrator()
g.load(p)
g.set_options(max_iters=K)
g.iterate(3)


def timed(strat, mode, flush):
    g.set_options(strategy=strat)
    g.set_profiling(mode, flush)
    best, s = 1e9, None
    for _ in range(5):
        g.load(p)
        s = g.iterate(K)
        best = min(best, s["device_seconds"])
    return 1e6 * best / K, s["kernel_launches"]


for strat, mode, name in ((0, 0, "LM persistent"), (1, 0, "DOGLEG persistent"), (1, 4, "DOGLEG multi-launch")):
    for flush in (False, True):
        us, launches = timed(strat, mode, flush)
        print(f"{name:22s} {'L2 flushed' if flush else 'back to back':12s} {us:8.2f} us/iter  launches {launches}")
us, _ = timed(strategy, 8, False)
print(f"{'LM' if strategy == 0 else 'DOGLEG'} persistent+clocks {us:8.2f} us/iter")
for k, v in g.stage_times().items():
    if v[1]:
        print(f"    {k:14s} {1e3 * v[0] / v[1]:8.2f} us/iter")
g.set_options(strategy=strategy)
g.set_profiling(0, False)
for rep in range(3):
    t0 = time.perf_counter(); g.load(p); t1 = time.perf_counter(); s = g.iterate(K); t2 = time.perf_counter(); g.state()
    t3 = time.perf_counter()
    print(f"e2e: load {1e3*(t1-t0):.2f} ms  iterate({K}) {1e3*(t2-t1):.2f} ms (device {1e3*s['device_seconds']:.2f})  "
          f"state {1e3*(t3-t2):.2f} ms")
