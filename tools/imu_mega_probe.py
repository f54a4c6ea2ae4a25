"""Device phase clocks of the persistent inertial kernels (chain_solve_kernel / eval_mega_kernel), us per iteration.
   python tools/imu_mega_probe.py [workload] [K] [flush]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vicalib_b200 import synth
from vicalib_b200.capi import Calibrator

wl = sys.argv[1] if len(sys.argv) > 1 else "target"
K = int(sys.argv[2]) if len(sys.argv) > 2 else 20
flush = int(sys.argv[3]) if len(sys.argv) > 3 else 0
p = synth.make_config(wl)
g = Calibrator()
g.load(p)
g.set_flags(inertial=1, bias_active=1, scale_active=1, optimize_ts=1)
g.set_options(max_iters=K)
g.iterate(3)
for prof, name in ((0, "persistent"), (4, "multi-launch")):
    g.load(p)
    g.set_profiling(prof, flush)
    s = g.iterate(K)
    print(f"{name}: {1e6 * s['device_seconds'] / K:.1f} us/iteration, {s['kernel_launches']} launches, accepted {s['successful_steps']}")
g.load(p)
g.set_profiling(8, flush)
s = g.iterate(K)
ns = g.phase_clocks().astype(float) / K / 1e3
# the back-substitution slots count levels from the top (slot 12: the level just below the dense system); the last one
# used is level 0, shared out among whichever CTAs are there (the ones still working the weights queue join later)
names = {10: "schur reduce", 11: "dense", 22: "step stats", 23: "weights (solver CTAs)", 32: "eval tasks", 33: "imu accumulate", 34: "reduce", 35: "decide", 36: "weights"}
# chunk phase clocks: level 1 on CTA 0 (slots 40..47), level 0 on CTA 0's first group (slots 56..63); above level 0 the
# couplings are written in the pass that adds the Schur terms from the left
chunk = ("wait prev", "async copies + wait", "scale / damp / add in place", "couplings", "forward sweep (+ Z, last node)",
         "backward sweep (+ Z)", "Schur acc", "separator update + stores")
cyc = {53: "dense: LDL^T", 54: "dense: back-substitution", 55: "dense: write + top update"}
for base, lv in ((40, 1), (56, 0)):
    cyc.update({base + k: f"level {lv} chunk: {nm}" for k, nm in enumerate(chunk)})
for k in range(64):
    if k in cyc:
        if ns[k] > 0:
            print(f"  [{k:2d}] {cyc[k]:46s} {ns[k] * 1e3 / 1980.0:8.2f} us (cycles / 1980 MHz, the H100 SXM maximum SM clock)")
        continue
    if ns[k] > 0:
        nm = names.get(k, f"eliminate level {k}" if k < 10 else f"backsub, level {k - 11} from the top")
        print(f"  [{k:2d}] {nm:26s} {ns[k]:8.2f} us")
print(f"  sum {ns[:40].sum():.1f} us; with clocks on: {1e6 * s['device_seconds'] / K:.1f} us/iteration")
