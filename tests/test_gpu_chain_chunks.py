"""GPU: the partitioned chain solve of the inertial problem on every branch of its dispatch.

The frame counts come from the host model of the plan (chain_plan.py) for this device's SM count, so that every row of
the dispatch table is reached: narrow levels (one chunk per CTA), a wide level 0 in one round and in two, four
elimination levels, a wide level 1, a last chunk that is a separator alone, and 4 top nodes in the dense solve.  With
chunks of 8 on 132 SMs: 5, 8, 9, 10, 15, 17, 32, 33, 65, 66, 256, 257, 1056, 1057, 2049, 2113 and 8449
frames.

Each case is checked three ways:
- forward: the step against the oracle's sequential block Cholesky (1e-7 relative);
- backward error against a plain long-double reference: the scaled system (S H S + diag(D2)) x = -S g is assembled
  block-wise from the device's own normal equations and the residual of the device's step is computed in
  np.longdouble.  ||r||_inf / (||A||_inf ||x||_inf + ||S g||_inf) does not depend on the conditioning, so it catches a
  dropped coupling block that the forward check can miss.  The largest measured on an H100 80GB HBM3: 5.3e-17;
- engines: the persistent solve, the multi-launch engine (vc_chain.cuh) and the persistent solve with every level
  forced wide (VCGPU_NO_NARROW, read on every call) agree within 1e-9 relative (largest measured: 1.7e-12).
"""
import numpy as np
import pytest

import chain_plan
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu

ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
MULTI_LAUNCH = 4       # vcgpu_set_profiling bit 2
FORWARD_BAR = 1e-7
BACKWARD_BAR = 1e-12   # ~2e4 x the largest backward error measured (5.3e-17, H100 80GB HBM3)
ENGINE_BAR = 1e-9

SMS, _ = chain_plan.device_or_h100()
CASES = chain_plan.chain_cases(SMS)


def _relerr(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("n_frames,claims", CASES, ids=[str(n) for n, _ in CASES])
def test_chain_solve_chunk_boundaries(n_frames, claims, monkeypatch):
    from oracle.binding import Oracle
    from vicalib_b200.capi import Calibrator

    assert claims <= chain_plan.branches(n_frames, SMS)
    long_chain = n_frames >= 1000  # one camera and a small board keep the oracle cheap
    p = synth.make_problem(models=("poly2",), n_frames=n_frames, grid=(4, 3) if long_chain else (14, 10), inertial=True,
                           seed=21)
    o = Oracle(p, **ALL_ON)
    g = Calibrator()
    g.load(p)
    g.set_flags(**ALL_ON)
    ne_o = o.normal_equations()
    diag = np.concatenate([np.einsum("fii->fi", ne_o["B"]).ravel(), np.diag(ne_o["C"])])
    scale = 1.0 / (1.0 + np.sqrt(diag))
    D2 = np.clip(diag * scale * scale, 1e-6, 1e32) / 1e4
    x_o = o.solve_arrow(scale, D2)
    x_g = g.solve_arrow(scale, D2)
    fwd = _relerr(x_g, x_o)
    assert fwd <= FORWARD_BAR

    eta = chain_plan.backward_error(g.normal_equations(), scale, D2, x_g)
    assert eta <= BACKWARD_BAR

    g.set_profiling(MULTI_LAUNCH, False)
    x_m = g.solve_arrow(scale, D2)
    g.set_profiling(0, False)
    monkeypatch.setenv("VCGPU_NO_NARROW", "1")
    x_w = g.solve_arrow(scale, D2)
    monkeypatch.delenv("VCGPU_NO_NARROW")
    ab = max(_relerr(x_m, x_g), _relerr(x_w, x_g))
    print(f"\nchain n={n_frames}: forward {fwd:.2e}, backward {eta:.2e}, engines {ab:.2e}")
    assert ab <= ENGINE_BAR, (_relerr(x_m, x_g), _relerr(x_w, x_g))
