"""IMU streams and frames stamped with Unix time, as a recording made with the host clock reaches vcgpu_set_imu and
vcgpu_set_frames, each builder asserting the regime it claims.

At E = 1.76e9 s, in [2^30, 2^31), one binary64 ulp is 2^-22 s (2.4e-7 s).  Every time sum the reference forms rounds
there: t_i + ts, the RK4 midpoint z0.time + dt/2 (so the midpoint weight alpha departs from 0.5 by up to ulp/2 / dt:
2.4e-5 at 200 Hz, 1.2e-4 at 1 kHz) and z0.time + dt.  At the small origins of synth (t ~ 1-70 s) the same sums are
exact to ~1e-13 of a step, so a kernel that reassociated them, or rebased the stamps, would pass every other test.

restamp(p)   p with ftime and imu_t moved to fl(t + E).  The signals stay the ones synth drew at the small origin: a
             stamp moves by at most 2^-23 s, and synth's trajectory is never evaluated at absolute time (its sin(f t)
             and h = 1e-4 differences would lose seven digits there).
twin(p)      (small, epoch): the same stream with every stamp and ts on the 2^-21 s grid, epoch = small + E.  On that
             grid every sum the reference forms is exact at both origins: t_i + ts and t_i + E need bits from 2^30
             down to 2^-21 (52 places); dt is a multiple of 2^-21, dt / 2 of 2^-22, and z0.time + dt / 2 lands on the
             2^-22 ulp of [2^30, 2^31); differences of nearby stamps are exact (Sterbenz).  Every inertial result is
             therefore a function of the same bits at both origins and must be bit-identical: a product with a stamp,
             a stamp narrowed to float, or any other dependence on the absolute time would show.  The twins do not see
             the rounding itself (every sum is exact on the grid); realistic() does.
realistic()  every imu_streams and imu_motion problem restamped at E with an off-grid ts: >= 90 % of the sums
             t_i + ts inexact and max |alpha_mid - 0.5| >= 1e-5 * (200 Hz / rate).
rounding_tie()  an IMU-triggered camera at E with ts = 6e-8 < 2^-23: every t_j + ts rounds back to t_j, so every frame
             is tied in binary64 and none in exact arithmetic, and HasElement covers frame 0 only by rounding.
"""
import dataclasses
from fractions import Fraction

import numpy as np

import imu_motion
import imu_streams
from vicalib_b200 import synth

E = 1_760_000_000.0  # a 2025 Unix time, in [2^30, 2^31): ulp 2^-22 s
GRID = 2.0 ** -21
assert 2.0 ** 30 <= E < 2.0 ** 31 and np.spacing(E) == 2.0 ** -22


def restamp(p, e=E):
    """p with ftime and imu_t replaced by fl(t + e); signals, poses and ts as they were"""
    return dataclasses.replace(p, ftime=np.asarray(p.ftime, dtype=np.float64) + e,
                               imu_t=np.asarray(p.imu_t, dtype=np.float64) + e)


def on_grid(x):
    return np.round(np.asarray(x, dtype=np.float64) / GRID) * GRID


def twin(p):
    """(small, epoch) of p's stream with ftime, imu_t and ts on the 2^-21 s grid.  Ties of p (t_i + ts == ftime[k]) are
    kept: the tied frame is set to the rounded sample's stamp plus the rounded ts, which is on the grid and exact."""
    ts = float(on_grid(p.ts))
    t, ft = on_grid(p.imu_t), on_grid(p.ftime)
    tt0 = np.asarray(p.imu_t, dtype=np.float64) + float(p.ts)
    for k, f in enumerate(p.ftime):
        j = np.flatnonzero(tt0 == f)
        if len(j):
            ft[k] = t[j[0]] + ts
    small = dataclasses.replace(p, imu_t=t, ftime=ft, ts=ts)
    epoch = restamp(small)
    for q in (small, epoch):
        assert np.all(np.diff(q.imu_t) > 0) and np.all(np.diff(q.ftime) > 0)
        assert exact_sums(q), "a stamp off the grid"
    assert np.array_equal(epoch.imu_t - E, small.imu_t) and np.array_equal(epoch.ftime - E, small.ftime)
    cs, ce = imu_streams.classify(small), imu_streams.classify(epoch)
    for k in cs:
        assert np.array_equal(cs[k], ce[k]), k
    c0 = imu_streams.classify(p)
    for k in ("covered", "tie_start", "tie_end", "clamped", "single"):  # the grid kept the stream's edges
        assert np.array_equal(cs[k], c0[k]), k
    return small, epoch


def exact_sums(p):
    """every stamp and ts on the grid, so that no t_i + ts and no RK4 midpoint rounds in binary64"""
    on = all(np.array_equal(on_grid(x), np.asarray(x, dtype=np.float64)) for x in (p.imu_t, p.ftime, p.ts))
    return on and inexact_fraction(p) == 0.0 and alpha_departure(p)[0] == 0.0


def inexact_fraction(p):
    """the fraction of the sums t_i + ts that round in binary64: (t + ts) - t != ts, the subtraction exact by Sterbenz"""
    t = np.asarray(p.imu_t, dtype=np.float64)
    ts = float(p.ts)
    return float(np.mean((t + ts) - t != ts)) if len(t) else 0.0


def alpha_departure(p):
    """(max |alpha_mid - 0.5|, median sample spacing): the RK4 midpoint weight of every pair of adjacent samples,
    alpha = (z1 - (z0 + dt / 2)) / (z1 - z0) with z = t + ts, in binary64 as the kernels form it"""
    tt = np.asarray(p.imu_t, dtype=np.float64) + float(p.ts)
    if len(tt) < 2:
        return 0.0, np.inf
    dt = tt[1:] - tt[:-1]
    alpha = (tt[1:] - (tt[:-1] + dt / 2.0)) / (tt[1:] - tt[:-1])
    return float(np.abs(alpha - 0.5).max()), float(np.median(np.diff(p.imu_t)))


@dataclasses.dataclass
class Epoch:
    name: str
    p: synth.Problem        # at E
    small: synth.Problem    # the same problem at its small origin
    cls: dict               # imu_streams.classify(p)
    changed: dict           # classification keys whose value differs from the small origin's: {key: intervals}
    inexact: float
    alpha: float


REALISTIC = tuple(imu_streams.NAMES) + tuple(imu_motion.NAMES)


def _source(name):
    if name in imu_streams.BUILDERS:
        return imu_streams.perturbed(imu_streams.build(name).p)
    return imu_motion.build(name).p  # already perturbed


def realistic(name):
    """imu_streams / imu_motion problem `name` at E.  Streams whose own ts is 0 (on every grid) take imu_streams.TS."""
    small = _source(name)
    if float(small.ts) == 0.0:
        small = dataclasses.replace(small, ts=imu_streams.TS)
    p = restamp(small)
    t = np.concatenate([p.imu_t, p.ftime])
    assert np.all((t >= 2.0 ** 30) & (t < 2.0 ** 31))
    assert np.all(np.diff(p.imu_t) > 0) and np.all(np.diff(p.ftime) > 0)
    frac = inexact_fraction(p)
    alpha, spacing = alpha_departure(p)
    if len(p.imu_t):
        assert frac >= 0.9, (name, frac)
    if len(p.imu_t) >= 20:  # ulp / 2 / dt: the bar scales with the sample spacing (1e-5 at 200 Hz)
        assert alpha >= 1e-5 * 0.005 / spacing, (name, alpha, spacing)
    c, c0 = imu_streams.classify(p), imu_streams.classify(small)
    changed = {k: np.flatnonzero(c[k] != c0[k]).tolist() for k in c if not np.array_equal(c[k], c0[k])}
    return Epoch(name, p, small, c, changed, frac, alpha)


RT_TS = 6e-8  # below 2^-23 s, half an ulp at E: fl(t + RT_TS) == t there


def rounding_tie(n_frames=16, grid=(10, 7), seed=39):
    """An IMU-triggered camera at E: each frame stamped with the stamp of the 1 kHz sample nearest to it (moved by at
    most 0.5 ms), frame 0 on the first sample, ts = 6e-8."""
    p = synth.make_problem(models=("poly3",), n_frames=n_frames, grid=grid, inertial=True, seed=seed,
                           imu_rate=imu_streams.RATE)
    ft = p.ftime.copy()
    j = [int(np.argmin(np.abs(p.imu_t - f))) for f in ft]
    assert len(set(j)) == n_frames
    ft = p.imu_t[j].copy()
    assert np.abs(ft - p.ftime).max() <= 0.0005 + 1e-12
    p = dataclasses.replace(p, ftime=ft, imu_t=p.imu_t[j[0]:].copy(), imu_w=p.imu_w[j[0]:].copy(),
                            imu_a=p.imu_a[j[0]:].copy())
    small = imu_streams.perturbed(p)
    small.ts = RT_TS
    e = restamp(small)
    assert RT_TS < 2.0 ** -23
    tt = e.imu_t + RT_TS
    ties = np.isin(e.ftime, tt)
    assert ties.all() and np.array_equal(tt, e.imu_t)  # every frame a tie in binary64 ...
    exact = {Fraction(float(t)) + Fraction(RT_TS) for t in e.imu_t}
    assert not any(Fraction(float(f)) in exact for f in e.ftime)  # ... and none in exact arithmetic
    # HasElement at frame 0: ftime[0] >= t_0 + ts holds in binary64, not in exact arithmetic
    assert e.ftime[0] == e.imu_t[0] and e.ftime[0] >= e.imu_t[0] + RT_TS
    assert not Fraction(float(e.ftime[0])) >= Fraction(float(e.imu_t[0])) + Fraction(RT_TS)
    c, c0 = imu_streams.classify(e), imu_streams.classify(small)
    assert c["covered"].all() and c["tie_start"].all() and c["tie_end"].all() and c["comparable"].all()
    assert not np.isin(small.ftime, small.imu_t + RT_TS).any()  # no tie at the small origin
    assert not c0["tie_start"].any() and not c0["tie_end"].any()
    assert not c0["covered"][0] and c0["covered"][1:].all()
    changed = {k: np.flatnonzero(c[k] != c0[k]).tolist() for k in c if not np.array_equal(c[k], c0[k])}
    return Epoch("rounding_tie", e, small, c, changed, inexact_fraction(e), alpha_departure(e)[0])


# the twins of test_gpu_imu_epoch.py: a gentle 200 Hz rig, the vigorous 1 kHz one, and an inertial rig one of whose
# cameras no frame sees
def twin_source(name):
    if name == "gentle200":
        p = synth.make_problem(models=("poly3", "kb4"), n_frames=24, grid=(10, 7), inertial=True, seed=51)
        p.ts = 0.0021
        return imu_streams.perturbed(p)
    if name == "imu1000":
        return imu_motion.build("imu1000").p
    if name == "unseen_camera":
        import target_views

        p = target_views.unseen_camera(True).p
        p.ts = 0.0021
        return imu_streams.perturbed(p)
    raise KeyError(name)


TWINS = ("gentle200", "imu1000", "unseen_camera")
