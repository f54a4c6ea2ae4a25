"""IMU streams of the kinds real recordings produce, cut from one 1 kHz synthetic stream, with a per-interval
classification that each builder checks against the edge it claims.

synth.make_problem's stream is uniform (200 Hz by default) and never lands a sample on a frame time.  Recordings have
dropped packets, IMUs that start after the camera, hardware-synchronised timestamps, IMUs slower than the camera and
dropped frames.  Each builder here starts from make_problem(..., imu_rate=1000.0) and keeps a subset of its samples (so
the signal stays consistent with the trajectory), then asserts that the stream really has its edge: a later change to
synth cannot quietly remove the edge from a test.

The classification restates, in binary64 as the kernels compute it, what the interpolation buffer does with interval
k = [ftime[k], ftime[k+1]] at time offset ts (interpolation-buffer.h: HasElement, GetElement, GetNext, GetRange):
  covered    HasElement(ftime[k]): ftime[k] in [t_0 + ts, t_last + ts].  Uncovered intervals have no measurements:
             zero residual rows, weights left as they are.
  interior   samples with ftime[k] < t_i + ts < min(ftime[k+1], t_last + ts): the end is clamped to the last sample.
  steps      RK4 steps of nonzero length: interior + 1 on a covered interval that does not start at the last sample.
             A tied sample adds a zero-length step, which both integrators skip.
  tie_start, tie_end   some t_i + ts == ftime[k] (resp. ftime[k+1]) exactly.
  clamped    ftime[k+1] > t_last + ts on a covered interval.
An interval with steps == 1 ("single": no interior sample, one step between two interpolated ends) has a 9 x 9
covariance of rank <= 6 (one step maps the 6 noise channels): its weight is decided by rounding (DESIGN.md,
UpdateImuWeights).  Weights are comparable between implementations where steps >= 2.
"""
import dataclasses

import numpy as np

from vicalib_b200 import synth

RATE = 1000.0
TS = 0.0021  # the time offset of the streams that do not fix their own
MODELS = ("poly3",)


@dataclasses.dataclass
class Stream:
    name: str
    p: synth.Problem
    cls: dict
    untouched_frames: tuple = ()  # frames no covered interval touches (partial coverage)


def _base(n_frames, grid, seed):
    return synth.make_problem(models=MODELS, n_frames=n_frames, grid=grid, inertial=True, seed=seed, imu_rate=RATE)


def _keep(p, idx):
    idx = np.asarray(idx, dtype=np.int64)
    return dataclasses.replace(p, imu_t=p.imu_t[idx].copy(), imu_w=p.imu_w[idx].copy(), imu_a=p.imu_a[idx].copy())


def classify(p, ts=None):
    """Per-interval classification of p's stream at offset ts (default p.ts); see the module docstring."""
    ts = float(p.ts if ts is None else ts)
    t, ft = np.asarray(p.imu_t, dtype=np.float64), np.asarray(p.ftime, dtype=np.float64)
    ni, n = len(ft) - 1, len(t)
    tt = t + ts
    out = {k: np.zeros(ni, dtype=bool) for k in ("covered", "tie_start", "tie_end", "clamped")}
    out["interior"] = np.zeros(ni, dtype=np.int64)
    out["steps"] = np.zeros(ni, dtype=np.int64)
    for k in range(ni):
        t0, t1 = ft[k], ft[k + 1]
        cov = n > 0 and t0 >= t[0] + ts and t0 <= t[-1] + ts
        out["covered"][k] = cov
        out["tie_start"][k] = bool(np.any(tt == t0))
        out["tie_end"][k] = bool(np.any(tt == t1))
        if not cov:
            continue
        t_end = min(t1, tt[-1])
        out["clamped"][k] = t1 > tt[-1]
        out["interior"][k] = int(np.count_nonzero((tt > t0) & (tt < t_end)))
        out["steps"][k] = out["interior"][k] + (1 if t_end > t0 else 0)
    out["single"] = out["covered"] & (out["steps"] == 1)
    out["comparable"] = out["covered"] & (out["steps"] >= 2)
    return out


def guess_offsets(p, ts=None):
    """GetElement's first guess minus the index it settles on, at every frame time inside the stream: how far the walk
    goes (the guess is (time - t_0 + ts) / average_dt with the running average of AddElement)."""
    ts = float(p.ts if ts is None else ts)
    t = np.asarray(p.imu_t, dtype=np.float64)
    avg = 0.0
    for i in range(len(t)):
        avg = (avg * i + (t[i] - t[i - 1] if i else 0.0)) / (i + 1)
    off = []
    for f in p.ftime:
        if not (t[0] + ts < f < t[-1] + ts):
            continue
        guess = min(int((f - t[0] + ts) / avg), len(t) - 1)
        off.append(guess - (int(np.searchsorted(t + ts, f, side="left")) - 1))
    return np.array(off)


def _check_stream(p):
    assert np.all(np.diff(p.imu_t) > 0), "timestamps must strictly increase"
    assert len(p.imu_t) == len(p.imu_w) == len(p.imu_a)


def jittered(n_frames=16, grid=(10, 7), seed=31):
    """A random quarter of the 1 kHz samples: gaps of 1-10+ ms, so GetElement's guess walks several samples back and
    forward."""
    p = _base(n_frames, grid, seed)
    rng = np.random.default_rng(seed)
    p = _keep(p, np.sort(rng.choice(len(p.imu_t), len(p.imu_t) // 4, replace=False)))
    p.ts = TS
    _check_stream(p)
    off = guess_offsets(p)
    assert off.max() >= 3 and off.min() <= -3, off  # long walks in both directions
    c = classify(p)
    assert c["covered"].all() and c["comparable"].all()
    return Stream("jittered", p, c)


def short_gaps(n_frames=16, grid=(10, 7), seed=32):
    """Holes of 20-25 ms around every third frame time; every interval keeps interior samples."""
    p = _base(n_frames, grid, seed)
    keep = np.ones(len(p.imu_t), dtype=bool)
    holes = []
    for i, f in enumerate(range(2, n_frames - 1, 3)):
        a = p.ftime[f] - 0.012 + 0.001 * (i % 3)
        keep &= ~((p.imu_t > a) & (p.imu_t < a + 0.0215 + 0.001 * (i % 3)))
        holes.append(f)
    p = _keep(p, np.flatnonzero(keep))
    p.ts = TS
    _check_stream(p)
    gaps = np.diff(p.imu_t)
    big = gaps[gaps > 0.005]
    assert len(big) == len(holes) and big.min() >= 0.020 and big.max() <= 0.025, big
    c = classify(p)
    assert c["covered"].all() and c["comparable"].all()
    assert np.abs(guess_offsets(p)).max() >= 5  # the guess lands across a hole
    return Stream("short_gaps", p, c)


LONG_GAP = (4, 5, 6)


def long_gap(n_frames=16, grid=(10, 7), seed=33):
    """No samples from 10 ms before frame 4 to 2 ms after frame 7: intervals 4, 5, 6 have no interior sample (one RK4
    step between two interpolated ends)."""
    p = _base(n_frames, grid, seed)
    gap = (p.imu_t > p.ftime[4] - 0.01) & (p.imu_t < p.ftime[7] + 0.002)
    p = _keep(p, np.flatnonzero(~gap))
    p.ts = TS
    _check_stream(p)
    c = classify(p)
    assert c["covered"].all()
    assert tuple(np.flatnonzero(c["single"])) == LONG_GAP, np.flatnonzero(c["single"])
    assert c["comparable"].sum() == len(c["covered"]) - len(LONG_GAP)
    return Stream("long_gap", p, c)


def slow(hz, n_frames=16, grid=(10, 7), seed=34):
    """Every (1000 / hz)-th sample: an IMU slower than the 30 Hz camera.  45 Hz leaves 1-2 interior samples per
    interval (two- and three-step intervals), 20 Hz 0-1 (one- and two-step intervals)."""
    p = _base(n_frames, grid, seed)
    p = _keep(p, np.arange(0, len(p.imu_t), int(round(RATE / hz))))
    p.ts = TS
    _check_stream(p)
    c = classify(p)
    assert c["covered"].all()
    want = {45: {1, 2}, 20: {0, 1}}[hz]
    assert set(c["interior"].tolist()) == want, c["interior"]
    return Stream(f"imu{hz}", p, c)


def partial(n_frames=20, grid=(10, 7), seed=35):
    """The IMU starts after frame 2 and ends 10 ms before frame n-3: intervals 0-2 and n-3, n-2 have no measurements
    (HasElement is false), interval n-4 ends on the last sample (the end-of-buffer clamp).  Intervals 2 (uncovered) and
    3 (covered) share a warp of the weights kernel (intervals 2k, 2k+1), and so do n-4 (covered) and n-3 (uncovered).
    Frames 0-2, n-2 and n-1 are touched by no covered interval."""
    assert n_frames % 2 == 0
    p = _base(n_frames, grid, seed)
    p = _keep(p, np.flatnonzero((p.imu_t > p.ftime[2] + 0.004) & (p.imu_t < p.ftime[n_frames - 3] - 0.01)))
    p.ts = 0.0
    _check_stream(p)
    c = classify(p)
    ni = n_frames - 1
    want = np.zeros(ni, dtype=bool)
    want[3:ni - 2] = True
    assert np.array_equal(c["covered"], want), c["covered"]
    assert np.flatnonzero(c["clamped"]).tolist() == [ni - 3]
    assert np.array_equal(c["comparable"], want)
    assert (ni - 3) % 2 == 0  # the clamped interval and the uncovered one after it share a warp
    return Stream("partial", p, c, untouched_frames=(0, 1, 2, n_frames - 2, n_frames - 1))


def tied(exact_ts, n_frames=16, grid=(10, 7), seed=36):
    """Frame times set onto sample times at every other frame, so that t_j + ts == ftime[f] in binary64: with ts = 0
    (exact_ts False) and with ts = TS (ftime[f] = fl(t_j + TS)).  A tied frame ends one interval and starts the next:
    zero-length RK4 steps in both integrators, and GetElement's index on a tie.  250 Hz stream."""
    p = _base(n_frames, grid, seed)
    p = _keep(p, np.arange(0, len(p.imu_t), 4))
    ts = TS if exact_ts else 0.0
    ft = p.ftime.copy()
    tied_frames = list(range(1, n_frames - 1, 2))
    for f in tied_frames:
        j = int(np.argmin(np.abs(p.imu_t + ts - ft[f])))
        ft[f] = p.imu_t[j] + ts
        assert p.imu_t[j] + ts == ft[f] and abs(ft[f] - p.ftime[f]) < 0.0021
    p.ftime, p.ts = ft, ts
    _check_stream(p)
    assert np.all(np.diff(p.ftime) > 0)
    c = classify(p)
    for f in tied_frames:
        assert c["tie_end"][f - 1] and c["tie_start"][f], f
    assert c["covered"].all() and c["comparable"].all()
    return Stream("tied_ts" if exact_ts else "tied_ts0", p, c)


DROPPED = range(5, 20)  # frames removed: interval 4 spans 0.53 s


def dropped(n_frames=32, grid=(10, 7), seed=37):
    """Frames 5-19 dropped (observations re-indexed): interval 4 runs over ~530 samples, its warp mate, interval 5,
    over ~33; the two 16-lane teams of that warp run very unequal step counts."""
    p = _base(n_frames, grid, seed)
    keep_f = np.array([f for f in range(n_frames) if f not in DROPPED])
    remap = -np.ones(n_frames, dtype=np.int32)
    remap[keep_f] = np.arange(len(keep_f), dtype=np.int32)
    sel = remap[p.obs_frame] >= 0
    truth = dict(p.truth, T_wp=p.truth["T_wp"][keep_f], v_w=p.truth["v_w"][keep_f])
    p = dataclasses.replace(p, T_wp=p.T_wp[keep_f].copy(), v_w=p.v_w[keep_f].copy(), ftime=p.ftime[keep_f].copy(),
                            obs_frame=remap[p.obs_frame[sel]], obs_cam=p.obs_cam[sel].copy(), p_w=p.p_w[sel].copy(),
                            p_c=p.p_c[sel].copy(), grid_idx=p.grid_idx[sel].copy(), truth=truth)
    p.ts = TS
    _check_stream(p)
    c = classify(p)
    assert c["covered"].all() and c["comparable"].all()
    assert c["interior"][4] >= 450 and c["interior"][5] <= 40, c["interior"][4:6]
    assert c["interior"][4] >= 10 * c["interior"][np.arange(len(c["interior"])) != 4].max()
    return Stream("dropped", p, c)


def few_samples(n, n_frames=12, grid=(10, 7), seed=38):
    """0, 1 or 2 samples.  One sample sits exactly on frame 3: HasElement holds for interval 3 alone (a zero-step
    interval), and average_dt is 0.  Two samples straddle frames 4 and 5: intervals 4 and 5 are single-step (the second
    ends on the buffer's clamp), average_dt is half their spacing.  Every other interval has no measurements."""
    p = _base(n_frames, grid, seed)
    ft = p.ftime
    if n == 0:
        idx = []
    elif n == 1:
        idx = [int(np.argmin(np.abs(p.imu_t - ft[3])))]
    else:
        idx = [int(np.searchsorted(p.imu_t, 0.5 * (ft[3] + ft[4]))), int(np.searchsorted(p.imu_t, 0.5 * (ft[5] + ft[6])))]
    p = _keep(p, idx)
    if n == 1:
        p.ftime = ft.copy()
        p.ftime[3] = p.imu_t[0]
    p.ts = 0.0
    _check_stream(p)
    c = classify(p)
    want = {0: [], 1: [3], 2: [4, 5]}[n]
    assert np.flatnonzero(c["covered"]).tolist() == want
    assert np.all(c["steps"][want] == (0 if n == 1 else 1))
    return Stream(f"samples{n}", p, c)


BUILDERS = {
    "jittered": jittered,
    "short_gaps": short_gaps,
    "long_gap": long_gap,
    "imu45": lambda: slow(45),
    "imu20": lambda: slow(20),
    "partial": partial,
    "tied_ts0": lambda: tied(False),
    "tied_ts": lambda: tied(True),
    "dropped": dropped,
    "samples0": lambda: few_samples(0),
    "samples1": lambda: few_samples(1),
    "samples2": lambda: few_samples(2),
}
NAMES = tuple(BUILDERS)
# every covered interval has >= 2 steps: weights comparable everywhere, live-weight solves compared with the oracle
COMPARABLE = ("jittered", "short_gaps", "imu45", "partial", "tied_ts0", "tied_ts", "dropped")


def build(name):
    return BUILDERS[name]()


def ts_kinks(z):
    """Intervals with a sample exactly on an end (t_i + ts == ftime).  The residual has a kink in ts there: the
    interpolated signal's slope jumps at the sample, so the central difference averages two one-sided derivatives, and
    the dual-number derivative follows the branch GetElement / GetNext take (a zero-length step, whose derivative the
    integrator drops).  Column 32 (ts) of those intervals is not compared; all other columns are."""
    tt = z["imu_t"] + float(z["ts"])
    return np.array([np.isin(z["ftime"][k:k + 2], tt).any() for k in range(len(z["ftime"]) - 1)])


def perturbed(p, seed=3):
    """p with a state away from the truth, so that every Jacobian column is exercised: biases, scale factors and
    velocities perturbed (the poses already are)."""
    rng = np.random.default_rng(seed)
    q = dataclasses.replace(p)
    q.b = 1e-2 * rng.standard_normal(6)
    q.sf = 1 + 1e-2 * rng.standard_normal(6)
    q.v_w = p.truth["v_w"] + 1e-2 * rng.standard_normal(p.v_w.shape)
    return q
