"""Generates the known-answer fixtures in tests/golden/ (run once, here; fixtures are committed).

The reference pins nothing for this path (its only test needs a tarball fetched at configure time
and uses the linear model, testing/vi_sim_test.cpp:18-21), and none of Ceres / Calibu / Sophus /
Eigen can be imported in this container.  These vectors are therefore produced by an INDEPENDENT
restatement in 60-digit mpmath arithmetic — rotation matrices instead of quaternions, Rodrigues
formulae instead of Sophus' quaternion exp/log, exact central differences (h = 1e-25) instead of
dual numbers — of the same published formulas:
    reprojection  r = Project(R_ck R_wk^T (p_w - t_wk) + p_ck) - z       ceres-cost-functions.h:361-370
    IMU           r = W^T [log(T_end T_2^-1); v_end - v2], RK4 integration ceres-cost-functions.h:138-177,402-484
Both the oracle (C++, float64 dual numbers) and the CUDA kernels are checked against them.

    python tests/golden/make_golden.py
"""
import os
import sys

import mpmath as mp
import numpy as np

mp.mp.dps = 60
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

LINEAR, FOV, POLY2, POLY3, KB4 = range(5)
NUM_INTR = {LINEAR: 4, FOV: 5, POLY2: 6, POLY3: 7, KB4: 8}


def M(a):
    return mp.matrix([[mp.mpf(float(x)) for x in row] for row in np.atleast_2d(a)])


def V(a):
    return mp.matrix([mp.mpf(float(x)) for x in a])


def quat_R(q):
    x, y, z, w = [mp.mpf(float(v)) for v in q]
    n = mp.sqrt(x * x + y * y + z * z + w * w)
    x, y, z, w = x / n, y / n, z / n, w / n
    return mp.matrix([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def hat(w):
    return mp.matrix([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])


def so3_exp(w):
    th = mp.sqrt(w[0] ** 2 + w[1] ** 2 + w[2] ** 2)
    W = hat(w)
    if th == 0:
        return mp.eye(3)
    return mp.eye(3) + mp.sin(th) / th * W + (1 - mp.cos(th)) / th ** 2 * W * W


def so3_V(w):
    th = mp.sqrt(w[0] ** 2 + w[1] ** 2 + w[2] ** 2)
    W = hat(w)
    if th == 0:
        return mp.eye(3)
    return mp.eye(3) + (1 - mp.cos(th)) / th ** 2 * W + (th - mp.sin(th)) / th ** 3 * W * W


def so3_log(R):
    c = (R[0, 0] + R[1, 1] + R[2, 2] - 1) / 2
    th = mp.acos(c)
    if th == 0:
        return mp.matrix([0, 0, 0])
    f = th / (2 * mp.sin(th))
    return mp.matrix([f * (R[2, 1] - R[1, 2]), f * (R[0, 2] - R[2, 0]), f * (R[1, 0] - R[0, 1])])


def se3_log(R, t):
    w = so3_log(R)
    return list(mp.inverse(so3_V(w)) * t) + list(w)


def se3_plus(R, t, d):  # T * exp(upsilon, omega)   (local-param-se3.h:14-26)
    ups, om = mp.matrix(d[:3]), mp.matrix(d[3:])
    return R * so3_exp(om), t + R * (so3_V(om) * ups)


def project(model, p, k):
    X, Y, Z = p
    if model == KB4:
        rho = mp.sqrt(X * X + Y * Y)
        th = mp.atan2(rho, Z)
        d = th + k[4] * th ** 3 + k[5] * th ** 5 + k[6] * th ** 7 + k[7] * th ** 9
        return [k[0] * d * X / rho + k[2], k[1] * d * Y / rho + k[3]]
    u, v = X / Z, Y / Z
    r2 = u * u + v * v
    if model == LINEAR:
        f = 1
    elif model == FOV:  # Calibu FovCamera::Factor: the two small-argument branches are part of the model
        w = k[4]
        if w * w > mp.mpf("1e-5"):
            if r2 < mp.mpf("1e-5"):
                f = 2 * mp.tan(w / 2) / w
            else:
                rad = mp.sqrt(r2)
                f = mp.atan(rad * 2 * mp.tan(w / 2)) / (rad * w)
        else:
            f = mp.mpf(1)
    elif model == POLY2:
        f = 1 + k[4] * r2 + k[5] * r2 ** 2
    else:
        f = 1 + k[4] * r2 + k[5] * r2 ** 2 + k[6] * r2 ** 3
    return [k[0] * f * u + k[2], k[1] * f * v + k[3]]


def reproj(model, Rwk, twk, Rck, pck, intr, pw, z):
    pc = Rck * (Rwk.T * (pw - twk)) + pck
    pr = project(model, pc, intr)
    return [pr[0] - z[0], pr[1] - z[1]]


def random_sample(rng, model, tgt=None, dist=None):
    """(T_wk, T_ck, intrinsics, world point, measurement); tgt = the point's camera-frame coordinates."""
    K = NUM_INTR[model]
    from vicalib_b200.synth import TRUTH_DIST, quat_to_mat, so3_exp as np_exp
    q = np_exp(rng.normal(0, 0.6, 3)); t = rng.normal(0, 0.2, 3) + np.array([0, 0, -0.6])
    qc = np_exp(rng.normal(0, 0.3, 3)); pc = rng.normal(0, 0.05, 3)
    intr = np.zeros(10)
    intr[:4] = [300 + 30 * rng.random(), 310 + 30 * rng.random(), 320 + 5 * rng.random(), 240 + 5 * rng.random()]
    intr[4:K] = np.array(TRUTH_DIST[model]) * (1 + 0.2 * rng.random(K - 4))
    if dist is not None:
        intr[4:K] = dist
    # a world point in front of the camera: p_w = R_wk (R_ck^T (pc_target - p_ck)) + t
    if tgt is None:
        tgt = np.array([rng.uniform(-0.25, 0.25), rng.uniform(-0.2, 0.2), rng.uniform(0.4, 0.8)])
    pw = quat_to_mat(q) @ (quat_to_mat(qc).T @ (np.asarray(tgt, float) - pc)) + t
    z = rng.uniform(100, 500, 2)
    return q, t, qc, pc, intr, pw, z


def reproj_kat(rng, model, n=12, samples=None):
    K = NUM_INTR[model]
    rows = []
    if samples is None:
        samples = [random_sample(rng, model) for _ in range(n)]
    for q, t, qc, pc, intr, pw, z in samples:
        Rwk, Rck = quat_R(q), quat_R(qc)
        a = (model, Rwk, V(t), Rck, V(pc), [mp.mpf(float(x)) for x in intr], V(pw), V(z))
        r = reproj(*a)
        h = mp.mpf(10) ** -25
        J = np.zeros((2, 12 + K))
        col = 0

        def fd(fp, fm):
            return [(x - y) / (2 * h) for x, y in zip(fp, fm)]

        for k in range(6):  # frame pose, right perturbation
            d = [mp.mpf(0)] * 6
            d[k] = h
            Rp, tp = se3_plus(Rwk, V(t), d)
            d[k] = -h
            Rm, tm = se3_plus(Rwk, V(t), d)
            g = fd(reproj(model, Rp, tp, Rck, V(pc), a[5], V(pw), V(z)), reproj(model, Rm, tm, Rck, V(pc), a[5], V(pw), V(z)))
            J[:, col] = [float(x) for x in g]; col += 1
        for k in range(3):  # R_ck * exp(w)
            w = [mp.mpf(0)] * 3
            w[k] = h
            Rp = Rck * so3_exp(mp.matrix(w))
            w[k] = -h
            Rm = Rck * so3_exp(mp.matrix(w))
            g = fd(reproj(model, Rwk, V(t), Rp, V(pc), a[5], V(pw), V(z)), reproj(model, Rwk, V(t), Rm, V(pc), a[5], V(pw), V(z)))
            J[:, col] = [float(x) for x in g]; col += 1
        for k in range(3):
            e = mp.matrix([0, 0, 0]); e[k] = h
            g = fd(reproj(model, Rwk, V(t), Rck, V(pc) + e, a[5], V(pw), V(z)), reproj(model, Rwk, V(t), Rck, V(pc) - e, a[5], V(pw), V(z)))
            J[:, col] = [float(x) for x in g]; col += 1
        for k in range(K):
            ip, im = list(a[5]), list(a[5])
            ip[k] += h; im[k] -= h
            g = fd(reproj(model, Rwk, V(t), Rck, V(pc), ip, V(pw), V(z)), reproj(model, Rwk, V(t), Rck, V(pc), im, V(pw), V(z)))
            J[:, col] = [float(x) for x in g]; col += 1
        rows.append(dict(T_wk=np.concatenate([q, t]), q_ck=qc, p_ck=pc, intr=intr, p_w=pw, z=z,
                         r=np.array([float(x) for x in r]), J=J))
    return {k: np.stack([r_[k] for r_ in rows]) for k in rows[0]}


# ------------------------------------------------------------------ IMU
GRAV = mp.mpf("9.8007")


def gravity_vec(g):
    sp, cp, sq, cq = mp.sin(g[0]), mp.cos(g[0]), mp.sin(g[1]), mp.cos(g[1])
    return mp.matrix([-GRAV * cp * sq, GRAV * sp, -GRAV * cp * cq])


def get_range(t, w, a, ts, t0, t1):
    """[interp(t0), samples with t0 < t_i + ts <= t1, interp(t1)] (interpolation-buffer.h:208-226).  A time at or past
    the last sample gives that sample, at its own time (GetElement's end-of-buffer clamp)."""
    tt = [x + ts for x in t]

    def interp(time):
        if time >= tt[-1]:
            return (tt[-1], w[-1], a[-1])
        i = max(k for k in range(len(tt)) if tt[k] <= time)
        f = (time - tt[i]) / (tt[i + 1] - tt[i])
        return (time, w[i] * (1 - f) + w[i + 1] * f, a[i] * (1 - f) + a[i + 1] * f)

    out = [interp(t0)]
    i0 = max(k for k in range(len(tt)) if tt[k] <= t0)
    for k in range(i0 + 1, len(tt)):
        if tt[k] > t1:
            break
        out.append((tt[k], w[k], a[k]))
    out.append(interp(t1))
    return out


def imu_residual(t, w, a, t0, t1, R2, p2, v2, R1, p1, v1, g, b, sf, ts, W, switch, integrator=None):
    p, R, v = (integrator or integrate)(t, w, a, t0, t1, R1, p1, v1, g, b, sf, ts)
    Re = R * R2.T
    te = p - Re * p2
    raw = se3_log(Re, te) + list(v - v2)
    r = [sum(raw[i] * W[i, j] for i in range(9)) for j in range(9)]
    if switch:
        for j in (0, 1, 2, 6, 7, 8):
            r[j] = mp.mpf(0)
    return r


def integrate(t, w, a, t0, t1, R1, p1, v1, g, b, sf, ts):
    """(p, R, v) at t1 from (p1, R1, v1) at t0: RK4 over the measurements of get_range"""
    gv = gravity_vec(g)
    bg, ba = mp.matrix(b[:3]), mp.matrix(b[3:])
    meas = get_range(t, w, a, ts, t0, t1)
    p, R, v = p1, R1, v1

    def deriv(p_, R_, v_, z0, z1, dt):
        al = (z1[0] - (z0[0] + dt)) / (z1[0] - z0[0])
        zg = z0[1] * al + z1[1] * (1 - al)
        za = z0[2] * al + z1[2] * (1 - al)
        wv = R_ * mp.matrix([zg[i] * sf[i] + bg[i] for i in range(3)])
        av = R_ * mp.matrix([za[i] * sf[3 + i] + ba[i] for i in range(3)]) - gv
        return v_, wv, av

    def step(p_, R_, v_, k, dt):
        return p_ + k[0] * dt, so3_exp(k[1] * dt) * R_, v_ + k[2] * dt

    for z0, z1 in zip(meas[:-1], meas[1:]):
        dt = z1[0] - z0[0]
        if dt == 0:
            continue
        k1 = deriv(p, R, v, z0, z1, 0)
        y1 = step(p, R, v, k1, dt / 2)
        k2 = deriv(*y1, z0, z1, dt / 2)
        y2 = step(p, R, v, k2, dt / 2)
        k3 = deriv(*y2, z0, z1, dt / 2)
        y3 = step(p, R, v, k3, dt)
        k4 = deriv(*y3, z0, z1, dt)
        k = [k1[i] + 2 * k2[i] + 2 * k3[i] + k4[i] for i in range(3)]
        p, R, v = step(p, R, v, k, dt / 6)
    return p, R, v


def imu_kat(rng):
    from vicalib_b200.synth import so3_exp as np_exp
    n = 40
    t = 0.1 + 0.005 * np.arange(n) + 0.0003 * rng.random(n)
    w = rng.normal(0, 0.4, (n, 3)); a = rng.normal(0, 1.0, (n, 3)) + np.array([0.3, 9.7, 0.5])
    ftime = np.array([0.123, 0.151, 0.1837, 0.2169])
    nf = len(ftime)
    q = np.stack([np_exp(rng.normal(0, 0.5, 3)) for _ in range(nf)])
    p = rng.normal(0, 0.3, (nf, 3)); v = rng.normal(0, 0.5, (nf, 3))
    g = np.array([0.05, -0.03]); b = np.concatenate([rng.normal(0, 1e-2, 3), rng.normal(0, 1e-1, 3)])
    sf = 1 + 0.02 * rng.normal(size=6); ts = 0.0023
    W = 500 * np.eye(9) + 20 * rng.normal(size=(9, 9))
    out_r, out_J = imu_rows(t, w, a, ftime, q, p, v, g, b, sf, ts, W, (0, 1))
    return dict(imu_t=t, imu_w=w, imu_a=a, ftime=ftime, T_wp=np.concatenate([q, p], 1), v_w=v, g=g, b=b, sf=sf, ts=np.array(ts),
                W=W, r=np.array(out_r).reshape(2, nf - 1, 9), J=np.array(out_J).reshape(2, nf - 1, 9, 33))


def imu_rows(t, w, a, ftime, q, p, v, g, b, sf, ts, W, switches, integrator=None, jac=True):
    """residual and exact central-difference 9 x 33 Jacobian (jac) of every interval, for each switch value"""
    nf = len(ftime)
    tm, wm, am = [mp.mpf(float(x)) for x in t], [V(x) for x in w], [V(x) for x in a]
    Wm = M(W)
    h = mp.mpf(10) ** -25
    out_r, out_J = [], []
    for sw in switches:
        for k in range(nf - 1):
            base = dict(R2=quat_R(q[k + 1]), p2=V(p[k + 1]), v2=V(v[k + 1]), R1=quat_R(q[k]), p1=V(p[k]), v1=V(v[k]),
                        g=[mp.mpf(float(x)) for x in g], b=[mp.mpf(float(x)) for x in b], sf=[mp.mpf(float(x)) for x in sf],
                        ts=mp.mpf(ts))

            def ev(**kw):
                d = dict(base); d.update(kw)
                return imu_residual(tm, wm, am, mp.mpf(float(ftime[k])), mp.mpf(float(ftime[k + 1])), d["R2"], d["p2"], d["v2"],
                                    d["R1"], d["p1"], d["v1"], d["g"], d["b"], d["sf"], d["ts"], Wm, sw, integrator)

            r0 = ev()
            out_r.append([float(x) for x in r0])
            if not jac:
                continue
            cols = []

            def fd(kp, km):
                rp, rm = ev(**kp), ev(**km)
                cols.append([float((x - y) / (2 * h)) for x, y in zip(rp, rm)])

            for which in ("2", "1"):
                R, pp = base["R" + which], base["p" + which]
                for j in range(6):
                    d = [mp.mpf(0)] * 6
                    d[j] = h
                    Rp, tp = se3_plus(R, pp, d)
                    d[j] = -h
                    Rm, tm_ = se3_plus(R, pp, d)
                    fd({"R" + which: Rp, "p" + which: tp}, {"R" + which: Rm, "p" + which: tm_})
            for which in ("v2", "v1"):
                for j in range(3):
                    e = mp.matrix([0, 0, 0]); e[j] = h
                    fd({which: base[which] + e}, {which: base[which] - e})
            for name, cnt in (("g", 2), ("b", 6), ("sf", 6)):
                for j in range(cnt):
                    lp, lm = list(base[name]), list(base[name])
                    lp[j] += h; lm[j] -= h
                    fd({name: lp}, {name: lm})
            fd({"ts": base["ts"] + h}, {"ts": base["ts"] - h})
            out_J.append(np.array(cols).T)
    return out_r, out_J


# time unit of the edge stream: sample times, frame times and ts are multiples of U / 4, so every t_i + ts is exact in
# binary64 and in mpmath alike, and a tie is a tie in both
U = 1.0 / 1024
EDGE_SAMPLES = [0, 3, 5, 9, 10, 14, 20, 21, 27, 30, 38, 41, 44, 52, 55, 60, 61, 70]  # t_i = (100 + k) U
EDGE_TS = 3 * U
# interval 0 [108, 117]      a sample on each end (ties at start and end: zero-length RK4 steps)
# interval 1 [117, 118.25]   starts on a tie, no interior sample
# interval 2 [118.25, 122.5] no interior sample, two interpolated ends
# interval 3 [122.5, 130.5]  the sample at 130 U is inside at ts = 0 and pushed past the end (133 U) by ts
# interval 4 [130.5, 150.25] ordinary
# interval 5 [150.25, 180]   ends past the last sample (173 U): the end-of-buffer clamp
EDGE_FTIME = [108, 117, 118.25, 122.5, 130.5, 150.25, 180]


def imu_edge_kat():
    """The interpolation buffer's edges on an irregular stream (tests/golden/imu_edge_kat.npz, keys of imu_kat.npz with
    one switch value, 0)."""
    from vicalib_b200.synth import so3_exp as np_exp
    rng = np.random.default_rng(20261016)
    t = (100 + np.array(EDGE_SAMPLES, dtype=np.float64)) * U
    n = len(t)
    w = rng.normal(0, 0.4, (n, 3)); a = rng.normal(0, 1.0, (n, 3)) + np.array([0.3, 9.7, 0.5])
    ftime = np.array(EDGE_FTIME) * U
    nf = len(ftime)
    tt = t + EDGE_TS
    assert tt[EDGE_SAMPLES.index(5)] == ftime[0] and tt[EDGE_SAMPLES.index(14)] == ftime[1]  # the ties, in binary64
    for k in (1, 2):
        assert not np.any((tt > ftime[k]) & (tt < ftime[k + 1]))  # no interior sample
    j = EDGE_SAMPLES.index(30)
    assert ftime[3] < t[j] < ftime[4] < tt[j]  # moved across the end by ts
    assert ftime[-1] > tt[-1] and ftime[-2] < tt[-1]  # the last interval ends past the last sample
    q = np.stack([np_exp(rng.normal(0, 0.5, 3)) for _ in range(nf)])
    p = rng.normal(0, 0.3, (nf, 3)); v = rng.normal(0, 0.5, (nf, 3))
    g = np.array([0.05, -0.03]); b = np.concatenate([rng.normal(0, 1e-2, 3), rng.normal(0, 1e-1, 3)])
    sf = 1 + 0.02 * rng.normal(size=6)
    W = 500 * np.eye(9) + 20 * rng.normal(size=(9, 9))
    out_r, out_J = imu_rows(t, w, a, ftime, q, p, v, g, b, sf, EDGE_TS, W, (0,))
    return dict(imu_t=t, imu_w=w, imu_a=a, ftime=ftime, T_wp=np.concatenate([q, p], 1), v_w=v, g=g, b=b, sf=sf,
                ts=np.array(EDGE_TS), W=W, r=np.array(out_r).reshape(1, nf - 1, 9), J=np.array(out_J).reshape(1, nf - 1, 9, 33))


# interval k of the vigorous fixture: frame k + 1 = sign * (integrated end state of interval k) * Exp(angle * axis), so
# that the rotation of log(T_end T_2^-1) is `angle` and its quaternion has w = sign * cos(angle / 2) as the kernels
# compute it (the integrated end keeps the sign of frame k)
VIGOROUS_CASES = [
    (-1, 3e-11),  # converged, frame 2 of the opposite sign: w ~ -1, SO3 log's Taylor branch (|vec| < 1e-10)
    (-1, 0.9),    # opposite sign, large residual
    (+1, 2.6),    # large angle: the V^-1 coefficient far from its small-angle limit
    (-1, 2.95),   # large angle, opposite sign: w ~ -0.1
    (+1, 0.2),
    (-1, 2.75),
    (+1, 3e-11),  # converged, same sign
]
VIGOROUS_RATE = 300.0
VIGOROUS_TS = 0.0031


def imu_vigorous_kat():
    """The IMU residual under vigorous motion and across the quaternion double cover (tests/golden/imu_vigorous_kat.npz,
    keys of imu_kat.npz with both switch values): a ~300 Hz jittered stream with |w| up to ~9 rad/s (|w| dt up to ~0.03
    per RK4 step) and |a| up to ~25 m/s^2, 21-36 steps per interval, frame quaternions of both signs (frame 0 has w < 0)
    and the residual rotations of VIGOROUS_CASES."""
    from vicalib_b200.synth import mat_to_quat, quat_mul, quat_to_mat, so3_exp as np_exp
    rng = np.random.default_rng(20261018)
    nf = len(VIGOROUS_CASES) + 1
    lengths = rng.uniform(0.07, 0.12, nf - 1)
    ftime = 0.15 + np.concatenate([[0.0], np.cumsum(lengths)])
    n = int((ftime[-1] - 0.1) * VIGOROUS_RATE) + 15
    t = 0.1 + (np.arange(n) + 0.25 * rng.random(n)) / VIGOROUS_RATE
    f, ph = rng.uniform(1.5, 3.0, (2, 3)), rng.uniform(0, 2 * np.pi, (2, 3))
    w = np.array([6.0, 5.0, 6.5]) * np.sin(2 * np.pi * f[0] * t[:, None] + ph[0]) + rng.normal(0, 0.05, (n, 3))
    a = np.array([0.3, 9.7, 0.5]) + np.array([12.0, 10.0, 13.0]) * np.sin(2 * np.pi * f[1] * t[:, None] + ph[1])
    a += rng.normal(0, 0.05, (n, 3))
    tt = t + VIGOROUS_TS
    assert np.all(np.diff(t) > 0) and tt[0] < ftime[0] and tt[-1] > ftime[-1]
    assert np.abs(tt[:, None] - ftime[None, :]).min() > 1e-5  # no sample near a frame time: no ts kink
    g = np.array([0.05, -0.03]); b = np.concatenate([rng.normal(0, 1e-2, 3), rng.normal(0, 1e-1, 3)])
    sf = 1 + 0.02 * rng.normal(size=6)
    W = 500 * np.eye(9) + 20 * rng.normal(size=(9, 9))
    q = np.zeros((nf, 4)); p = np.zeros((nf, 3)); v = np.zeros((nf, 3))
    q[0] = -np_exp(rng.normal(0, 0.5, 3)); p[0] = rng.normal(0, 0.3, 3); v[0] = rng.normal(0, 0.5, 3)
    assert q[0, 3] < 0
    tm, wm, am = [mp.mpf(float(x)) for x in t], [V(x) for x in w], [V(x) for x in a]
    mpl = lambda x: [mp.mpf(float(y)) for y in x]  # noqa: E731
    for k, (sign, angle) in enumerate(VIGOROUS_CASES):
        pe, Re, ve = integrate(tm, wm, am, mp.mpf(float(ftime[k])), mp.mpf(float(ftime[k + 1])), quat_R(q[k]), V(p[k]), V(v[k]),
                               mpl(g), mpl(b), mpl(sf), mp.mpf(VIGOROUS_TS))
        Rk = quat_to_mat(q[k])
        Re = np.array(Re.tolist(), dtype=np.float64)
        dq = mat_to_quat(Rk.T @ Re)  # the interval's rotation (< pi), w >= 0: the end keeps frame k's sign
        qe = quat_mul(q[k], dq)
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        q[k + 1] = sign * quat_mul(qe, np_exp(angle * axis))
        tiny = angle < 1e-6
        p[k + 1] = np.array([float(x) for x in pe]) + (1e-9 if tiny else 0.05) * rng.normal(size=3)
        v[k + 1] = np.array([float(x) for x in ve]) + (1e-8 if tiny else 0.1) * rng.normal(size=3)
        rel = quat_mul(qe, q[k + 1] * np.array([-1, -1, -1, 1.0]))
        assert np.sign(rel[3]) == sign and abs(2 * np.arccos(min(1.0, abs(rel[3]))) - angle) < 1e-6 + 1e-3 * angle, (k, rel)
        steps = np.count_nonzero((tt > ftime[k]) & (tt < ftime[k + 1])) + 1
        assert 20 <= steps <= 50, steps
    wdt = np.linalg.norm(w[1:], axis=1) * np.diff(t)
    print(f"vigorous: max |w| {np.linalg.norm(w, axis=1).max():.2f} rad/s, max |w| dt {wdt.max():.4f}, "
          f"max |a| {np.linalg.norm(a, axis=1).max():.1f} m/s^2", flush=True)
    out_r, out_J = imu_rows(t, w, a, ftime, q, p, v, g, b, sf, VIGOROUS_TS, W, (0, 1))
    return dict(imu_t=t, imu_w=w, imu_a=a, ftime=ftime, T_wp=np.concatenate([q, p], 1), v_w=v, g=g, b=b, sf=sf,
                ts=np.array(VIGOROUS_TS), W=W, r=np.array(out_r).reshape(2, nf - 1, 9),
                J=np.array(out_J).reshape(2, nf - 1, 9, 33))


# ------------------------------------------------------------------ IMU at Unix time
EPOCH = 1_760_000_000.0  # in [2^30, 2^31): one binary64 ulp is 2^-22 s
EPOCH_RATE = 300.0
EPOCH_TS = 0.0031


class T64:
    """A time as the reference's Jet<double> carries it: a binary64 scalar part f, which every sum rounds, and an
    exact part d, the derivative part times (ts - ts0), which never rounds; its value is f + d.  Decisions (which
    samples an interval takes, zero-length steps) read f alone, as GetElement, GetNext and HasElement read the scalar."""

    def __init__(self, f, d=0):
        self.f, self.d = float(f), mp.mpf(d)

    @property
    def v(self):
        return mp.mpf(self.f) + self.d

    def __add__(self, o):  # the scalar sum rounds to binary64 (Python float)
        return T64(self.f + o.f, self.d + o.d)

    def __sub__(self, o):  # exact: the stamps here are within a factor 2 of each other (Sterbenz)
        f = self.f - o.f
        assert mp.mpf(f) == mp.mpf(self.f) - mp.mpf(o.f)
        return T64(f, self.d - o.d)


def integrate_rounded(t, w, a, t0, t1, R1, p1, v1, g, b, sf, ts):
    """integrate() with every time sum the reference forms in binary64, in its order: t_i + ts, dt / 2 then
    z0.time + dt / 2, and z0.time + dt.  ts - ts0 (the perturbation of the ts column's differences) is carried as the
    exact part, so that each rounded sum s(ts0) continues as s(ts0) + (ts - ts0): the Jet semantics."""
    ts0 = float(ts)
    dts = ts - mp.mpf(ts0)
    assert abs(dts) < mp.mpf(10) ** -20
    tt = [T64(float(x) + ts0, dts) for x in t]
    t0, t1 = float(t0), float(t1)

    def interp(time):  # GetElement; no sample ties a frame and the frames lie inside the stream
        i = max(k for k in range(len(tt)) if tt[k].f <= time)
        tm = T64(time)
        fr = (tm - tt[i]).v / (tt[i + 1] - tt[i]).v
        return (tm, w[i] * (1 - fr) + w[i + 1] * fr, a[i] * (1 - fr) + a[i + 1] * fr)

    assert tt[0].f < t0 and t1 < tt[-1].f
    meas = [interp(t0)] + [(x, w[k], a[k]) for k, x in enumerate(tt) if t0 < x.f <= t1] + [interp(t1)]
    gv = gravity_vec(g)
    bg, ba = mp.matrix(b[:3]), mp.matrix(b[3:])
    p, R, v = p1, R1, v1

    def deriv(p_, R_, v_, z0, z1, st):
        al = (z1[0] - (z0[0] + st)).v / (z1[0] - z0[0]).v
        zg = z0[1] * al + z1[1] * (1 - al)
        za = z0[2] * al + z1[2] * (1 - al)
        wv = R_ * mp.matrix([zg[i] * sf[i] + bg[i] for i in range(3)])
        av = R_ * mp.matrix([za[i] * sf[3 + i] + ba[i] for i in range(3)]) - gv
        return v_, wv, av

    def step(p_, R_, v_, k, dt):
        return p_ + k[0] * dt, so3_exp(k[1] * dt) * R_, v_ + k[2] * dt

    for z0, z1 in zip(meas[:-1], meas[1:]):
        dt = z1[0] - z0[0]
        if dt.f == 0:
            continue
        half = T64(dt.f / 2, dt.d / 2)
        k1 = deriv(p, R, v, z0, z1, T64(0.0))
        y1 = step(p, R, v, k1, dt.v / 2)
        k2 = deriv(*y1, z0, z1, half)
        y2 = step(p, R, v, k2, dt.v / 2)
        k3 = deriv(*y2, z0, z1, half)
        y3 = step(p, R, v, k3, dt.v)
        k4 = deriv(*y3, z0, z1, dt)
        k = [k1[i] + 2 * k2[i] + 2 * k3[i] + k4[i] for i in range(3)]
        p, R, v = step(p, R, v, k, dt.v / 6)
    return p, R, v


def imu_epoch_kat():
    """The IMU residual at Unix time (tests/golden/imu_epoch_kat.npz, keys of imu_kat.npz with both switch values, and
    r_exact): a ~300 Hz jittered stream and 7 frames stamped near EPOCH, ts = 0.0031 off the 2^-22 s grid, no sample
    within 1e-5 s of a frame time.  r and J follow the reference's binary64 time sums (integrate_rounded); r_exact is
    the same residual with exact sums, at least 1e3 x the KATs' 1e-9 relative bar away from r."""
    from vicalib_b200.synth import mat_to_quat, quat_mul, so3_exp as np_exp
    rng = np.random.default_rng(20261019)
    nf = 7
    ftime = EPOCH + 0.15 + np.concatenate([[0.0], np.cumsum(rng.uniform(0.03, 0.05, nf - 1))])
    n = int((ftime[-1] - EPOCH - 0.1) * EPOCH_RATE) + 15
    t = EPOCH + 0.1 + (np.arange(n) + 0.5 * rng.random(n)) / EPOCH_RATE
    w = rng.normal(0, 0.4, (n, 3)); a = rng.normal(0, 1.0, (n, 3)) + np.array([0.3, 9.7, 0.5])
    tt = t + EPOCH_TS
    assert np.all(np.diff(t) > 0) and tt[0] < ftime[0] and tt[-1] > ftime[-1]
    assert np.abs(tt[:, None] - ftime[None, :]).min() > 1e-5  # no sample near a frame time: no ts kink
    assert np.mean((t + EPOCH_TS) - t != EPOCH_TS) >= 0.9  # the sums t_i + ts round
    g = np.array([0.05, -0.03]); b = np.concatenate([rng.normal(0, 1e-2, 3), rng.normal(0, 1e-1, 3)])
    sf = 1 + 0.02 * rng.normal(size=6)
    W = 500 * np.eye(9) + 20 * rng.normal(size=(9, 9))
    # each frame near the exact integration of the one before, so that |r| is small beside the rounding's effect on it
    q = np.zeros((nf, 4)); p = np.zeros((nf, 3)); v = np.zeros((nf, 3))
    q[0] = np_exp(rng.normal(0, 0.5, 3)); p[0] = rng.normal(0, 0.3, 3); v[0] = rng.normal(0, 0.5, 3)
    tm, wm, am = [mp.mpf(float(x)) for x in t], [V(x) for x in w], [V(x) for x in a]
    mpl = lambda x: [mp.mpf(float(y)) for y in x]  # noqa: E731
    for k in range(nf - 1):
        pe, Re, ve = integrate(tm, wm, am, mp.mpf(float(ftime[k])), mp.mpf(float(ftime[k + 1])), quat_R(q[k]), V(p[k]),
                               V(v[k]), mpl(g), mpl(b), mpl(sf), mp.mpf(EPOCH_TS))
        qe = mat_to_quat(np.array(Re.tolist(), dtype=np.float64))
        qe = qe if qe @ q[k] >= 0 else -qe
        q[k + 1] = quat_mul(qe, np_exp(0.02 * rng.normal(size=3)))
        p[k + 1] = np.array([float(x) for x in pe]) + 0.002 * rng.normal(size=3)
        v[k + 1] = np.array([float(x) for x in ve]) + 0.005 * rng.normal(size=3)
    out_r, out_J = imu_rows(t, w, a, ftime, q, p, v, g, b, sf, EPOCH_TS, W, (0,), integrator=integrate_rounded)
    r_exact, _ = imu_rows(t, w, a, ftime, q, p, v, g, b, sf, EPOCH_TS, W, (0,), jac=False)
    r0, J0, rx = np.array(out_r), np.array(out_J), np.array(r_exact)
    rot = [0, 1, 2, 6, 7, 8]  # rotation_only zeroes these residual rows (imu_residual's switch)
    r1, J1, rx1 = r0.copy(), J0.copy(), rx.copy()
    r1[:, rot], J1[:, rot], rx1[:, rot] = 0.0, 0.0, 0.0
    r, J, rx = np.stack([r0, r1]), np.stack([J0, J1]), np.stack([rx, rx1])
    sep = [np.abs(r[s] - rx[s]).max() / np.abs(r[s]).max() for s in (0, 1)]
    print(f"epoch: |r| max {np.abs(r0).max():.3g}, |r - r_exact| / |r| {sep[0]:.2e} / {sep[1]:.2e}", flush=True)
    assert min(sep) >= 1e3 * 1e-9, sep
    return dict(imu_t=t, imu_w=w, imu_a=a, ftime=ftime, T_wp=np.concatenate([q, p], 1), v_w=v, g=g, b=b, sf=sf,
                ts=np.array(EPOCH_TS), W=W, r=r, J=J, r_exact=rx)


def edge_kat():
    """Branch and boundary cases of the camera models (each model's own small-argument branches, the image
    centre, the image border).  Written to reproj_edge_kat.npz with the keys of reproj_kat.npz."""
    rng = np.random.default_rng(20260925)
    out = {}
    cases = {
        "fov": [dict(tgt=[1e-4, -2e-4, 0.5]),                      # rad^2 < 1e-5:  2 tan(w/2) / w
                dict(dist=[2e-3]),                                   # w^2 <= 1e-5:  factor 1
                dict(tgt=[-3e-5, 1e-5, 0.7], dist=[1e-3]),          # both
                dict(tgt=[0.45, -0.3, 0.4])],                        # wide angle (rad ~ 1.35)
        "kb4": [dict(tgt=[1e-5, -2e-5, 0.5]), dict(tgt=[0.5, 0.35, 0.35])],
        "poly3": [dict(tgt=[1e-6, 2e-6, 0.6]), dict(tgt=[0.35, 0.25, 0.4])],
        "poly2": [dict(tgt=[0.0, 0.0, 0.5]), dict(tgt=[-0.35, 0.25, 0.4])],
        "linear": [dict(tgt=[0.0, 0.0, 0.5]), dict(tgt=[0.4, -0.3, 0.4])],
    }
    ids = dict(linear=LINEAR, fov=FOV, poly2=POLY2, poly3=POLY3, kb4=KB4)
    for name, specs in cases.items():
        samples = [random_sample(rng, ids[name], **sp) for sp in specs]
        kat = reproj_kat(rng, ids[name], samples=samples)
        for k, v in kat.items():
            out[f"{name}_{k}"] = v
        print(name, "edge done", flush=True)
    np.savez_compressed(os.path.join(HERE, "reproj_edge_kat.npz"), **out)


# ------------------------------------------------------------------ wide-angle and fisheye lenses
KB4_FISHEYE = [0.04, -0.02, 0.005, -0.0005]  # d(theta) monotone to ~139 degrees
POLY2_BARREL = [-0.32, 0.04]                 # fold (first maximum of r f(r^2)) at r = 1.236
POLY3_BARREL = [-0.3, 0.06, -0.005]          # fold at r = 1.932
WIDE_KB4_THETA = [10.0, 45.0, 80.0, 89.9, 90.0, 95.0, 100.0]  # degrees; 90 exactly: Z = 0
WIDE_FOV_W = [0.9, 1.2]
WIDE_FOV_RAD = [1e-3, 0.1, 0.5, 1.0, 2.0, 3.5, float(np.tan(np.radians(80.0)))]
WIDE_POLY_RAD = {POLY2: [0.05, 0.4, 0.8, 1.1, 1.2], POLY3: [0.05, 0.6, 1.2, 1.6, 1.85]}
WIDE_LINEAR_RAD = [0.5, 1.5, 2.2, 3.0]


def wide_kat():
    """The camera models far from the axis (tests/golden/reproj_wide_kat.npz, keys of reproj_kat.npz): KB4 at fisheye
    distortion at WIDE_KB4_THETA, behind the image plane included; FOV at both WIDE_FOV_W from rad = 1e-3 (its small-
    argument branch) to tan 80 degrees; strong barrel poly2 / poly3 up to 0.97 of the fold; linear to rad = 3.  The
    90-degree KB4 row has identity poses, so that Z is exactly 0 in binary64 as in mpmath."""
    rng = np.random.default_rng(20261020)
    out = {}

    def ray(rad, scale=0.5):
        phi = rng.uniform(0, 2 * np.pi)
        return [scale * rad * np.cos(phi), scale * rad * np.sin(phi), scale]

    def kb4_samples():
        for th in WIDE_KB4_THETA:
            if th == 90.0:
                s = random_sample(rng, KB4, tgt=[0.3, -0.4, 0.0], dist=KB4_FISHEYE)
                ident = np.array([0.0, 0.0, 0.0, 1.0])
                _, _, _, _, intr, _, z = s
                yield ident, np.zeros(3), ident, np.zeros(3), intr, np.array([0.3, -0.4, 0.0]), z
                continue
            phi, t = rng.uniform(0, 2 * np.pi), np.radians(th)
            yield random_sample(rng, KB4, tgt=0.5 * np.array([np.sin(t) * np.cos(phi), np.sin(t) * np.sin(phi),
                                                                 np.cos(t)]), dist=KB4_FISHEYE)

    cases = {
        "kb4": (KB4, list(kb4_samples())),
        "fov": (FOV, [random_sample(rng, FOV, tgt=ray(r), dist=[w]) for w in WIDE_FOV_W for r in WIDE_FOV_RAD]),
        "poly2": (POLY2, [random_sample(rng, POLY2, tgt=ray(r), dist=POLY2_BARREL) for r in WIDE_POLY_RAD[POLY2]]),
        "poly3": (POLY3, [random_sample(rng, POLY3, tgt=ray(r), dist=POLY3_BARREL) for r in WIDE_POLY_RAD[POLY3]]),
        "linear": (LINEAR, [random_sample(rng, LINEAR, tgt=ray(r)) for r in WIDE_LINEAR_RAD]),
    }
    for name, (model, samples) in cases.items():
        for k, v in reproj_kat(rng, model, samples=samples).items():
            out[f"{name}_{k}"] = v
        print(name, "wide done", flush=True)
    return out


if __name__ == "__main__":
    if "--edge" in sys.argv:  # only the branch / boundary fixture (the others are unchanged)
        edge_kat()
        sys.exit(0)
    if "--wide" in sys.argv:  # only the wide-angle / fisheye fixture (the others are unchanged)
        np.savez_compressed(os.path.join(HERE, "reproj_wide_kat.npz"), **wide_kat())
        sys.exit(0)
    if "--imu-edge" in sys.argv:  # only the interpolation-buffer edge fixture (the others are unchanged)
        np.savez_compressed(os.path.join(HERE, "imu_edge_kat.npz"), **imu_edge_kat())
        sys.exit(0)
    if "--imu-vigorous" in sys.argv:  # only the vigorous-motion fixture (the others are unchanged)
        np.savez_compressed(os.path.join(HERE, "imu_vigorous_kat.npz"), **imu_vigorous_kat())
        sys.exit(0)
    if "--imu-epoch" in sys.argv:  # only the Unix-time fixture (the others are unchanged)
        np.savez_compressed(os.path.join(HERE, "imu_epoch_kat.npz"), **imu_epoch_kat())
        sys.exit(0)
    rng = np.random.default_rng(20260924)
    out = {}
    for name, m in (("linear", LINEAR), ("fov", FOV), ("poly2", POLY2), ("poly3", POLY3), ("kb4", KB4)):
        kat = reproj_kat(rng, m)
        for k, v in kat.items():
            out[f"{name}_{k}"] = v
        print(name, "done", flush=True)
    np.savez_compressed(os.path.join(HERE, "reproj_kat.npz"), **out)
    kat = imu_kat(rng)
    np.savez_compressed(os.path.join(HERE, "imu_kat.npz"), **kat)
    print("imu done")
