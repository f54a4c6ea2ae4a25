"""A numpy restatement of vcgpu_align_imu (include/vcgpu.h): hand-eye alignment of the gyro stream with the frame poses.
  a_f         log(R_f^T R_f+1) of the frame poses
  b_f(s, b_g) log of the attitude the reference's IntegrateImu RK4 reaches from the identity over GetRange(t_f, t_f+1, s)
              (the oracle's GetRange), with the gyro scale sf[0..2] and bias b_g
  grid        Horn's closed form per candidate s (and, as a cross-check, an SVD Kabsch fit)
  refinement  Gauss-Newton on (dtheta, s, b_g) with the call's acceptance rule: a step only where it lowers the cost,
              halved at most HALVINGS times, s clamped to [ts_lo, ts_hi]; the s and b_g columns by central differences.
Everything here is float64 numpy; nothing is shared with the device code."""
import numpy as np

from vicalib_b200 import synth

HALVINGS = 10


def qmul(a, b):
    """(x y z w) Hamilton product in the device's (and the host apply's) order"""
    return np.array([a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1],
                     a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2],
                     a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0],
                     a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]])


def qconj(q):
    return np.array([-q[0], -q[1], -q[2], q[3]])


def so3_log(q):
    n = np.linalg.norm(q[:3])
    if n < 1e-300:
        return 2.0 * q[:3] / q[3]
    return 2.0 * np.arctan(n / q[3]) / n * q[:3]


def rot(q):
    return synth.quat_to_mat(np.asarray(q) / np.linalg.norm(q))


def rig_turns(T_wp, ivs):
    """a_f of the intervals ivs (their first frames)"""
    return np.array([so3_log(qmul(qconj(T_wp[f, :4]), T_wp[f + 1, :4])) for f in ivs]).reshape(-1, 3)


def attitude(meas, sfg, bg):
    """IntegrateImu's RK4 of the attitude alone (types.h; ceres-cost-functions.h:79-177) over GetRange's measurements
    (rows time | w (3) | a (3)), from the identity; returns log(dR)"""
    q = np.array([0.0, 0.0, 0.0, 1.0])
    for z0, z1 in zip(meas[:-1], meas[1:]):
        if z1[0] == z0[0]:
            continue
        dt = z1[0] - z0[0]

        def rate(y, h):
            alpha = (z1[0] - (z0[0] + h)) / (z1[0] - z0[0])
            zg = z0[1:4] * alpha + z1[1:4] * (1.0 - alpha)
            return rot(y) @ (zg * sfg + bg)

        k1 = rate(q, 0.0)
        y1 = qmul(synth.so3_exp(k1 * dt * 0.5), q)
        k2 = rate(y1, dt / 2.0)
        y2 = qmul(synth.so3_exp(k2 * dt * 0.5), q)
        k3 = rate(y2, dt / 2.0)
        y3 = qmul(synth.so3_exp(k3 * dt), q)
        k4 = rate(y3, dt)
        q = qmul(synth.so3_exp((k1 + 2 * k2 + 2 * k3 + k4) * dt / 6.0), q)
    return so3_log(q)


class Rig:
    """a problem's usable intervals and its gyro turns through the oracle's GetRange"""

    def __init__(self, p, oracle, s_lo, s_hi, active=None):
        self.p, self.o = p, oracle
        seen = np.zeros(p.n_frames, bool)
        seen[p.obs_frame if active is None else p.obs_frame[active]] = True
        lo, hi = p.imu_t[0] + s_hi, p.imu_t[-1] + s_lo
        t = p.ftime
        self.ivs = [f for f in range(p.n_frames - 1) if seen[f] and seen[f + 1] and t[f] >= lo and t[f + 1] <= hi]
        self.a = rig_turns(p.T_wp, self.ivs)
        self.sfg = np.asarray(p.sf[:3], float)

    def turns(self, s, bg):
        t = self.p.ftime
        return np.array([attitude(self.o.imu_get_range(t[f], t[f + 1], s), self.sfg, bg) for f in self.ivs]).reshape(-1, 3)


def horn(a, b):
    """(cost, Q (x y z w)) of the least mean |a - Q b|^2, by Horn's 4 x 4 matrix"""
    S = b.T @ a  # S[x][y] = sum b_x a_y
    N = np.array([
        [S[0, 0] + S[1, 1] + S[2, 2], S[1, 2] - S[2, 1], S[2, 0] - S[0, 2], S[0, 1] - S[1, 0]],
        [S[1, 2] - S[2, 1], S[0, 0] - S[1, 1] - S[2, 2], S[0, 1] + S[1, 0], S[2, 0] + S[0, 2]],
        [S[2, 0] - S[0, 2], S[0, 1] + S[1, 0], -S[0, 0] + S[1, 1] - S[2, 2], S[1, 2] + S[2, 1]],
        [S[0, 1] - S[1, 0], S[2, 0] + S[0, 2], S[1, 2] + S[2, 1], -S[0, 0] - S[1, 1] + S[2, 2]]])
    lam, V = np.linalg.eigh(N)
    v = V[:, -1]
    cost = ((a * a).sum() + (b * b).sum() - 2.0 * lam[-1]) / len(a)
    return cost, np.array([v[1], v[2], v[3], v[0]])


def kabsch(a, b):
    """(cost, R) of the same fit by the SVD of sum b a^T"""
    U, _, Vt = np.linalg.svd(b.T @ a)
    d = np.sign(np.linalg.det(Vt.T @ U.T))
    R = Vt.T @ np.diag([1.0, 1.0, d]) @ U.T
    return ((a - b @ R.T) ** 2).sum(1).mean(), R


def candidates(ts_lo, ts_hi, n_ts):
    return np.linspace(ts_lo, ts_hi, n_ts)


def cost_at(rig, Q, s, bg):
    b = rig.turns(s, bg)
    return ((rig.a - b @ rot(Q).T) ** 2).sum(1).mean()


def align(p, oracle, ts_lo=-0.05, ts_hi=0.05, n_ts=41, find_time_offset=True, max_iters=20, active=None):
    """vcgpu_align_imu at p's state: dict(Q, ts, b_g, rms, excitation, n_intervals, iterations, curve, status)"""
    bg0 = np.asarray(p.b[:3], float)
    s_lo, s_hi = (ts_lo, ts_hi) if find_time_offset else (p.ts, p.ts)
    rig = Rig(p, oracle, s_lo, s_hi, active)
    n = len(rig.ivs)
    cands = candidates(ts_lo, ts_hi, n_ts) if find_time_offset else np.array([p.ts])
    fits = [horn(rig.a, rig.turns(s, bg0)) for s in cands]
    curve = np.array([c for c, _ in fits])
    out = dict(n_intervals=n, curve=curve if find_time_offset else None, iterations=0, status=0)
    m = int(np.nanargmin(curve)) if np.isfinite(curve).any() else 0
    Q, s, bg = fits[m][1], float(cands[m]), bg0.copy()
    if n < 3:
        out.update(status=-3)
    else:
        cost = cost_at(rig, Q, s, bg)
        for _ in range(max_iters):
            b = rig.turns(s, bg)
            R = rot(Q)
            qb = b @ R.T
            r = (rig.a - qb).ravel()
            J = np.zeros((3 * n, 7))
            for f in range(n):
                x, y, z = qb[f]
                J[3 * f:3 * f + 3, :3] = [[0, -z, y], [z, 0, -x], [-y, x, 0]]
            h = 1e-7
            if find_time_offset:
                db = (rig.turns(s + h, bg) - rig.turns(s - h, bg)) / (2 * h)
                J[:, 3] = -(db @ R.T).ravel()
            for k in range(3):
                e = np.zeros(3)
                e[k] = h
                db = (rig.turns(s, bg + e) - rig.turns(s, bg - e)) / (2 * h)
                J[:, 4 + k] = -(db @ R.T).ravel()
            H, g = J.T @ J, -J.T @ r
            if not find_time_offset:
                H[3, :] = H[:, 3] = 0.0
                H[3, 3], g[3] = 1.0, 0.0
            try:
                d = np.linalg.solve(np.linalg.cholesky(H).T, np.linalg.solve(np.linalg.cholesky(H), g))
            except np.linalg.LinAlgError:
                out.update(status=-3)
                break
            alpha, accepted = 1.0, False
            for _ in range(HALVINGS + 1):
                Qc = qmul(synth.so3_exp(alpha * d[:3]), Q)
                Qc = Qc / np.linalg.norm(Qc)
                sc = min(max(s + alpha * d[3], ts_lo), ts_hi) if find_time_offset else s
                bc = bg + alpha * d[4:]
                c2 = cost_at(rig, Qc, sc, bc)
                if c2 < cost:
                    Q, s, bg, cost, accepted = Qc, sc, bc, c2, True
                    break
                alpha *= 0.5
            if not accepted:
                break
            out["iterations"] += 1
    b = rig.turns(s, bg)
    out["excitation"] = np.sort(np.linalg.eigvalsh(b.T @ b / n)) if n else np.full(3, np.nan)
    if out["status"]:
        out.update(Q=np.full(4, np.nan), ts=np.nan, b_g=np.full(3, np.nan), rms=np.nan)
    else:
        Q = Q if Q[3] >= 0 else -Q
        out.update(Q=Q, ts=s, b_g=bg, rms=float(np.sqrt(cost_at(rig, Q, s, bg))))
    return out


def angle(q1, q2):
    """the angle in radians between two rotations given as quaternions"""
    return 2.0 * np.arccos(min(1.0, abs(float(np.dot(q1, q2)) / (np.linalg.norm(q1) * np.linalg.norm(q2)))))


def camera0_start(p, T_ck0=None):
    """p re-expressed with camera 0 as the rig frame, as the reference starts without a cameras.xml: q_ck[0] the identity
    and p_ck[0] zero, every frame pose T_wk T_ck0^-1, every other camera T_ck T_ck0^-1.  T_ck0: (q, p) of the transform
    (default p's truth).  The rotation the alignment should then find is q_ck0."""
    import dataclasses

    q0, p0 = (p.truth["q_ck"][0], p.truth["p_ck"][0]) if T_ck0 is None else T_ck0
    q0i = qconj(q0)
    T = p.T_wp.copy()
    for f in range(p.n_frames):
        T[f, :4] = qmul(p.T_wp[f, :4], q0i)
        T[f, 4:] = p.T_wp[f, 4:] - rot(T[f, :4]) @ p0
    qc, pc = p.q_ck.copy(), p.p_ck.copy()
    for c in range(p.n_cams):
        qc[c] = qmul(p.q_ck[c], q0i) if c else np.array([0.0, 0.0, 0.0, 1.0])
        pc[c] = p.p_ck[c] - rot(qc[c]) @ p0 if c else np.zeros(3)
    return dataclasses.replace(p, T_wp=T, q_ck=qc, p_ck=pc)
