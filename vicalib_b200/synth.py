"""Seeded synthetic calibration problems (SURVEY.md §8d).

Produces the flat arrays both the CUDA path (through the C-ABI) and the CPU oracle consume:
cameras, frames, grid-corner observations, IMU samples, plus the ground truth they were drawn
from.  Geometry follows the reference's conventions:

* p_w = spacing * (gx, gy, 0)                      (vicalib-task.cc:357-358; spacing 0.01355 m,
                                                     vicalib-engine.cc:46)
* residual = Project(T_ck * (T_wk^-1 * p_w)) - p_c (ceres-cost-functions.h:361-370)
* frames are the rig ("k") poses T_wk; with an IMU the rig frame is the IMU frame
* IMU model used by the integrator                  (ceres-cost-functions.h:95-102):
      w_world = R_wk (sf_g * w_meas + b_g),  v' = R_wk (sf_a * a_meas + b_a) - g_vec
* sample i of the IMU buffer is valid at frame-clock time t_i + ts
                                                    (interpolation-buffer.h:150-153)

This module is host-side product code (numpy only); it never touches oracle/.
"""
from __future__ import annotations

import dataclasses

import numpy as np

LINEAR, FOV, POLY2, POLY3, KB4 = 0, 1, 2, 3, 4
MODEL_IDS = {"linear": LINEAR, "fov": FOV, "poly2": POLY2, "poly3": POLY3, "kb4": KB4}
NUM_INTR = {LINEAR: 4, FOV: 5, POLY2: 6, POLY3: 7, KB4: 8}
GRAVITY = 9.8007  # types.h:40-42
GYRO_SIGMA = 5.3088444e-5  # types.h:34
ACCEL_SIGMA = 0.001883649  # types.h:35
GRID_SPACING = 0.01355  # reference default (vicalib-engine.cc:46)
SYNTH_SPACING = 0.03  # synthetic default: fills the 640x480 image so distortion is observable


# ----------------------------------------------------------------------------- small Lie helpers
def quat_mul(a, b):
    """Hamilton product, coefficients (x, y, z, w) as in Eigen/Sophus."""
    ax, ay, az, aw = np.moveaxis(a, -1, 0)
    bx, by, bz, bw = np.moveaxis(b, -1, 0)
    return np.stack(
        [
            aw * bx + ax * bw + ay * bz - az * by,
            aw * by + ay * bw + az * bx - ax * bz,
            aw * bz + az * bw + ax * by - ay * bx,
            aw * bw - ax * bx - ay * by - az * bz,
        ],
        axis=-1,
    )


def quat_conj(q):
    return q * np.array([-1.0, -1.0, -1.0, 1.0])


def quat_to_mat(q):
    x, y, z, w = np.moveaxis(q, -1, 0)
    return np.stack(
        [
            np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
            np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
            np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1),
        ],
        axis=-2,
    )


def mat_to_quat(R):
    """Rotation matrices (..., 3, 3) -> unit quaternions (x, y, z, w), w >= 0."""
    R = np.asarray(R, dtype=np.float64)
    out = np.empty(R.shape[:-2] + (4,))
    flat_R = R.reshape(-1, 3, 3)
    flat_o = out.reshape(-1, 4)
    for i, m in enumerate(flat_R):
        t = np.trace(m)
        if t > 0:
            s = np.sqrt(t + 1.0) * 2
            q = [(m[2, 1] - m[1, 2]) / s, (m[0, 2] - m[2, 0]) / s, (m[1, 0] - m[0, 1]) / s, 0.25 * s]
        elif m[0, 0] > m[1, 1] and m[0, 0] > m[2, 2]:
            s = np.sqrt(1.0 + m[0, 0] - m[1, 1] - m[2, 2]) * 2
            q = [0.25 * s, (m[0, 1] + m[1, 0]) / s, (m[0, 2] + m[2, 0]) / s, (m[2, 1] - m[1, 2]) / s]
        elif m[1, 1] > m[2, 2]:
            s = np.sqrt(1.0 + m[1, 1] - m[0, 0] - m[2, 2]) * 2
            q = [(m[0, 1] + m[1, 0]) / s, 0.25 * s, (m[1, 2] + m[2, 1]) / s, (m[0, 2] - m[2, 0]) / s]
        else:
            s = np.sqrt(1.0 + m[2, 2] - m[0, 0] - m[1, 1]) * 2
            q = [(m[0, 2] + m[2, 0]) / s, (m[1, 2] + m[2, 1]) / s, 0.25 * s, (m[1, 0] - m[0, 1]) / s]
        q = np.array(q)
        if q[3] < 0:
            q = -q
        flat_o[i] = q / np.linalg.norm(q)
    return out


def so3_exp(w):
    w = np.asarray(w, dtype=np.float64)
    th = np.linalg.norm(w, axis=-1, keepdims=True)
    small = th < 1e-10
    ths = np.where(small, 1.0, th)
    imag = np.where(small, 0.5 - th * th / 48.0, np.sin(0.5 * ths) / ths)
    real = np.where(small, 1.0 - th * th / 8.0, np.cos(0.5 * ths))
    return np.concatenate([imag * w, real], axis=-1)


def se3_apply_right(T, delta):
    """T * exp(delta) for small deltas (first-order V = I is exact enough for perturbing guesses)."""
    q, t = T[..., :4], T[..., 4:]
    dq = so3_exp(delta[..., 3:])
    R = quat_to_mat(q)
    t2 = t + np.einsum("...ij,...j->...i", R, delta[..., :3])
    q2 = quat_mul(q, dq)
    q2 /= np.linalg.norm(q2, axis=-1, keepdims=True)
    return np.concatenate([q2, t2], axis=-1)


def gravity_vector(g2):
    sp, cp, sq, cq = np.sin(g2[0]), np.cos(g2[0]), np.sin(g2[1]), np.cos(g2[1])
    return -GRAVITY * np.array([cp * sq, -sp, cp * cq])


# ----------------------------------------------------------------------------- camera models
def project(model: int, ray: np.ndarray, p: np.ndarray) -> np.ndarray:
    """Vectorised forward projection, restating SURVEY App. A.2 (Calibu `Project`)."""
    X, Y, Z = ray[..., 0], ray[..., 1], ray[..., 2]
    if model == KB4:
        rho = np.sqrt(X * X + Y * Y)
        th = np.arctan2(rho, Z)
        th2 = th * th
        d = th * (1 + th2 * (p[4] + th2 * (p[5] + th2 * (p[6] + th2 * p[7]))))
        rs = np.where(rho > 0, rho, 1.0)
        return np.stack([p[0] * d * X / rs + p[2], p[1] * d * Y / rs + p[3]], -1)
    u, v = X / Z, Y / Z
    r2 = u * u + v * v
    if model == LINEAR:
        f = np.ones_like(u)
    elif model == FOV:
        w = p[4]
        rad = np.sqrt(r2)
        m = 2.0 * np.tan(w / 2.0)
        rs = np.where(r2 < 1e-5, 1.0, rad)
        f = np.where(r2 < 1e-5, m / w, np.arctan(rs * m) / (rs * w))
    elif model == POLY2:
        f = 1 + p[4] * r2 + p[5] * r2 * r2
    elif model == POLY3:
        f = 1 + p[4] * r2 + p[5] * r2 * r2 + p[6] * r2 * r2 * r2
    else:
        raise ValueError(model)
    return np.stack([p[0] * f * u + p[2], p[1] * f * v + p[3]], -1)


TRUTH_DIST = {
    LINEAR: [],
    FOV: [0.9],
    POLY2: [-0.15, 0.03],
    POLY3: [-0.15, 0.03, -0.004],
    KB4: [-0.02, 0.004, -0.001, 0.0002],
}
SEED_DIST = {LINEAR: [], FOV: [0.2], POLY2: [0, 0], POLY3: [0, 0, 0], KB4: [0, 0, 0, 0]}


@dataclasses.dataclass
class Problem:
    """Flat problem arrays (initial guess) + truth."""

    models: np.ndarray  # int32 [n_cams]
    intr: np.ndarray  # f64 [n_cams, 10]
    q_ck: np.ndarray  # f64 [n_cams, 4]
    p_ck: np.ndarray  # f64 [n_cams, 3]
    T_wp: np.ndarray  # f64 [n_frames, 7]  (qx qy qz qw tx ty tz)
    v_w: np.ndarray  # f64 [n_frames, 3]
    ftime: np.ndarray  # f64 [n_frames]
    obs_frame: np.ndarray  # int32 [n_obs]
    obs_cam: np.ndarray  # int32 [n_obs]
    p_w: np.ndarray  # f64 [n_obs, 3]
    p_c: np.ndarray  # f64 [n_obs, 2]
    grid_idx: np.ndarray  # int32 [n_obs, 2]  integer corner indices (gx, gy)
    imu_t: np.ndarray  # f64 [n_imu]
    imu_w: np.ndarray  # f64 [n_imu, 3]
    imu_a: np.ndarray  # f64 [n_imu, 3]
    g: np.ndarray  # f64 [2]
    b: np.ndarray  # f64 [6]
    sf: np.ndarray  # f64 [6]
    ts: float
    truth: dict
    inertial: bool

    @property
    def n_obs(self):
        return int(self.obs_frame.shape[0])

    @property
    def n_frames(self):
        return int(self.T_wp.shape[0])

    @property
    def n_cams(self):
        return int(self.models.shape[0])


def _look_at(cam_pos, target, roll):
    """Camera-to-world rotations with +z towards target, x right, y down; extra roll about z."""
    z = target - cam_pos
    z /= np.linalg.norm(z, axis=-1, keepdims=True)
    up = np.array([0.0, 1.0, 0.0])  # world y is image-down
    x = np.cross(np.broadcast_to(up, z.shape), z)
    x /= np.linalg.norm(x, axis=-1, keepdims=True)
    y = np.cross(z, x)
    R = np.stack([x, y, z], axis=-1)
    c, s = np.cos(roll), np.sin(roll)
    Rz = np.zeros(R.shape)
    Rz[..., 0, 0], Rz[..., 0, 1], Rz[..., 1, 0], Rz[..., 1, 1], Rz[..., 2, 2] = c, -s, s, c, 1.0
    return R @ Rz


def _vigorous_cam0_pose(t, centre, ph):
    """Camera 0 of a handheld recording that excites every axis, still looking at the grid: translations at 1.3-2 Hz
    (up to ~13 m/s^2 along the optical axis, so the specific force departs from g by more than 10 m/s^2), tilts at
    1.1-1.4 Hz and a roll of -0.5 +- 1.4 rad about the optical axis at 0.7 Hz (up to 6 rad/s), which carries the
    rig's attitude across pi from the world frame (near a roll of -pi/2)."""
    t = np.asarray(t, dtype=np.float64)
    w = 2 * np.pi * np.array([1.3, 1.7, 2.0, 1.1, 1.4, 0.7])
    pos = np.stack(
        [
            centre[0] + 0.10 * np.sin(w[0] * t + ph[0]),
            centre[1] + 0.08 * np.sin(w[1] * t + ph[1]),
            -(0.47 + 0.08 * np.sin(w[2] * t + ph[2])),
        ],
        -1,
    )
    tgt = np.stack(
        [
            centre[0] + 0.06 * np.sin(w[3] * t + ph[3]),
            centre[1] + 0.05 * np.sin(w[4] * t + ph[4]),
            np.zeros_like(t),
        ],
        -1,
    )
    roll = -0.5 + 1.4 * np.sin(w[5] * t + ph[5])
    return _look_at(pos, tgt, roll), pos


def make_problem(
    models=("poly3",),
    n_frames=50,
    grid=(14, 10),
    inertial=False,
    seed=20260924,
    pixel_sigma=0.1,
    intr_init="perturbed",  # "perturbed" (truth + 1 %), "seed" (reference seeds), "truth"
    pose_noise=(2e-3, 5e-3),  # (metres, radians) on the initial frame poses
    ts_truth=0.0,
    frame_rate=30.0,
    imu_rate=200.0,
    width=640,
    height=480,
    imu_noise=True,
    spacing=None,
    motion="gentle",  # "gentle" (the default trajectory) or "vigorous" (_vigorous_cam0_pose)
    focal=None,  # truth focal length in pixels, one or one per camera (default 320), each drawn within +-5 %
    dist=None,  # truth distortion, one list per camera (default TRUTH_DIST of its model)
    standoff=None,  # (mean, amplitude) of camera 0's distance from the grid plane in metres (default (0.47, 0.11))
    tilt=None,  # (mean, amplitude) in radians of camera 0's turn away from the grid, about an axis that rotates
    #             in the image plane: the grid moves from the image centre towards the rim (default: no turn)
    cull=False,  # drop corners outside the image, and (every model but KB4) corners not in front of the camera
) -> Problem:
    rng = np.random.default_rng(seed)
    models = np.array([MODEL_IDS[m] if isinstance(m, str) else int(m) for m in models], dtype=np.int32)
    n_cams = len(models)
    gx, gy = np.meshgrid(np.arange(grid[0]), np.arange(grid[1]), indexing="xy")
    gidx = np.stack([gx.ravel(), gy.ravel()], -1).astype(np.int32)
    M = gidx.shape[0]
    if spacing is None:
        spacing = SYNTH_SPACING * 14.0 / grid[0]
    pw_grid = np.concatenate([spacing * gidx.astype(np.float64), np.zeros((M, 1))], -1)
    centre = pw_grid.mean(0)

    # ---- truth intrinsics / extrinsics
    intr_t = np.zeros((n_cams, 10))
    focals = np.broadcast_to(np.asarray(320.0 if focal is None else focal, dtype=np.float64), (n_cams,))
    for c, m in enumerate(models):
        f = focals[c] * (1 + 0.05 * rng.uniform(-1, 1))
        intr_t[c, :4] = [f, f * (1 + 0.002 * rng.uniform(-1, 1)), width / 2 + rng.uniform(-5, 5),
                         height / 2 + rng.uniform(-5, 5)]
        d = TRUTH_DIST[int(m)] if dist is None else dist[c]
        if len(d) != NUM_INTR[int(m)] - 4:
            raise ValueError(f"camera {c}: {len(d)} distortion parameters for model {int(m)}")
        intr_t[c, 4:4 + len(d)] = d
    R_rdf = np.array([[0.0, 1, 0], [0, 0, 1], [1, 0, 0]])  # RdfRobotics (vi_sim_test.cpp:71-74)
    q_ck_t = np.zeros((n_cams, 4))
    p_ck_t = np.zeros((n_cams, 3))
    for c in range(n_cams):
        if inertial:
            dR = quat_to_mat(so3_exp(0.02 * rng.standard_normal(3)))
            Rck = dR @ R_rdf
            p_ck_t[c] = np.array([0.02, -0.01, 0.015]) + np.array([0.10 * c, 0, 0]) if c == 0 else \
                np.array([0.02 + 0.10 * c, -0.01, 0.015]) + 0.003 * rng.standard_normal(3)
        else:
            Rck = np.eye(3) if c == 0 else quat_to_mat(so3_exp(0.02 * rng.standard_normal(3)))
            p_ck_t[c] = np.zeros(3) if c == 0 else np.array([0.10 * c, 0, 0]) + 0.003 * rng.standard_normal(3)
        q_ck_t[c] = mat_to_quat(Rck)

    # ---- smooth trajectory of camera 0 (sum of sinusoids), 0.35-0.6 m from the grid
    ftime = 1.0 + np.arange(n_frames) / frame_rate
    ph = rng.uniform(0, 2 * np.pi, 8)
    fr = 2 * np.pi * np.array([0.31, 0.23, 0.17, 0.41, 0.29, 0.13, 0.37, 0.19])
    if motion not in ("gentle", "vigorous"):
        raise ValueError(motion)
    if motion == "vigorous" and (standoff is not None or tilt is not None):
        raise ValueError("standoff and tilt shape the gentle trajectory only")
    d0, d1 = (0.47, 0.11) if standoff is None else standoff

    def turned(R, t):
        """R turned by tilt about an image-plane axis whose direction rotates with time"""
        if tilt is None:
            return R
        phi = fr[6] * t + ph[6]
        ang = tilt[0] + tilt[1] * np.sin(fr[7] * t + ph[7])
        axis = np.stack([np.cos(phi), np.sin(phi), np.zeros_like(phi)], -1)
        return R @ quat_to_mat(so3_exp(ang[..., None] * axis))

    def cam0_pose(t):
        if motion == "vigorous":
            return _vigorous_cam0_pose(t, centre, ph)
        t = np.asarray(t, dtype=np.float64)
        pos = np.stack(
            [
                centre[0] + 0.16 * np.sin(fr[0] * t + ph[0]),
                centre[1] + 0.12 * np.sin(fr[1] * t + ph[1]),
                -(d0 + d1 * np.sin(fr[2] * t + ph[2])),
            ],
            -1,
        )
        tgt = np.stack(
            [
                centre[0] + 0.03 * np.sin(fr[3] * t + ph[3]),
                centre[1] + 0.03 * np.sin(fr[4] * t + ph[4]),
                np.zeros_like(t),
            ],
            -1,
        )
        roll = 0.35 * np.sin(fr[5] * t + ph[5])
        return turned(_look_at(pos, tgt, roll), t), pos

    R_ck0 = quat_to_mat(q_ck_t[0])

    def rig_pose(t):
        """T_wk = T_wc0 * T_ck0 (p_c = R_ck p_k + p_ck  =>  T_wc = T_wk T_ck^-1)."""
        Rwc, pwc = cam0_pose(t)
        Rwk = Rwc @ R_ck0
        pwk = pwc + np.einsum("...ij,j->...i", Rwc, p_ck_t[0])
        return Rwk, pwk

    Rwk, pwk = rig_pose(ftime)
    T_wp_t = np.concatenate([mat_to_quat(Rwk), pwk], -1)
    h = 1e-4
    v_w_t = (rig_pose(ftime + h)[1] - rig_pose(ftime - h)[1]) / (2 * h)

    # ---- observations, sorted by (cam, frame, corner)
    obs_frame, obs_cam, p_w, p_c, g_idx = [], [], [], [], []
    for c in range(n_cams):
        Rck = quat_to_mat(q_ck_t[c])
        pk = np.einsum("fji,fmj->fmi", Rwk, pw_grid[None, :, :] - pwk[:, None, :])  # R^T (p_w - t)
        pc = np.einsum("ij,fmj->fmi", Rck, pk) + p_ck_t[c]
        with np.errstate(divide="ignore", invalid="ignore"):  # corners behind a pinhole-type camera are culled below
            z = project(int(models[c]), pc, intr_t[c]) + pixel_sigma * rng.standard_normal((n_frames, M, 2))
        sel = np.ones(n_frames * M, dtype=bool)
        if cull:
            zf = z.reshape(-1, 2)
            sel = np.isfinite(zf).all(1) & (zf[:, 0] >= 0) & (zf[:, 0] < width) & (zf[:, 1] >= 0) & (zf[:, 1] < height)
            if int(models[c]) != KB4:
                sel &= pc.reshape(-1, 3)[:, 2] > 0
        obs_frame.append(np.repeat(np.arange(n_frames, dtype=np.int32), M)[sel])
        obs_cam.append(np.full(n_frames * M, c, dtype=np.int32)[sel])
        p_w.append(np.tile(pw_grid, (n_frames, 1))[sel])
        p_c.append(z.reshape(-1, 2)[sel])
        g_idx.append(np.tile(gidx, (n_frames, 1))[sel])
    obs_frame = np.concatenate(obs_frame)
    obs_cam = np.concatenate(obs_cam)
    p_w = np.concatenate(p_w)
    p_c = np.concatenate(p_c)
    g_idx = np.concatenate(g_idx)

    # ---- IMU
    g_t = np.array([0.05, -0.03]) if inertial else np.zeros(2)
    b_t = np.concatenate([1e-3 * rng.standard_normal(3), 1e-2 * rng.standard_normal(3)]) if inertial else np.zeros(6)
    sf_t = 1 + 0.01 * rng.uniform(-1, 1, 6) if inertial else np.ones(6)
    if inertial:
        t0, t1 = ftime[0] - 0.2, ftime[-1] + 0.2
        n_imu = int(np.floor((t1 - t0) * imu_rate))
        imu_t = t0 + 0.001234 + np.arange(n_imu) / imu_rate  # phase offset: no exact frame/sample ties
        tt = imu_t + ts_truth  # frame-clock time at which sample i is valid
        Rm, _ = rig_pose(tt)
        Rp, pp = rig_pose(tt + h)
        Rn, pn = rig_pose(tt - h)
        _, p0 = rig_pose(tt)
        acc_w = (pp - 2 * p0 + pn) / (h * h)
        # world-frame angular velocity from R' R^T
        dR = (Rp - Rn) / (2 * h)
        Wx = np.einsum("nij,nkj->nik", dR, Rm)
        w_world = np.stack([Wx[:, 2, 1], Wx[:, 0, 2], Wx[:, 1, 0]], -1)
        w_body = np.einsum("nji,nj->ni", Rm, w_world)
        a_body = np.einsum("nji,nj->ni", Rm, acc_w + gravity_vector(g_t))
        imu_w = (w_body - b_t[:3]) / sf_t[:3]
        imu_a = (a_body - b_t[3:]) / sf_t[3:]
        if imu_noise:
            imu_w = imu_w + GYRO_SIGMA * rng.standard_normal(imu_w.shape)
            imu_a = imu_a + ACCEL_SIGMA * rng.standard_normal(imu_a.shape)
    else:
        imu_t = np.zeros(0)
        imu_w = np.zeros((0, 3))
        imu_a = np.zeros((0, 3))

    # ---- initial guess
    intr0 = intr_t.copy()
    if intr_init == "perturbed":
        for c, m in enumerate(models):
            K = NUM_INTR[int(m)]
            intr0[c, :4] *= 1 + 0.01 * rng.uniform(-1, 1, 4)
            intr0[c, 4:K] *= 1 + 0.05 * rng.uniform(-1, 1, K - 4)
    elif intr_init == "seed":  # vicalib-engine.cc:207-247
        for c, m in enumerate(models):
            K = NUM_INTR[int(m)]
            intr0[c, :4] = [300, 300, width / 2.0, height / 2.0]
            intr0[c, 4:K] = SEED_DIST[int(m)]
    delta = np.concatenate(
        [pose_noise[0] * rng.standard_normal((n_frames, 3)), pose_noise[1] * rng.standard_normal((n_frames, 3))], -1
    )
    T_wp0 = se3_apply_right(T_wp_t, delta)
    q_ck0, p_ck0 = q_ck_t.copy(), p_ck_t.copy()
    for c in range(n_cams):
        if c == 0 and not inertial:
            continue  # cam0 extrinsics are held constant without an IMU (vicalibrator.h:572-576)
        q = quat_mul(q_ck_t[c], so3_exp(0.01 * rng.standard_normal(3)))
        q_ck0[c] = q / np.linalg.norm(q)
        p_ck0[c] = p_ck_t[c] + 0.003 * rng.standard_normal(3)
    truth = dict(intr=intr_t, q_ck=q_ck_t, p_ck=p_ck_t, T_wp=T_wp_t, v_w=v_w_t, g=g_t, b=b_t, sf=sf_t, ts=ts_truth)
    return Problem(
        models=models, intr=intr0, q_ck=q_ck0, p_ck=p_ck0, T_wp=T_wp0,
        v_w=np.zeros((n_frames, 3)),  # AddFrame seeds velocities with zero (vicalibrator.h:359)
        ftime=ftime, obs_frame=obs_frame, obs_cam=obs_cam, p_w=p_w, p_c=p_c, grid_idx=g_idx,
        imu_t=imu_t, imu_w=imu_w, imu_a=imu_a,
        g=np.zeros(2) if not inertial else g_t + 0.01 * rng.standard_normal(2),
        b=np.zeros(6), sf=np.ones(6), ts=0.0, truth=truth, inertial=inertial,
    )


# BASELINE.json `configs`, in order, plus the north_star target configuration.
CONFIGS = {
    "config1": dict(models=("poly3",), n_frames=50, grid=(14, 10), inertial=False),
    "config2": dict(models=("poly3",), n_frames=2000, grid=(14, 10), inertial=False),
    "config3": dict(models=("fov", "fov"), n_frames=2000, grid=(14, 10), inertial=True),
    "config4": dict(models=("kb4", "kb4"), n_frames=5000, grid=(20, 15), inertial=True, ts_truth=0.003),
    "config5": dict(models=("poly3",) * 4, n_frames=10000, grid=(20, 15), inertial=True),
    "target": dict(models=("poly3", "poly3"), n_frames=2000, grid=(14, 10), inertial=True),
}


def make_config(name: str, **overrides) -> Problem:
    kw = dict(CONFIGS[name])
    idx = list(CONFIGS).index(name)
    kw.setdefault("seed", 20260924 + idx + 1)
    kw.update(overrides)
    return make_problem(**kw)


def shard_frames(n_frames: int, rank: int, world: int):
    """Contiguous frame range [f0, f1) owned by `rank` (SURVEY §8e: frames shard naturally)."""
    base, rem = divmod(n_frames, world)
    f0 = rank * base + min(rank, rem)
    return f0, f0 + base + (1 if rank < rem else 0)


def shard(p: Problem, rank: int, world: int) -> Problem:
    """Rank-local slice: the rank's frames (re-indexed from 0) and the observations of those frames;
    cameras / globals / the IMU stream are replicated.  With inertial terms every rank but the last
    also gets the next rank's first frame appended as a ghost (no observations): the IMU factor
    between its last frame and that frame is owned by this rank."""
    f0, f1 = shard_frames(p.n_frames, rank, world)
    g1 = f1 + (1 if (p.inertial and rank < world - 1) else 0)
    sel = (p.obs_frame >= f0) & (p.obs_frame < f1)
    truth = dict(p.truth)
    truth["T_wp"] = p.truth["T_wp"][f0:g1]
    truth["v_w"] = p.truth["v_w"][f0:g1]
    return dataclasses.replace(
        p, T_wp=p.T_wp[f0:g1].copy(), v_w=p.v_w[f0:g1].copy(), ftime=p.ftime[f0:g1].copy(),
        obs_frame=(p.obs_frame[sel] - f0).astype(np.int32), obs_cam=p.obs_cam[sel].copy(), p_w=p.p_w[sel].copy(),
        p_c=p.p_c[sel].copy(), grid_idx=p.grid_idx[sel].copy(), truth=truth)
