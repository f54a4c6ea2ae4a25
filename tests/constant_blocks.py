"""Host model of the constant parameter blocks (shared by test_cpu_constant_blocks.py and test_gpu_constant_blocks.py).

Ceres minimises over the parameter blocks that are neither constant nor unused (Program::RemoveFixedBlocks): it never
moves the others, and its parameter tolerance, step_norm <= param_tol * (x_norm + param_tol), takes x_norm over the
blocks it keeps.  Which blocks ViCalibrator::SetupProblem holds constant (vicalibrator.h:572-600, 657-676) is restated
here from the flags, and which frames and cameras no residual uses from the observations, independently of the
oracle's GlobalMask and the device's fill_mask.
"""
import numpy as np

from vicalib_b200 import synth

STAGE_ROT_ONLY = dict(inertial=1, rotation_only=1, bias_active=0, scale_active=0, optimize_ts=1)
FIX = dict(fix_intrinsics=1)
INERTIAL_FIX = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=0, optimize_ts=0, fix_intrinsics=1)


def vision_problem(seed=3, n_frames=24):
    """Two cameras; cam0's rotation and one unseen frame's pose are quaternions that renormalisation would move."""
    p = synth.make_problem(models=("poly3", "fov"), n_frames=n_frames, grid=(14, 10), seed=seed)
    return unseen_frame(unfix_cam0_rotation(p), n_frames // 2)


def inertial_problem(seed=21, n_frames=24):
    return synth.make_problem(models=("poly3",), n_frames=n_frames, grid=(14, 10), inertial=True, seed=seed)


# the parameter-tolerance cases: fixed intrinsics (vision, inertial) and a rotation-only stage
PT_CASES = [("vision_fix", vision_problem, FIX), ("inertial_fix", inertial_problem, INERTIAL_FIX),
            ("rotation_only", inertial_problem, STAGE_ROT_ONLY)]


def uploaded(p):
    """the state a problem uploads, as a state dict"""
    return dict(intr=p.intr, q_ck=p.q_ck, p_ck=p.p_ck, T_wp=p.T_wp, v_w=p.v_w, g=p.g, b=p.b, sf=p.sf, ts=p.ts)


def num_intr(models):
    return [synth.NUM_INTR[int(m)] for m in models]


def frames_used(p, flags):
    """1 per frame a residual uses: every frame of an inertial run, else the frames an observation sees."""
    if flags.get("inertial", 0):
        return np.ones(p.n_frames, bool)
    used = np.zeros(p.n_frames, bool)
    used[np.asarray(p.obs_frame)] = True
    return used


def cams_used(p, active=None):
    """1 per camera an active observation sees: the IMU residual takes no camera block, so a camera without one is in
    no residual at all (vision or inertial)"""
    used = np.zeros(p.n_cams, bool)
    cam = np.asarray(p.obs_cam)
    used[cam if active is None else cam[np.asarray(active) > 0]] = True
    return used


def free_blocks(flags):
    """{block name: free?} for the global blocks (cam0's extrinsics are listed separately from the other cameras')"""
    inertial = bool(flags.get("inertial", 0))
    rot_only = bool(flags.get("rotation_only", 0))
    return dict(q0=inertial, p0=inertial and not rot_only, intr=not flags.get("fix_intrinsics", 0),
                g=inertial and not rot_only, b=inertial and bool(flags.get("bias_active", 0)),
                sf=inertial and bool(flags.get("scale_active", 0)), ts=inertial and bool(flags.get("optimize_ts", 0)))


def state_norms(st, p, flags):
    """(x_norm over the free blocks a residual uses, x_norm over every block) of a state dict"""
    inertial = bool(flags.get("inertial", 0))
    free = free_blocks(flags)
    used = frames_used(p, flags)
    cams = cams_used(p)
    K = num_intr(p.models)
    s_free = s_all = 0.0

    def add(v, is_free):
        nonlocal s_free, s_all
        v2 = float(np.sum(np.square(v)))
        s_all += v2
        if is_free:
            s_free += v2

    for f in range(p.n_frames):
        add(st["T_wp"][f], used[f])
        if inertial:
            add(st["v_w"][f], used[f])
    for c in range(p.n_cams):
        add(st["q_ck"][c], cams[c] and (c > 0 or free["q0"]))
        add(st["p_ck"][c], cams[c] and (c > 0 or free["p0"]))
        add(st["intr"][c, :K[c]], cams[c] and free["intr"])
    if inertial:
        for k in ("g", "b", "sf"):
            add(st[k], free[k])
        add(st["ts"], free["ts"])
    return np.sqrt(s_free), np.sqrt(s_all)


def constant_parts(st, p, flags):
    """{name: array} of every constant block of a state (to compare bit for bit with the uploaded values)"""
    free = free_blocks(flags)
    out = {}
    if not free["intr"]:
        out["intr"] = st["intr"]
    if not free["q0"]:
        out["q_ck0"] = st["q_ck"][0]
    if not free["p0"]:
        out["p_ck0"] = st["p_ck"][0]
    unused = ~frames_used(p, flags)
    if unused.any():
        out["T_wp_unused"] = st["T_wp"][unused]
    for c in np.flatnonzero(~cams_used(p)):
        out[f"q_ck{c}"], out[f"p_ck{c}"], out[f"intr{c}"] = st["q_ck"][c], st["p_ck"][c], st["intr"][c]
    if flags.get("inertial", 0):
        for k in ("g", "b", "sf"):
            if not free[k]:
                out[k] = st[k]
        if not free["ts"]:
            out["ts"] = np.array([st["ts"]])
    return out


def renormalised(q):
    return q / np.sqrt(np.sum(q * q))


def moves_on_renormalisation(q):
    return not np.array_equal(renormalised(q), q)


def unfix(q):
    """q (in place), one ulp at a time off unit norm until renormalising it changes its bits (synth writes quaternions
    that are fixed points, cam0's identity among them)"""
    k = 0
    while not moves_on_renormalisation(q):
        q[k % 4] = np.nextafter(q[k % 4], np.inf)
        k += 1
    return q


def unfix_cam0_rotation(p):
    unfix(p.q_ck[0])
    return p


def drop_frame(p, f):
    """Remove every observation of frame f: a frame no camera sees."""
    keep = p.obs_frame != f
    p.obs_frame, p.obs_cam, p.p_w, p.p_c = p.obs_frame[keep], p.obs_cam[keep], p.p_w[keep], p.p_c[keep]
    if getattr(p, "grid_idx", None) is not None:
        p.grid_idx = p.grid_idx[keep]
    return p


def unseen_frame(p, f):
    """Frame f made unseen, with a pose quaternion that renormalisation would change."""
    unfix(p.T_wp[f, :4])
    return drop_frame(p, f)


def param_tol_window(rows, norms, margin=1 + 1e-6):
    """A parameter tolerance under which the free-block rule stops at iteration k while the all-block rule stops at some
    j < k.  rows: the iteration rows of a solve with every tolerance at 0 (column 5: step norm); norms[it]: (free, all)
    x_norm of the state iteration it starts from.  Returns (tol, k, j) for the widest such window, with every decision
    at least `margin` (relative) away from its threshold, or None.  The window is at most as wide as the ratio of the
    two norms: 1 + 8e-6 for a rotation-only stage, whose constant blocks are small."""
    sn = rows[:, 5]
    valid = [it for it in range(1, len(rows)) if sn[it] > 0]
    best = None
    for i, k in enumerate(valid[1:], 1):
        before = valid[:i]
        rf = {it: sn[it] / norms[it][0] for it in valid[: i + 1]}
        ra = {it: sn[it] / norms[it][1] for it in before}
        lo, hi = max(rf[k], min(ra.values())), min(rf[it] for it in before)
        if hi > lo * margin ** 2 and (best is None or hi / lo > best[0]):
            tol = float(np.sqrt(lo * hi))
            best = (hi / lo, tol, k, next(it for it in before if ra[it] <= tol))
    return None if best is None else best[1:]


def param_tol_case(p, flags, strategy=0, n_iters=14):
    """(rows, norms, (tol, k, j) or None) of an oracle solve with every tolerance at 0: norms[it] = (free, all) x_norm of
    the state iteration it starts from, from oracle solves stopped after it - 1 iterations"""
    from oracle.binding import Oracle

    def run(max_iters):
        o = Oracle(p, **flags)
        o.set_options(max_iters=max_iters, function_tol=0.0, gradient_tol=0.0, param_tol=0.0, strategy=strategy)
        return o, o.solve()

    rows = run(n_iters)[1]["rows"]
    norms = {it: state_norms(run(it - 1)[0].state(), p, flags) for it in range(1, len(rows))}
    return rows, norms, param_tol_window(rows, norms)


def stops_at(rows, norms, tol, which):
    """The first iteration whose step passes step_norm <= tol * (x_norm + tol) with x_norm = norms[it][which]"""
    return next((it for it in range(1, len(rows)) if rows[it, 5] > 0 and rows[it, 5] <= tol * (norms[it][which] + tol)),
                None)
