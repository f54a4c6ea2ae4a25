"""Host model of the inertial chain solve's plan, in plain Python.

It restates what the host and the kernels decide from the problem's shape alone: the level table of `imu_prepare`
(vc_imu_host.inl), the per-level dispatch of `chain_solve_kernel` (narrow or wide, rounds of chunks, which CTAs leave
for the deferred weight update), the dense solve's tile count, the persistent-fit decision of `imu_mega_prepare`
(vc_engine.inl) and the dynamic shared memory every chain kernel asks for, and the loop shapes of the DOGLEG kernels
(vc_dogleg.cuh).  The tests use it to pick frame counts and rigs that land on a given branch, and to check that branch
is the one the numbers say.  Its plain reference (`arrow_matvec`, `backward_error`) works on the block normal equations
in long double.

The shape constants (`kCsChunk`, `kCsTop`, ...) are read from the CUDA sources, so a change of chunk length moves the
test cases with it.
"""
import ctypes
import itertools
import math
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "vicalib_b200", "csrc")

FD = 9                 # inertial frame block: pose 6 + velocity 3
IMU_GLOBALS = 15       # g 2 | b 6 | sf 6 | ts 1
H100_SMS = 132         # H100 SXM
H100_SMEM_OPTIN = 232448  # cudaDevAttrMaxSharedMemoryPerBlockOptin on sm_90
# static shared memory a chain kernel of the multi-launch engine declares next to its dynamic request (one int flag,
# rounded up generously); it counts against the same per-block opt-in
CHAIN_STATIC_SMEM = 64
MODEL_K = {"linear": 4, "fov": 5, "poly2": 6, "poly3": 7, "kb4": 8}
MAX_CAMS = 8

_CONST = re.compile(r"constexpr\s+(?:int|size_t)\s+(\w+)\s*=\s*([^;]+);")


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _constants():
    """Every `constexpr int NAME = <integer arithmetic>;` of the headers the plan depends on, evaluated."""
    raw = {}
    for name in ("vc_internal.h", "vc_kernels.cuh", "vc_fused.cuh", "vc_mega.cuh", "vc_imu_weights.cuh", "vc_imu_mega.cuh",
                 "vc_imu_eval_mega.cuh", "vc_dogleg.cuh"):
        for k, expr in _CONST.findall(_read(name)):
            raw.setdefault(k, re.sub(r"//.*", "", expr).strip())
    vals, busy = {}, set()

    def ev(k):
        if k not in vals:
            if k in busy:  # a function-local constant that shadows another one: not a plan constant
                raise ValueError(f"{k} refers to itself")
            busy.add(k)
            expr = raw[k]
            for name in set(re.findall(r"[A-Za-z_]\w*", expr)):
                if name not in raw:
                    raise ValueError(f"{k} = {expr}: {name} is not an integer constant")
                expr = re.sub(rf"\b{name}\b", str(ev(name)), expr)
            if not re.fullmatch(r"[\d\s+\-*/()]+", expr):
                raise ValueError(f"{k} = {raw[k]}: not integer arithmetic")
            vals[k] = int(eval(expr.replace("/", "//")))  # integer arithmetic of literals only (checked above)
        return vals[k]

    out = {}
    for k in raw:
        try:
            out[k] = ev(k)
        except ValueError:
            pass
    return out


K = _constants()
CHUNK, TOP, GROUP, THREADS, MAX_LEVELS = (K[k] for k in ("kCsChunk", "kCsTop", "kCsGroup", "kCsThreads", "kMaxChainLevels"))
GROUPS = THREADS // GROUP


def _work_doubles():
    """sizeof(wts::Work) / sizeof(double): the weight team's shared-memory workspace."""
    body = re.search(r"struct Work \{(.*?)\};", _read("vc_imu_weights.cuh"), re.S).group(1)
    size = 0
    for typ, decls in re.findall(r"(double|int)\s+([^;]+);", body):
        n = sum(int(d) for d in re.findall(r"\[(\d+)\]", decls))
        size += n * (8 if typ == "double" else 4)
    return math.ceil(size / 8)


WORK_DOUBLES = _work_doubles()


# ------------------------------------------------------------------------------------------------ the level table
def level_sizes(n_frames, top=TOP):
    """Nodes per level on one GPU (imu_prepare): every CHUNK-th node of a level is a separator, and the level of at most
    `top` nodes joins the dense solve."""
    sizes, m = [], n_frames
    while True:
        sizes.append(m)
        if m <= top:
            return sizes
        m = (m + CHUNK - 1) // CHUNK


def elimination_levels(n_frames):
    return len(level_sizes(n_frames)) - 1


def top_nodes(n_frames):
    return level_sizes(n_frames)[-1]


def lone_separator_levels(n_frames):
    """Elimination levels whose last chunk has no interior node: a separator alone ((m - 1) mod CHUNK == 0)."""
    sizes = level_sizes(n_frames)
    return [l for l in range(len(sizes) - 1) if (sizes[l] - 1) % CHUNK == 0]


def weight_tasks(n_frames):
    """16-interval tasks of the deferred UpdateImuWeights queue (one 16-lane team per interval)."""
    return (n_frames - 1 + THREADS // 16 - 1) // (THREADS // 16)


def n_solver(n_frames, sms=H100_SMS):
    """CTAs that stay with the solve while the others work the weights queue (imu_mega_solve)."""
    return min(32, max(8, sms - weight_tasks(n_frames) - 4))


def levels(n_frames, sms=H100_SMS, narrow_ok=True, weights=False):
    """Per elimination level: nodes, chunks (nsep), wide or narrow, rounds of chunks, CTAs leaving after it.

    `weights`: the deferred weight update is pending (an LM iteration after an accepted step), so CTAs leave."""
    sizes = level_sizes(n_frames)
    nl = len(sizes)
    ns = min(n_solver(n_frames, sms), sms) if weights else sms
    n_act, out = sms, []
    for l in range(nl - 1):
        nsep = sizes[l + 1]
        wide = nsep > sms or not narrow_ok
        rounds = math.ceil(nsep / (sms * GROUPS)) if wide else math.ceil(nsep / sms)
        n_next = ns
        if l + 2 < nl:
            nsep2 = sizes[l + 2]
            n_next = sms if (nsep2 > sms or not narrow_ok) else max(ns, nsep2)
        n_next = min(n_next, n_act)
        out.append(dict(level=l, n=sizes[l], nsep=nsep, wide=wide, rounds=rounds, active=n_act, leaving=n_act - n_next,
                        lone_last=(sizes[l] - 1) % CHUNK == 0))
        n_act = n_next
    return out


def leaving_ctas(n_frames, sms=H100_SMS):
    """CTAs that leave the solve for the weights queue during the elimination of an LM iteration with weights (all but
    the n_solver that go on; without an elimination level they leave at the barrier before the Schur reduction)."""
    return sms - min(n_solver(n_frames, sms), sms)


BRANCHES = ("narrow", "wide0", "wide0_rounds2", "levels4", "wide1", "lone_last", "top4")


def branches(n_frames, sms=H100_SMS):
    """The branches of chain_solve_kernel's elimination a frame count reaches (names as in BRANCHES):
    narrow          a level with at most one chunk per CTA (the whole CTA on a chunk)
    wide0           level 0 with more chunks than CTAs (two chunks per CTA in flight)
    wide0_rounds2   ... and more chunks than groups: a group takes a second chunk
    levels4         four elimination levels or more
    wide1           level 1 wide too
    lone_last       a level whose last chunk is a separator without interior nodes
    top4            kCsTop nodes join the dense solve (the most it takes)"""
    lv = levels(n_frames, sms)
    out = set()
    if any(not x["wide"] for x in lv):
        out.add("narrow")
    if lv and lv[0]["wide"]:
        out.add("wide0")
    if lv and lv[0]["rounds"] >= 2:
        out.add("wide0_rounds2")
    if len(lv) >= 4:
        out.add("levels4")
    if len(lv) >= 2 and lv[1]["wide"]:
        out.add("wide1")
    if any(x["lone_last"] for x in lv):
        out.add("lone_last")
    if top_nodes(n_frames) == TOP:
        out.add("top4")
    return out


def chain_cases(sms=H100_SMS):
    """(frame count, branches it is there for) of test_gpu_chain_chunks.py; with chunks of 8, kCsTop = 4 and 132 SMs:
    5, 8, 9, 10, 15, 17, 32, 33, 65, 66, 256, 257, 1056, 1057, 2049, 2113, 8449 frames."""
    c, t, g = CHUNK, TOP, GROUPS
    return [
        (t + 1, {"narrow"}),                  # one ragged chunk
        (c, {"narrow"}),                      # one full chunk, no right separator
        (c + 1, {"lone_last"}),
        (c + 2, {"narrow"}),                  # a last chunk of one interior node
        (2 * c - 1, {"narrow"}),              # two chunks, the last one ragged
        (2 * c + 1, {"lone_last"}),
        (t * c, {"top4"}),
        (t * c + 1, {"lone_last"}),
        (c * c + 1, {"lone_last"}),           # on two levels
        (c * c + 2, {"narrow"}),
        (t * c * c, {"top4"}),
        (t * c * c + 1, {"lone_last"}),
        (c * sms, {"narrow"}),                # the widest narrow level 0: one chunk per CTA
        (c * sms + 1, {"wide0"}),
        (t * c ** 3 + 1, {"levels4"}),
        (c * sms * g + 1, {"wide0_rounds2", "levels4"}),
        (c * c * sms + 1, {"wide1"}),
    ]


# ------------------------------------------------------------------------------------------------ the dense solve
def dense_n(G, n_frames):
    return G + FD * top_nodes(n_frames)


def dense_tiles(N):
    """16 x 16 register tiles of chain_solve_kernel's dense L D L^T (0: the shared-memory version)."""
    t = (N + 1 + 15) // 16
    return 6 if t <= 6 else 7 if t <= 7 else 9 if t <= 9 else 0


def dense_rows(N):
    return 16 * dense_tiles(N) if dense_tiles(N) else N + 1


def dense_ld(N):
    return 16 * dense_tiles(N) + 1 if dense_tiles(N) else (N | 1)


# ------------------------------------------------------------------------------------------------ persistent engine
def chain_group_doubles(G):
    c = CHUNK
    VW = FD + 2 * FD + G + 1
    sacc = G * (G + 1) // 2 + G
    return sacc + FD * FD + FD * G + FD + (2 * (c - 1) + 1) * FD * FD + (c - 1) * FD * VW + (c - 1) * FD * G


def chain_solve_smem_bytes(G):
    grp = GROUPS * chain_group_doubles(G)
    N = G + TOP * FD
    dense = dense_rows(N) * dense_ld(N) + N + 2
    wts = (THREADS // 16) * (WORK_DOUBLES + 1)
    return (max(grp, dense, wts) + 16) * 8


def eval_mega_smem_bytes(G):
    NS = G * G + G
    m = max(NS, K["kEvWarps"] * K["kWarpDoubles"], (K["kEvThreads"] // 16) * (WORK_DOUBLES + 1))
    return (m + K["kMaxCams"] * (K["kCamStateStride"] + 9) + 16) * 8


def persistent_fits(G, n_frames, smem_optin=H100_SMEM_OPTIN):
    """imu_mega_prepare on one GPU: both persistent kernels' requests fit the opt-in, the level table fits, and a
    group's threads cover a V row (3 FD + G + 1 columns)."""
    return (chain_solve_smem_bytes(G) <= smem_optin and eval_mega_smem_bytes(G) <= smem_optin
            and len(level_sizes(n_frames)) <= MAX_LEVELS and 3 * FD + G + 1 <= GROUP)


# ------------------------------------------------------------------------------------------------ multi-launch engine
def chain_eliminate_smem_bytes(G, c=CHUNK):
    """chain_eliminate_kernel: Sacc [G^2 + G] | Al Ap Uc [3 x 81] | El [9 G] | gl [9] | V [(c - 1) 9 (G + 28)]."""
    return (G * G + G + 3 * FD * FD + FD * G + FD + (c - 1) * FD * (FD + 2 * FD + G + 1)) * 8


def chain_dense_smem_bytes(N):
    """dense_solve_kernel: S [N^2] | rhs [N]."""
    return (N * N + N) * 8


def multi_launch_requests(G, inertial=True, top=TOP):
    """Dynamic shared memory (bytes) of every multi-launch kernel whose request grows with G."""
    NS = G * G + G
    out = {"reduce_finalize_kernel": NS * 8}
    if inertial:
        out["chain_eliminate_kernel"] = chain_eliminate_smem_bytes(G)
        out["dense_solve_kernel"] = chain_dense_smem_bytes(G + FD * top)
    else:
        out["frame_solve_kernel"] = (NS + (K["kSolveThreads"] // 32) * 2 * 6 * (G + 1)) * 8
        out["global_solve_kernel"] = NS * 8
    return out


def rig_globals(models, inertial=True):
    return sum(6 + MODEL_K[m] for m in models) + (IMU_GLOBALS if inertial else 0)


def rig_with_globals(G, inertial=True):
    """The first rig (fewest cameras, then models in MODEL_K order) with G globals."""
    for n in range(1, MAX_CAMS + 1):
        for models in itertools.combinations_with_replacement(MODEL_K, n):
            if rig_globals(models, inertial) == G:
                return models
    raise ValueError(f"no rig of at most {MAX_CAMS} cameras has {G} globals")


# ------------------------------------------------------------------------------------------------ the DOGLEG kernels
DL_BLOCKS, MV_WARPS = K["kDlBlocks"], K["kMvWarps"]


def matvec_parts(n_frames):
    """Per-CTA partials of E^T w_f that arrow_matvec_globals_kernel sums (one warp per frame)."""
    return (n_frames + MV_WARPS - 1) // MV_WARPS


def dot_passes(n):
    """Passes of dl_dots_kernel's 256-thread loop over the largest of its DL_BLOCKS slices of n entries."""
    width = max((n * (b + 1)) // DL_BLOCKS - (n * b) // DL_BLOCKS for b in range(DL_BLOCKS))
    return (width + 255) // 256


def engine_smem_optin(device_optin=H100_SMEM_OPTIN):
    """The dynamic shared memory the multi-launch engine opts its chain kernels in to (kernel_smem_optin): the device's
    per-block opt-in less the kernel's static shared memory, unless the source names a fixed size."""
    src = _read("vc_engine.inl")
    body = re.search(r"static int kernel_smem_optin\(vcgpu_handle\* h\) \{(.*?)\n\}", src, re.S).group(1)
    fixed = re.search(r"=\s*(\d+)\s*\*\s*1024\s*;", body)
    if fixed:
        return int(fixed.group(1)) * 1024
    return device_optin - CHAIN_STATIC_SMEM


# ------------------------------------------------------------------------------------------------ plain reference
def scaled_blocks(ne, scale):
    """The blocks of S H S and S g in long double.  H is block tridiagonal + arrow: B[f] on the diagonal,
    U[f] = H[f-1, f], E[f] = H[f, globals], C = H[globals, globals]; returns U[k] = H[k, k+1], k = 0 .. nf-2."""
    ld = np.longdouble
    nf, fd, _ = ne["B"].shape
    nfp = nf * fd
    sf, sc = scale[:nfp].reshape(nf, fd).astype(ld), scale[nfp:].astype(ld)
    return dict(B=ne["B"].astype(ld) * sf[:, :, None] * sf[:, None, :],
                U=ne["U"][1:].astype(ld) * sf[:-1, :, None] * sf[1:, None, :],
                E=ne["E"].astype(ld) * sf[:, :, None] * sc[None, None, :],
                C=ne["C"].astype(ld) * sc[:, None] * sc[None, :],
                gf=ne["gf"].astype(ld) * sf, gc=ne["gc"].astype(ld) * sc)


def arrow_matvec(ne, scale, x):
    """y = S H S x in long double, x and y of length nf fd + G (frames first, then the globals)."""
    sb = scaled_blocks(ne, scale)
    nf, fd, _ = ne["B"].shape
    nfp = nf * fd
    x = np.asarray(x)
    xf, xc = x[:nfp].reshape(nf, fd).astype(np.longdouble), x[nfp:].astype(np.longdouble)
    yf = np.einsum("fij,fj->fi", sb["B"], xf) + np.einsum("fij,j->fi", sb["E"], xc)
    yf[:-1] += np.einsum("kij,kj->ki", sb["U"], xf[1:])
    yf[1:] += np.einsum("kji,kj->ki", sb["U"], xf[:-1])
    yc = sb["C"] @ xc + np.einsum("fij,fi->j", sb["E"], xf)
    return np.concatenate([yf.ravel(), yc])


def backward_error(ne, scale, D2, x):
    """Normwise backward error of x as a solution of (S H S + diag(D2)) x = -S g, in long double."""
    ld = np.longdouble
    nf, fd, _ = ne["B"].shape
    G = ne["C"].shape[0]
    nfp = nf * fd
    sb = scaled_blocks(ne, scale)
    B, U, E, C, gf, gc = (sb[k] for k in ("B", "U", "E", "C", "gf", "gc"))
    df, dc = D2[:nfp].reshape(nf, fd).astype(ld), D2[nfp:].astype(ld)
    xf, xc = x[:nfp].reshape(nf, fd).astype(ld), x[nfp:].astype(ld)
    r = arrow_matvec(ne, scale, x) + D2.astype(ld) * x.astype(ld)
    rf, rc = r[:nfp].reshape(nf, fd) + gf, r[nfp:] + gc
    nrm_f = np.abs(B).sum(2) + np.abs(df) + np.abs(E).sum(2)
    nrm_f[:-1] += np.abs(U).sum(2)
    nrm_f[1:] += np.abs(U).sum(1)
    nrm_c = np.abs(C).sum(1) + np.abs(dc) + np.abs(E).sum((0, 1))
    r = max(np.abs(rf).max(), np.abs(rc).max())
    a = max(nrm_f.max(), nrm_c.max())
    xn = max(np.abs(xf).max(), np.abs(xc).max())
    gn = max(np.abs(gf).max(), np.abs(gc).max())
    assert G == xc.shape[0]
    return float(r / (a * xn + gn))


# ------------------------------------------------------------------------------------------------ the device
def device_attrs():
    """(SM count, per-block shared-memory opt-in) of CUDA device 0, from the driver (no torch import)."""
    cuda = ctypes.CDLL("libcuda.so.1")
    assert cuda.cuInit(0) == 0
    dev = ctypes.c_int(0)
    assert cuda.cuDeviceGet(ctypes.byref(dev), 0) == 0
    sms, optin = ctypes.c_int(0), ctypes.c_int(0)
    assert cuda.cuDeviceGetAttribute(ctypes.byref(sms), 16, dev) == 0     # CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT
    assert cuda.cuDeviceGetAttribute(ctypes.byref(optin), 97, dev) == 0   # ..._MAX_SHARED_MEMORY_PER_BLOCK_OPTIN
    return sms.value, optin.value


def device_or_h100():
    """device_attrs(), or the H100's values where there is no device (test collection on a CPU-only machine)."""
    try:
        return device_attrs()
    except (OSError, AssertionError):
        return H100_SMS, H100_SMEM_OPTIN
