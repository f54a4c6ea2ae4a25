"""Host model of the persistent vision kernel's fit (mega_fit, vcgpu.cu), in plain Python.

It restates how many warps per CTA `lm_mega_kernel` runs with for a rig, per strategy (0 LM, 1 DOGLEG), or 0 where the
solve takes the multi-launch engine.  The shape constants are read from the CUDA sources through chain_plan's reader,
so a change of slab or table size moves the answer with it.
"""
import re

from chain_plan import H100_SMEM_OPTIN, K, _read

# the kernel's own (static) shared memory: group table int2[kGtabMax], triangle look-up [128], two flags (ptxas: 2192 B)
MEGA_STATIC_SMEM = 8 * K["kGtabMax"] + 128 + 16


def _sc_count():
    """kScCount of the step-scalar enum (vc_kernels.cuh)"""
    return int(re.search(r"kScCount\s*=\s*(\d+)", _read("vc_kernels.cuh")).group(1))


def _ctl_doubles():
    """sizeof(Ctl) / sizeof(double) (vc_internal.h): its int and double members, in order, 8-byte aligned"""
    body = re.search(r"struct Ctl \{(.*?)\};", _read("vc_internal.h"), re.S).group(1)
    size = 0
    for typ, decls in re.findall(r"^\s*(double|int)\s+([^;]+);", body, re.M):
        n = len(decls.split(","))
        if typ == "double":
            size = (size + 7) // 8 * 8
        size += n * (8 if typ == "double" else 4)
    return (size + 7) // 8


def mega_smem_bytes(G, n_cams, warps, strategy=0):
    """lm_mega_kernel's dynamic shared memory (mega_smem_doubles, vc_mega.cuh); strategy 1 (DOGLEG) adds u_g, D_g, g~_g
    and its scalars"""
    NS = G * G + G
    d = (warps * (K["kWarpDoubles"] + n_cams * K["kCgStride"]) + 3 * NS + G + K["kMaxCams"] * (K["kCamStateStride"] + 9)
         + _sc_count() + 8 * K["kMegaMaxWarps"] + n_cams * K["kCgStride"] + K["kMegaPartExtra"] + _ctl_doubles() + 8
         + (3 * G + 8 if strategy == 1 else 0))
    return 8 * d


def mega_warps(G, n_cams, smem_optin=H100_SMEM_OPTIN, strategy=0, nranks=1, static_smem=MEGA_STATIC_SMEM):
    """Warps per CTA of the persistent vision kernel, 0 where the solve takes the multi-launch engine: the most (up to
    kMegaMaxWarps) whose dynamic shared memory, next to the kernel's static share, fits the per-block opt-in, if a warp's
    slab holds the frame solve's [E | g] and X (12 (G + 1) doubles) and the totals fit the exchange buffer.  (The
    occupancy check that follows on the device passes wherever this fits: one CTA of kMegaMaxThreads threads at 128
    registers.)"""
    w = K["kMegaMaxWarps"]
    while w > 0 and mega_smem_bytes(G, n_cams, w, strategy) > smem_optin - static_smem:
        w -= 1
    PS = G * G + G + K["kMegaPartExtra"]
    PC = n_cams * K["kCgStride"] + K["kMegaPartExtra"]
    if (w == 0 or 12 * (G + 1) > K["kWarpDoubles"] or PS > 32768 or 4 * nranks * PS > K["kXchgCOff"]
            or 4 * nranks * PC > K["kXchgCtlOff"] - K["kXchgCOff"]):
        return 0
    return w
