"""Host model of vcgpu_solve_batch's launch plan (batch_cluster_size and the grouping of run_solve_batch, vc_batch.inl),
in plain Python.

A rig runs inside one thread-block cluster.  How many CTAs the cluster has is a function of the rig alone: the fewest
of 1, 2, 4, 8 whose warp slots (CTAs x warps per CTA) hold its frames, 8 beyond that.  Rigs of one strategy, cluster
size and warp count share a launch.
"""
import mega_plan
from chain_plan import H100_SMEM_OPTIN

MAX_CLUSTER = 8  # the portable maximum cluster size
# static shared memory of lm_mega_batch_kernel: lm_mega_kernel's, plus the rig's staged arguments (ptxas: 2944 B)
BATCH_STATIC_SMEM = mega_plan.MEGA_STATIC_SMEM + 752


def cluster_size(n_frames, warps):
    size = 1
    while size < MAX_CLUSTER and size * warps < n_frames:
        size *= 2
    return size


def batch_warps(G, n_cams, strategy=0, smem_optin=H100_SMEM_OPTIN):
    """warps per CTA of the batch kernel for a rig (0: the rig does not fit, the batch is refused)"""
    return mega_plan.mega_warps(G, n_cams, smem_optin, strategy, static_smem=BATCH_STATIC_SMEM)


def groups(rigs):
    """rigs: [(strategy, n_frames, warps)] -> launch groups in launch order, each (key, [rig indices]) with
    key = (strategy, cluster size, warps); a group starts at its first rig"""
    out = {}
    for i, (strategy, n_frames, warps) in enumerate(rigs):
        out.setdefault((strategy, cluster_size(n_frames, warps), warps), []).append(i)
    return list(out.items())
