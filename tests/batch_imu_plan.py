"""Host model of vcgpu_solve_batch_inertial's launch plan (imu_batch_cluster_size and the grouping of
run_solve_batch_inertial, vc_batch.inl), in plain Python.

A rig runs inside one thread-block cluster of the persistent inertial kernels.  How many CTAs the cluster has is a
function of the rig alone: the fewest of 1, 2, 4, 8 whose elimination groups (GROUPS per CTA) take the chunks of level
0 in one round, 8 beyond that.  Rigs of one cluster size share a group: per iteration one solve launch and one
evaluation launch for the whole group, the groups in increasing cluster size.
"""
import chain_plan

MAX_CLUSTER = 8  # the portable maximum cluster size


def level0_chunks(n_frames):
    return -(-n_frames // chain_plan.CHUNK)


def cluster_size(n_frames):
    size = 1
    while size < MAX_CLUSTER and size * chain_plan.GROUPS < level0_chunks(n_frames):
        size *= 2
    return size


def groups(frames):
    """frame counts of the rigs, in handle order -> [(cluster size, [rig indices])] in launch order"""
    out = {}
    for i, n in enumerate(frames):
        out.setdefault(cluster_size(n), []).append(i)
    return sorted(out.items())


def launches(iterations, weights, jacobi_scaling=True, rotation_only=False):
    """kernel_launches of a rig that ran `iterations` iterations, each queued for it: the Jacobi scale, with live
    weights three UpdateImuWeights launches (before the solve, after iteration 0, after the last iteration), the
    start point's evaluation and one solve and one evaluation launch per iteration.  vcgpu_solve's count alike."""
    own = (1 if jacobi_scaling else 0) + (3 if weights and not rotation_only else 0)
    return own + 1 + 2 * iterations

