"""CPU checks of vcgpu_solve_batch_inertial: the cluster-size rule and the grouping (batch_imu_plan.py) at their
boundaries, the C++ rule against that restatement, and the entry points at the library boundary."""
import ctypes as C
import os
import re

import batch_imu_plan
import chain_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cluster_size_boundaries():
    cs = batch_imu_plan.cluster_size
    assert chain_plan.CHUNK == 8 and chain_plan.GROUPS == 2  # 16 frames of level 0 per CTA
    assert cs(2) == 1 and cs(16) == 1                   # two chunks: one CTA's two groups
    assert cs(17) == 2 and cs(32) == 2
    assert cs(33) == 4 and cs(64) == 4 and cs(65) == 8
    assert cs(128) == 8 and cs(129) == 8 and cs(2000) == 8 and cs(40000) == 8  # the cap: groups then loop over chunks
    assert [cs(n) for n in (24, 200, 256)] == [2, 8, 8]


def test_batch_source_states_the_same_rule():
    src = open(os.path.join(ROOT, "vicalib_b200", "csrc", "vc_batch.inl")).read()
    body = re.search(r"static int imu_batch_cluster_size\(int n_frames\) \{(.*?)\n\}", src, re.S).group(1)
    assert "const int chunks = (n_frames + kCsChunk - 1) / kCsChunk;" in body
    assert "while (size < 8 && size * kCsGroups < chunks) size *= 2;" in body


def test_grouping_of_a_mixed_batch():
    g = batch_imu_plan.groups([200, 24, 12, 50, 2000, 30, 16])
    assert g == [(1, [2, 6]), (2, [1, 5]), (4, [3]), (8, [0, 4])]
    assert batch_imu_plan.groups([100] * 40) == [(8, list(range(40)))]  # like rigs: one group


def test_launch_count():
    assert batch_imu_plan.launches(6, 0) == 1 + 1 + 12
    assert batch_imu_plan.launches(6, 1) == 1 + 3 + 1 + 12
    assert batch_imu_plan.launches(6, 1, rotation_only=True) == batch_imu_plan.launches(6, 0)
    assert batch_imu_plan.launches(4, 0, jacobi_scaling=False) == 1 + 8


def test_entry_points_at_the_boundary():
    from vicalib_b200 import capi

    for name in ("vcgpu_solve_batch_inertial", "vcgpu_batch_plan_inertial"):
        assert name in capi.EXPORTS
    L = capi.lib()
    hdr = open(os.path.join(ROOT, "include", "vcgpu.h")).read()
    assert re.search(r"int vcgpu_solve_batch_inertial\(vcgpu_handle\* const\* handles, int n, vcgpu_summary\* out", hdr)
    assert re.search(r"int vcgpu_batch_plan_inertial\(vcgpu_handle\* h, int\* cluster_size, int\* resident_clusters\)", hdr)
    assert L.vcgpu_solve_batch_inertial(None, C.c_int(1), None) == -1  # VCGPU_ERR_INVALID
    one = (C.c_void_p * 1)(None)
    assert L.vcgpu_solve_batch_inertial(one, C.c_int(0), None) == -1
    assert L.vcgpu_solve_batch_inertial(one, C.c_int(-3), None) == -1
    assert L.vcgpu_solve_batch_inertial(one, C.c_int(1), None) == -1  # a null handle in the list
    assert L.vcgpu_batch_plan_inertial(None, None, None) == -1
