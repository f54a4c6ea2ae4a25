"""CPU checks of vcgpu_solve_batch: the cluster-size rule and the grouping (batch_plan.py) at their boundaries, the
C++ rule against that restatement, and the entry point at the library boundary."""
import ctypes as C
import os
import re

import batch_plan
import chain_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cluster_size_boundaries():
    cs = batch_plan.cluster_size
    assert cs(1, 16) == 1 and cs(16, 16) == 1          # warp slots exactly full
    assert cs(17, 16) == 2 and cs(32, 16) == 2         # one frame over
    assert cs(33, 16) == 4 and cs(64, 16) == 4 and cs(65, 16) == 8
    assert cs(128, 16) == 8 and cs(129, 16) == 8 and cs(40000, 16) == 8  # the cap: warps then loop over frames
    # 15 against 16 warps per CTA: the same rig can take a larger cluster
    assert cs(16, 15) == 2 and cs(30, 15) == 2 and cs(31, 15) == 4 and cs(31, 16) == 2
    assert cs(60, 15) == 4 and cs(61, 15) == 8 and cs(61, 16) == 4
    assert cs(10, 1) == 8


def test_batch_source_states_the_same_rule():
    src = open(os.path.join(ROOT, "vicalib_b200", "csrc", "vc_batch.inl")).read()
    body = re.search(r"static int batch_cluster_size\(int n_frames, int warps\) \{(.*?)\n\}", src, re.S).group(1)
    assert "while (size < 8 && size * warps < n_frames) size *= 2;" in body


def test_batch_kernel_fit_next_to_its_static_share():
    """the batch kernel stages the rig's arguments in shared memory, so a rig at the edge runs one warp fewer than in
    the grid kernel (a rig that has a single warp there is beyond the batch kernel's fit and is refused)"""
    import mega_plan

    assert batch_plan.BATCH_STATIC_SMEM > mega_plan.MEGA_STATIC_SMEM
    seen_less = False
    for n_cams in range(1, 9):
        for K in (4, 5, 6, 7, 8):
            G = n_cams * (6 + K)
            for st in (0, 1):
                wg, wb = mega_plan.mega_warps(G, n_cams, strategy=st), batch_plan.batch_warps(G, n_cams, st)
                assert wb in (wg, max(wg - 1, 0)), (G, n_cams, st, wg, wb)
                seen_less |= wb < wg
    assert batch_plan.batch_warps(chain_plan.rig_globals(("poly3",), False), 1) == 16
    assert seen_less


def test_grouping_of_a_mixed_batch():
    rigs = [(0, 50, 16), (1, 50, 16), (0, 60, 16), (0, 10, 16), (0, 50, 15), (1, 64, 16), (0, 3000, 16), (0, 120, 16)]
    g = batch_plan.groups(rigs)
    assert g == [((0, 4, 16), [0, 2]), ((1, 4, 16), [1, 5]), ((0, 1, 16), [3]), ((0, 4, 15), [4]), ((0, 8, 16), [6, 7])]
    assert batch_plan.groups([(0, 50, 16)] * 40) == [((0, 4, 16), list(range(40)))]  # like rigs: one launch


def test_entry_point_at_the_boundary():
    from vicalib_b200 import capi

    assert "vcgpu_solve_batch" in capi.EXPORTS
    L = capi.lib()
    assert hasattr(L, "vcgpu_solve_batch")
    hdr = open(os.path.join(ROOT, "include", "vcgpu.h")).read()
    assert re.search(r"int vcgpu_solve_batch\(vcgpu_handle\* const\* handles, int n, vcgpu_summary\* out", hdr)
    assert L.vcgpu_solve_batch(None, C.c_int(1), None) == -1          # VCGPU_ERR_INVALID
    one = (C.c_void_p * 1)(None)
    assert L.vcgpu_solve_batch(one, C.c_int(0), None) == -1
    assert L.vcgpu_solve_batch(one, C.c_int(1), None) == -1           # a null handle in the list
