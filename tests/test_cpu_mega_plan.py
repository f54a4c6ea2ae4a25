"""CPU: the host model of the persistent vision kernel's fit (tests/mega_plan.py) on the rigs the GPU tests rely on."""
import chain_plan
import mega_plan


def test_large_rig_does_not_fit():
    models = chain_plan.rig_with_globals(104, False)
    assert [mega_plan.mega_warps(104, len(models), strategy=s) for s in (0, 1)] == [0, 0]


def test_four_cameras_fit_both_strategies():
    assert [mega_plan.mega_warps(51, 4, strategy=s) for s in (0, 1)] == [12, 12]


def test_dogleg_adds_three_global_vectors():
    for G, n in ((13, 1), (36, 3), (51, 4)):
        assert mega_plan.mega_smem_bytes(G, n, 8, 1) - mega_plan.mega_smem_bytes(G, n, 8, 0) == 8 * (3 * G + 8)


def test_static_share_counts():
    """G = 36 on three cameras: 16 DOGLEG warps fit the opt-in only if the kernel's static shared memory is left out"""
    G = chain_plan.rig_globals(("poly3", "poly2", "fov"), False)
    assert G == 36
    assert mega_plan.mega_warps(G, 3, strategy=0) == 16
    assert mega_plan.mega_warps(G, 3, strategy=1) == 15
    assert mega_plan.mega_warps(G, 3, strategy=1, static_smem=0) == 16
