"""CPU: the host model of the inertial chain solve's plan (tests/chain_plan.py) against the figures DESIGN states, the
branches the GPU tests claim to reach, the persistent engine's fit boundary, and the shared memory the multi-launch
engine's chain kernels ask for on every rig the C API accepts.  Assumes an H100 SXM: 132 SMs, 227 KB opt-in."""
import itertools

import pytest

import chain_plan as cp


def test_constants_come_from_the_source():
    assert cp.CHUNK >= 2 and cp.TOP >= 1 and cp.THREADS == cp.GROUPS * cp.GROUP and cp.MAX_LEVELS >= 2
    assert cp.WORK_DOUBLES == 472  # wts::Work: 460 doubles + 8 rotations + 8 int pairs


def test_target_workload_matches_design():
    """DESIGN §4.4 on the 2000-frame target: 2000 -> 250 -> 32 -> 4 nodes, level 0 runs 250 chunks on 264 groups in
    one round, and 100 of the 132 CTAs leave for the weights queue after level 0."""
    assert cp.level_sizes(2000) == [2000, 250, 32, 4]
    lv = cp.levels(2000, weights=True)
    assert [x["nsep"] for x in lv] == [250, 32, 4]
    assert lv[0]["wide"] and lv[0]["rounds"] == 1 and cp.H100_SMS * cp.GROUPS == 264
    assert not lv[1]["wide"] and not lv[2]["wide"]
    assert lv[0]["leaving"] == 100
    assert cp.n_solver(2000) == 8 and cp.leaving_ctas(2000) == 124
    assert cp.dense_n(41, 2000) == 77 and cp.dense_tiles(77) == 6


def test_level_table_edges():
    assert cp.level_sizes(2) == [2]  # nothing to eliminate: the chain joins the dense solve
    for n in range(2, 3000):
        sizes = cp.level_sizes(n)
        assert sizes[-1] <= cp.TOP and all(s > cp.TOP for s in sizes[:-1])
        assert all(b == -(-a // cp.CHUNK) for a, b in zip(sizes, sizes[1:]))


@pytest.mark.parametrize("n_frames,claims", cp.chain_cases(), ids=[str(n) for n, _ in cp.chain_cases()])
def test_chain_cases_reach_their_branch(n_frames, claims):
    assert claims <= cp.branches(n_frames), (n_frames, cp.branches(n_frames))


def test_chain_cases_cover_every_branch():
    assert set().union(*(c for _, c in cp.chain_cases())) == set(cp.BRANCHES)
    assert set().union(*(cp.branches(n) for n, _ in cp.chain_cases())) == set(cp.BRANCHES)


def test_branch_thresholds():
    """The first frame counts of the dispatch table: each branch appears exactly at its threshold."""
    first = {}
    for n in range(2, 9000):
        for b in cp.branches(n):
            first.setdefault(b, n)
    assert first["wide0"] == cp.CHUNK * cp.H100_SMS + 1 == 1057
    assert first["wide0_rounds2"] == cp.CHUNK * cp.H100_SMS * cp.GROUPS + 1 == 2113
    assert first["levels4"] == cp.TOP * cp.CHUNK ** 3 + 1 == 2049
    assert first["wide1"] == cp.CHUNK ** 2 * cp.H100_SMS + 1 == 8449
    assert first["lone_last"] == cp.CHUNK + 1
    assert first["top4"] == cp.TOP


def test_engine_cases():
    """The shapes of test_gpu_imu_engines.py land where they claim."""
    # G = 67 with 4 top nodes: N = 103 takes the 7-tile register L D L^T; fewer top nodes would not
    G = cp.rig_globals(("poly3",) * 4)
    assert G == 67 and cp.top_nodes(256) == 4 and cp.dense_tiles(cp.dense_n(G, 256)) == 7
    assert all(cp.dense_tiles(G + 9 * t) == 6 for t in (1, 2, 3))
    assert cp.persistent_fits(G, 256)
    # wide level 0 in two rounds, four levels, on the persistent engine
    assert {"wide0_rounds2", "levels4"} <= cp.branches(2113) and cp.persistent_fits(cp.rig_globals(("poly3",)), 2113)
    # the deferred weights queue has more tasks than leaving CTAs from 1986 frames on (5000: 313 tasks, 124 CTAs)
    assert cp.weight_tasks(5000) == 313 and cp.leaving_ctas(5000) == 124
    assert min(n for n in range(2, 6000) if cp.weight_tasks(n) > cp.leaving_ctas(n)) == 1986
    # the largest rigs: 4 top nodes at 32 frames, one at 33
    assert cp.rig_globals(("kb4",) * 8) == 127 and cp.rig_globals(("kb4",) * 3 + ("poly3",) * 5) == 122
    assert cp.top_nodes(32) == 4 and cp.top_nodes(33) == 1


def test_persistent_fit_boundary():
    """G = 67 fits the persistent inertial kernels on an H100 (231 472 of 232 448 B), G = 68 falls back."""
    assert cp.rig_globals(("kb4",) * 3 + ("linear",)) == 67
    assert cp.rig_globals(("kb4",) * 3 + ("fov",)) == 68
    assert cp.chain_solve_smem_bytes(67) == 231472 <= cp.H100_SMEM_OPTIN < cp.chain_solve_smem_bytes(68)
    assert cp.persistent_fits(67, 40) and not cp.persistent_fits(68, 40)
    assert all(cp.eval_mega_smem_bytes(G) <= cp.H100_SMEM_OPTIN for G in range(1, 128))


def test_backward_error_reference():
    """The long-double backward error of the GPU chain tests: ~1e-16 for a float64 dense solve of the same system, and
    far above its bar when one coupling block is dropped from the solve."""
    import numpy as np

    rng = np.random.default_rng(7)
    nf, fd, G = 11, 9, 5
    n = nf * fd + G
    J = rng.standard_normal((3 * n, n))
    H = J.T @ J
    mask = np.ones((n, n), bool)  # block tridiagonal frames + dense globals: no coupling of frames further apart
    for f in range(nf):
        for h in range(nf):
            if abs(f - h) > 1:
                mask[f * fd:(f + 1) * fd, h * fd:(h + 1) * fd] = False
    H = np.where(mask, H, 0.0) + n * np.eye(n)
    g = rng.standard_normal(n)
    scale, D2 = 1.0 / (1.0 + np.sqrt(np.diag(H))), np.full(n, 1e-3)
    ne = dict(B=np.stack([H[f * fd:(f + 1) * fd, f * fd:(f + 1) * fd] for f in range(nf)]),
              U=np.stack([np.zeros((fd, fd))] + [H[(f - 1) * fd:f * fd, f * fd:(f + 1) * fd] for f in range(1, nf)]),
              E=np.stack([H[f * fd:(f + 1) * fd, nf * fd:] for f in range(nf)]),
              gf=g[:nf * fd].reshape(nf, fd), C=H[nf * fd:, nf * fd:], gc=g[nf * fd:])
    A = scale[:, None] * H * scale[None, :] + np.diag(D2)
    x = np.linalg.solve(A, -scale * g)
    assert cp.backward_error(ne, scale, D2, x) <= 1e-15
    A_cut = A.copy()
    A_cut[4 * fd:5 * fd, 5 * fd:6 * fd] = 0.0  # the solve forgets H[4, 5]
    A_cut[5 * fd:6 * fd, 4 * fd:5 * fd] = 0.0
    assert cp.backward_error(ne, scale, D2, np.linalg.solve(A_cut, -scale * g)) > 1e-6


def _rig_globals_accepted():
    """Every G of a rig vcgpu_set_cameras accepts: 1..8 cameras with 4..8 intrinsics each."""
    Gs = set()
    for n_cams in range(1, cp.MAX_CAMS + 1):
        for ks in itertools.combinations_with_replacement(sorted(set(cp.MODEL_K.values())), n_cams):
            Gs.add(sum(6 + k for k in ks))
    return sorted(Gs)


@pytest.mark.parametrize("inertial", [False, True])
def test_multi_launch_requests_fit_every_rig(inertial):
    """Every multi-launch kernel's dynamic shared memory, for every accepted rig and 1..4 top nodes, is at most what the
    engine opts in to.  The largest rig (8 x kb4 + IMU, G = 127) asks 219 328 B for the chain elimination and 213 856 B
    for the dense solve with 4 top nodes: more than a fixed 200 KB, less than the H100's 227 KB."""
    limit = cp.engine_smem_optin(cp.H100_SMEM_OPTIN)
    worst = {}
    for Gv in _rig_globals_accepted():
        G = Gv + (cp.IMU_GLOBALS if inertial else 0)
        for top in range(1, cp.TOP + 1):
            for k, v in cp.multi_launch_requests(G, inertial, top).items():
                if v > worst.get(k, (0, 0))[0]:
                    worst[k] = (v, G)
    over = {k: v for k, v in worst.items() if v[0] > limit}
    assert not over, f"requests (bytes, G) above the {limit} B opt-in: {over}"
    if inertial:
        assert worst["chain_eliminate_kernel"] == (219328, 127)
        assert worst["dense_solve_kernel"] == (213856, 127)
