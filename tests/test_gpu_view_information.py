"""GPU: vcgpu_get_view_information, the information candidate views would add (view_prior_kernel, view_info_kernel).
  parity      n_seen exactly, gain, var and post against tests/view_info_ref.py on the matrix vcgpu_get_covariance
              returns: five models, vision and inertial, fix_intrinsics, a camera no observation sees, two wide-lens
              rigs, G = 67 and G = 112
  end to end  the candidate appended to the problem at its predicted pixels: vcgpu_get_covariance of that problem
              gives var and gain, independently of the reference's S
  exact       no contributing corner: 0.0 and Sigma's bits; 1-3 corners: NaN; duplicates and the other candidates
              of a call do not change a candidate's bits
  chaining    post as the next prior matches the two-frame dense reference; a passed-in matrix gives the same bits
  errors      no side effects; refusals name the candidate, point or camera and write nothing"""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import chain_plan
import target_views as tv
import view_info_ref as V
import wide_lenses as W
from vicalib_b200 import synth

pytestmark = pytest.mark.gpu
ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)
# Bars, relative: gain to max(1, |gain|), var and post to sqrt(Sigma_ii Sigma_jj).  Measured on an H100 80GB HBM3
# (700 W): gain 2.3e-10, var and post 6.0e-10 (G = 67 inertial, G = 112 vision, poly3 + kb4 inertial), 2.6e-11 and below
# on the vision rigs.
GAIN_BAR, COV_BAR = 1e-8, 1e-8


def _solved(p, flags, iters=15):
    from vicalib_b200.capi import Calibrator

    g = Calibrator()
    g.models = np.asarray(p.models)
    g.load(p)
    g.set_flags(**flags)
    g.set_options(function_tol=1e-12, max_iters=iters)
    g.solve()
    return g


def _target(p):
    return np.unique(p.p_w, axis=0)[:400]


def _candidates(p, n, seed, dw=0.08, dt=0.03):
    rng = np.random.default_rng(seed)
    out = []
    for k in rng.integers(0, p.n_frames, n):
        T = p.T_wp[k]
        w = rng.normal(0, dw, 3)
        th = np.linalg.norm(w)
        dq = np.r_[np.sin(th / 2) * w / th, np.cos(th / 2)]
        q = synth.quat_mul(T[:4], dq)
        out.append(np.r_[q / np.linalg.norm(q), T[4:] + rng.normal(0, dt, 3)])
    return np.array(out)


def _used(g, p):
    return np.array([(p.obs_cam == c).any() for c in range(g.n_cams)])


def _ref(g, p, S, T, pw, flags, width=640, height=480, facing=None):
    st = g.state()
    mask = (np.diag(S) != 0).astype(float)
    return V.information(S, g.models, st["intr"], st["q_ck"], st["p_ck"], _used(g, p), mask, T, pw, width, height,
                         facing=facing, visual_mult=flags.get("visual_mult", 1.0))


def _errors(r, ref, S):
    ok = np.isfinite(ref["gain"])
    assert np.array_equal(np.isnan(r["gain"]), ~ok)
    sd = np.sqrt(np.abs(np.diag(S)))
    sc = np.where(np.outer(sd, sd) > 0, np.outer(sd, sd), 1.0)
    eg = (np.abs(r["gain"][ok] - ref["gain"][ok]) / np.maximum(1.0, np.abs(ref["gain"][ok]))).max(initial=0.0)
    ev = (np.abs(r["var"][ok] - ref["var"][ok]) / np.diag(sc)[None, :]).max(initial=0.0)
    ep = (np.abs(r["post"][ok] - ref["post"][ok]) / sc[None]).max(initial=0.0) if "post" in r else 0.0
    return eg, ev, ep


def _check(g, p, flags, T, pw, post=True, S=None, width=640, height=480, facing=None):
    S = g.covariance() if S is None else S
    r = g.view_information(T, pw, width, height, facing=facing, var=True, post=post, cov=S)
    ref = _ref(g, p, S, T, pw, flags, width, height, facing)
    assert np.array_equal(r["n_seen"], ref["n_seen"])  # every camera's, an unused one's included
    eg, ev, ep = _errors(r, ref, S)
    assert eg <= GAIN_BAR and ev <= COV_BAR and ep <= COV_BAR, (eg, ev, ep)
    assert np.array_equal(r["var"], np.diagonal(r["post"], axis1=1, axis2=2)) if post else True
    if post:
        assert np.array_equal(r["post"], np.swapaxes(r["post"], 1, 2))
    return r, (eg, ev, ep)


CASES = {
    "linear": (("linear",), False, {}),
    "fov": (("fov",), False, {}),
    "poly2": (("poly2",), False, {}),
    "poly3": (("poly3",), False, {}),
    "kb4": (("kb4",), False, {}),
    "poly3_fov_fixed": (("poly3", "fov"), False, dict(fix_intrinsics=1)),
    "poly3_kb4_inertial": (("poly3", "kb4"), True, ALL_ON),
}


@pytest.mark.parametrize("name", list(CASES))
def test_parity(name):
    models, inertial, flags = CASES[name]
    p = synth.make_problem(models=models, n_frames=60 if inertial else 18, inertial=inertial, seed=15)
    g = _solved(p, flags)
    r, e = _check(g, p, flags, _candidates(p, 24, 1), _target(p))
    print(f"{name}: gain {e[0]:.1e}, var {e[1]:.1e}, post {e[2]:.1e}, gains {np.nanmin(r['gain']):.3f}..{np.nanmax(r['gain']):.3f}")
    assert np.isfinite(r["gain"]).sum() > 12 and (r["gain"][np.isfinite(r["gain"])] >= 0).all()


@pytest.mark.parametrize("name", ["fov_kb4", "kb4_poly3_inertial"])
def test_wide_lens_rig(name):
    lens = W.build(name)
    g = _solved(lens.p, lens.flags, iters=10)
    _, e = _check(g, lens.p, lens.flags, _candidates(lens.p, 16, 2, dw=0.3), _target(lens.p))
    print(f"{name}: gain {e[0]:.1e}, var {e[1]:.1e}, post {e[2]:.1e}")


def test_unseen_camera():
    v = tv.build("unseen_camera")
    g = _solved(v.p, v.flags)
    r, e = _check(g, v.p, v.flags, _candidates(v.p, 12, 3), _target(v.p))
    assert r["n_seen"][:, v.unseen_cam].sum() > 0  # counted, though it adds nothing
    print(f"unseen camera: gain {e[0]:.1e}, var {e[1]:.1e}, post {e[2]:.1e}")


def test_facing_and_image_sizes():
    """the facing test with the target's normal towards the cameras (+n: as without a normal) and away from them (-n:
    nothing seen, so gain 0.0 and Sigma's bits), and cameras of different image sizes that cut corners off"""
    p = synth.make_problem(models=("poly3", "kb4"), n_frames=18, seed=17)
    g = _solved(p, {})
    S = g.covariance()
    pw = _target(p)
    T = _candidates(p, 16, 11)
    n = np.array([0.0, 0.0, np.sign(np.mean(p.T_wp[:, 6]))])
    front, e = _check(g, p, {}, T, pw, S=S, facing=n)
    plain = g.view_information(T, pw, 640, 480, var=True, post=True, cov=S)
    assert all(front[k].tobytes() == plain[k].tobytes() for k in plain)
    back, _ = _check(g, p, {}, T, pw, S=S, facing=-n)
    assert not back["n_seen"].any() and (back["gain"] == 0.0).all() and back["post"].tobytes() == np.broadcast_to(S, back["post"].shape).tobytes()
    # a tilted normal: some views see the target from behind
    tilted, _ = _check(g, p, {}, _candidates(p, 16, 12, dw=0.4, dt=0.15), pw, S=S, facing=n + np.array([0.9, 0.0, 0.0]))
    sized, e2 = _check(g, p, {}, T, pw, S=S, width=[600, 520], height=[430, 380])
    assert (sized["n_seen"] < plain["n_seen"]).any() and (sized["n_seen"] <= plain["n_seen"]).all()
    print(f"facing: gain {e[0]:.1e}, var {e[1]:.1e}; sizes: gain {e2[0]:.1e}, var {e2[1]:.1e}; tilted seen {tilted['n_seen'].sum()}")


@pytest.mark.parametrize("G,inertial,kw", [(67, True, dict(n_frames=48, grid=(14, 10))),
                                           (112, False, dict(n_frames=40))], ids=["inertial_G67", "vision_G112"])
def test_large_rigs(G, inertial, kw):
    models = chain_plan.rig_with_globals(67) if inertial else ("kb4",) * 8
    p = synth.make_problem(models=models, inertial=inertial, seed=G, **kw)
    flags = ALL_ON if inertial else {}
    g = _solved(p, flags)
    assert g.G == G
    _, e = _check(g, p, flags, _candidates(p, 6, 4), _target(p))
    print(f"G = {G}: gain {e[0]:.1e}, var {e[1]:.1e}, post {e[2]:.1e}")


def test_end_to_end_against_appended_problem():
    """var and gain from vcgpu_get_covariance of the problem with the candidate appended, on a fresh handle at the same
    state"""
    from vicalib_b200.capi import Calibrator

    p = synth.make_problem(models=("poly3", "kb4"), n_frames=18, seed=21)
    g = _solved(p, {})
    st = g.state()
    S = g.covariance()
    pw = _target(p)
    T = _candidates(p, 3, 5)
    r = g.view_information(T, pw, 640, 480, var=True)
    base = dataclasses.replace(p, T_wp=st["T_wp"], intr=st["intr"], q_ck=st["q_ck"], p_ck=st["p_ck"])
    F = np.diag(S) != 0
    for i, Ti in enumerate(T):
        seen, pix = V.visibility(g.models, st["intr"], st["q_ck"], st["p_ck"], Ti, pw, 640, 480)
        sel = [(c, j) for c in range(g.n_cams) for j in np.flatnonzero(seen[c])]
        q = dataclasses.replace(
            base, T_wp=np.vstack([st["T_wp"], Ti]), v_w=np.vstack([p.v_w, np.zeros(3)]), ftime=np.r_[p.ftime, p.ftime[-1] + 1.0],
            obs_frame=np.r_[p.obs_frame, np.full(len(sel), p.n_frames)].astype(np.int32),
            obs_cam=np.r_[p.obs_cam, [c for c, _ in sel]].astype(np.int32), p_w=np.vstack([p.p_w, [pw[j] for _, j in sel]]),
            p_c=np.vstack([p.p_c, [pix[c, j] for c, j in sel]]))
        h = Calibrator()
        h.load(q)
        Sq = h.covariance()
        sd = np.sqrt(np.diag(S)[F])
        assert (np.abs(r["var"][i][F] - np.diag(Sq)[F]) / sd ** 2).max() < 1e-7
        gain = 0.5 * (np.linalg.slogdet(S[np.ix_(F, F)])[1] - np.linalg.slogdet(Sq[np.ix_(F, F)])[1])
        assert abs(r["gain"][i] - gain) < 1e-7 * max(1.0, gain), (r["gain"][i], gain)


def test_exact_cases_and_bits():
    p = synth.make_problem(models=("poly3", "fov"), n_frames=18, seed=15)
    g = _solved(p, {})
    S = g.covariance()
    pw = _target(p)
    T = _candidates(p, 6, 6)
    away = T[0].copy()
    away[4:] += np.array([0.0, 0.0, 50.0]) * np.sign(np.mean(p.T_wp[:, 6]))  # far behind: nothing seen
    away[:4] = synth.quat_mul(away[:4], np.array([1.0, 0.0, 0.0, 0.0]))
    # few corners: keep only 1..3 target points
    r = g.view_information(np.vstack([T, away, T[2]]), pw, 640, 480, var=True, post=True)
    k = len(T)
    assert r["gain"][k] == 0.0 and r["var"][k].tobytes() == np.diag(S).copy().tobytes() and r["post"][k].tobytes() == S.tobytes()
    assert r["gain"][2].tobytes() == r["gain"][k + 1].tobytes() and r["post"][2].tobytes() == r["post"][k + 1].tobytes()
    alone = g.view_information(T[3:4], pw, 640, 480, var=True, post=True)
    assert alone["gain"].tobytes() == r["gain"][3:4].tobytes() and alone["post"].tobytes() == r["post"][3:4].tobytes()
    # 1 to 3 corners of a single-camera rig do not fix the view's pose: NaN; 4 do
    p1 = synth.make_problem(models=("poly3",), n_frames=18, seed=15)
    g1 = _solved(p1, {})
    pw1 = _target(p1)
    T1 = _candidates(p1, 1, 13, dw=0.02, dt=0.005)
    central = pw1[np.argsort(np.abs(pw1 - pw1.mean(0)).sum(1))]
    for n in (1, 2, 3, 4):
        few = g1.view_information(T1, central[:n], 640, 480, var=True, post=True)
        assert few["n_seen"].sum() == n
        bad = np.isnan(few["gain"]).all() and np.isnan(few["var"]).all() and np.isnan(few["post"]).all()
        assert bad == (n < 4), n
    assert few["gain"][0] > 0


def test_chaining_and_passed_matrix():
    p = synth.make_problem(models=("kb4", "poly2"), n_frames=18, seed=16)
    g = _solved(p, {})
    S = g.covariance()
    pw = _target(p)
    T = _candidates(p, 2, 7)
    a = g.view_information(T, pw, 640, 480, var=True, post=True)
    b = g.view_information(T, pw, 640, 480, var=True, post=True, cov=S)
    assert all(a[k].tobytes() == b[k].tobytes() for k in a)
    # chain: view 0's post as the prior of view 1, against the reference applied twice
    r1 = g.view_information(T[1:2], pw, 640, 480, var=True, post=True, cov=a["post"][0])
    ref0 = _ref(g, p, S, T[:1], pw, {})
    ref1 = _ref(g, p, ref0["post"][0], T[1:2], pw, {})
    eg, ev, ep = _errors(r1, ref1, S)
    assert eg <= GAIN_BAR and ev <= COV_BAR and ep <= COV_BAR, (eg, ev, ep)


def _snapshot(g, inertial):
    W_ = g.imu_weights() if inertial else np.zeros(0)
    return {k: np.asarray(v).tobytes() for k, v in g.state().items()}, W_.tobytes()


@pytest.mark.parametrize("inertial", [False, True], ids=["vision", "inertial"])
def test_no_side_effects(inertial):
    from vicalib_b200.capi import Calibrator

    def make():
        g = Calibrator()
        p = synth.make_problem(models=("poly3", "kb4"), n_frames=60 if inertial else 20, inertial=inertial, seed=8)
        g.load(p)
        g.set_flags(**(ALL_ON if inertial else {}))
        g.set_options(max_iters=4)
        return g, p

    (g, p), (fresh, _) = make(), make()
    g.solve()
    fresh.solve()
    before = _snapshot(g, inertial)
    g.view_information(_candidates(p, 8, 8), _target(p), 640, 480, var=True, post=True)
    assert _snapshot(g, inertial) == before
    s, s0 = g.solve(free_running=True), fresh.solve(free_running=True)
    for k in ("iterations", "successful_steps", "termination", "initial_cost", "final_cost"):
        assert s[k] == s0[k], k
    assert _snapshot(g, inertial) == _snapshot(fresh, inertial)


def test_errors():
    from vicalib_b200.capi import VcgpuError, ViewCandidates, _view_candidates, lib

    p = synth.make_problem(models=("poly3", "fov"), n_frames=18, seed=15)
    g = _solved(p, {}, iters=2)
    pw = _target(p)
    T = _candidates(p, 4, 9)

    def refused(match, T_=T, pw_=pw, w=640, h=480, facing=None):
        with pytest.raises(VcgpuError, match=match):
            g.view_information(T_, pw_, w, h, facing=facing)

    bad = T.copy(); bad[2, 5] = np.nan
    refused("candidate 2: pose not finite", bad)
    bad = T.copy(); bad[1, :4] *= 1.01
    refused("candidate 1: quaternion norm", bad)
    refused("camera 1: width or height", w=[640, 0])
    refused("camera 0: width or height", h=[-1, 480])
    bad = pw.copy(); bad[3, 0] = np.inf
    refused("point 3: not finite", pw_=bad)
    refused("n_pts 401 above 400", pw_=np.vstack([pw] * 5)[:401])
    refused("facing: not finite", facing=[0.0, np.nan, 1.0])
    L = lib()
    keep, v = _view_candidates(T, pw, 640, 480, None, True, False, g.n_cams, g.G)
    for field, value, match in (("n_cand", -1, "n_cand < 0"), ("n_pts", 0, "n_pts <= 0"), ("gain", None, "null T_wp")):
        b = ViewCandidates.from_buffer_copy(v)
        setattr(b, field, value)
        assert L.vcgpu_get_view_information(g.h, None, C.byref(b)) == -1
        assert match in L.vcgpu_last_error(g.h).decode()
        assert not keep[6].any() and not keep[5].any()  # nothing written
    assert L.vcgpu_get_view_information(g.h, None, None) == -1
    assert "null candidates" in L.vcgpu_last_error(g.h).decode()
    # a prior that is not positive definite: VCGPU_ERR_NUMERIC, nothing written
    S = g.covariance()
    F = np.flatnonzero(np.diag(S) != 0)
    S[F[0], F[1]] = S[F[1], F[0]] = 2 * np.sqrt(S[F[0], F[0]] * S[F[1], F[1]])
    keep, v = _view_candidates(T, pw, 640, 480, None, True, False, g.n_cams, g.G)
    assert L.vcgpu_get_view_information(g.h, S.ctypes.data_as(C.POINTER(C.c_double)), C.byref(v)) == -3
    assert not keep[6].any() and not keep[5].any()
    # no candidates: nothing written, success
    assert g.view_information(np.zeros((0, 7)), pw, 640, 480)["gain"].shape == (0,)



def test_host_method(tmp_path):
    """ViCalibrator::GetViewInformation (image sizes from its cameras) against vcgpu_get_view_information on the same
    handle, through tests/cpp/view_information_main.cc"""
    import os
    import subprocess

    from test_gpu_host_mirror import _write_problem

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "view_information")
    subprocess.run([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-Wall", "-o", exe,
                    os.path.join(root, "tests", "cpp", "view_information_main.cc"),
                    "-L" + os.path.join(root, "vicalib_b200"), "-lvcgpu", "-lpthread",
                    "-Wl,-rpath," + os.path.join(root, "vicalib_b200")], check=True, timeout=300)
    p = synth.make_problem(models=("poly3", "kb4"), n_frames=18, seed=22)
    pw, T = _target(p), _candidates(p, 8, 14)
    width, height = np.array([640, 560], np.int32), np.array([480, 400], np.int32)
    facing = np.array([0.0, 0.0, np.sign(np.mean(p.T_wp[:, 6]))])
    prob, views, res = (str(tmp_path / n) for n in ("problem.bin", "views.bin", "result.bin"))
    _write_problem(prob, p, True, 15, 0)
    with open(views, "wb") as f:
        np.array([len(T), len(pw), 1], np.int64).tofile(f)
        width.tofile(f)
        height.tofile(f)
        for a in (T, pw, facing):
            np.ascontiguousarray(a, dtype=np.float64).tofile(f)
    subprocess.run([exe, prob, views, res], check=True, timeout=600)
    out = np.fromfile(res, dtype=np.float64)
    G = int(out[:1].view(np.int64)[0])
    n, nc = len(T), p.n_cams
    per = n + n * G + n * nc
    a, b = out[1:1 + per], out[1 + per:1 + 2 * per]
    assert a.tobytes() == b.tobytes()
    gain, seen = a[:n], a[n + n * G:].reshape(n, nc)
    assert np.isfinite(gain).sum() >= n // 2 and (seen > 0).any()
