"""Worker for the multi-GPU parity test: run under torchrun with N ranks (one GPU each).

Every rank solves its frame shard of the same seeded problem jointly (NCCL all-reduce inside
libvcgpu), then reads the covariance of the globals on its shard; rank 0 additionally solves the whole problem on its
own GPU and compares both.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch.distributed as dist  # noqa: E402

from test_gpu_covariance_batch import BAR, _corr_err  # noqa: E402
from vicalib_b200 import synth  # noqa: E402
from vicalib_b200.capi import Calibrator  # noqa: E402


ALL_ON = dict(inertial=1, rotation_only=0, bias_active=1, scale_active=1, optimize_ts=1)


def run_case(rank, world, local, inertial, strategy=0):
    if inertial:
        p = synth.make_problem(models=("poly3", "fov"), n_frames=67, seed=34, inertial=True, ts_truth=0.002)
        flags, iters = ALL_ON, 12
    else:
        p = synth.make_problem(models=("poly3", "fov"), n_frames=64, seed=33)
        flags, iters = {}, 30
    uid = [Calibrator.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    g = Calibrator(device=local)
    g.comm_init(uid[0], rank, world)
    ps = synth.shard(p, rank, world)
    g.load(ps)
    g.set_flags(**flags)
    g.set_options(function_tol=1e-14, max_iters=iters, strategy=strategy)
    s = g.solve()
    st = g.state()
    cov = g.covariance()  # every rank, on its shard
    n_own = synth.shard_frames(p.n_frames, rank, world)
    n_own = n_own[1] - n_own[0]
    out = [None] * world
    dist.all_gather_object(out, dict(cost=s["final_cost"], iters=s["iterations"], intr=st["intr"], p_ck=st["p_ck"],
                                     q_ck=st["q_ck"], T=st["T_wp"][:n_own], v=st["v_w"][:n_own], b=st["b"], ts=st["ts"],
                                     cov=cov))
    ok = True
    if rank == 0:
        ref = Calibrator(device=local)
        ref.load(p)
        ref.set_flags(**flags)
        ref.set_options(function_tol=1e-14, max_iters=iters, strategy=strategy)
        sr = ref.solve()
        sref = ref.state()
        T = np.concatenate([o["T"] for o in out])
        checks = {
            "cost": abs(out[0]["cost"] - sr["final_cost"]) <= 1e-9 * sr["final_cost"],
            "iters": all(o["iters"] == sr["iterations"] for o in out),
            "ranks_agree": all(np.array_equal(o["intr"], out[0]["intr"]) and o["cost"] == out[0]["cost"] for o in out),
            "intr": np.abs(out[0]["intr"] - sref["intr"]).max() <= 1e-6 * np.abs(sref["intr"]).max(),
            "p_ck": np.abs(out[0]["p_ck"] - sref["p_ck"]).max() <= 1e-8,
            "poses": np.abs(T - sref["T_wp"]).max() <= 1e-8,
            "cov": _corr_err(out[0]["cov"], ref.covariance()) <= BAR[inertial],
            "cov_ranks_agree": all(np.array_equal(o["cov"], out[0]["cov"]) for o in out),
        }
        if inertial:
            V = np.concatenate([o["v"] for o in out])
            checks["vel"] = np.abs(V - sref["v_w"]).max() <= 1e-7
            checks["bias"] = np.abs(out[0]["b"] - sref["b"]).max() <= 1e-8
            checks["ts"] = abs(out[0]["ts"] - sref["ts"]) <= 1e-10
        ok = all(checks.values())
        print("MG_CHECK", ("inertial" if inertial else "vision") + (" dogleg" if strategy else ""), "PASS" if ok else "FAIL", checks, "cost", out[0]["cost"],
              sr["final_cost"], flush=True)
    flag = [ok]
    dist.broadcast_object_list(flag, src=0)
    return flag[0]


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dist.init_process_group("gloo")
    ok = run_case(rank, world, local, False)
    ok = run_case(rank, world, local, True) and ok
    ok = run_case(rank, world, local, False, strategy=1) and ok  # the reference's DOGLEG on frame shards (vision stages)
    if rank == 0:
        print("MG_CHECK", "ALL PASS" if ok else "SOME FAIL", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
