"""Worker of the two-rank test of estimated rig extrinsics (test_gpu_rig_sensors.py): one process per GPU (torchrun),
landmarks sharded over the ranks, every rank given the same rigs, sensors and camera priors; the sharded step (the NCCL
hand-over with the rig and sensor contraction after the all-reduce) compared on rank 0 with a single-rank handle of the same
problem, and the cameras bit-identical across the ranks.
Usage: torchrun --nproc-per-node N multirank_rig_sensors_worker.py <out.json> <f32|f64> <JACOBI|SCHUR_JACOBI>"""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def rel(a, b):
    a = np.asarray(a, np.float64).ravel(); b = np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / (np.linalg.norm(a) + np.linalg.norm(b) + 1e-300))


def rigs(nc):
    """rigs of 3 consecutive cameras, every 7th camera free"""
    return np.where(np.arange(nc) % 7 == 0, -1, np.arange(nc) // 3).astype(np.int32)


def sensors(rig):
    """the last camera of every rig of 3 is a capture of one estimated sensor"""
    c = np.arange(len(rig))
    return np.where((rig >= 0) & (c % 3 == 2), 5, -1).astype(np.int32)


def camera_prior(arrays):
    import camera_prior_model as pm
    rng = np.random.default_rng(18)
    mean = pm.mean_at(arrays.cams)
    mean[:, 4:7] += rng.normal(0, 0.05, (arrays.nc, 3))
    L = np.stack([pm.sqrt_info_kind(["dense", "centre", "intrinsics", "none"][c % 4], rng) for c in range(arrays.nc)])
    return mean, L


def main():
    out_path, sfx, precond = sys.argv[1], sys.argv[2], sys.argv[3]
    dtype = np.float32 if sfx == "f32" else np.float64
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import rootba_b200 as rb
    import camera_rig_model as rm
    from rootba_b200.synthetic import synth_bal
    arrays = synth_bal(300, 6000, 4.5, seed=17, locality=2.0, max_track=40)
    rig, prior = rigs(arrays.nc), camera_prior(arrays)
    E = rm.rig_case(arrays.nc, seed=4)
    lam = 1e-3

    def run(nranks, rk, comm):
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        bp.camera_prior = prior
        bp.camera_rig = (rig, E)
        bp.rig_sensor = sensors(rig)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(device=local, rank=rk, nranks=nranks, preconditioner_type=precond))
        if comm:
            uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
            if rank == 0:
                uid.copy_(torch.frombuffer(bytearray(rb.nccl_unique_id()), dtype=torch.uint8))
            dist.broadcast(uid, 0)
            lin.comm_init(bytes(uid.cpu().numpy().tobytes()))
            mine = torch.frombuffer(bytearray(lin.ipc_export()), dtype=torch.uint8).cuda()
            allh = [torch.zeros(len(mine), dtype=torch.uint8, device="cuda") for _ in range(world)]
            dist.all_gather(allh, mine)
            lin.ipc_import(b"".join(bytes(t.cpu().numpy().tobytes()) for t in allh))  # mapped peers: still NCCL with sensors
        st = lin.stats()
        cost0 = lin.compute_error()["all"]["error"]
        lin.linearize()
        inc = lin.solve(lam)
        b = lin.get_rhs()
        l_diff = lin.apply(inc)
        lin.download_state()
        cost = lin.compute_error()["all"]["error"]
        lin.close()
        return bp, st, inc, b, l_diff, cost0, cost

    bp, st, inc, b, l_diff, cost0, cost = run(world, rank, True)
    lms = torch.from_numpy(np.where(np.arange(arrays.nl)[:, None] >= st["landmark_begin"], bp.lms, 0) *
                           (np.arange(arrays.nl)[:, None] < st["landmark_end"])).double().cuda()
    dist.all_reduce(lms)
    chk = torch.from_numpy(np.concatenate([inc, b, bp.cams.ravel()]).astype(np.float64)).cuda()
    mx, mn = chk.clone(), chk.clone()
    dist.all_reduce(mx, op=dist.ReduceOp.MAX); dist.all_reduce(mn, op=dist.ReduceOp.MIN)
    res = {"rank": rank, "world": world, "replicas_identical": bool(torch.equal(mx, mn))}
    if rank == 0:
        bp1, _, inc1, b1, l1, c01, c1 = run(1, 0, False)
        res.update(b=rel(b, b1), inc=rel(inc, inc1), l_diff=abs(l_diff - l1) / abs(l1), lms=rel(lms.cpu().numpy(), bp1.lms),
                   cams=rel(bp.cams, bp1.cams), cost0=abs(cost0 - c01) / c01, cost=abs(cost - c1) / c1)
        with open(out_path, "w") as f:
            json.dump(res, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
