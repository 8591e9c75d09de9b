"""Worker of the two-rank test of camera rigs (test_gpu_camera_rigs.py): one process per GPU (torchrun), landmarks sharded
over the ranks, every rank given the same rigs (and camera priors, whose terms are contracted too); the sharded step (the
NCCL hand-over with the rig contraction after the all-reduce; with SCHUR_JACOBI also the cross-rank sum of the blocks D_u is
built from) compared on rank 0 with a single-rank handle of the same problem, the cameras bit-identical across the ranks
and every member at M_j T_lead.
Usage: torchrun --nproc-per-node N multirank_camera_rigs_worker.py <out.json> <f32|f64> <JACOBI|SCHUR_JACOBI>"""
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
            lin.ipc_import(b"".join(bytes(t.cpu().numpy().tobytes()) for t in allh))  # mapped peers: still NCCL with rigs
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
        lead = rm.leads(rig)
        M = rm.maps(np.asarray(np.asarray(E, dtype), np.float64), lead)
        cams = np.asarray(bp.cams, np.float64)
        u = 1e-15 if dtype == np.float64 else 1e-6
        rigid = 0.0
        for c in np.flatnonzero((lead >= 0) & (lead != np.arange(arrays.nc))):
            q, t = rm.relative(cams[c], cams[lead[c]])
            q *= np.sign(q[3]) * np.sign(M[c, 3])
            rigid = max(rigid, np.max(np.abs(q - M[c, :4])) / u,
                        np.max(np.abs(t - M[c, 4:])) / (u * (1.0 + np.linalg.norm(cams[lead[c], 4:7]))))
        res.update(b=rel(b, b1), inc=rel(inc, inc1), l_diff=abs(l_diff - l1) / abs(l1), lms=rel(lms.cpu().numpy(), bp1.lms),
                   cams=rel(bp.cams, bp1.cams), cost0=abs(cost0 - c01) / c01, cost=abs(cost - c1) / c1, rigid=float(rigid))
        with open(out_path, "w") as f:
            json.dump(res, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
