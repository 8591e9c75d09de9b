"""Worker of the two-rank test of per-observation losses (test_gpu_observation_loss.py): one process per GPU (torchrun),
landmarks sharded over the ranks, every rank given the same full arrays (kind, scale) of mixed kinds; one LM step and the
residual read-back compared on rank 0 with a single-rank handle of the same problem.  An observation weighed by another
observation's loss shows up in the cost, b and the step; a read-back that writes outside the rank's shard in
`readback_covers_own_shard_only`.
Usage: torchrun --nproc-per-node N multirank_observation_loss_worker.py <out.json> <f32|f64>"""
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


def main():
    out_path, sfx = sys.argv[1], sys.argv[2]
    dtype = np.float32 if sfx == "f32" else np.float64
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import observation_loss_model as lm
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_bal
    arrays = synth_bal(300, 6000, 4.5, seed=17, locality=2.0, max_track=40)
    kind, scale = lm.mixed(arrays.nobs, seed=23)
    lam = 1e-3

    def run(nranks, rk, comm):
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        bp.observation_loss = (kind, scale)
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(device=local, rank=rk, nranks=nranks))
        if comm:
            uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
            if rank == 0:
                uid.copy_(torch.frombuffer(bytearray(rb.nccl_unique_id()), dtype=torch.uint8))
            dist.broadcast(uid, 0)
            lin.comm_init(bytes(uid.cpu().numpy().tobytes()))
            mine = torch.frombuffer(bytearray(lin.ipc_export()), dtype=torch.uint8).cuda()
            allh = [torch.zeros(len(mine), dtype=torch.uint8, device="cuda") for _ in range(world)]
            dist.all_gather(allh, mine)
            lin.ipc_import(b"".join(bytes(t.cpu().numpy().tobytes()) for t in allh))  # no-op with RBA_PEER_AR=0
        st = lin.stats()
        cost0 = lin.compute_error()["all"]["error"]
        readback = lin.observation_residuals()
        lin.linearize()
        inc = lin.solve(lam)
        b = lin.get_rhs()
        l_diff = lin.apply(inc)
        lin.download_state()
        cost = lin.compute_error()["all"]["error"]
        lin.close()
        return bp, st, inc, b, l_diff, cost0, cost, readback

    bp, st, inc, b, l_diff, cost0, cost, (res, hw, flags) = run(world, rank, True)
    own_lm = (np.arange(arrays.nl) >= st["landmark_begin"]) & (np.arange(arrays.nl) < st["landmark_end"])
    own_obs = np.repeat(own_lm, np.diff(arrays.lm_off))
    # in its shard every observation is in use with a positive weight or a Tukey rejection; outside nothing was written
    covers = bool(np.all(flags[own_obs] & 2) and np.all(hw[own_obs] >= 0) and np.all(hw[~own_obs] == 0) and np.all(res[~own_obs] == 0)
                  and np.all(flags[~own_obs] == 0))
    ok = torch.tensor([int(covers)], device="cuda")
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    lms = torch.from_numpy(np.where(own_lm[:, None], bp.lms, 0)).double().cuda()
    dist.all_reduce(lms)
    res_all = torch.from_numpy(np.where(own_obs[:, None], res, 0)).double().cuda()
    dist.all_reduce(res_all)
    chk = torch.from_numpy(np.concatenate([inc, b, bp.cams.ravel()]).astype(np.float64)).cuda()
    mx, mn = chk.clone(), chk.clone()
    dist.all_reduce(mx, op=dist.ReduceOp.MAX); dist.all_reduce(mn, op=dist.ReduceOp.MIN)
    out = {"rank": rank, "world": world, "replicas_identical": bool(torch.equal(mx, mn)), "readback_covers_own_shard_only": bool(ok.item())}
    if rank == 0:
        bp1, _, inc1, b1, l1, c01, c1, (res1, _, _) = run(1, 0, False)
        out.update(b=rel(b, b1), inc=rel(inc, inc1), l_diff=abs(l_diff - l1) / abs(l1), lms=rel(lms.cpu().numpy(), bp1.lms),
                   cams=rel(bp.cams, bp1.cams), cost0=abs(cost0 - c01) / c01, cost=abs(cost - c1) / c1,
                   residuals=rel(res_all.cpu().numpy(), res1))
        with open(out_path, "w") as f:
            json.dump(out, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
