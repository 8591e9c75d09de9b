"""Worker of the two-rank test of rba_triangulate_landmarks (test_gpu_triangulation.py): one process per GPU (torchrun),
landmarks sharded over the ranks, every rank given the same full list; the union of the shards' positions, status, angle
and cost compared bit for bit on rank 0 with a single-rank handle of the same problem, with observation information,
losses and landmark priors on.  An output written outside the rank's shard shows up in `covers_own_shard_only`.
Usage: torchrun --nproc-per-node N multirank_triangulation_worker.py <out.json> <f32|f64>"""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    out_path, sfx = sys.argv[1], sys.argv[2]
    dtype = np.float32 if sfx == "f32" else np.float64
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import observation_loss_model as lm
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_bal
    arrays = synth_bal(300, 6000, 4.5, seed=19, locality=2.0, max_track=40, perturb_lm=1.0)
    kind, scale = lm.mixed(arrays.nobs, seed=29)
    rng = np.random.default_rng(5)
    W = np.broadcast_to(np.eye(2), (arrays.nobs, 2, 2)).copy()
    W[rng.random(arrays.nobs) < 0.1] = 0.0
    pidx = np.arange(0, arrays.nl, 7, dtype=np.int32)
    prior = (pidx, arrays.lms[pidx] + rng.normal(0, 0.1, (len(pidx), 3)), np.broadcast_to(np.eye(3) * 3.0, (len(pidx), 3, 3)))
    lst = rng.permutation(arrays.nl)[: arrays.nl // 2].astype(np.int32)

    def run(nranks, rk):
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        bp.observation_sqrt_info = W
        bp.observation_loss = (kind, scale)
        bp.landmark_prior = prior
        lin = rb.LinearizorQR.create(bp, rb.SolverOptions(device=local, rank=rk, nranks=nranks))
        st = lin.stats()
        full = lin.triangulate()
        sub = lin.triangulate(lst, mode="refine")
        lin.close()
        return bp, st, full, sub

    bp, st, full, sub = run(world, rank)
    own = (np.arange(arrays.nl) >= st["landmark_begin"]) & (np.arange(arrays.nl) < st["landmark_end"])
    own_sub = own[lst]
    covers = all(np.all(a[~own] == 0) for a in full) and all(np.all(a[~own_sub] == 0) for a in sub)
    ok = torch.tensor([int(covers)], device="cuda")
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    gather = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).cuda()  # noqa: E731
    lms = gather(np.where(own[:, None], bp.lms, 0))
    outs = [gather(a) for a in full + sub]
    for t in [lms] + outs:
        dist.all_reduce(t)  # every entry is non-zero on exactly one rank: the sum is that rank's value, bit for bit
    out = {"rank": rank, "world": world, "covers_own_shard_only": bool(ok.item())}
    if rank == 0:
        bp1, _, full1, sub1 = run(1, 0)
        same = [bool(np.array_equal(t.cpu().numpy(), np.asarray(a, np.float64))) for t, a in zip(outs, full1 + sub1)]
        out.update(lms_identical=bool(np.array_equal(lms.cpu().numpy(), np.asarray(bp1.lms, np.float64))), outputs_identical=same,
                   written=int(np.count_nonzero(full1[0] & 1)))
        with open(out_path, "w") as f:
            json.dump(out, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
