"""Worker of the two-rank tests of the held-camera and prior features (objective_checks.check_two_rank_step): one process per
GPU (torchrun), landmarks sharded over the ranks, every rank given the same held-camera flags or the same full list of priors
of one kind; compared on rank 0 with a single-rank handle of the same problem.  A prior term counted on every rank, or on
none, would show up in the cost, l_diff and the step; a held parameter moved by one shard in the step and the state.
Usage: torchrun --nproc-per-node N multirank_step_worker.py <out.json> <f32|f64> <fixed|camera|pair|landmark>"""
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


def feature(kind, arrays):
    """the BalProblem attribute and value of `kind` on the shared problem"""
    import rootba_b200 as rb
    if kind == "fixed":
        flags = np.zeros(arrays.nc, np.uint8)
        flags[::3] = rb.FIX_INTRINSICS
        flags[::7] = rb.FIX_ALL
        flags[1::11] = rb.FIX_POSE | rb.FIX_K2
        return "camera_fixed", flags
    if kind == "landmark":
        import landmark_prior_model as lp
        return "landmark_prior", lp.prior_case(arrays.lms, every=7, seed=19)
    rng = np.random.default_rng(18)
    if kind == "camera":
        import camera_prior_model as pm
        mean = pm.mean_at(arrays.cams)
        mean[:, 4:7] += rng.normal(0, 0.05, (arrays.nc, 3))
        L = np.stack([pm.sqrt_info_kind(["dense", "centre", "intrinsics", "none"][c % 4], rng) for c in range(arrays.nc)])
        return "camera_prior", (mean, L)
    assert kind == "pair", kind
    import pair_prior_model as qm
    pairs = np.array([(c, c + 1) for c in range(arrays.nc - 1)] + [(c + 7, c) for c in range(0, arrays.nc - 7, 5)], np.int32)
    mean = qm.mean_at(arrays.cams, pairs)
    mean[:, 4:7] += rng.normal(0, 0.05, (len(pairs), 3))
    L = np.stack([qm.sqrt_info_kind(["dense", "translation", "rotation", "none"][p % 4], rng) for p in range(len(pairs))])
    return "camera_pair_prior", (pairs, mean, L)


def main():
    out_path, sfx, kind = sys.argv[1], sys.argv[2], sys.argv[3]
    dtype = np.float32 if sfx == "f32" else np.float64
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_bal
    arrays = synth_bal(300, 6000, 4.5, seed=17, locality=2.0, max_track=40)
    name, value = feature(kind, arrays)
    lam = 1e-3

    def run(nranks, rk, comm):
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        setattr(bp, name, value)
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
        lin.linearize()
        inc = lin.solve(lam)
        b = lin.get_rhs()
        l_diff = lin.apply(inc)
        lin.download_state()
        cost = lin.compute_error()["all"]["error"]
        lin.close()
        return bp, st, inc, b, l_diff, cost0, cost

    cams0 = arrays.cams.astype(dtype)
    bp, st, inc, b, l_diff, cost0, cost = run(world, rank, True)
    lms = torch.from_numpy(np.where(np.arange(arrays.nl)[:, None] >= st["landmark_begin"], bp.lms, 0) *
                           (np.arange(arrays.nl)[:, None] < st["landmark_end"])).double().cuda()
    dist.all_reduce(lms)
    chk = torch.from_numpy(np.concatenate([inc, b, bp.cams.ravel()]).astype(np.float64)).cuda()
    mx, mn = chk.clone(), chk.clone()
    dist.all_reduce(mx, op=dist.ReduceOp.MAX); dist.all_reduce(mn, op=dist.ReduceOp.MIN)
    res = {"rank": rank, "world": world, "replicas_identical": bool(torch.equal(mx, mn))}
    if kind == "landmark":  # priors in every shard
        in_shard = (value[0] >= st["landmark_begin"]) & (value[0] < st["landmark_end"])
        nmine = torch.tensor([int(in_shard.sum())], device="cuda")
        nall = [torch.zeros_like(nmine) for _ in range(world)]
        dist.all_gather(nall, nmine)
        res["priors_per_shard"] = [int(t.item()) for t in nall]
    if rank == 0:
        bp1, _, inc1, b1, l1, c01, c1 = run(1, 0, False)
        res.update(b=rel(b, b1), inc=rel(inc, inc1), l_diff=abs(l_diff - l1) / abs(l1), lms=rel(lms.cpu().numpy(), bp1.lms),
                   cams=rel(bp.cams, bp1.cams))
        if kind == "fixed":
            from objective_checks import fixed_entries, fixed_params
            fp = fixed_params(value)
            res.update(fixed_inc_zero=bool(np.all(inc[fixed_entries(value)] == 0)),
                       fixed_params_identical=bool(np.array_equal(bp.cams[fp], cams0[fp])))
        else:
            res.update(cost0=abs(cost0 - c01) / c01, cost=abs(cost - c1) / c1)
        with open(out_path, "w") as f:
            json.dump(res, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
