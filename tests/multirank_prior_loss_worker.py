"""Worker of the two-rank test of the robust losses on the priors (test_gpu_prior_loss.py): one process per GPU (torchrun),
landmarks sharded over the ranks, every rank given the same full lists of camera, pair and landmark priors (zero-L ones among
them) and the same losses in the caller's order; one LM step and the read-back of every prior kind compared on rank 0 with a
single-rank handle of the same problem, and each rank's landmark read-back with the float64 model.  A landmark loss mapped
to the wrong item of a shard shows up in the cost, b and the step; a read-back that writes outside the rank's shard in
`landmark_readback_covers_own_shard_only`.
Usage: torchrun --nproc-per-node N multirank_prior_loss_worker.py <out.json> <f32|f64>"""
import ctypes as C
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
    import multirank_step_worker as sw
    import prior_loss_model as plm
    import rootba_b200 as rb
    from rootba_b200 import _lib
    from rootba_b200.synthetic import synth_bal
    arrays = synth_bal(300, 6000, 4.5, seed=17, locality=2.0, max_track=40)
    priors = {"camera": sw.feature("camera", arrays)[1], "pairs": sw.feature("pair", arrays)[1],
              "landmarks": sw.feature("landmark", arrays)[1]}
    state = (np.asarray(arrays.cams, np.float64), np.asarray(arrays.lms, np.float64))
    losses = {k: plm.losses_around(k, state, priors[name], seed=29 + k) for k, name in enumerate(plm.KINDS)}
    lam = 1e-3

    def readback(lin, k, n):
        """rba_get_prior_residuals into NaN-filled buffers: entries the handle does not write stay NaN"""
        res = np.full((n, _lib.PRIOR_ROWS[k]), np.nan, lin.dtype)
        w = np.full(n, np.nan, lin.dtype)
        _lib.check(_lib.lib().rba_get_prior_residuals(lin.h, k, C.c_void_p(res.ctypes.data), C.c_void_p(w.ctypes.data)))
        return res, w

    def run(nranks, rk, comm):
        bp = rb.BalProblem.from_arrays(arrays, dtype)
        bp.camera_prior, bp.camera_pair_prior, bp.landmark_prior = priors["camera"], priors["pairs"], priors["landmarks"]
        bp.camera_prior_loss, bp.camera_pair_prior_loss, bp.landmark_prior_loss = losses[0], losses[1], losses[2]
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
        rb_all = [readback(lin, k, len(priors[name][-1])) for k, name in enumerate(plm.KINDS)]
        lin.linearize()
        inc = lin.solve(lam)
        b = lin.get_rhs()
        l_diff = lin.apply(inc)
        lin.download_state()
        cost = lin.compute_error()["all"]["error"]
        lin.close()
        return bp, st, inc, b, l_diff, cost0, cost, rb_all

    bp, st, inc, b, l_diff, cost0, cost, rb_all = run(world, rank, True)
    idx = priors["landmarks"][0]
    own = (idx >= st["landmark_begin"]) & (idx < st["landmark_end"])
    lres, lw = rb_all[2]
    covers = bool(np.all(np.isfinite(lres[own])) and np.all(np.isfinite(lw[own])) and np.all(np.isnan(lres[~own]))
                  and np.all(np.isnan(lw[~own])) and own.any() and (~own).any())
    # this rank's landmark read-back against the float64 model at the state rounded to the handle's scalar
    f = lambda a: np.asarray(np.asarray(a, dtype), np.float64)
    model = (idx, f(priors["landmarks"][1]), f(priors["landmarks"][2]))
    st0 = (f(arrays.cams), f(arrays.lms))
    want_r = plm.whitened(plm.LANDMARK, st0, model)
    want_w = np.where(plm.dropped(plm.LANDMARK, model), 1.0, plm.weights(plm.LANDMARK, st0, model, losses[2])[2])
    model_err = max(rel(lres[own], want_r[own]), float(np.max(np.abs(lw[own] - want_w[own]))))
    ok = torch.tensor([int(covers)], device="cuda")
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    merr = torch.tensor([model_err], device="cuda", dtype=torch.float64)
    dist.all_reduce(merr, op=dist.ReduceOp.MAX)
    lms = torch.from_numpy(np.where(np.arange(arrays.nl)[:, None] >= st["landmark_begin"], bp.lms, 0) *
                           (np.arange(arrays.nl)[:, None] < st["landmark_end"])).double().cuda()
    dist.all_reduce(lms)
    lres_all = torch.from_numpy(np.where(own[:, None], lres, 0)).double().cuda()
    lw_all = torch.from_numpy(np.where(own, lw, 0)).double().cuda()
    dist.all_reduce(lres_all); dist.all_reduce(lw_all)
    chk = torch.from_numpy(np.concatenate([inc, b, bp.cams.ravel()] + [np.concatenate([r.ravel(), w]) for r, w in rb_all[:2]])
                           .astype(np.float64)).cuda()
    mx, mn = chk.clone(), chk.clone()
    dist.all_reduce(mx, op=dist.ReduceOp.MAX); dist.all_reduce(mn, op=dist.ReduceOp.MIN)
    out = {"rank": rank, "world": world, "replicas_identical": bool(torch.equal(mx, mn)),
           "landmark_readback_covers_own_shard_only": bool(ok.item()), "landmark_readback_model": float(merr.item())}
    if rank == 0:
        bp1, _, inc1, b1, l1, c01, c1, rb1 = run(1, 0, False)
        out.update(b=rel(b, b1), inc=rel(inc, inc1), l_diff=abs(l_diff - l1) / abs(l1), lms=rel(lms.cpu().numpy(), bp1.lms),
                   cams=rel(bp.cams, bp1.cams), cost0=abs(cost0 - c01) / c01, cost=abs(cost - c1) / c1,
                   camera_readback=rel(np.concatenate([rb_all[0][0].ravel(), rb_all[0][1]]), np.concatenate([rb1[0][0].ravel(), rb1[0][1]])),
                   pair_readback=rel(np.concatenate([rb_all[1][0].ravel(), rb_all[1][1]]), np.concatenate([rb1[1][0].ravel(), rb1[1][1]])),
                   landmark_readback=rel(np.concatenate([lres_all.cpu().numpy().ravel(), lw_all.cpu().numpy()]),
                                         np.concatenate([rb1[2][0].ravel(), rb1[2][1]])))
        with open(out_path, "w") as fh:
            json.dump(out, fh)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
