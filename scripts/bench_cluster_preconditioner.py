#!/usr/bin/env python
"""SCHUR_JACOBI against CLUSTER_JACOBI at cluster sizes K = 4, 8 and 16 (preconditioner_type, DESIGN.md section 28).

    python scripts/bench_cluster_preconditioner.py [--lm-iterations 20] [--seed 38401] [--only NAME,...]

Workloads: the synthetic stand-ins of Ladybug-1723 (f32, the bench.py workload) and Trafalgar-257 (f64)
(rootba_b200.synthetic.synth_config), and a sequential synthetic problem of 500 cameras (60 landmarks per camera, 4
observations per landmark, local visibility) with an odometry pair prior between every two consecutive cameras (f64).

Per workload and arm, rba_lm_run for --lm-iterations iterations from the same start: PCG iterations per solve, the solves
that stop at the 500-iteration cap, the cost after the fixed number of iterations and the device time per LM iteration
(rba_lm_run's per-iteration CUDA-event times).  Then, from a torch.profiler run of one solve at lambda = 1e-4 after the
run, the kernel time of the cluster assembly and factorisation (k_cluster_build, and the L^-1 b it is followed by) and of
the apply per PCG iteration (k_cluster_back + k_cluster_fwd).  Prints one JSON line per workload and the card's name and
power limit, read in the same call.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

ARMS = [("SCHUR_JACOBI", None), ("CLUSTER_JACOBI", 4), ("CLUSTER_JACOBI", 8), ("CLUSTER_JACOBI", 16)]
CAP = 500


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        sys.exit("bench_cluster_preconditioner.py: nvidia-smi found no GPU; this measurement needs an H100")
    name, power = [s.strip() for s in q.stdout.strip().split("\n")[0].split(",")]
    return name, power


def kernel_ms(lin, lam):
    """kernel milliseconds of one solve by kernel family, from torch.profiler's CUDA activity"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        lin.solve(lam)
        torch.cuda.synchronize()
    out = {"build": 0.0, "fwd": 0.0, "back": 0.0, "fwd_calls": 0, "all": 0.0}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = (e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total) / 1e3
        out["all"] += t
        for k in ("build", "fwd", "back"):
            if f"k_cluster_{k}" in e.name:
                out[k] += t
                if k == "fwd":
                    out["fwd_calls"] += 1
    return out, int(lin.last_cg.num_iterations)


def sequential(seed):
    """500 cameras along a path, each landmark seen by nearby cameras, and an odometry prior on every consecutive pair"""
    import pair_prior_model as qm
    from rootba_b200.synthetic import synth_bal
    prob = synth_bal(500, 30000, 4.0, seed, locality=2.0)
    pairs = np.array([(i + 1, i) for i in range(prob.nc - 1)], np.int32)
    mean = qm.mean_at(prob.cams, pairs)
    L = np.tile(np.eye(6) * 10.0, (len(pairs), 1, 1))
    return prob, (pairs, mean, L)


def arm_run(prob, dtype, pairs, pc, k, args):
    import rootba_b200 as rb
    so = rb.SolverOptions(max_num_iterations=args.lm_iterations, preconditioner_type=pc)
    bp = rb.BalProblem.from_arrays(prob, dtype)
    if pairs is not None:
        bp.camera_pair_prior = pairs
    lin = rb.LinearizorQR.create(bp, so)
    if k is not None:
        lin.set_camera_clusters(rb.cluster_cameras(bp, k))
    lin.lm_run(2, so)  # warm-up: modules, the assembled operator's first build
    bp2 = rb.BalProblem.from_arrays(prob, dtype)
    lin.bal_problem.cams[:] = bp2.cams
    lin.bal_problem.lms[:] = bp2.lms
    lin.upload_state()
    its, _, _ = lin.lm_run(args.lm_iterations, so)
    out = {"lm_iterations": len(its), "accepted": sum(it["accepted"] for it in its),
           "pcg_per_solve": round(float(np.mean([it["cg_iterations"] for it in its])), 1),
           "solves_at_cap": sum(it["cg_iterations"] >= CAP for it in its),
           "cost": lin.compute_error()["all"]["error"],
           "ms_per_lm_iteration": round(1e3 * float(np.mean([it["device_seconds"] for it in its])), 3)}
    lin.linearize()
    km, iters = kernel_ms(lin, 1e-4)
    if k is not None:
        out["assembly_factor_ms"] = round(km["build"] + km["fwd"] / max(km["fwd_calls"], 1), 3)
        out["apply_ms_per_pcg_iteration"] = round((km["back"] + km["fwd"] * (1 - 1 / max(km["fwd_calls"], 1))) / max(iters, 1), 4)
    out["profiled_solve_kernel_ms"] = round(km["all"], 3)
    out["profiled_solve_pcg_iterations"] = iters
    lin.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lm-iterations", type=int, default=20)
    ap.add_argument("--seed", type=int, default=38401)
    ap.add_argument("--only", default="", help="comma-separated workload names to run (default: all)")
    args = ap.parse_args()
    name, power = card()
    import torch
    torch.cuda.init()
    from rootba_b200.synthetic import synth_config
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    runs = [("ladybug-1723", lambda: (synth_config("ladybug-1723", seed=args.seed), None), np.float32),
            ("trafalgar-257", lambda: (synth_config("trafalgar-257", seed=args.seed), None), np.float64),
            ("sequential-500-pairs", lambda: sequential(args.seed), np.float64)]
    only = set(s for s in args.only.split(",") if s)
    for wname, make, dtype in runs:
        if only and wname not in only:
            continue
        prob, pairs = make()
        out = {"workload": wname, "dtype": np.dtype(dtype).name, "num_cameras": prob.nc, "num_observations": prob.nobs}
        for pc, k in ARMS:
            out[pc if k is None else f"{pc}-{k}"] = arm_run(prob, dtype, pairs, pc, k, args)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
