#!/usr/bin/env python
"""The exact solve of the reduced camera system (linear_solver_type = DENSE_SCHUR, DESIGN.md section 27).

    python scripts/bench_dense_solver.py [--solves 3] [--lm-iterations 50] [--sweep 100,250,500,1000] [--seed 38401]

Workloads: the synthetic stand-ins of Trafalgar-257 (f64) and Ladybug-1723 (f32, f64) (rootba_b200.synthetic.synth_config),
and a sweep of camera counts from the generator with the Ladybug stand-in's sequence-like visibility (60 landmarks per
camera, 4 observations per landmark, f64), which is where PCG needs the most iterations.

Per workload:
  * one DENSE_SCHUR solve at lambda = 1e-4 after a warm-up solve, --solves times: the solve's CUDA-event time
    (solve_reduced_system_time, which covers the whole dense path) and, from a separate torch.profiler run of one solve, the
    kernel time of each phase by kernel name: the landmark pass (k_dense_landmark), the assembly (k_cov_assemble, the
    priors, the group and rig passes, the scaling, k_cov_equil, k_dense_gather), potrf (k_cov_tile_*, k_cov_dgemm) and the
    triangular solves (k_dense_trsv_*, k_dense_finish).  The copies and memsets between them are not in the phases.  FP64
    TFLOP/s of the factorisation = (N^3 / 3) / potrf kernel time, N = 9 nc rounded up to 64.
  * rba_lm_run to convergence (or --lm-iterations) with ITERATIVE_SCHUR (the default options) and with DENSE_SCHUR: LM
    iterations, accepted steps, PCG iterations, final cost and the device time summed over the iterations.
Prints one JSON line per workload and the card's name and power limit, read in the same call.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PHASES = {"landmark": ("k_dense_landmark",),
          "assembly": ("k_cov_assemble", "k_cov_priors", "k_cov_group", "k_cov_rig", "k_sensor_tie", "k_dense_scaling",
                       "k_dense_tied_scaling", "k_cov_equil", "k_dense_gather"),
          "potrf": ("k_cov_tile_potrf", "k_cov_tile_trtri", "k_cov_dgemm"),
          "trsv": ("k_dense_trsv", "k_dense_finish")}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        sys.exit("bench_dense_solver.py: nvidia-smi found no GPU; this measurement needs an H100")
    name, power = [s.strip() for s in q.stdout.strip().split("\n")[0].split(",")]
    return name, power


def phase_times(lin, lam):
    """kernel milliseconds per phase of one solve, from torch.profiler's CUDA activity"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        lin.solve(lam)
        torch.cuda.synchronize()
    out = {k: 0.0 for k in PHASES}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for k, names in PHASES.items():
            if any(n in e.name for n in names):
                out[k] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
                break
    return out


def workload(name, prob, dtype, args):
    import rootba_b200 as rb
    out = {"workload": name, "dtype": np.dtype(dtype).name, "num_cameras": prob.nc, "num_observations": prob.nobs}
    n = (9 * prob.nc + 63) // 64 * 64
    out["N"] = n
    dense = dict(linear_solver_type="DENSE_SCHUR")
    lin = rb.LinearizorQR.create(rb.BalProblem.from_arrays(prob, dtype), rb.SolverOptions(**dense))
    lin.compute_error()
    lin.linearize()
    lin.solve(1e-4)  # warm-up
    ms = []
    for _ in range(args.solves):
        lin.solve(1e-4)
        ms.append(1e3 * lin.timings()["solve_reduced_system_time"])
    out["solve_ms_min_median_max"] = [round(min(ms), 3), round(float(np.median(ms)), 3), round(max(ms), 3)]
    out["solve_termination"] = int(lin.last_cg.termination_type)
    ph = phase_times(lin, 1e-4)
    out["phase_kernel_ms"] = {k: round(v, 3) for k, v in ph.items()}
    if ph["potrf"] > 0:
        out["potrf_fp64_tflops"] = round(n ** 3 / 3 / (ph["potrf"] * 1e-3) / 1e12, 2)
    out["dense_matrix_gb"] = round(8 * n * n / 1e9, 3)
    lin.close()
    for arm, cfg in (("iterative", {}), ("dense", dense)):
        so = rb.SolverOptions(max_num_iterations=args.lm_iterations, **cfg)
        lin = rb.LinearizorQR.create(rb.BalProblem.from_arrays(prob, dtype), so)
        its, _, _ = lin.lm_run(args.lm_iterations, so)
        out[f"lm_{arm}"] = {"iterations": len(its), "accepted": sum(it["accepted"] for it in its),
                            "pcg_iterations": sum(it["cg_iterations"] for it in its),
                            "final_cost": lin.compute_error()["all"]["error"],
                            "device_s": round(sum(it["device_seconds"] for it in its), 4)}
        lin.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solves", type=int, default=3)
    ap.add_argument("--lm-iterations", type=int, default=50)
    ap.add_argument("--sweep", default="100,250,500,1000")
    ap.add_argument("--seed", type=int, default=38401)
    ap.add_argument("--only", default="", help="comma-separated workload names to run (default: all)")
    args = ap.parse_args()
    name, power = card()
    import torch
    torch.cuda.init()
    from rootba_b200.synthetic import synth_bal, synth_config
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    runs = [("trafalgar-257", lambda: synth_config("trafalgar-257", seed=args.seed), np.float64),
            ("ladybug-1723", lambda: synth_config("ladybug-1723", seed=args.seed), np.float32),
            ("ladybug-1723", lambda: synth_config("ladybug-1723", seed=args.seed), np.float64)]
    for nc in [int(s) for s in args.sweep.split(",") if s]:
        runs.append((f"sweep-{nc}", lambda nc=nc: synth_bal(nc, 60 * nc, 4.0, args.seed, locality=2.0), np.float64))
    only = set(s for s in args.only.split(",") if s)
    for wname, make, dtype in runs:
        if only and wname not in only:
            continue
        print(json.dumps(workload(wname, make(), dtype, args)), flush=True)


if __name__ == "__main__":
    main()
