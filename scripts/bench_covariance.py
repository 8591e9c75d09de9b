#!/usr/bin/env python
"""Device time of rba_compute_covariance (DESIGN.md section 16) on a synthetic stand-in.

    python scripts/bench_covariance.py [--workload ladybug-1723|venice-1778] [--lm-steps 10] [--reps 3] [--profile DIR]

Set-up: the stand-in in float32 with a centre prior on every camera, as scripts/bench_camera_priors.py sets them (they fix the
gauge), after an LM run of --lm-steps iterations.  Then one untimed call (it builds the term list cached on the handle) and
--reps calls timed with the handle's CUDA-event timer.  The dense work of the factorisation and inversion is N^3 flops for
N = 9 Nc (computed, not measured); the rate printed is N^3 over the summed device time of the dense kernels when --profile
gives per-kernel times, else N^3 over the whole call (a lower bound of the dense kernels' rate).  The data-sheet FP64 tensor
rate of an H100 SXM is 67 TFLOP/s at 700 W.  --profile DIR runs torch.profiler over one more call, in a separate pass after the
timed ones, and writes its trace there.  Prints one JSON line.
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_camera_priors import camera_centre_priors  # noqa: E402

DENSE_KERNELS = ("k_cov_dgemm", "k_cov_tile_potrf", "k_cov_tile_trtri", "k_cov_tile_lauu2")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="ladybug-1723", choices=["ladybug-1723", "venice-1778"])
    ap.add_argument("--seed", type=int, default=38401)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--lm-steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--profile", default=None, metavar="DIR")
    args = ap.parse_args()

    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_config
    arrays = synth_config(args.workload, seed=args.seed, scale=args.scale)
    bp = rb.BalProblem.from_arrays(arrays, np.float32)
    bp.camera_prior = camera_centre_priors(arrays)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(use_double=False))
    its, _, _ = lin.lm_run(args.lm_steps)
    n = 9 * lin.nc
    lin.covariance()  # warm-up: term list, module load
    times = []
    for _ in range(args.reps):
        lin.timer_start()
        cam, lm = lin.covariance()
        times.append(lin.timer_stop())
    call = float(np.median(times))
    flops = float(n) ** 3
    out = {"workload": args.workload, "card": card(), "num_cameras": lin.nc, "num_landmarks": lin.nl, "N": n,
           "lm_steps": len(its), "call_seconds": times, "call_seconds_median": call, "dense_flops_computed": flops,
           "fp64_tflops_whole_call": flops / call / 1e12,
           "finite_camera_blocks": int(np.isfinite(cam).all(axis=(1, 2)).sum()),
           "finite_landmark_blocks": int(np.isfinite(lm).all(axis=(1, 2)).sum())}
    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            lin.covariance()
            torch.cuda.synchronize()
        os.makedirs(args.profile, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.profile, f"covariance_{args.workload}.pt.trace.json"))
        per = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            if t > 0 and "k_cov" in ev.key:
                name = ev.key.split("(")[0].replace("void ", "").replace("rba::", "").split("<")[0]
                d = per.setdefault(name, {"us": 0.0, "count": 0})
                d["us"] += t
                d["count"] += ev.count
        out["kernels_us"] = per
        dense_us = sum(v["us"] for k, v in per.items() if k in DENSE_KERNELS)
        if dense_us > 0:
            out["dense_kernels_seconds"] = dense_us * 1e-6
            out["fp64_tflops_dense_kernels"] = flops / (dense_us * 1e-6) / 1e12
    lin.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
