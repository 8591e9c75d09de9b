#!/usr/bin/env python
"""Robust losses on the pair priors (rba_set_prior_loss, DESIGN.md section 22) on bench.py's flagship workload.

    python scripts/bench_prior_loss.py [--rounds 3] [--steps 10] [--warmup 3] [--profile DIR]

The Ladybug-1723 stand-in in float32 with a centre prior on every camera and the 1722 consecutive pair priors of
scripts/bench_camera_priors.py --pair-priors, plus N_FALSE false loop closures: pairs of distant cameras whose measured
relative pose is their initial one rotated by 30 degrees about a random axis and moved by 4 scene units in a random direction.  Two arms, alternated `rounds` times in one process on the same
problem: NONE on every pair, and CAUCHY with a = 3.55 (a 95 % gate on 6 degrees of freedom) on every pair.  Prints one JSON
line per arm and round (ms per LM iteration, over `steps` rba_lm_step calls after `warmup`) and the card's name and power
limit.  --profile DIR runs a separate pass of linearisations under torch.profiler and reports the time of the weighting
kernel (k_prior_weight) and of a whole linearisation.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_camera_priors import _rotations, camera_centre_priors, consecutive_pair_priors  # noqa: E402

N_FALSE = 16  # false loop closures
A_CAUCHY = 3.55


def pair_priors_with_false_closures(arrays, seed=5):
    """the consecutive pair priors, then N_FALSE pairs (i, j) between the two halves of the sequence at their initial
    relative pose T_i T_j^-1 = (M, t_i - M t_j), M = R_i R_j^T, rotated by 30 degrees and moved by 4 units"""
    from scipy.spatial.transform import Rotation
    pairs, mean, L = consecutive_pair_priors(arrays)
    rng = np.random.default_rng(seed)
    cams = np.asarray(arrays.cams, np.float64)
    nc = len(cams)
    fp = np.stack([rng.integers(0, nc // 2, N_FALSE), rng.integers(nc // 2, nc, N_FALSE)], 1).astype(np.int32)
    R = _rotations(cams)
    M = np.einsum("cab,cdb->cad", R[fp[:, 0]], R[fp[:, 1]])
    t = cams[fp[:, 0], 4:7] - np.einsum("cab,cb->ca", M, cams[fp[:, 1], 4:7])
    axis = rng.normal(size=(N_FALSE, 3))
    dirs = rng.normal(size=(N_FALSE, 3))
    fm = np.zeros((N_FALSE, 7))
    fm[:, :4] = (Rotation.from_rotvec(np.radians(30) * axis / np.linalg.norm(axis, axis=1, keepdims=True)) * Rotation.from_matrix(M)).as_quat()
    fm[:, 4:7] = t + 4.0 * dirs / np.linalg.norm(dirs, axis=1, keepdims=True)
    return np.vstack([pairs, fp]), np.vstack([mean, fm]), np.concatenate([L, L[:N_FALSE]])


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def handle(arrays, loss):
    import rootba_b200 as rb
    bp = rb.BalProblem.from_arrays(arrays, np.float32)
    bp.camera_prior = camera_centre_priors(arrays)
    bp.camera_pair_prior = pair_priors_with_false_closures(arrays)
    if loss != "NONE":
        bp.camera_pair_prior_loss = (loss, A_CAUCHY)
    return bp, rb.LinearizorQR.create(bp, rb.SolverOptions(use_double=False))


def ms_per_iteration(arrays, loss, warmup, steps):
    import torch
    bp, lin = handle(arrays, loss)
    lam, out = 1e-4, []
    for k in range(warmup + steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        lin.lm_step(lam, True)  # one LM inner iteration at a fixed lambda: linearize, solve, apply, cost
        torch.cuda.synchronize()
        if k >= warmup:
            out.append(1e3 * (time.perf_counter() - t0))
    cost = lin.compute_error()["all"]["error"]
    lin.close()
    return float(np.median(out)), float(np.min(out)), cost


def profile(arrays, out_dir, n=20):
    import torch
    from torch.profiler import ProfilerActivity
    bp, lin = handle(arrays, "CAUCHY")
    for _ in range(3):
        lin.linearize()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        for _ in range(n):
            lin.linearize()
        torch.cuda.synchronize()
    lin.close()
    os.makedirs(out_dir, exist_ok=True)
    prof.export_chrome_trace(os.path.join(out_dir, "prior_loss_trace.json"))
    tot = {}
    for ev in prof.key_averages():
        if ev.device_type.name == "CUDA" or getattr(ev, "device_time_total", 0) > 0:
            tot[ev.key] = tot.get(ev.key, 0.0) + getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0))
    weight = sum(v for k, v in tot.items() if "k_prior_weight" in k) / n
    lin_all = sum(tot.values()) / n
    return {"k_prior_weight_us_per_linearize": weight, "all_kernels_us_per_linearize": lin_all}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", default=None, metavar="DIR")
    args = ap.parse_args()
    from rootba_b200.synthetic import synth_config
    arrays = synth_config("ladybug-1723", seed=38401, scale=1.0)
    print(json.dumps({"card": card(), "workload": "synthetic ladybug-1723, float32", "pairs": len(arrays.cams) - 1 + N_FALSE,
                      "false_closures": N_FALSE}), flush=True)
    for r in range(args.rounds):
        for loss in ("NONE", "CAUCHY"):
            med, best, cost = ms_per_iteration(arrays, loss, args.warmup, args.steps)
            print(json.dumps({"round": r, "pair_loss": loss, "ms_per_lm_iteration_median": round(med, 3),
                              "ms_per_lm_iteration_min": round(best, 3), "final_cost": cost}), flush=True)
    if args.profile:
        print(json.dumps({"profile": profile(arrays, args.profile)}), flush=True)


if __name__ == "__main__":
    main()
