#!/usr/bin/env python
"""Device time of rba_compute_covariance_blocks (DESIGN.md section 20) on a synthetic stand-in.

    python scripts/bench_covariance_blocks.py [--workload ladybug-1723|venice-1778] [--lm-steps 10] [--reps 3]

Set-up as scripts/bench_covariance.py: the stand-in in float32 with a centre prior on every camera, after an LM run of
--lm-steps iterations, then one untimed call (term list, module load).  The call with cam_cov only (the factorisation and the
camera marginals) is timed with the handle's CUDA-event timer, --reps calls, median.  The call-to-call spread of that time
(tens of ms) is larger than the extraction, so the extra device time of 10^3, 10^4 and 10^5 random requests of each kind
(camera pairs, camera-landmark pairs, landmark pairs, relative poses) is the device time of that kind's extraction kernel and
the copies of its requests and outputs, read from torch.profiler over one call per kind and count (after the timed calls).
Prints one JSON line.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_camera_priors import camera_centre_priors  # noqa: E402
from bench_covariance import card  # noqa: E402

COUNTS = (10 ** 3, 10 ** 4, 10 ** 5)
KERNEL = {"cameras": "k_cov_cam_cross", "camera_landmark": "k_cov_cam_lm", "landmarks": "k_cov_lm_cross",
          "relative": "k_cov_rel_pose"}


def requests(rng, kind, m, nc, nl):
    if kind == "cameras":
        return rng.integers(0, nc, (m, 2))
    if kind == "camera_landmark":
        return np.stack([rng.integers(0, nc, m), rng.integers(0, nl, m)], 1)
    if kind == "landmarks":
        return rng.integers(0, nl, (m, 2))
    i = rng.integers(0, nc, m)
    return np.stack([i, (i + rng.integers(1, nc, m)) % nc], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="ladybug-1723", choices=["ladybug-1723", "venice-1778"])
    ap.add_argument("--seed", type=int, default=38401)
    ap.add_argument("--lm-steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()

    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_config
    arrays = synth_config(args.workload, seed=args.seed)
    bp = rb.BalProblem.from_arrays(arrays, np.float32)
    bp.camera_prior = camera_centre_priors(arrays)
    lin = rb.LinearizorQR.create(bp, rb.SolverOptions(use_double=False))
    its, _, _ = lin.lm_run(args.lm_steps)

    times = []
    lin.covariance(landmarks=False)  # warm-up: term list, module load
    for _ in range(args.reps):
        lin.timer_start()
        lin.covariance(landmarks=False)
        times.append(lin.timer_stop())
    base = float(np.median(times))

    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    rng = np.random.default_rng(1)
    extra = {}
    for kind in ("cameras", "camera_landmark", "landmarks", "relative"):
        for m in COUNTS:
            req = requests(rng, kind, m, lin.nc, lin.nl)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                lin.covariance_blocks(**{kind: req})
                torch.cuda.synchronize()
            us = {"kernel": 0.0, "copies": 0.0}
            for ev in prof.key_averages():
                t = getattr(ev, "device_time_total", None)
                t = ev.cuda_time_total if t is None else t
                if KERNEL[kind] in ev.key:
                    us["kernel"] += t
                elif "Memcpy" in ev.key and ("HtoD" in ev.key or "DtoH" in ev.key):
                    us["copies"] += t
            extra[f"{kind}_{m}"] = {"kernel_seconds": us["kernel"] * 1e-6, "copy_seconds": us["copies"] * 1e-6}
    out = {"workload": args.workload, "card": card(), "num_cameras": lin.nc, "num_landmarks": lin.nl, "N": 9 * lin.nc,
           "lm_steps": len(its), "cam_cov_call_seconds": base, "cam_cov_call_seconds_all": times,
           "extra_device_seconds": extra}
    lin.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
