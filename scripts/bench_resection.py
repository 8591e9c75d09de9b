#!/usr/bin/env python
"""Resection of every camera from the current landmarks (rba_resect_cameras, DESIGN.md section 26).

    python scripts/bench_resection.py [--rounds 3] [--model-sample 20] [--lm-iterations 30] [--seed 38401]

Workload: the synthetic Ladybug-1723 stand-in (rootba_b200.synthetic.synth_config("ladybug-1723"), the shape of BAL
problem-1723-156502) with its perturbed cameras.  In f32 and f64, each mode (linear, refine, linear+refine) is timed on
every camera over --rounds rounds, a fresh handle per round, after one warm-up call on another handle.  The time is that of
the whole rba_resect_cameras call between two CUDA events on the handle's stream: the host's checks, unit building and
sort, the camera snapshot, the scratch allocation and release, the uploads, the launch and the copies of the outputs; not
the kernel alone.  The minimum, median and maximum over the rounds are printed.  The float64 numpy model
(tests/resection_model.py) does the same work camera by camera in Python: it is timed on the first --model-sample cameras
and the time is scaled to all of them.  Then, in f64, an LM solve (rba_lm_run, capped at --lm-iterations) is run from the
stand-in's perturbed cameras, from the same after a linear+refine resection, and after a resection then a linear+refine
triangulation: the LM iterations and the final cost of each.  Prints one JSON line with the card's name and power limit
read in the same call.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        sys.exit("bench_resection.py: nvidia-smi found no GPU; this measurement needs an H100")
    name, power = [s.strip() for s in q.stdout.strip().split("\n")[0].split(",")]
    return name, power


def whole_call(lin, mode):
    """(seconds, status) of one rba_resect_cameras call on every camera, CUDA events around it"""
    import ctypes as C
    from rootba_b200 import _lib
    o = _lib.ResectOpts()
    _lib.lib().rba_default_resect_opts(C.byref(o))
    o.mode = _lib.RESECT_MODES[mode]
    status = np.zeros(lin.nc, np.uint8)
    lin.timer_start()
    _lib.check(_lib.lib().rba_resect_cameras(lin.h, C.byref(o), lin.nc, None, status.ctypes.data, None, None))
    return lin.timer_stop(), status


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--model-sample", type=int, default=20)
    ap.add_argument("--lm-iterations", type=int, default=30)
    ap.add_argument("--seed", type=int, default=38401)
    args = ap.parse_args()
    name, power = card()
    import resection_model as rm
    import rootba_b200 as rb
    from rootba_b200.synthetic import synth_config
    prob = synth_config("ladybug-1723", seed=args.seed)
    out = {"card": name, "power_limit": power, "num_cameras": prob.nc, "num_observations": prob.nobs}
    for dtype, sfx in ((np.float32, "f32"), (np.float64, "f64")):
        warm = rb.LinearizorQR.create(rb.BalProblem.from_arrays(prob, dtype), rb.SolverOptions())
        warm.resect()
        warm.close()
        for mode in ("linear", "refine", "linear+refine"):
            ms = []
            for _ in range(args.rounds):
                lin = rb.LinearizorQR.create(rb.BalProblem.from_arrays(prob, dtype), rb.SolverOptions())
                sec, status = whole_call(lin, mode)
                ms.append(1e3 * sec)
                lin.close()
            out[f"{sfx}_{mode}_ms_min_median_max"] = [round(min(ms), 3), round(float(np.median(ms)), 3), round(max(ms), 3)]
            out[f"{sfx}_{mode}_written"] = int(np.count_nonzero(status & rm.WRITTEN))
    k = min(args.model_sample, prob.nc)
    model = rm.Problem(prob.cams, prob.lms, prob.obs_cam, np.repeat(np.arange(prob.nl), np.diff(prob.lm_off)), prob.obs_xy)
    for mode, m in (("linear", rm.LINEAR), ("refine", rm.REFINE), ("linear+refine", rm.LINEAR | rm.REFINE)):
        t0 = time.perf_counter()
        for c in range(k):
            model.resect(c, m)
        out[f"model_{mode}_s_all"] = round((time.perf_counter() - t0) / k * prob.nc, 1)
    opts = rb.SolverOptions(max_num_iterations=args.lm_iterations)
    for arm, res, tri in (("perturbed", False, False), ("resected", True, False), ("resected_triangulated", True, True)):
        lin = rb.LinearizorQR.create(rb.BalProblem.from_arrays(prob, np.float64), opts)
        if res:
            lin.resect()
        if tri:
            lin.triangulate()
        log, _, _ = lin.lm_run(args.lm_iterations, opts)
        out[f"lm_{arm}_iterations"] = len(log)
        out[f"lm_{arm}_cost"] = lin.compute_error()["all"]["error"]
        lin.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
