#!/usr/bin/env python
"""Triangulation of every landmark from the current cameras (rba_triangulate_landmarks, DESIGN.md section 25).

    python scripts/bench_triangulation.py [--rounds 3] [--model-sample 300] [--lm-iterations 30] [--seed 38401]

Workload: the synthetic Ladybug-1723 stand-in (rootba_b200.synthetic.synth_config("ladybug-1723"), the shape of BAL
problem-1723-156502) with its perturbed landmarks.  In f32 and f64, each mode (linear, refine, linear+refine) is timed on
every landmark over --rounds rounds, a fresh handle per round, after one warm-up call on another handle.  The time is that of
the whole rba_triangulate_landmarks call between two CUDA events on the handle's stream: the host's checks and sort, the
scratch allocation and release, the item upload, the launch and the copies of the outputs; not the kernel alone.  The
minimum, median and maximum over the rounds are printed.  A long-track case times the same whole call on 64 landmarks
seen by 350 cameras each (61 075 ray pairs per landmark in the angle pass), near the longest track a float64 handle
accepts (its dense-operator scratch bounds the track length).  The
float64 numpy model (tests/triangulation_model.py) does the same work landmark by landmark in Python: it is timed on the
first --model-sample landmarks and the time is scaled to all of them.  Then, in f64, an LM solve (rba_lm_run) from
landmarks scrambled by N(0, 5) is run with and without a linear+refine triangulation first, and one from the stored
landmarks as the reference: the LM iterations and the final cost of each.  Prints one JSON line with the card's name and
power limit read in the same call.
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
        sys.exit("bench_triangulation.py: nvidia-smi found no GPU; this measurement needs an H100")
    name, power = [s.strip() for s in q.stdout.strip().split("\n")[0].split(",")]
    return name, power


def whole_call(lin, mode):
    """(seconds, status) of one rba_triangulate_landmarks call on every landmark, CUDA events around it"""
    import ctypes as C
    from rootba_b200 import _lib
    o = _lib.TriangulateOpts()
    _lib.lib().rba_default_triangulate_opts(C.byref(o))
    o.mode = _lib.TRIANGULATE_MODES[mode]
    status = np.zeros(lin.nl, np.uint8)
    lin.timer_start()
    _lib.check(_lib.lib().rba_triangulate_landmarks(lin.h, C.byref(o), lin.nl, None, status.ctypes.data, None, None))
    return lin.timer_stop(), status


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--model-sample", type=int, default=300)
    ap.add_argument("--lm-iterations", type=int, default=30)
    ap.add_argument("--seed", type=int, default=38401)
    args = ap.parse_args()
    name, power = card()
    import rootba_b200 as rb
    import triangulation_model as tm
    from rootba_b200.synthetic import BalArrays, synth_bal, synth_config
    prob = synth_config("ladybug-1723", seed=args.seed)
    out = {"card": name, "power_limit": power, "num_landmarks": prob.nl, "num_observations": prob.nobs}
    for dtype, sfx in ((np.float32, "f32"), (np.float64, "f64")):
        warm = rb.LinearizorQR.create(rb.BalProblem.from_arrays(prob, dtype), rb.SolverOptions())
        warm.triangulate()
        warm.close()
        for mode in ("linear", "refine", "linear+refine"):
            ms = []
            for _ in range(args.rounds):
                lin = rb.LinearizorQR.create(rb.BalProblem.from_arrays(prob, dtype), rb.SolverOptions())
                sec, status = whole_call(lin, mode)
                ms.append(1e3 * sec)
                lin.close()
            out[f"{sfx}_{mode}_ms_min_median_max"] = [round(min(ms), 3), round(float(np.median(ms)), 3), round(max(ms), 3)]
            out[f"{sfx}_{mode}_written"] = int(np.count_nonzero(status & tm.WRITTEN))
    longp = synth_bal(400, 64, 2.0, seed=args.seed, track_lengths=[350] * 64, lm_spread=0.5, perturb_lm=0.2)
    for dtype, sfx in ((np.float32, "f32"), (np.float64, "f64")):
        ms = []
        for _ in range(args.rounds):
            lin = rb.LinearizorQR.create(rb.BalProblem.from_arrays(longp, dtype), rb.SolverOptions())
            ms.append(1e3 * whole_call(lin, "linear+refine")[0])
            lin.close()
        out[f"long_track_350_{sfx}_ms_min_median_max"] = [round(min(ms), 3), round(float(np.median(ms)), 3), round(max(ms), 3)]
    k = min(args.model_sample, prob.nl)
    o = int(prob.lm_off[k])
    trs = tm.tracks(BalArrays(prob.cams, prob.lms[:k], prob.lm_off[: k + 1], prob.obs_cam[:o], prob.obs_xy[:o]))
    for mode, m in (("linear", tm.LINEAR), ("refine", tm.REFINE), ("linear+refine", tm.LINEAR | tm.REFINE)):
        t0 = time.perf_counter()
        for l, tr in enumerate(trs):
            tr.triangulate(prob.lms[l], m)
        out[f"model_{mode}_s_all"] = round((time.perf_counter() - t0) / len(trs) * prob.nl, 1)
    opts = rb.SolverOptions(max_num_iterations=args.lm_iterations)
    scrambled = BalArrays(prob.cams, prob.lms + np.random.default_rng(1).normal(0, 5.0, prob.lms.shape), prob.lm_off,
                          prob.obs_cam, prob.obs_xy)
    for arm, arrays, tri in (("stored", prob, False), ("scrambled", scrambled, False), ("scrambled_triangulated", scrambled, True)):
        lin = rb.LinearizorQR.create(rb.BalProblem.from_arrays(arrays, np.float64), opts)
        if tri:
            lin.triangulate()
        log, _, _ = lin.lm_run(args.lm_iterations, opts)
        out[f"lm_{arm}_iterations"] = len(log)
        out[f"lm_{arm}_cost"] = lin.compute_error()["all"]["error"]
        lin.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
