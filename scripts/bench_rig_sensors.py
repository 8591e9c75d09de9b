#!/usr/bin/env python
"""Rig bundle adjustment with estimated extrinsics (rba_set_rig_sensors, DESIGN.md section 24) on a synthetic rig capture.

    python scripts/bench_rig_sensors.py [--sensors 6] [--placements 290] [--landmarks 60000] [--lm-iterations 15] [--seed 5]

The capture (rootba_b200.synthetic.synth_rig_capture: a ring of `--sensors` outward-looking cameras placed `--placements`
times along a path, ~1740 cameras by default, near the Ladybug-1723 stand-in's size) has observations with 0.5 px noise,
landmarks moved by 1 cm, and the scale and gauge fixed by centre priors (sigma 1 cm) on sensor 0's cameras at their true
centres.  Three arms, in f32 and in f64, each a fresh handle in this one process:
  held_true       rigs held at the true extrinsics (rba_set_camera_rigs alone);
  held_perturbed  rigs held at extrinsics perturbed by N(0, 2 deg) and N(0, 3 cm) per sensor but sensor 0 (the only option
                  without sensors);
  estimated       the perturbed extrinsics as the start, every sensor but sensor 0 estimated (rba_set_rig_sensors).
Per arm: the final cost after rba_lm_run(--lm-iterations), the largest extrinsic error (rotation in degrees, translation in
units) of rba_get_rig_extrinsics against the truth, ms per LM iteration (device seconds of the run), the PCG iterations of
the run, the kernel launches of one LM step, and the microseconds per PCG iteration at exactly 50 iterations (min = max
linear solver iterations, the median of 5 solves).  Prints one JSON line with the card's name and power limit read in the
same call.
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

FIXED_PCG = 50


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        sys.exit("bench_rig_sensors.py: nvidia-smi found no GPU; this measurement needs an H100")
    name, power = [s.strip() for s in q.stdout.strip().split("\n")[0].split(",")]
    return name, power


def ext_error(got, true, rigged):
    from scipy.spatial.transform import Rotation
    g, t = np.asarray(got, np.float64)[rigged], np.asarray(true, np.float64)[rigged]
    rot = (Rotation.from_quat(g[:, :4]) * Rotation.from_quat(t[:, :4]).inv()).magnitude()
    return float(np.rad2deg(rot.max())), float(np.linalg.norm(g[:, 4:] - t[:, 4:], axis=1).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sensors", type=int, default=6)
    ap.add_argument("--placements", type=int, default=290)
    ap.add_argument("--landmarks", type=int, default=60000)
    ap.add_argument("--lm-iterations", type=int, default=15)
    ap.add_argument("--seed", type=int, default=5)
    args = ap.parse_args()
    name, power = card()
    import rootba_b200 as rb
    from scipy.spatial.transform import Rotation
    from rootba_b200.synthetic import quat_to_rot, synth_rig_capture
    cap = synth_rig_capture(args.sensors, args.placements, args.landmarks, seed=args.seed, max_depth=6.0)
    rng = np.random.default_rng(args.seed)
    prob = cap.prob
    prob.obs_xy = prob.obs_xy + rng.normal(0, 0.5, prob.obs_xy.shape)
    prob.lms = prob.lms + rng.normal(0, 0.01, prob.lms.shape)
    nc = prob.nc
    # the perturbed extrinsics: every sensor but sensor 0 turned and shifted
    E = cap.cam_from_rig.copy()
    for k in range(1, args.sensors):
        m = cap.sensor == k
        E[m, :4] = (Rotation.from_rotvec(np.deg2rad(rng.normal(0, 2.0, 3))) * Rotation.from_quat(E[m][0, :4])).as_quat()
        E[m, 4:] = E[m][0, 4:] + rng.normal(0, 0.03, 3)
    # centre priors on sensor 0's cameras at their true centres
    mean = np.array(prob.cams, np.float64)
    R = quat_to_rot(mean[:, :4])
    mean[:, 4:7] = -np.einsum("nji,nj->ni", R, mean[:, 4:7])
    L = np.zeros((nc, 9, 9))
    held = np.flatnonzero(cap.sensor == 0)
    L[held, 0, 0] = L[held, 1, 1] = L[held, 2, 2] = 100.0
    sensor = np.where(cap.sensor == 0, -1, cap.sensor).astype(np.int32)
    arms = {"held_true": (cap.cam_from_rig, None), "held_perturbed": (E, None), "estimated": (E, sensor)}
    out = {"card": name, "power_limit": power, "workload": {**prob.stats(), "sensors": args.sensors, "placements": args.placements,
                                                            "lm_iterations": args.lm_iterations},
           "fixed_pcg_iterations": FIXED_PCG, "arms": {}}
    for dtype, sfx in ((np.float32, "f32"), (np.float64, "f64")):
        for arm, (ext, sen) in arms.items():
            def handle(**opts):
                bp = rb.BalProblem.from_arrays(prob, dtype)
                bp.camera_prior = (mean, L)
                bp.camera_rig = (cap.rig, ext)
                if sen is not None:
                    bp.rig_sensor = sen
                return rb.LinearizorQR.create(bp, rb.SolverOptions(**opts))
            lin = handle()
            lin._backup()
            lin.linearize(); lin.solve(1e-4); lin.apply(None)  # warm-up of every kernel of a step
            lin._restore()
            before = lin.timings()["kernel_launches"]
            lin.linearize(); lin.solve(1e-4); lin.apply(None)
            launches = lin.timings()["kernel_launches"] - before
            lin._restore()
            its, _, _ = lin.lm_run(args.lm_iterations)
            cost = lin.compute_error()["all"]["error"]
            rot, trans = ext_error(lin.rig_extrinsics(), cap.cam_from_rig, cap.rig >= 0)
            lin.close()
            fixed = handle(min_linear_solver_iterations=FIXED_PCG, max_linear_solver_iterations=FIXED_PCG)
            fixed.linearize()
            fixed.solve(1e-4)  # warm-up
            us = []
            for _ in range(5):
                fixed.solve(1e-4)
                us.append(1e6 * fixed.timings()["solve_reduced_system_time"] / FIXED_PCG)
            fixed.close()
            r = {"final_cost": cost, "extrinsic_error_deg": rot, "extrinsic_error_translation": trans,
                 "ms_per_lm_iteration": 1e3 * sum(i["device_seconds"] for i in its) / max(len(its), 1),
                 "lm_iterations": len(its), "pcg_iterations": int(sum(i["cg_iterations"] for i in its)),
                 "launches_per_lm_step": int(launches), "pcg_us_per_iteration_fixed": float(np.median(us))}
            out["arms"][f"{arm}/{sfx}"] = r
            print(f"{arm}/{sfx}: {r}", file=sys.stderr, flush=True)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
