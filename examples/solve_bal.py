#!/usr/bin/env python
"""Solve a BAL (or Bundler) problem with the square-root solver on one H100 and write the reference's ba_log.json.

    python examples/solve_bal.py problem-49-7776-pre.txt [--float] [--max-num-iterations 20] [--operator-form DENSE|IMPLICIT]

Mirrors what `bal_qr --input ...` of the reference does (src/app/bal_qr.cpp): load + normalise (bal_problem.cpp:773-852),
optimize_lm_ours with the QR linearizor (solver/bal_bundle_adjustment.cpp:249-544), log (bal/ba_log.hpp)."""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rootba_b200 as rb  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("input")
    ap.add_argument("--float", action="store_true", help="float32 instead of float64 (--no-use-double of the reference)")
    ap.add_argument("--max-num-iterations", type=int, default=20)
    ap.add_argument("--preconditioner-type", default="SCHUR_JACOBI", choices=["JACOBI", "SCHUR_JACOBI"])
    ap.add_argument("--operator-form", default="DENSE", choices=["DENSE", "IMPLICIT"])
    ap.add_argument("--init-depth-threshold", type=float, default=0.0)
    ap.add_argument("--log-path", default="ba_log.json")
    args = ap.parse_args()

    t0 = time.perf_counter()
    dtype = np.float32 if args.float else np.float64
    problem = rb.BalProblem.load_bal(args.input, dtype, normalize=True, init_depth_threshold=args.init_depth_threshold)
    t_load = time.perf_counter() - t0
    print(f"Loaded {problem.num_cameras()} cams, {problem.num_landmarks()} lms, {problem.num_observations()} obs in {t_load:.2f}s")
    options = rb.SolverOptions(max_num_iterations=args.max_num_iterations, preconditioner_type=args.preconditioner_type,
                               operator_form=args.operator_form, use_double=not args.float)
    summary = rb.bundle_adjust_manual(problem, options, verbose=True)
    print(summary["termination_type"], summary["message"])
    rb.save_ba_log(args.log_path, summary, problem, args.input, {"load": t_load, "optimize": summary["total_time"]})
    print("wrote", args.log_path)


if __name__ == "__main__":
    main()
