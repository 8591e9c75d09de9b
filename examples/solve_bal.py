#!/usr/bin/env python
"""Solve a BAL (or Bundler) problem with the square-root solver on one H100 and write the reference's ba_log.json.

    python examples/solve_bal.py problem-49-7776-pre.txt [--float] [--max-num-iterations 20] [--operator-form DENSE|IMPLICIT]
        [--fix-intrinsics] [--fix-cameras I,J,...] [--camera-prior FILE.npz] [--camera-pair-prior FILE.npz]
        [--landmark-prior FILE.npz] [--shared-intrinsics | --intrinsics-groups FILE.npy] [--camera-rigs FILE.npz] [--rig-extrinsics OUT.npy] [--covariance OUT.npz]
        [--relative-covariance PAIRS.npy] [--observation-info FILE.npy] [--observation-loss KIND:SCALE | FILE.npz]
        [--residuals OUT.npz] [--camera-prior-loss KIND:SCALE | FILE.npz] [--pair-prior-loss KIND:SCALE | FILE.npz]
        [--landmark-prior-loss KIND:SCALE | FILE.npz] [--prior-residuals OUT.npz]
        [--triangulate linear|refine|linear+refine [--triangulation OUT.npz]]
        [--resect linear|refine|linear+refine [--resect-intrinsics] [--resection OUT.npz]]

Mirrors what `bal_qr --input ...` of the reference does (src/app/bal_qr.cpp): load + normalise (bal_problem.cpp:773-852),
optimize_lm_ours with the QR linearizor (solver/bal_bundle_adjustment.cpp:249-544), log (bal/ba_log.hpp)."""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rootba_b200 as rb  # noqa: E402
from rootba_b200 import _lib  # noqa: E402


def read_loss(ap, flag, value):
    """(kind, scale) of a KIND:SCALE or FILE.npz (arrays `kind`, `scale`) loss argument"""
    if value.endswith(".npz"):
        with np.load(value) as f:
            if "kind" not in f or "scale" not in f:
                ap.error(f"{flag}: {value} must hold the arrays `kind` and `scale`")
            return f["kind"], f["scale"]
    kind, sep, scale = value.partition(":")
    if not sep:
        ap.error(f"{flag}: expected KIND:SCALE (e.g. CAUCHY:2) or FILE.npz")
    try:
        return kind, float(scale)
    except ValueError:
        ap.error(f"{flag}: the scale of {value!r} is not a number")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("input")
    ap.add_argument("--float", action="store_true", help="float32 instead of float64 (--no-use-double of the reference)")
    ap.add_argument("--max-num-iterations", type=int, default=20)
    ap.add_argument("--preconditioner-type", default="SCHUR_JACOBI", choices=["JACOBI", "SCHUR_JACOBI", "CLUSTER_JACOBI"],
                    help="CLUSTER_JACOBI: the block diagonal of the reduced camera matrix over clusters of co-visible cameras")
    ap.add_argument("--cluster-size", type=int, default=None,
                    help="with CLUSTER_JACOBI: cluster the cameras with at most K per cluster (1..16; default: the library's)")
    ap.add_argument("--clusters", default=None, help="with CLUSTER_JACOBI: one int32 cluster id per camera (.npy)")
    ap.add_argument("--operator-form", default="DENSE", choices=["DENSE", "IMPLICIT"])
    ap.add_argument("--linear-solver-type", default="ITERATIVE_SCHUR", choices=["ITERATIVE_SCHUR", "DENSE_SCHUR"],
                    help="the camera increment by truncated PCG, or exactly by a dense Cholesky factorisation of the reduced "
                         "camera matrix (needs (9 cameras)^2 x 8 bytes of device memory)")
    ap.add_argument("--init-depth-threshold", type=float, default=0.0)
    ap.add_argument("--log-path", default="ba_log.json")
    ap.add_argument("--fix-intrinsics", action="store_true", help="hold f, k1, k2 of every camera constant")
    ap.add_argument("--fix-cameras", default="", metavar="I,J,...",
                    help="hold every parameter of the listed cameras constant; indices refer to the loaded problem "
                         "(a Bundler file's cameras with focal length 0 are dropped by the loader first)")
    ap.add_argument("--camera-prior", default=None, metavar="FILE.npz",
                    help="Gaussian camera priors: arrays `mean` [nc, 10] (qx,qy,qz,qw, camera centre, f, k1, k2) and `sqrt_info` "
                         "[nc, 9, 9] in the coordinates of the loaded (normalised) problem (DESIGN.md section 14)")
    ap.add_argument("--camera-pair-prior", default=None, metavar="FILE.npz",
                    help="relative pose priors between pairs of cameras: arrays `pairs` [m, 2] (i, j), `mean` [m, 7] (qx,qy,qz,qw, t "
                         "of T_i T_j^-1) and `sqrt_info` [m, 6, 6] in the coordinates of the loaded (normalised) problem "
                         "(DESIGN.md section 15)")
    ap.add_argument("--landmark-prior", default=None, metavar="FILE.npz",
                    help="Gaussian priors on landmark positions (e.g. ground control points): arrays `idx` [m], `mean` [m, 3] and "
                         "`sqrt_info` [m, 3, 3] in the coordinates of the loaded (normalised) problem (DESIGN.md section 17)")
    groups = ap.add_mutually_exclusive_group()
    groups.add_argument("--shared-intrinsics", action="store_true",
                        help="every camera shares one f, k1, k2, those of camera 0 at the start (DESIGN.md section 18)")
    groups.add_argument("--intrinsics-groups", default=None, metavar="FILE.npy",
                        help="an int array [nc] of intrinsics group ids, -1 = the camera keeps its own; the cameras of a group "
                             "share one f, k1, k2, those of its lowest-index camera at the start (DESIGN.md section 18)")
    ap.add_argument("--camera-rigs", default=None, metavar="FILE.npz",
                    help="rigid camera rigs: arrays `rig` [nc] int (rig id, -1 = free camera) and `cam_from_rig` [nc, 7] "
                         "(qx,qy,qz,qw, tx,ty,tz per camera, in the coordinates of the loaded (normalised) problem); every member "
                         "is kept at its extrinsics relative to its rig's lowest-index camera (DESIGN.md section 23); an "
                         "optional array `sensor` [nc] int (-1 = held extrinsics) names the physical camera of each capture, "
                         "whose extrinsics are estimated and shared by its captures (DESIGN.md section 24)")
    ap.add_argument("--rig-extrinsics", default=None, metavar="OUT.npy",
                    help="with --camera-rigs: after the solve, write every camera's refined cam_from_rig [nc, 7] (held ones as "
                         "given, estimated sensors' from the final state, free cameras the identity)")
    ap.add_argument("--covariance", default=None, metavar="OUT.npz",
                    help="after the solve, write the marginal covariances `cam` [nc, 9, 9] (tx,ty,tz, rx,ry,rz, f,k1,k2) and `lm` "
                         "[nl, 3, 3] at the final state (DESIGN.md section 16); the gauge must be fixed by priors or held "
                         "parameters")
    ap.add_argument("--relative-covariance", default=None, metavar="PAIRS.npy",
                    help="with --covariance: an int array [m, 2] of camera pairs (i, j), i != j; adds to the --covariance file "
                         "`relative` [m, 6, 6], the covariance of the relative pose T_i T_j^-1 as the residual (e_t, e_r) of "
                         "--camera-pair-prior at the final state, and `relative_pairs` (DESIGN.md section 20)")
    ap.add_argument("--observation-info", default=None, metavar="FILE.npy",
                    help="square-root information of the keypoints: an array [Nobs] (1 / sigma per observation) or [Nobs, 2, 2] "
                         "(a square root W of the inverse 2x2 keypoint covariance) in the order of the loaded problem's "
                         "observations, in the units of the loaded (normalised) image coordinates; zero switches an observation "
                         "off (DESIGN.md section 19)")
    ap.add_argument("--observation-loss", default=None, metavar="KIND:SCALE | FILE.npz",
                    help="a robust loss per observation (DESIGN.md section 21): KIND:SCALE for every observation (KIND one of "
                         "NONE, HUBER, CAUCHY, SOFT_L1, TUKEY; SCALE the inlier threshold in units of sigma), or a .npz with the "
                         "arrays `kind` [Nobs] (names or RBA_LOSS_* ints) and `scale` [Nobs] in the order of the loaded problem's "
                         "observations")
    ap.add_argument("--residuals", default=None, metavar="OUT.npz",
                    help="after the solve, write per observation `residual` [Nobs, 2] (W r), `robust_weight` [Nobs] and `flags` "
                         "[Nobs] (bit 0 = projection valid, bit 1 = in use) at the final state (DESIGN.md section 19)")
    for flag, what in (("--camera-prior-loss", "camera of --camera-prior"), ("--pair-prior-loss", "pair of --camera-pair-prior"),
                       ("--landmark-prior-loss", "prior of --landmark-prior")):
        ap.add_argument(flag, default=None, metavar="KIND:SCALE | FILE.npz",
                        help=f"a robust loss per {what} (DESIGN.md section 22): KIND:SCALE for every one (KIND as for "
                             "--observation-loss; SCALE the threshold on |L e|, e.g. 2.80 for a 95 %% gate on 3 degrees of freedom, "
                             "3.55 on 6), or a .npz with the arrays `kind` and `scale`, one entry each in the prior's order")
    ap.add_argument("--prior-residuals", default=None, metavar="OUT.npz",
                    help="after the solve, write per prior kind given `<kind>_residual` [num, 9 | 6 | 3] (L e) and "
                         "`<kind>_robust_weight` [num] at the final state, kind camera, pair or landmark (DESIGN.md section 22)")
    ap.add_argument("--triangulate", default=None, choices=["linear", "refine", "linear+refine"],
                    help="before the solve, re-initialise every landmark from the loaded cameras (DESIGN.md section 25)")
    ap.add_argument("--triangulation", default=None, metavar="OUT.npz",
                    help="with --triangulate, write per landmark `status` (RBA_TRI_* bits), `angle` [rad] and `cost`")
    ap.add_argument("--resect", default=None, choices=["linear", "refine", "linear+refine"],
                    help="before the solve (and before --triangulate), re-initialise every camera (rig) from the loaded "
                         "landmarks (DESIGN.md section 26)")
    ap.add_argument("--resect-intrinsics", action="store_true",
                    help="with --resect: also refine the free f, k1, k2 of cameras outside rigs and intrinsics groups")
    ap.add_argument("--resection", default=None, metavar="OUT.npz",
                    help="with --resect, write per camera `status` (RBA_RES_* bits), `points` and `cost`")
    args = ap.parse_args()
    if args.resection and not args.resect:
        ap.error("--resection requires --resect")
    if args.resect_intrinsics and not args.resect:
        ap.error("--resect-intrinsics requires --resect")
    if args.triangulation and not args.triangulate:
        ap.error("--triangulation requires --triangulate")
    if args.relative_covariance and not args.covariance:
        ap.error("--relative-covariance requires --covariance")
    rel_pairs = None
    if args.relative_covariance:
        rel_pairs = np.load(args.relative_covariance)
        if rel_pairs.ndim != 2 or rel_pairs.shape[1] != 2 or not np.issubdtype(rel_pairs.dtype, np.integer):
            ap.error(f"--relative-covariance: {args.relative_covariance} must hold an int array [m, 2], got {rel_pairs.dtype} "
                     f"{rel_pairs.shape}")
    try:
        fix_cameras = [int(v) for v in args.fix_cameras.split(",")] if args.fix_cameras else []
    except ValueError:
        ap.error(f"--fix-cameras expects a comma-separated list of camera indices, got {args.fix_cameras!r}")

    t0 = time.perf_counter()
    dtype = np.float32 if args.float else np.float64
    problem = rb.BalProblem.load_bal(args.input, dtype, normalize=True, init_depth_threshold=args.init_depth_threshold)
    t_load = time.perf_counter() - t0
    print(f"Loaded {problem.num_cameras()} cams, {problem.num_landmarks()} lms, {problem.num_observations()} obs in {t_load:.2f}s")
    if args.fix_intrinsics or fix_cameras:
        bad = [c for c in fix_cameras if not 0 <= c < problem.num_cameras()]
        if bad:
            ap.error(f"--fix-cameras: {bad} out of range (the loaded problem has {problem.num_cameras()} cameras)")
        flags = np.full(problem.num_cameras(), rb.FIX_INTRINSICS if args.fix_intrinsics else 0, np.uint8)
        flags[fix_cameras] = rb.FIX_ALL
        problem.camera_fixed = flags
    if args.camera_prior:
        with np.load(args.camera_prior) as f:
            if "mean" not in f or "sqrt_info" not in f:
                ap.error(f"--camera-prior: {args.camera_prior} must hold the arrays `mean` and `sqrt_info`")
            try:
                problem.camera_prior = (f["mean"], f["sqrt_info"])
            except ValueError as e:
                ap.error(f"--camera-prior: {e}")
    if args.camera_pair_prior:
        with np.load(args.camera_pair_prior) as f:
            if "pairs" not in f or "mean" not in f or "sqrt_info" not in f:
                ap.error(f"--camera-pair-prior: {args.camera_pair_prior} must hold the arrays `pairs`, `mean` and `sqrt_info`")
            try:
                problem.camera_pair_prior = (f["pairs"], f["mean"], f["sqrt_info"])
            except ValueError as e:
                ap.error(f"--camera-pair-prior: {e}")
    if args.landmark_prior:
        with np.load(args.landmark_prior) as f:
            if "idx" not in f or "mean" not in f or "sqrt_info" not in f:
                ap.error(f"--landmark-prior: {args.landmark_prior} must hold the arrays `idx`, `mean` and `sqrt_info`")
            try:
                problem.landmark_prior = (f["idx"], f["mean"], f["sqrt_info"])
            except ValueError as e:
                ap.error(f"--landmark-prior: {e}")
    if args.shared_intrinsics:
        problem.intrinsics_group = np.zeros(problem.num_cameras(), np.int32)
    elif args.intrinsics_groups:
        try:
            problem.intrinsics_group = np.load(args.intrinsics_groups)
        except ValueError as e:
            ap.error(f"--intrinsics-groups: {e}")
    if args.camera_rigs:
        with np.load(args.camera_rigs) as f:
            try:
                problem.camera_rig = (f["rig"], f["cam_from_rig"])
                if "sensor" in f.files:
                    problem.rig_sensor = f["sensor"]
            except ValueError as e:
                ap.error(f"--camera-rigs: {e}")
    if args.observation_info:
        info = np.load(args.observation_info)
        nobs = problem.num_observations()
        if info.shape not in ((nobs,), (nobs, 2, 2)):
            ap.error(f"--observation-info: {args.observation_info} has shape {info.shape}; the loaded problem has {nobs} observations"
                     + (f" after --init-depth-threshold {args.init_depth_threshold} removed some" if args.init_depth_threshold > 0 else "")
                     + f", so the array must have shape ({nobs},) or ({nobs}, 2, 2)")
        try:
            problem.observation_sqrt_info = info
        except ValueError as e:
            ap.error(f"--observation-info: {e}")
    for flag, value, attr in (("--observation-loss", args.observation_loss, "observation_loss"),
                              ("--camera-prior-loss", args.camera_prior_loss, "camera_prior_loss"),
                              ("--pair-prior-loss", args.pair_prior_loss, "camera_pair_prior_loss"),
                              ("--landmark-prior-loss", args.landmark_prior_loss, "landmark_prior_loss")):
        if value:
            loss = read_loss(ap, flag, value)
            try:
                setattr(problem, attr, loss)
            except ValueError as e:
                ap.error(f"{flag}: {e}")
    options = rb.SolverOptions(max_num_iterations=args.max_num_iterations, preconditioner_type=args.preconditioner_type,
                               operator_form=args.operator_form, linear_solver_type=args.linear_solver_type,
                               use_double=not args.float)
    if args.resect:
        lin_res = rb.LinearizorQR.create(problem, options)  # the new cameras go back into `problem`
        status, points, cost = lin_res.resect(mode=args.resect, intrinsics=args.resect_intrinsics)
        lin_res.close()
        written = int(np.count_nonzero(status & _lib.RES_WRITTEN))
        print(f"resected ({args.resect}{', intrinsics' if args.resect_intrinsics else ''}): {written} of {len(status)} "
              f"cameras written, {int(np.count_nonzero(status & _lib.RES_FEW_POINTS))} with fewer than 3 usable points")
        if args.resection:
            np.savez(args.resection, status=status, points=points, cost=cost)
            print("wrote", args.resection)
    if args.triangulate:
        lin_tri = rb.LinearizorQR.create(problem, options)  # the new positions go back into `problem`
        status, angle, cost = lin_tri.triangulate(mode=args.triangulate)
        lin_tri.close()
        written = int(np.count_nonzero(status & _lib.TRI_WRITTEN))
        print(f"triangulated ({args.triangulate}): {written} of {len(status)} landmarks written, "
              f"{int(np.count_nonzero(status & _lib.TRI_FEW_RAYS))} with fewer than 2 usable rays")
        if args.triangulation:
            np.savez(args.triangulation, status=status, angle=angle, cost=cost)
            print("wrote", args.triangulation)
    if args.rig_extrinsics and problem.camera_rig is None:
        ap.error("--rig-extrinsics needs --camera-rigs")
    if (args.cluster_size is not None or args.clusters) and args.preconditioner_type != "CLUSTER_JACOBI":
        ap.error("--cluster-size and --clusters need --preconditioner-type CLUSTER_JACOBI")
    if args.cluster_size is not None and args.clusters:
        ap.error("give --cluster-size or --clusters, not both")
    clusters = None
    if args.cluster_size is not None:
        try:
            clusters = rb.cluster_cameras(problem, args.cluster_size)
        except rb.RbaError as e:
            ap.error(f"--cluster-size: {e}")
    elif args.clusters:
        clusters = np.load(args.clusters)
    lin_ba = rb.LinearizorQR.create(problem, options) if args.rig_extrinsics or clusters is not None else None
    if clusters is not None:
        try:
            lin_ba.set_camera_clusters(clusters)
        except (ValueError, rb.RbaError) as e:
            ap.error(f"--clusters: {e}")
    summary = rb.bundle_adjust_manual(problem, options, linearizor=lin_ba, verbose=True)
    if lin_ba is not None and args.rig_extrinsics:
        extrinsics = lin_ba.rig_extrinsics()
        np.save(args.rig_extrinsics, extrinsics)
    if lin_ba is not None:
        lin_ba.close()
        print("wrote", args.rig_extrinsics)
        if problem.rig_sensor is not None:  # a later handle ties the sensors' captures to the refined extrinsics
            sensor = problem.rig_sensor
            problem.camera_rig = (problem.camera_rig[0], extrinsics)
            problem.rig_sensor = sensor
    print(summary["termination_type"], summary["message"])
    rb.save_ba_log(args.log_path, summary, problem, args.input, {"load": t_load, "optimize": summary["total_time"]})
    print("wrote", args.log_path)
    if args.covariance or args.residuals or args.prior_residuals:
        lin = rb.LinearizorQR.create(problem, options)  # at the final state, with the same priors, information and held parameters
        try:
            if args.covariance:  # one factorisation for the marginals and the relative poses
                blocks = lin.covariance_blocks(relative=rel_pairs, marginals=True)
            if args.residuals:
                res, hw, flags = lin.observation_residuals()
            prior_res = {}
            if args.prior_residuals:
                for kind, prior in (("camera", problem.camera_prior), ("pair", problem.camera_pair_prior),
                                    ("landmark", problem.landmark_prior)):
                    if prior is not None:
                        prior_res[kind + "_residual"], prior_res[kind + "_robust_weight"] = lin.prior_residuals(kind)
        finally:
            lin.close()
        if args.covariance:
            extra = {} if rel_pairs is None else dict(relative=blocks["relative"], relative_pairs=rel_pairs)
            np.savez(args.covariance, cam=blocks["cam"], lm=blocks["lm"], **extra)
            print("wrote", args.covariance)
        if args.residuals:
            np.savez(args.residuals, residual=res, robust_weight=hw, flags=flags)
            print("wrote", args.residuals)
        if args.prior_residuals:
            np.savez(args.prior_residuals, **prior_res)
            print("wrote", args.prior_residuals)


if __name__ == "__main__":
    main()
