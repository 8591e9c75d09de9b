/*
 * rootba_b200.h -- C ABI of the H100-native square-root bundle-adjustment inner loop.
 *
 * This is the drop-in boundary for the ONE hot path of NikolausDemmel/rootba that this
 * repository accelerates: the QR (square-root) Levenberg-Marquardt inner loop.  The
 * reference has no C ABI; its seam is the C++ strategy interface
 *     rootba::Linearizor<Scalar>          (src/rootba/solver/linearizor.hpp:47-83)
 * implemented for the QR solver by
 *     rootba::LinearizorQR<Scalar>        (src/rootba/solver/linearizor_qr.cpp:52-291)
 * on top of
 *     rootba::LinearizationQR<Scalar, 9>  (src/rootba/qr/linearization_qr.hpp:54-841).
 * Every entry point below names the reference member function it replaces.  A reference
 * maintainer binds them from a `LinearizorQR_B200 : LinearizorBase<Scalar>` shim -- see
 * INTEGRATION.md.
 *
 * Conventions
 *  - plain pointers and sizes only; all pointers are HOST pointers unless the name says _dev;
 *  - Scalar-typed arrays are `float` for handles created with rba_create_f32 and `double`
 *    for rba_create_f64 (the reference instantiates float and double, linearizor.cpp:67-73);
 *  - camera state = 10 scalars (qx,qy,qz,qw, tx,ty,tz, f,k1,k2)  (bal_problem.hpp:72,84-89),
 *    landmark = 3 scalars, observation = 2 scalars (already in the loaded convention);
 *  - every function returns RBA_OK (0), RBA_NUMERICAL_FAILURE (1: the reference returns an
 *    empty vector / NaN, linearization_qr.hpp:702-711, linearizor_qr.cpp:275-277) or a negative
 *    fatal code (the reference CHECK/LOG(FATAL)-aborts; we return instead);
 *  - there is NO CPU fallback: without a CUDA device rba_create_* fails with RBA_ERR_NO_DEVICE.
 */
#ifndef ROOTBA_B200_H_
#define ROOTBA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RBA_OK 0
#define RBA_NUMERICAL_FAILURE 1
#define RBA_ERR_INVALID_ARGUMENT (-1)
#define RBA_ERR_NO_DEVICE (-2)
#define RBA_ERR_CUDA (-3)
#define RBA_ERR_UNSUPPORTED (-4)
#define RBA_ERR_NCCL (-5)
#define RBA_ERR_STATE (-6)

#define RBA_ABI_VERSION 1

typedef struct rba_handle rba_handle; /* opaque; one per (problem, rank) */

/* BalProblem topology + observations (bal/bal_problem.hpp:61-234) in CSR-by-landmark form.
 * Per landmark the observations are ordered by ascending camera index -- the std::map order
 * the reference iterates in (bal_problem.hpp:137, landmark_block_dynamic.hpp:49-54). */
typedef struct {
  int32_t num_cameras;
  int32_t num_landmarks;
  int64_t num_observations;
  const int64_t* lm_obs_offset; /* [num_landmarks + 1] */
  const int32_t* obs_cam_idx;   /* [num_observations] */
  const void* obs_xy;           /* [2 * num_observations] Scalar */
} rba_problem_view;

/* Subset of SolverOptions (bal/solver_options.hpp:46-284) read by the QR path, plus placement. */
typedef struct {
  int32_t use_householder_marginalization; /* :258 ; 1 = Householder (ipp:717-743), 0 = Givens (ipp:700-715); both run on the device */
  int32_t use_valid_projections_only;      /* SolverOptions::use_projection_validity_check() */
  int32_t robust_norm;                     /* 0 NONE, 1 HUBER  (bal_residual_options.hpp:52) */
  double huber_parameter;                  /* bal_residual_options.hpp:58 */
  double jacobi_scaling_epsilon;           /* :208 ; 0 -> Sophus epsilonSqrt (linearizor_base.cpp:72-79) */
  int32_t preconditioner_type;             /* 0 JACOBI, 1 SCHUR_JACOBI (:217), 2 CLUSTER_JACOBI (:73-75): the block diagonal
                                              of the reduced camera matrix over clusters of co-visible cameras, each
                                              (9k) x (9k) block with its cross blocks factorised in float64 once per solve
                                              (DESIGN.md section 28; rba_cluster_cameras, rba_set_camera_clusters).  Other
                                              values -> RBA_ERR_INVALID_ARGUMENT; CLUSTER_JACOBI with solver_type = 2 or
                                              linear_solver_type = DENSE_SCHUR (no PCG) -> RBA_ERR_INVALID_ARGUMENT, with
                                              nranks > 1 -> RBA_ERR_UNSUPPORTED. */
  int32_t min_linear_solver_iterations;    /* :180 */
  int32_t max_linear_solver_iterations;    /* :184 */
  double eta;                              /* :189 */
  int32_t residual_reset_period;           /* ConjugateGradientsSolver::Options (conjugate_gradient.hpp:87) = 10 */
  /* placement */
  int32_t device;                          /* CUDA device ordinal, -1 = current */
  int32_t rank;                            /* landmark shard owned by this handle */
  int32_t nranks;                          /* 1 = single GPU */
  int32_t pcg_check_period;                /* CG iterations the host enqueues ahead of the progress the device publishes (NCCL exchange: poll period) (0 -> 4) */
  int32_t use_cuda_graphs;                 /* reserved, ignored: the kernels of a PCG iteration are chained with programmatic
                                              dependent launch + a device-side convergence flag instead of graph capture */
  int32_t operator_form;                   /* PCG operator (Q2^T Jp)^T (Q2^T Jp) x: 0 = dense Q2 panels, as the reference
                                              (ipp:400-441; default, the contract kernel); 1 = implicit
                                              Jp^T Jp x - (Q1d^T Jp)^T (Q1d^T Jp) x from the per-observation records
                                              (same result up to rounding, ~n/2.7 x fewer bytes, but the subtraction gives
                                              up the float32 robustness of the square-root form: recommended with f64) */
  int32_t stage2_form;                     /* gradient b and SCHUR_JACOBI blocks of the reduced system: 0 = from the stored Q2 panels
                                              like the reference (ipp:443-466, :520-552: sums of squares, no cancellation;
                                              default), 1 = through the orthogonality identities Jp^T r - Q1d^T (Q1^T r)_d and
                                              Jp^T Jp - Q1d^T Q1d (O(n) per landmark, but they cancel: float64 only).  With
                                              operator_form = 1 no panels exist and form 1 is used. */
  int32_t solver_type;                     /* SolverOptions::solver_type (:63-76): 0 = SQUARE_ROOT (LinearizorQR, default), 1 = SCHUR_COMPLEMENT
                                              (LinearizorSC, solver/linearizor_sc.cpp: landmark eliminated through the normal equations,
                                              PCG on the reduced camera system), 2 = POWER_SCHUR_COMPLEMENT (LinearizorPowerSC,
                                              solver/linearizor_power_sc.cpp: power-series solve, sc/linearization_power_sc.hpp:130-160;
                                              one GPU).  Types 1 and 2 store no Q2 panels; same entry points, same protocol. */
  int32_t power_order;                     /* :270 ; maximum number of terms of the power series (0 -> 20) */
  int32_t linear_solver_type;              /* SolverOptions::linear_solver_type (bal/solver_options.hpp:77-80, 225-230): how rba_solve
                                              gets the camera increment.  0 = ITERATIVE_SCHUR (default): truncated PCG, or the power
                                              series with solver_type = 2.  1 = DENSE_SCHUR: the exact increment -H_ff^-1 b_f of the
                                              same reduced system, by a dense float64 Cholesky factorisation of the Jacobi-scaled,
                                              damped reduced camera matrix on the device, re-linearised in float64 at the current
                                              state for either Scalar (DESIGN.md section 27).  eta, min/max_linear_solver_iterations,
                                              residual_reset_period and pcg_check_period are then ignored; the summary is
                                              SUCCESS with reason 7, or FAILURE with reason 8 (a pivot <= 0 or not finite; the free
                                              entries of the increment are then NaN), with 0 iterations and matvecs.  The dense
                                              (9 nc rounded up to 64)^2 float64 matrix and the per-slot scratch are allocated by
                                              rba_create_* (counted in device_bytes): RBA_ERR_UNSUPPORTED when they do not fit in
                                              the free device memory.  Other values, or DENSE_SCHUR with solver_type = 2 ->
                                              RBA_ERR_INVALID_ARGUMENT; DENSE_SCHUR with nranks > 1 -> RBA_ERR_UNSUPPORTED. */
  int32_t reserved[1];
} rba_solver_opts;

/* ResidualInfo (bal/residual_info.hpp:59-89) */
typedef struct {
  int64_t all_num_obs;
  double all_error;
  double all_residual_sum;
  int64_t valid_num_obs;
  double valid_error;
  double valid_residual_sum;
  int32_t is_numerically_valid;
  int32_t pad_;
} rba_residual_info;

/* ConjugateGradientsSolver::Summary (cg/conjugate_gradient.hpp:97-107) */
typedef struct {
  int32_t termination_type; /* 0 NO_CONVERGENCE, 1 SUCCESS, 2 FAILURE */
  int32_t num_iterations;
  int32_t num_matvecs;
  int32_t reason;           /* detail code for the message (see DESIGN.md); with linear_solver_type = DENSE_SCHUR:
                               7 = the dense Cholesky solve succeeded (SUCCESS), 8 = a pivot of the scaled, damped reduced
                               camera matrix was <= 0 or not finite (FAILURE, the free entries of the increment are NaN) */
} rba_cg_summary;

/* Device times (CUDA events on the solver stream) of the IterationSummary fields
 * (solver/solver_summary.hpp:165-205), in seconds, for the LAST call of each entry point. */
typedef struct {
  double stage1_time;               /* linearize */
  double stage2_time;               /* solve: damping + gradient + precond blocks */
  double compute_preconditioner_time; /* solve: block inversion */
  double solve_reduced_system_time; /* solve: PCG */
  double back_substitution_time;    /* apply */
  double update_cameras_time;       /* apply */
  double residual_evaluation_time;  /* compute_error */
  double matvec_time;               /* inside PCG: sum over all rcs_matvec launches */
  int64_t matvec_launches;
  int64_t kernel_launches;          /* cumulative number of kernels launched by this handle since create */
} rba_stage_timings;

/* Workload statistics (computed at create; per rank) */
typedef struct {
  int64_t num_landmarks_local;
  int64_t num_observations_local;
  int64_t sum_n2;                 /* M2 = sum n_l^2 over local landmarks */
  int32_t max_n;
  int32_t num_tiles;
  int64_t panel_scalars;          /* allocated (padded) Q2 panel size in scalars */
  int64_t panel_scalars_algorithmic; /* 18 * M2 */
  int64_t device_bytes;           /* total device allocation */
  int64_t matvec_algorithmic_bytes;  /* 18*M2*s + 18*Nobs*s + 4*Nobs (SURVEY 8d) */
  int32_t landmark_begin, landmark_end; /* shard [begin, end) in problem order */
  int32_t num_matvec_items;
  int32_t reserved_;
} rba_workload_stats;

/* ---- lifecycle -------------------------------------------------------------------------- */

int32_t rba_abi_version(void);
/* message of the last failure on this thread */
const char* rba_last_error(void);
void rba_default_solver_opts(rba_solver_opts* opts);

/* replaces LinearizorQR ctor (linearizor_qr.cpp:52-72) + LinearizationQR ctor (linearization_qr.hpp:80-111):
 * uploads topology, classifies landmark blocks by track length (the reference's static n=2..8 / dynamic
 * split, qr/landmark_block.cpp:51-80, becomes sub-warp group classes), allocates device storage. */
int32_t rba_create_f32(const rba_problem_view* problem, const rba_solver_opts* opts, rba_handle** out);
int32_t rba_create_f64(const rba_problem_view* problem, const rba_solver_opts* opts, rba_handle** out);
int32_t rba_destroy(rba_handle* h);
int32_t rba_get_workload_stats(const rba_handle* h, rba_workload_stats* out);
/* 4 = float32, 8 = float64 */
int32_t rba_scalar_size(const rba_handle* h);

/* contiguous landmark shards equalising sum n^2 (SURVEY 8e); bounds[nranks + 1]; pure host code */
int32_t rba_partition_landmarks(int32_t num_landmarks, const int64_t* lm_obs_offset, int32_t nranks,
                                int32_t* bounds);

/* Host-only self check of the data model built for (problem, rank, nranks): every observation is assigned to exactly one
 * slot with the right camera, tiles are homogeneous in track length, the matvec row chunks tile every panel exactly once,
 * the camera-major CSRs list every (y) slot exactly once under its camera, shards cover the landmarks.  Needs no GPU.
 * scalar_size selects the float (4) or double (8) class limits.  Returns RBA_OK or RBA_ERR_STATE (see rba_last_error). */
int32_t rba_layout_selftest(const rba_problem_view* problem, int32_t rank, int32_t nranks, int32_t scalar_size);

/* ---- BAL file loader (SURVEY 8f row 1; host only, no GPU) ----------------------------------- */

/* load_normalized_bal_problem (bal/bal_problem.cpp:773-852) = load_bal (:189-282: whitespace-separated
 * "Nc Nl Nobs", Nobs x (cam lm x y), 9 values per camera, 3 per landmark; y of the image and y/z of the camera frame
 * flipped; observations of a landmark in ascending camera order like the reference's std::map, bal_problem.hpp:137;
 * duplicate observation / short or malformed file -> RBA_ERR_INVALID_ARGUMENT where the reference LOG(FATAL)s)
 * + normalize(scale) (:428-469, median-centre + MAD-scale, in double) when `normalize` != 0.
 * A file whose name contains "bundle" is read as a Bundler "bundle.out" v0.3 file instead (load_bundler :284-404, chosen like
 * autodetect_input_type :124-135; cameras with focal length 0 are dropped).
 * The file is parsed by `num_threads` threads (<= 0: all hardware threads) straight into the flat arrays of
 * rba_problem_view; the result is bit-identical to a one-fscanf-per-line loader (from_chars and "%lf" both round
 * correctly).  All values are double, as in the reference (cast to float happens after normalisation, :813-832). */
typedef struct rba_bal_file rba_bal_file;
int32_t rba_bal_load(const char* path, int32_t normalize, double scale, int32_t num_threads, rba_bal_file** out);
/* BalProblem::filter_obs (bal_problem.cpp:471-505; BalDatasetOptions::init_depth_threshold): drop the observations whose
 * landmark is closer than `threshold` in front of the camera, then the landmarks left with fewer than 2 observations
 * (landmark indices are compacted).  Call after rba_bal_load, before rba_bal_dims / rba_bal_copy; threshold <= 0: no-op. */
int32_t rba_bal_filter_obs(rba_bal_file* f, double threshold);
/* BalProblem::perturb (bal_problem.cpp:507-554; BalDatasetOptions rotation_sigma / translation_sigma / point_sigma /
 * random_seed, default seed 38401): Gaussian perturbation of the camera centres (world frame), the camera rotations
 * (left-multiplied exp) and the landmarks, drawn from one std::default_random_engine exactly as the reference draws them
 * (same random stream when the reference is built against libstdc++).  Call after rba_bal_load (which normalises) and
 * before rba_bal_filter_obs -- the order of load_normalized_bal_problem (bal_problem.cpp:813-826).  seed < 0: random device. */
int32_t rba_bal_perturb(rba_bal_file* f, double rotation_sigma, double translation_sigma, double point_sigma, int32_t seed);
/* sizes, to allocate the arrays for rba_bal_copy */
int32_t rba_bal_dims(const rba_bal_file* f, int32_t* num_cameras, int32_t* num_landmarks, int64_t* num_observations);
/* cams [10*Nc] (qx,qy,qz,qw,t,f,k1,k2 = Camera::params(), bal_problem.hpp:84-89), lms [3*Nl], lm_obs_offset [Nl+1],
 * obs_cam_idx [Nobs], obs_xy [2*Nobs]; any pointer may be NULL */
int32_t rba_bal_copy(const rba_bal_file* f, double* cams, double* lms, int64_t* lm_obs_offset, int32_t* obs_cam_idx, double* obs_xy);
/* seconds spent reading / counting tokens / parsing / building the CSR / normalising in rba_bal_load */
int32_t rba_bal_load_timings(const rba_bal_file* f, double* out5);
int32_t rba_bal_free(rba_bal_file* f);

/* ---- optimisation state: BalProblem cameras()/landmarks() mirror ------------------------- */

/* host -> device; cams [10*Nc], lms [3*Nl] (full problem; a sharded handle reads its slice) */
int32_t rba_set_state(rba_handle* h, const void* cams, const void* lms);
/* device -> host; a sharded handle writes only its landmark slice of lms */
int32_t rba_get_state(rba_handle* h, void* cams, void* lms);
/* BalProblem::backup / restore (bal/bal_problem.cpp:590-608) on device */
int32_t rba_backup(rba_handle* h);
int32_t rba_restore(rba_handle* h);

/* ---- camera parameters held constant ---------------------------------------------------- */

/* One byte of flags per camera.  Bit order follows the 9-entry increment of a camera
 * (tx,ty,tz, rx,ry,rz, f, k1, k2).  The pose is one group: the increment is a left-multiplied SE(3)
 * exponential, so a free rotation would move a "fixed" translation. */
#define RBA_FIX_POSE 1u       /* increment entries 0..5; camera parameters qx,qy,qz,qw, tx,ty,tz */
#define RBA_FIX_F 2u          /* entry 6; f  */
#define RBA_FIX_K1 4u         /* entry 7; k1 */
#define RBA_FIX_K2 8u         /* entry 8; k2 */
#define RBA_FIX_INTRINSICS 14u
#define RBA_FIX_ALL 15u

/* Not in the reference (its fix_pose_gauge is unimplemented, bal/solver_options.hpp:106-108).
 * flags [num_cameras of the full problem]: RBA_FIX_* bits per camera; NULL = every parameter free (the default).
 * Every rank of a sharded problem passes the same array.  Takes effect at the next rba_solve; the device-resident
 * increment of an earlier solve is discarded (rba_apply(h, NULL) then returns RBA_ERR_STATE until the next solve).
 * A solve then gives the LM step with the flagged parameters held constant: their increment entries are exactly 0, the
 * free entries solve H_ff x_f = -b_f (the reduced camera system restricted to the free rows and columns), and the flagged
 * camera parameters stay bit-identical through rba_apply / rba_lm_step / rba_lm_run, also when rba_apply is given a host
 * increment with non-zero entries there (they are zeroed before the back-substitution).  Landmarks are all free.
 * A flag with a bit above 3 set -> RBA_ERR_INVALID_ARGUMENT, and the previous flags stay in force. */
int32_t rba_set_camera_fixed(rba_handle* h, const uint8_t* flags);

/* ---- Gaussian priors on the cameras (DESIGN.md section 14) -------------------------------- */

/* Not in the reference.  A soft prior on each camera's centre, orientation and intrinsics.
 * mean [10*Nc] Scalar per camera: qx,qy,qz,qw (world->camera rotation R0, the state's convention), cx,cy,cz (camera
 *   CENTRE c0 in the world frame, not t), f0, k1_0, k2_0.
 * sqrt_info [81*Nc] Scalar: per camera a row-major 9x9 square-root information L_c.  Residual order
 *   e = (c - c0 [3], Log(R R0^T) [3], f - f0, k1 - k1_0, k2 - k2_0),  c = -R^T t.
 *   The prior cost is 1/2 |L_c e_c|^2, in the same convention as the reprojection terms (err = 1/2 r^2); a robust loss per
 *   camera is set by rba_set_prior_loss (DESIGN.md section 22).
 *   An all-zero L_c means no prior on camera c.  Partial priors are rows of L (e.g. centre only).
 * Both NULL: no priors, the default.  Every rank of a sharded problem passes the same arrays.
 * The prior Jacobian is part of the linearisation: the Jacobi scaling is computed from the whole Jacobian (reprojection and
 * prior columns), and rba_get_jacobian_scaling, rba_get_rhs, rba_get_preconditioner and rba_right_multiply include the
 * prior terms.  After a call, rba_solve returns RBA_ERR_STATE until the next rba_linearize, the device-resident increment
 * is discarded and the next rba_compute_error is evaluated afresh.
 * rba_compute_error adds sum_c 1/2 |L_c e_c|^2 (accumulated in double) to all_error and valid_error; a non-finite prior
 * cost clears is_numerically_valid; the observation counts and residual sums are unchanged.  So every optimized_cost,
 * rba_lm_step, rba_lm_run and the host LM loops minimise the total (reprojection + prior) cost with no change of their own.
 * With rba_set_camera_fixed the solve gives the restricted system of the total problem.
 * Exactly one NULL pointer, a non-finite entry, or a mean quaternion whose norm is not within 1e-3 of 1 ->
 * RBA_ERR_INVALID_ARGUMENT, and the previous priors stay in force.  A valid quaternion is normalised in double. */
int32_t rba_set_camera_prior(rba_handle* h, const void* mean, const void* sqrt_info);

/* ---- Relative pose priors between pairs of cameras (DESIGN.md section 15) ------------------ */

/* Not in the reference.  A soft prior on the relative pose of two cameras (odometry, rig extrinsics, loop closures,
 * pose-graph results).  Poses are world->camera, T = [R | t], as in the state.  Pair p joins cameras (i, j), i != j:
 * pairs [2*num_pairs] int32 (i, j); mean [7*num_pairs] Scalar (qx,qy,qz,qw of R0, t0): the measured Z = (R0, t0) with
 *   T_i T_j^-1 ~ Z;  sqrt_info [36*num_pairs] Scalar, row-major 6x6 L.  num_pairs == 0 (pointers ignored): no pair priors,
 *   the default.  Residual (split form, not the SE(3) logarithm)
 *     e_t = t_i - R_i R_j^T t_j - t0   (= R_i (c_j - c_i) - t0, the centre of j seen from camera i),
 *     e_r = Log(R_i R_j^T R0^T)        (angle in [0, pi]),
 *   cost 1/2 |L (e_t, e_r)|^2 (a robust loss per pair: rba_set_prior_loss, DESIGN.md section 22).  An all-zero L has no effect.  Several pairs on the same cameras, and both
 *   (i, j) and (j, i), are allowed: each is one more measurement.  Every rank of a sharded problem passes the same arrays.
 * Like the absolute priors the pair priors are part of the linearisation (Jacobi scaling, rba_get_rhs,
 * rba_get_preconditioner, rba_right_multiply, rba_compute_error include them), combine with rba_set_camera_prior and
 * rba_set_camera_fixed, and after a call rba_solve returns RBA_ERR_STATE until the next rba_linearize; the device-resident
 * increment and the cached error are discarded.
 * num_pairs < 0, a NULL array when num_pairs > 0, a camera index outside [0, Nc) or i == j, a non-finite entry, or a mean
 * quaternion whose norm is not within 1e-3 of 1 -> RBA_ERR_INVALID_ARGUMENT, and the previous pair priors stay in force.
 * A valid quaternion is normalised in double. */
int32_t rba_set_camera_pair_prior(rba_handle* h, int32_t num_pairs, const int32_t* pairs, const void* mean,
                                  const void* sqrt_info);

/* ---- Gaussian priors on landmark positions (DESIGN.md section 17) ------------------------- */

/* Not in the reference.  A soft prior on the world position of selected landmarks (surveyed ground control points, depth
 * or LiDAR points, points of an earlier map).  Prior p is on landmark lm_idx[p] (problem order):
 *   lm_idx [num] int32;  mean [3*num] Scalar, the prior position x0 (world frame);  sqrt_info [9*num] Scalar, row-major
 *   3x3 L.  num == 0 (pointers ignored): no landmark priors, the default.  Residual e = x - x0, cost 1/2 |L e|^2 (a
 *   robust loss per prior: rba_set_prior_loss, DESIGN.md section 22).  L need not have full rank (a height-only prior is one non-zero row); an all-zero L is dropped.  Every
 *   rank of a sharded problem passes the same full list and keeps the priors of its own landmark shard.
 * The priors are part of the linearisation: the landmark Jacobi scaling is that of the whole Jacobian, and the solve, the
 * back-substitution, l_diff of rba_apply, rba_compute_error and rba_compute_covariance include them (a prior can give a
 * landmark with fewer than 2 valid observations a full-rank block, and priors on three non-collinear landmarks can fix the
 * gauge).  They combine with the camera priors, the pair priors and rba_set_camera_fixed.  After a call rba_solve returns
 * RBA_ERR_STATE until the next rba_linearize; the device-resident increment and the cached error are discarded.
 * The 3 damping rows of a landmark with a prior (rba_debug_get_block's last 3 rows) are those of [C | 0 | c], the QR of the
 * prior rows and the damping rows, after the 6 damping rotations, instead of those of [sqrt(lambda) I | 0 | 0].
 * num < 0, a NULL array when num > 0, an index outside [0, Nl), a repeated index or a non-finite entry ->
 * RBA_ERR_INVALID_ARGUMENT, and the previous landmark priors stay in force. */
int32_t rba_set_landmark_prior(rba_handle* h, int32_t num, const int32_t* lm_idx, const void* mean, const void* sqrt_info);

/* ---- Intrinsics shared across groups of cameras (DESIGN.md section 18) -------------------- */

/* Not in the reference.  Images taken by one physical camera share one set of intrinsics (f, k1, k2 together).
 * group [num_cameras of the full problem] int32: -1 = the camera keeps its own intrinsics; g >= 0 = group id (any
 * non-negative value below Nc).  NULL = no groups (the default).  A group's lead is its lowest-index camera; a group of one
 * camera is an ungrouped camera, bit for bit.  Every rank of a sharded problem passes the same array.
 * The solve gives the LM step of the tied problem (a pose per camera, one f, k1, k2 per group): with x = P u (P copies a
 * group's intrinsics into every member), (P^T D J^T J D P + lambda I) u = -P^T D J^T r, D the Jacobi scaling of the merged
 * columns J P, lambda once per group.  The call copies the lead's f, k1, k2 into the other members of its group (state and
 * backup), and so does every later rba_set_state; the members then stay bit-identical through rba_apply, rba_lm_step,
 * rba_lm_run, rba_backup and rba_restore.  A host increment given to rba_apply / rba_back_substitute has the members'
 * entries 6..8 replaced by the lead's before the back-substitution.
 * rba_get_jacobian_scaling gives every member the group-summed norms; rba_get_rhs the contracted b (the lead's entries 6..8
 * hold the group's sum, the other members' are 0); rba_get_preconditioner the inverse PCG uses (the lead's block is
 * blkdiag(pose^-1, G^-1) with G the members' summed intrinsics blocks + lambda I, another member's the pose inverse with
 * zero intrinsics rows and columns).  rba_right_multiply stays the full, ungrouped operator; rba_compute_error is unchanged.
 * After a call rba_solve returns RBA_ERR_STATE until the next rba_linearize; the device-resident increment and the cached
 * error are discarded.
 * An id outside [-1, Nc), or RBA_FIX_F / K1 / K2 bits that differ between members of one group (checked here and by
 * rba_set_camera_fixed) -> RBA_ERR_INVALID_ARGUMENT, and the previous groups (or flags) stay in force.  Groups of >= 2
 * cameras with solver_type = 2 (POWER_SCHUR_COMPLEMENT: Hpp of the tied problem is not block-diagonal) -> RBA_ERR_UNSUPPORTED.
 * rba_compute_covariance gives the covariance of the tied problem, P (P^T H P)^-1 P^T: every member's 9x9 block carries the
 * group's intrinsics covariance and its own pose-intrinsics cross terms, and the landmark blocks use the same matrix. */
int32_t rba_set_intrinsics_groups(rba_handle* h, const int32_t* group);

/* ---- Rigid camera rigs (DESIGN.md section 23) --------------------------------------------- */

/* Not in the reference.  The cameras of a rigid multi-camera body (a stereo head, a vehicle's cameras, a spherical head)
 * exposed together: one placement of the body is one rig.  Camera c of a rig has fixed extrinsics E_c = [R_e | t_e]
 * (cam_from_rig) and pose T_c = E_c T_rig (world->camera, as in the state).
 * rig [num_cameras of the full problem] int32: -1 = free camera; r >= 0 = rig id (any non-negative value below Nc).
 * cam_from_rig [7*Nc] Scalar: qx,qy,qz,qw, tx,ty,tz of E_c (the entries of free cameras are ignored).  Both NULL = no rigs
 * (the default).  A rig's lead is its lowest-index camera; a rig of one camera is a free camera, bit for bit.  Every rank
 * of a sharded problem passes the same arrays.
 * Every member j is kept at T_j = M_j T_lead, M_j = E_j E_lead^-1: the call sets the members' poses so (state and backup),
 * and so does every later rba_set_state and every camera update of rba_apply / rba_lm_step / rba_lm_run (computed in
 * double, rounded to Scalar), so rigs stay exactly rigid.  The solve gives the LM step of the tied problem (one pose per
 * rig, every camera's own intrinsics): with x = P u, P mapping the rig's pose increment to member j through the adjoint
 * A_j = [[R_m, [t_m]x R_m], [0, R_m]] of M_j = [R_m | t_m], (D_u P^T J^T J P D_u + lambda I) u = -D_u P^T J^T r, D_u the
 * Jacobi scaling of the merged columns J P (the whole weighted Jacobian: observations, camera and pair priors), lambda
 * once per rig pose parameter.  Combines with rba_set_intrinsics_groups (rigs tie entries 0..5, groups entries 6..8).
 * A host increment given to rba_apply / rba_back_substitute has the members' pose entries replaced by D_j^-1 A_j D_lead
 * times the lead's, so the increment rba_solve returns round-trips.
 * rba_get_jacobian_scaling gives the per-camera scaling, unchanged; rba_get_rhs the contracted b (the members' pose
 * entries 0); rba_get_preconditioner the inverse PCG uses (the lead's pose block from sum_j P~_j^T B_j P~_j, without the
 * cross terms between members; the members' pose rows and columns 0); rba_right_multiply stays the full, untied operator;
 * rba_compute_error is unchanged.
 * After a call rba_solve returns RBA_ERR_STATE until the next rba_linearize; the device-resident increment and the cached
 * error are discarded.
 * Exactly one NULL pointer, an id outside [-1, Nc), a non-finite entry or a quaternion whose norm is not within 1e-3 of 1
 * on a camera with an id, or RBA_FIX_POSE bits that differ between members of one rig (checked here and by
 * rba_set_camera_fixed) -> RBA_ERR_INVALID_ARGUMENT, and the previous rigs (or flags) stay in force; so do they when an
 * allocation fails.  A valid quaternion is normalised in double.  Rigs of >= 2 cameras with solver_type = 2
 * (POWER_SCHUR_COMPLEMENT: Hpp of the tied problem is not block-diagonal) -> RBA_ERR_UNSUPPORTED.
 * rba_compute_covariance and rba_compute_covariance_blocks give the covariance of the tied problem, P (P^T H P)^-1 P^T with
 * the unscaled A_j: every member's block carries its rig's pose covariance mapped through A_j, and the relative-pose
 * covariance of two members of one rig is 0 to rounding. */
int32_t rba_set_camera_rigs(rba_handle* h, const int32_t* rig, const void* cam_from_rig);

/* ---- Estimated rig extrinsics (DESIGN.md section 24) ------------------------------------------ */

/* Not in the reference.  Rig bundle adjustment: the extrinsics of a physical camera of the rigs ("sensor") are estimated,
 * one cam_from_rig shared by every capture of that sensor and refined together with the rig poses and the landmarks.
 * sensor [num_cameras of the full problem] int32: -1 = the camera's cam_from_rig (rba_set_camera_rigs) is held, as before;
 * s >= 0 = camera c is a capture of sensor s (any non-negative value below Nc), whose extrinsics are estimated and shared by
 * every camera with id s.  NULL = no sensors (the default): rigs behave bit for bit as in section 23.  Every rank of a
 * sharded problem passes the same array.
 * Lead: with sensors a rig's lead (it carries the rig's pose) is its lowest-index camera with held extrinsics.  A held
 * member stays at T_j = M_j T_lead, M_j = E_j E_lead^-1.  Sensor s has a home, its lowest-index camera; the state defines
 * its extrinsics as the home's pose relative to its lead, E_s = T_home T_lead(home)^-1 E_lead(home), and every other camera
 * j of s is kept at T_j = E_s E_lead(j)^-1 T_lead(j) (computed in double, rounded to Scalar) after every camera update and
 * at every rba_set_state.  The extrinsics live in the camera state, so rba_backup / rba_restore, rba_get_state /
 * rba_set_state, rba_lm_step and rba_lm_run carry them unchanged.  The call re-ties every member from its (possibly new)
 * lead: held members through the extrinsics given to rba_set_camera_rigs, every camera of sensor s through those of s's home.
 * The solve gives the LM step of the tied problem J P with one pose per rig, one pose per sensor and every camera's own
 * intrinsics (or its group's): a sensor camera moves by A_j d_lead + d_s, d_s the left increment of E_s in the state's
 * convention (R' = Exp(w) R, t' = Exp(w) t + v) and A_j the adjoint of the current M_j; the Jacobi scaling is that of the
 * merged columns (with the pair-prior cross terms between two cameras of one sensor), lambda once per sensor pose parameter.
 * A pair prior between a rig's lead and a capture of an estimated sensor acts on that sensor's extrinsics: a way to feed a
 * factory calibration with its uncertainty.  RBA_FIX_POSE on a rig holds the rig's pose; the captures of an estimated
 * sensor still move with it (give them -1 to hold a sensor).
 * rba_get_rhs / rba_get_preconditioner give the contracted vectors, the home's pose entries holding the sensor's;
 * rba_right_multiply stays the full operator; a host increment's sensor entries are recovered from the home's and its
 * lead's entries, so the increment rba_solve returns round-trips through rba_apply.  rba_compute_covariance and
 * rba_compute_covariance_blocks give P (P^T H P)^-1 P^T for this P: the relative_cov of a lead and a capture of sensor s is
 * the uncertainty of that calibration.
 * After a call rba_solve returns RBA_ERR_STATE until the next rba_linearize.  An id outside [-1, Nc), an id on a camera
 * that is not in a rig of >= 2 cameras, two cameras of one rig with the same id, or a rig in which every camera has an id
 * -> RBA_ERR_INVALID_ARGUMENT, and the previous sensors stay in force; so do they when an allocation fails.  A later
 * successful rba_set_camera_rigs clears the sensors. */
int32_t rba_set_rig_sensors(rba_handle* h, const int32_t* sensor);
/* cam_from_rig [7*Nc] Scalar: every rigged camera's current extrinsics in the convention rba_set_camera_rigs takes, so the
 * output can be passed back in: held ones as given (normalised), a sensor's E_s from the current state; free cameras (and
 * rigs of one) the identity.  Needs no rba_linearize and changes nothing of the handle; a sharded handle writes every camera. */
int32_t rba_get_rig_extrinsics(rba_handle* h, void* cam_from_rig);

/* ---- Per-observation square-root information and residual read-back (DESIGN.md section 19) -- */

/* Not in the reference, where every reprojection term has unit weight.  Observation o (index in the problem's CSR order, the
 * order of obs_cam_idx / obs_xy) gets a row-major 2x2 W_o; its rows become sqrt(hw) W_o [Jp | Jl | r] and its cost
 * rho(|W_o r|^2), rho the handle's robust norm, so the Huber parameter is in units of sigma.  W_o = Sigma_o^-1/2 (any square
 * root: W need not be symmetric or triangular) is the Gaussian case, sqrt(w) I a scalar weight, rank 1 a constraint along one
 * image direction, and W_o = 0 switches the observation off: it gives the all-zero rows of a projection dropped by
 * use_valid_projections_only.  Projection validity (z >= eps_sqrt) does not depend on W.
 * sqrt_info [4*num_observations of the full problem] Scalar, row-major 2x2 per observation in problem order;
 * NULL = identity everywhere, the default.  Every rank of a sharded problem passes the same full array and keeps the
 * entries of its own landmark shard.  An array that is the identity bit for bit is the same as NULL: the unmodified kernels
 * run and every result is bit-identical to a handle that never had information set.
 * rba_compute_error: all_error / valid_error sum rho(|W r|^2), all_residual_sum / valid_residual_sum sum |W r|.  A switched-off
 * observation stays in all_num_obs (contributing 0) and is not counted in valid_num_obs, valid_error, valid_residual_sum,
 * whatever its projection validity; a projection of it that is not finite neither clears is_numerically_valid nor fails
 * rba_linearize.  Everything derived from the Jacobian uses the whitened rows: rba_get_jacobian_scaling, rba_get_rhs,
 * rba_get_preconditioner, rba_right_multiply, rba_debug_get_block, rba_compute_covariance.
 * After a successful call rba_solve returns RBA_ERR_STATE until the next rba_linearize; the device-resident increment and the
 * cached error are discarded.  A non-finite entry -> RBA_ERR_INVALID_ARGUMENT, and the previous information stays in force.
 * The information costs 4 Scalars per observation slot of device memory, counted in rba_workload_stats::device_bytes from
 * the first call that sets one on. */
int32_t rba_set_observation_info(rba_handle* h, const void* sqrt_info);

/* Per observation at the handle's CURRENT state, in problem order; any pointer may be NULL (all NULL ->
 * RBA_ERR_INVALID_ARGUMENT).  residual [2*Nobs] Scalar: the whitened residual W r (the raw r without observation
 * info); robust_weight [Nobs] Scalar: the robust weight w on |W r|^2 of the observation's own loss (rba_set_observation_loss;
 * without one the handle's robust norm, 1 with robust_norm NONE); flags [Nobs] uint8:
 * bit 0 = projection valid (z >= eps_sqrt), bit 1 = in use (W != 0).  A sharded handle writes only the observations of
 * its own landmark shard.  Needs no rba_linearize; changes nothing of the handle (scratch device memory is allocated for the
 * call and freed before it returns). */
int32_t rba_get_observation_residuals(rba_handle* h, void* residual, void* robust_weight, uint8_t* flags);

/* ---- Robust loss per observation (DESIGN.md section 21) ------------------------------------- */

#define RBA_LOSS_NONE    0
#define RBA_LOSS_HUBER   1
#define RBA_LOSS_CAUCHY  2
#define RBA_LOSS_SOFT_L1 3
#define RBA_LOSS_TUKEY   4

/* Not in the reference, where one robust norm (robust_norm, huber_parameter) applies to every observation.  Observation o
 * (index in the problem's CSR order) gets its own loss kind[o] with the scale a = scale[o], the inlier threshold in units of
 * sigma.  With s = |W r|^2 (W of rba_set_observation_info, or the identity) its cost is rho(s)/2, its robust weight
 * w = rho'(s) and its rows sqrt(w) W [Jp | Jl | r] (IRLS weighting as for Huber, no second-order correction):
 *   RBA_LOSS_NONE     rho = s                                                       w = 1           (scale ignored)
 *   RBA_LOSS_HUBER    rho = s if s < a^2, else 2 a sqrt(s) - a^2                    w = 1, else a / sqrt(s)
 *   RBA_LOSS_CAUCHY   rho = a^2 log1p(s / a^2)                                      w = 1 / (1 + s / a^2)
 *   RBA_LOSS_SOFT_L1  rho = 2 a^2 (sqrt(1 + s / a^2) - 1)                           w = 1 / sqrt(1 + s / a^2)
 *   RBA_LOSS_TUKEY    rho = (a^2 / 3) (1 - (1 - u)^3), u = s / a^2 < 1; else a^2/3  w = (1 - u)^2, else 0
 * Every rho has rho(s) ~ s and w -> 1 as s -> 0.  HUBER is exactly the handle's Huber norm; HUBER, CAUCHY and SOFT_L1 are
 * scipy.optimize.least_squares' losses with f_scale = a, and TUKEY is twice Ceres' TukeyLoss.
 * kind [Nobs] uint8 and scale [Nobs] Scalar of the full problem in problem order; both NULL = every observation uses the
 * handle's robust_norm / huber_parameter, the default.  Every rank of a sharded problem passes the same full arrays and keeps
 * the entries of its own landmark shard.  Arrays equal to the handle's own choice on every observation of the shard
 * ((RBA_LOSS_HUBER, (Scalar)huber_parameter) with robust_norm = 1, else RBA_LOSS_NONE) are the same as NULL: the unmodified
 * kernels run, bit for bit.  rba_solver_opts is unchanged.
 * A TUKEY observation beyond its scale (w = 0) has all-zero rows like a dropped projection, but still counts as valid in
 * rba_compute_error and adds a^2/6 to all_error / valid_error.  A switched-off observation (W = 0) stays off whatever its
 * loss.  A non-finite residual fails rba_linearize and clears is_numerically_valid as before, whatever the loss.
 * rba_get_observation_residuals returns each observation's own w; rba_compute_covariance and rba_compute_covariance_blocks
 * use it.  After a successful call rba_solve returns RBA_ERR_STATE until the next rba_linearize; the device-resident
 * increment and the cached error are discarded.
 * RBA_ERR_INVALID_ARGUMENT, with the previous losses kept in force: exactly one pointer NULL, a kind above RBA_LOSS_TUKEY, or
 * a kind other than RBA_LOSS_NONE with a scale that is not finite or <= 0.
 * The losses cost 8 bytes (float) or 9 bytes (double) per observation slot of device memory, counted in
 * rba_workload_stats::device_bytes from the first call that sets a loss other than the handle's own. */
int32_t rba_set_observation_loss(rba_handle* h, const uint8_t* kind, const void* scale);

/* ---- Robust losses on the priors (DESIGN.md section 22) ------------------------------------- */

#define RBA_PRIOR_CAMERA   0   /* rba_set_camera_prior:      one entry per camera, num = Nc            */
#define RBA_PRIOR_PAIR     1   /* rba_set_camera_pair_prior: one entry per pair, in the caller's order */
#define RBA_PRIOR_LANDMARK 2   /* rba_set_landmark_prior:    one entry per prior, in the caller's order */

/* Not in the reference.  Prior p of any kind has the whitened residual L_p e_p (e as defined for its kind) and
 * s_p = |L_p e_p|^2.  With a loss kind[p] and scale a = scale[p] (RBA_LOSS_*, the same rho as rba_set_observation_loss, from
 * the same device function) its cost is rho(s_p)/2, its robust weight w_p = rho'(s_p) and its rows sqrt(w_p) L_p de/d(inc)
 * and sqrt(w_p) L_p e_p (IRLS weighting, no second-order correction).  One weight per prior, on its whole squared
 * Mahalanobis distance (not per component): a is compared with |L e|.  A 95 % gate is a = sqrt(chi2_0.95(dof)): a ~ 3.55 for
 * a 6-DoF pair prior, a ~ 2.80 for a 3-DoF centre or landmark prior.  A TUKEY prior beyond its scale has w = 0: all-zero
 * rows, and a^2/6 in all_error and valid_error.
 * prior_kind RBA_PRIOR_*; kind [num] uint8 and scale [num] Scalar in the caller's order of that kind's setter: num = Nc for
 * camera priors, else the num (num_pairs) of the last successful call of its setter.  Priors dropped for an all-zero L, and
 * landmark priors of another shard, take their entries and ignore them.  Both NULL, or NONE on every entry, = no losses on
 * that kind, the default: the unmodified kernels run.  The handle's robust_norm never applies to priors; rba_solver_opts
 * is unchanged.  A later successful call of the kind's setter clears its losses back to NONE.
 * The rows and costs of every entry point (rba_linearize, rba_solve, rba_get_rhs, rba_get_preconditioner,
 * rba_right_multiply, rba_compute_error, l_diff) use the weighted priors, w taken at the state of rba_linearize for the
 * rows and at the current state for the cost; rba_compute_covariance and rba_compute_covariance_blocks evaluate w in
 * double at their current state.
 * After a successful call rba_solve returns RBA_ERR_STATE until the next rba_linearize; the device-resident increment and
 * the cached error are discarded.  RBA_ERR_INVALID_ARGUMENT, with the previous losses kept in force: an unknown prior_kind,
 * a num that does not match, exactly one pointer NULL, a kind above RBA_LOSS_TUKEY, or a kind other than RBA_LOSS_NONE with
 * a scale that is not finite or <= 0.
 * The losses cost the loss records (8 bytes (float) or 9 bytes (double) per prior) and a copy of the priors' L of device
 * memory, counted in rba_workload_stats::device_bytes from the first call that sets a loss other than NONE. */
int32_t rba_set_prior_loss(rba_handle* h, int32_t prior_kind, int32_t num, const uint8_t* kind, const void* scale);

/* Per prior of one kind at the handle's CURRENT state, in the caller's order of its setter (num entries as for
 * rba_set_prior_loss); either pointer may be NULL, not both (-> RBA_ERR_INVALID_ARGUMENT, as is an unknown prior_kind).
 * residual [9 / 6 / 3 * num] Scalar: L e, with the unweighted L; robust_weight [num] Scalar: w of the prior's loss (1 with
 * NONE).  A camera with an all-zero L, or a dropped pair or landmark prior, gives 0 and weight 1.  A sharded handle writes
 * every camera and pair entry, but only the landmark priors of its own shard.  Needs no rba_linearize; changes nothing of
 * the handle (scratch device memory is allocated for the call and freed before it returns). */
int32_t rba_get_prior_residuals(rba_handle* h, int32_t prior_kind, void* residual, void* robust_weight);

/* ---- Triangulation of landmarks from the current cameras (DESIGN.md section 25) ------------ */

#define RBA_TRIANGULATE_LINEAR 1   /* replace the position by the linear estimate from the rays */
#define RBA_TRIANGULATE_REFINE 2   /* minimise the landmark's own cost with the cameras held */

#define RBA_TRI_WRITTEN     1u     /* the landmark's position changed */
#define RBA_TRI_FEW_RAYS    2u     /* < 2 usable rays */
#define RBA_TRI_SMALL_ANGLE 4u     /* largest ray angle < min_angle */
#define RBA_TRI_AT_INFINITY 8u     /* linear estimate at (or beyond) infinity */
#define RBA_TRI_BEHIND      16u    /* linear estimate behind a camera of a usable ray */
#define RBA_TRI_REFINED     32u    /* the refinement accepted at least one step */
#define RBA_TRI_CONVERGED   64u    /* the refinement met function_tolerance */

typedef struct {
  int32_t mode;               /* RBA_TRIANGULATE_* bits, 1..3; default LINEAR | REFINE */
  int32_t max_iterations;     /* refinement iterations per landmark, rejected steps included; default 20 */
  double min_angle;           /* radians, >= 0; default 0 */
  double function_tolerance;  /* stop once a step changes the cost by less than this fraction; default 1e-10 */
  int32_t reserved[2];
} rba_triangulate_opts;       /* 32 bytes, no implicit padding */

void rba_default_triangulate_opts(rba_triangulate_opts* o);
/* Not in the reference.  Re-initialises landmark positions from the handle's current cameras, which are held: a problem
 * assembled from feature tracks, landmarks left behind by an outlier loop (W = 0) or by moved rig extrinsics.
 * lm_idx [num] int32 lists landmarks by problem index; NULL = every landmark, num must then be Nl.  Outputs are in the
 * caller's order and any of them may be NULL: status [num] RBA_TRI_* bits, angle [num] the largest angle (radians) between
 * two usable rays (0 with fewer than 2), cost [num] the landmark's share of rba_compute_error at its final stored position.
 * A sharded handle follows rba_set_landmark_prior: every rank passes the same full list, works on the entries of its own
 * shard and writes only those outputs.  Evaluated in float64 for either Scalar; a written position is rounded to Scalar.
 * A usable ray is an observation in use (W != 0) with f != 0 whose distortion inverts: rho (1 + k1 rho^2 + k2 rho^4) =
 * |obs| / |f| solved by Newton from rho = |obs / f| with a fixed iteration cap, failing when 1 + 3 k1 rho^2 + 5 k2 rho^4 <= 0
 * at an iterate or when it does not converge.  The ray is R^T (m, 1) from the centre c = -R^T t.
 * LINEAR: the homogeneous midpoint estimate (the smallest eigenvector of sum_i A_i^T A_i, A_i = (I - d d^T) [R | t], in
 * coordinates centred on the track's mean camera centre and scaled by their RMS distance), rejected as AT_INFINITY when
 * |X_h[3]| <= 1e-10 |X_h| and as BEHIND when its depth is below eps_sqrt of the Scalar in a camera of a usable ray; a
 * rejected estimate is not written.  REFINE: Levenberg-Marquardt on the landmark's share of the cost (its observations' own
 * losses or the handle's robust norm, the observation information, use_valid_projections_only, its landmark prior and that
 * prior's loss), IRLS-weighted normal equations; a step is accepted only when the cost decreases and no observation in use
 * goes from valid to invalid depth.  It starts from the position LINEAR left (or the current one without LINEAR), and its
 * result is written only when its cost, after rounding to Scalar, is below the cost at its start.  FEW_RAYS and
 * SMALL_ANGLE landmarks are left untouched, except that a FEW_RAYS landmark with a landmark prior is still refined.
 * The call is a state change: the state version is bumped, the error cache and the device-resident increment are
 * discarded and rba_solve returns RBA_ERR_STATE until the next rba_linearize.  rba_backup is untouched, so rba_restore
 * brings the previous landmarks back.  Cameras, rigs, sensors, groups, held flags and priors are read only.  Scratch device
 * memory is allocated for the call and freed before it returns.
 * RBA_ERR_INVALID_ARGUMENT before any device work, with nothing changed: o NULL, mode outside 1..3, max_iterations < 0,
 * min_angle or function_tolerance negative or not finite, num < 0, lm_idx NULL with num != Nl, an index outside [0, Nl) or
 * a repeated index. */
int32_t rba_triangulate_landmarks(rba_handle* h, const rba_triangulate_opts* o, int32_t num, const int32_t* lm_idx,
                                  uint8_t* status, double* angle, double* cost);

/* ---- Resection of cameras from the current landmarks (DESIGN.md section 26) ---------------- */

#define RBA_RESECT_LINEAR     1   /* replace the pose by the linear estimate from the 2D-3D correspondences */
#define RBA_RESECT_REFINE     2   /* minimise the camera's (rig's) own cost with the landmarks held */
#define RBA_RESECT_INTRINSICS 4   /* with REFINE: also refine the free f, k1, k2 of a single-camera unit */

#define RBA_RES_WRITTEN     1u    /* the unit's pose (or intrinsics) changed */
#define RBA_RES_FEW_POINTS  2u    /* < 3 usable points and no camera or pair prior on the unit: untouched */
#define RBA_RES_DEGENERATE  4u    /* LINEAR asked for, but < 6 usable points, near-planar points or a singular estimate */
#define RBA_RES_BEHIND      8u    /* linear estimate puts more than half of the usable points behind the camera */
#define RBA_RES_REFINED    16u    /* the refinement accepted at least one step */
#define RBA_RES_CONVERGED  32u    /* the refinement met function_tolerance */
#define RBA_RES_HELD       64u    /* the unit has no free entry (RBA_FIX_*): untouched */

typedef struct {
  int32_t mode;               /* RBA_RESECT_* bits; default LINEAR | REFINE */
  int32_t max_iterations;     /* refinement iterations per unit, rejected steps included; default 20 */
  double function_tolerance;  /* stop once a step changes the cost by less than this fraction; default 1e-10 */
  int32_t reserved[2];
} rba_resect_opts;            /* 24 bytes, no implicit padding */

void rba_default_resect_opts(rba_resect_opts* o);
/* Not in the reference.  Re-initialises and refines camera poses from the handle's current landmarks, which are held
 * (camera resection, motion-only bundle adjustment): an image registered against an existing map, cameras left behind by
 * moved landmarks, an outlier loop (W = 0) or new ground control points.
 * cam_idx [num] int32 lists cameras by index; NULL = every camera, num must then be Nc.  A free camera is a unit of one; a
 * camera in a rig of >= 2 cameras stands for its whole rig, whose free pose is the lead's, every member moving as
 * T_j = M_j T_lead (M_j the map of the re-tie: the held extrinsics, or for a capture of a sensor the sensor's map at the
 * call's start, the home included, so that every E_s stays unchanged to rounding).  Listing several members of one rig
 * resects it once and gives each of them the unit's outputs.  Outputs are in the caller's order and any of them may be NULL:
 * status [num] RBA_RES_* bits, points [num] the unit's usable points over its members, cost [num] the unit's share of
 * rba_compute_error at its final stored pose.  Evaluated in float64 for either Scalar; a written pose is rounded to Scalar.
 * Only the cameras of the listed units are written; every other camera stays bit-identical.
 * Free entries: the pose unless the unit has RBA_FIX_POSE; f, k1, k2 only with RBA_RESECT_INTRINSICS, for a single camera
 * outside any intrinsics group of >= 2 cameras, each unless its own RBA_FIX_* bit is set.  A unit without a free entry is
 * HELD and untouched.  A usable point is an observation in use (W != 0) of a camera with f != 0 whose distortion inverts
 * (as for rba_triangulate_landmarks).  A unit with fewer than 3 usable points is FEW_POINTS and untouched, unless it carries
 * a camera prior or a pair prior: then it is still refined.
 * LINEAR (a unit with a free pose): the DLT of one member, the one with the most usable points (ties to the lowest index):
 * p [12] = P row by row is the smallest eigenvector of M = sum_i G_i^T (I - v_i v_i^T) G_i with P X~_i = G_i p,
 * X~_i = ((X_i - Xbar) / s, 1) (Xbar the mean and s the RMS distance of the usable points) and v_i = (m, 1) / |(m, 1)| the
 * unit ray of the undistorted point m.  With P = [A | b] signed so that det A > 0, R is the polar factor of A, sigma the mean
 * singular value of A and t = s b / sigma - R Xbar; the lead's pose is M_j^-1 T_j.  DEGENERATE (not written) with fewer
 * than 6 usable points in that member, when the smallest principal standard deviation of the centred points is below 1e-3
 * of the largest, or when |det A| <= 1e-10 |A|_F^3; BEHIND (not written) when more than half of the member's usable points
 * lie at depth < eps_sqrt of the Scalar under the estimate.
 * REFINE: Levenberg-Marquardt on the unit's share of the cost with the landmarks held: rho(|W r|^2)/2 of every observation
 * in use by a member (its own loss or the handle's robust norm, use_valid_projections_only), the members' camera priors and
 * every pair prior with an endpoint in the unit, counted once, each with its loss.  A pair endpoint outside the unit is read
 * from the call's start, so a unit's result does not depend on which other cameras are listed.  The increment is the
 * state's left increment R' = Exp(w) R, t' = Exp(w) t + v of the lead, restricted to the free entries, a member's Jacobian
 * mapped through its adjoint A_j; IRLS-weighted normal equations, the damping, lambda schedule, acceptance (a strict cost
 * decrease with no observation in use going from valid to invalid depth) and convergence rules of
 * rba_triangulate_landmarks.  It starts from the pose LINEAR left (or the current one without LINEAR), and its result is
 * written only when its cost, after rounding to Scalar, is below the cost at its start.
 * The call is a state change: the state version is bumped, the error cache and the device-resident increment are
 * discarded and rba_solve returns RBA_ERR_STATE until the next rba_linearize.  rba_backup is untouched, so rba_restore
 * brings the previous cameras back.  Landmarks, rigs, sensors, groups, held flags and priors are read only.  Scratch device
 * memory is allocated for the call and freed before it returns.
 * RBA_ERR_INVALID_ARGUMENT before any device work, with nothing changed: o NULL, a mode with neither LINEAR nor REFINE,
 * INTRINSICS without REFINE or an unknown bit, max_iterations < 0, function_tolerance negative or not finite, num < 0,
 * cam_idx NULL with num != Nc, an index outside [0, Nc) or a repeated index.  RBA_ERR_UNSUPPORTED on a sharded handle
 * (nranks > 1): a camera's observations span every shard. */
int32_t rba_resect_cameras(rba_handle* h, const rba_resect_opts* o, int32_t num, const int32_t* cam_idx, uint8_t* status,
                           int32_t* points, double* cost);

/* ---- Marginal covariances (DESIGN.md section 16) ------------------------------------------ */

/* Not in the reference.  DESIGN.md section 16.  The covariance of the Gauss-Newton step of the total objective (reprojection
 * terms + camera priors + pair priors) at lambda = 0 and the handle's current state: the inverse of H = J^T J, with J the rows
 * rba_linearize would build (whitened by the observation information of rba_set_observation_info when it is set, sqrt(w)-weighted
 * by each observation's robust weight -- its own loss of rba_set_observation_loss, else the handle's robust norm -- the rows
 * use_valid_projections_only drops set to zero), and
 * the parameters held by rba_set_camera_fixed as constants (their rows and columns are exactly 0).  Evaluated in float64 for
 * either Scalar; unscaled (no Jacobi scaling); independent of solver_type, operator_form, stage2_form, preconditioner_type and
 * the QR variant (bit-identical output within one Scalar).
 *   cam_cov [81*Nc] double or NULL: per camera the 9x9 marginal block, row-major, in the order of the increment
 *     (tx,ty,tz, rx,ry,rz, f,k1,k2) = (v, w, f, k1, k2) with R' = Exp(w) R, t' = Exp(w) t + v;
 *   lm_cov [9*Nl] double or NULL: per landmark (problem order) its 3x3 marginal block; all NaN for a landmark whose Jl^T Jl has
 *     rank < 3 (e.g. one valid observation) -- it is eliminated with the pseudo-inverse and the other outputs stay valid.
 * No prior rba_linearize is needed, and nothing of the handle changes (state, linearisation, device-resident increment, error
 * cache, timings); scratch device memory is allocated for the call and freed before it returns.
 * RBA_NUMERICAL_FAILURE: a Cholesky pivot <= 1e-10 of the equilibrated reduced camera matrix (gauge not fixed, or a free camera
 *   without observations and prior); the outputs are not written and rba_last_error names the camera and increment entry.
 * RBA_ERR_UNSUPPORTED: nranks > 1, or the dense matrix and scratch do not fit in free device memory (the message gives the bytes).
 * RBA_ERR_INVALID_ARGUMENT: both pointers NULL. */
int32_t rba_compute_covariance(rba_handle* h, double* cam_cov, double* lm_cov);

/* ---- Covariance blocks (DESIGN.md section 20) ------------------------------------------------ */

/* Not in the reference.  DESIGN.md section 20.  Blocks of the same covariance H^-1 as rba_compute_covariance (same H, held
 * parameters, intrinsics groups, priors, observation information, per-observation robust weights and validity; float64 for either Scalar;
 * increments (tx,ty,tz, rx,ry,rz, f,k1,k2) per camera and (x,y,z) per landmark in problem order), for chosen pairs, from one
 * factorisation.  Output k belongs to request k; repeated requests and any order are allowed.
 *   camera_cross [81*k]: Cov(d_a, d_b), 9x9 row-major, rows of camera a; (a, a) is bit-identical to cam_cov[a], (b, a) is the
 *     transpose of (a, b) to one rounding; the rows and columns of held entries are 0.
 *   camera_landmark_cross [27*k]: Cov(d_c, d_l), 9x3 row-major.
 *   landmark_cross [9*k]: Cov(d_l, d_m), 3x3 row-major; (l, l) is bit-identical to lm_cov[l].
 *   relative_cov [36*k]: the 6x6 covariance of the pair-prior residual e = (e_t, e_r) of rba_set_camera_pair_prior for the
 *     pair (i, j) (i != j), linearised at the current state with its mean at the current relative pose
 *     (R0 = R_i R_j^T, t0 = t_i - R_i R_j^T t_j): A Sigma A^T with A = [[I, -[t_rel]x, -M, 0], [0, I, 0, -M]] on
 *     (v_i, w_i, v_j, w_j), M = R_i R_j^T.  That mean with any L with L^T L = relative_cov^-1, given to
 *     rba_set_camera_pair_prior, carries the same first-order information on that relative pose.  Exactly symmetric; 0 between
 *     two cameras whose poses are held.
 *   cam_cov, lm_cov: optional (NULL: skipped), exactly rba_compute_covariance's outputs.
 * Every block that involves a landmark whose Jl^T Jl has rank < 3 is all NaN; the other blocks stay valid.
 * No prior rba_linearize is needed and nothing of the handle changes; scratch device memory is allocated for the call and freed
 * before it returns.  On every failure the outputs are not written:
 * RBA_ERR_INVALID_ARGUMENT (checked before any device work): q NULL, a negative count, a NULL array with a positive count, an
 *   index out of range, i == j for a relative pose, or nothing requested (all counts 0 and both marginal pointers NULL).
 * RBA_NUMERICAL_FAILURE, RBA_ERR_UNSUPPORTED: as rba_compute_covariance (the byte count includes the requests and outputs). */
typedef struct {
  int32_t num_camera_pairs, num_camera_landmark, num_landmark_pairs, num_relative_poses;
  const int32_t* camera_pairs;      /* [2*num_camera_pairs]     (a, b), 0 <= a, b < Nc                    */
  const int32_t* camera_landmark;   /* [2*num_camera_landmark]  (c, l), camera c, landmark l (problem order) */
  const int32_t* landmark_pairs;    /* [2*num_landmark_pairs]   (l, m)                                     */
  const int32_t* relative_pairs;    /* [2*num_relative_poses]   (i, j), i != j                             */
  double* camera_cross;             /* [81*num_camera_pairs]                                                */
  double* camera_landmark_cross;    /* [27*num_camera_landmark]                                             */
  double* landmark_cross;           /* [9*num_landmark_pairs]                                               */
  double* relative_cov;             /* [36*num_relative_poses]                                              */
  double* cam_cov;                  /* [81*Nc] or NULL                                                      */
  double* lm_cov;                   /* [9*Nl] or NULL                                                       */
} rba_covariance_query;             /* no implicit padding: 16 + 10*8 = 96 bytes on LP64 */
int32_t rba_compute_covariance_blocks(rba_handle* h, const rba_covariance_query* q);

/* ---- Linearizor interface (solver/linearizor.hpp:56-82) ---------------------------------- */

/* LinearizorBase::compute_error (linearizor_base.cpp:59-67) -> BalBundleAdjustmentHelper::compute_error
 * (bal_bundle_adjustment_helper.cpp:68-109); + the camera and pair prior costs (sections 14 and 15) */
int32_t rba_compute_error(rba_handle* h, rba_residual_info* out);
/* LinearizorQR::linearize (linearizor_qr.cpp:78-138): stage 1 */
int32_t rba_linearize(rba_handle* h);
/* LinearizorQR::solve (linearizor_qr.cpp:140-265): stage 2 + preconditioner + PCG.
 * inc_out [9*Nc] (Jacobi-scaled space, already negated) may be NULL: the increment then stays on
 * the device for rba_apply(h, NULL, ...). */
int32_t rba_solve_f32(rba_handle* h, float lambda, float* inc_out, rba_cg_summary* cg);
int32_t rba_solve_f64(rba_handle* h, double lambda, double* inc_out, rba_cg_summary* cg);
/* LinearizorQR::apply (linearizor_qr.cpp:267-291): back-substitution, landmark and camera update.
 * inc == NULL uses the device-resident increment of the last rba_solve. l_diff is NaN on failure. */
int32_t rba_apply_f32(rba_handle* h, const float* inc, float* l_diff_out);
int32_t rba_apply_f64(rba_handle* h, const double* inc, double* l_diff_out);
/* One LM inner iteration of optimize_lm_ours (bal_bundle_adjustment.cpp:324-521) with a SINGLE host synchronisation
 * (SURVEY 8f row 2): [rba_linearize when linearize_first] + rba_solve(lambda) + rba_backup + rba_apply with the
 * device-resident increment + rba_compute_error, enqueued back to back.  Same kernels in the same order as the separate
 * calls: bit-identical results.  The caller keeps the reference's accept / reject and lambda logic and calls rba_restore
 * on a rejected step -- also when `solve_failed` is set (PCG FAILURE = the reference's non-finite increment, which it
 * does not apply; here the step is applied on the device first and undone by the restore).
 * Returns like rba_apply: RBA_NUMERICAL_FAILURE when l_diff is not finite (l_diff = NaN). */
typedef struct {
  rba_cg_summary cg;
  double l_diff;              /* model cost change (Scalar precision, widened) */
  rba_residual_info cost;     /* ResidualInfo after the step */
  int32_t solve_failed;
  int32_t pad_;
} rba_lm_step_result;
int32_t rba_lm_step_f32(rba_handle* h, int32_t linearize_first, float lambda, rba_lm_step_result* out);
int32_t rba_lm_step_f64(rba_handle* h, int32_t linearize_first, double lambda, rba_lm_step_result* out);
/* The LM loop itself, natively: optimize_lm_ours (solver/bal_bundle_adjustment.cpp:291-521) on top of rba_lm_step, so that
 * consecutive iterations are separated by one host synchronisation and a few scalar operations instead of an interpreter.
 * Starts a NEW solve at the handle's current state (lambda = 1 / initial_trust_region_radius, vee = initial_vee) and runs
 * until the reference's stopping rule fires -- |cost change| <= function_tolerance * cost after a successful step (:174-201),
 * lambda > 1 / min_trust_region_radius (:378-379), max_num_iterations (:291) -- or `max_steps` iterations have been done.
 * Same Scalar arithmetic for lambda / vee / step quality as the reference loop (and as the Python / C++ host mirrors, which
 * stay the tested restatements).  One rba_lm_iteration is written per iteration. */
typedef struct {
  double initial_trust_region_radius, min_trust_region_radius, max_trust_region_radius;  /* solver_options.hpp:119-133 */
  double min_relative_decrease, initial_vee, vee_factor, function_tolerance;              /* :146-148, :136-143, :113 */
  int32_t max_num_iterations;                                                              /* :106 */
  int32_t optimized_cost;                                                                  /* 0 ERROR, 1 ERROR_VALID, 2 ERROR_VALID_AVG (:80-96) */
} rba_lm_opts;
typedef struct {
  double lambda;             /* damping used for this iteration's solve */
  double cost;               /* optimized cost after the step (NaN when the solve failed) */
  double l_diff;             /* model cost change */
  double relative_decrease;  /* step quality */
  double device_seconds;     /* device time of this iteration's stages (CUDA events) */
  int32_t cg_iterations;
  int32_t cg_termination;
  int32_t accepted;          /* step_is_successful */
  int32_t terminated;        /* the stopping rule fired after this iteration */
} rba_lm_iteration;
void rba_default_lm_opts(rba_lm_opts* o);
/* phase_totals (may be NULL): sums of the stage timings over the iterations done (same fields as rba_get_timings) */
int32_t rba_lm_run_f32(rba_handle* h, const rba_lm_opts* o, int32_t max_steps, rba_lm_iteration* log, int32_t* steps_done,
                       int32_t* terminated, rba_stage_timings* phase_totals);
int32_t rba_lm_run_f64(rba_handle* h, const rba_lm_opts* o, int32_t max_steps, rba_lm_iteration* log, int32_t* steps_done,
                       int32_t* terminated, rba_stage_timings* phase_totals);
/* device timings of the last calls */
int32_t rba_get_timings(const rba_handle* h, rba_stage_timings* out);

/* ---- LinearizationQR-level access used by the parity tests -------------------------------- */

/* pose_jacobian_scaling_ (linearizor_qr.cpp:130-132) [9*Nc] and the squared column norms
 * LinearizationQR::get_stage1 returns (linearization_qr.hpp:634-712); with camera priors and pair priors their columns are
 * included */
int32_t rba_get_jacobian_scaling(rba_handle* h, void* scaling_out, void* diag2_out);
/* RHS b of the reduced camera system after the last rba_solve (get_stage2, linearization_qr.hpp:716-815);
 * + A^T r of the camera priors and the pair priors; the entries of parameters held by rba_set_camera_fixed are 0 */
int32_t rba_get_rhs(rba_handle* h, void* b_out);
/* explicit inverse of the block-Jacobi preconditioner (cg/preconditioner.hpp:79-120) [81*Nc] and the
 * blocks it was built from (damping and the camera and pair priors' diagonal A^T A blocks already added; the blocks are written with SCHUR_JACOBI) [81*Nc].  For a camera with rba_set_camera_fixed flags the inverse is
 * that of the free sub-block, embedded in the 9x9 slot with zero fixed rows and columns; the blocks are not masked. */
int32_t rba_get_preconditioner(rba_handle* h, void* inv_out, void* blocks_out);

/* ---- CLUSTER_JACOBI (preconditioner_type = 2, DESIGN.md section 28) ------------------------- */

#define RBA_CLUSTER_MAX_CAMERAS 16     /* 144 rows: a float64 cluster block fits in one CTA's shared memory */
#define RBA_CLUSTER_DEFAULT_CAMERAS 4  /* the cluster size rba_create_* clusters a CLUSTER_JACOBI handle's cameras with: the least slow of 4, 8 and 16 measured (DESIGN.md section 28) */

/* Deterministic single linkage with a size cap over the co-visibility graph; pure host code, no GPU.  The weight of an edge
 * (i, j) is the number of landmarks both cameras observe; the edges are merged in the order (weight descending, i, j) with
 * union-find, and a merge happens only when the joined size is at most max_cluster_size.  cluster_of_camera [Nc] receives
 * dense ids numbered by their smallest camera; a camera without observations is a cluster of its own.
 * RBA_ERR_INVALID_ARGUMENT: max_cluster_size outside [1, RBA_CLUSTER_MAX_CAMERAS], a camera index out of range, a NULL
 * pointer or no camera. */
int32_t rba_cluster_cameras(const rba_problem_view* problem, int32_t max_cluster_size, int32_t* cluster_of_camera);
/* Replaces the clustering of a CLUSTER_JACOBI handle from the next rba_solve on; NULL restores the default one
 * (rba_cluster_cameras with RBA_CLUSTER_DEFAULT_CAMERAS, made by rba_create_*).  Ids outside [0, Nc), ids that are not
 * dense (an unused id below the largest) or a cluster of more than RBA_CLUSTER_MAX_CAMERAS cameras ->
 * RBA_ERR_INVALID_ARGUMENT; another preconditioner_type -> RBA_ERR_STATE.  A rejected or failed call leaves the handle
 * untouched.  On a CLUSTER_JACOBI handle rba_set_intrinsics_groups and rba_set_camera_rigs with a group or rig of >= 2
 * cameras, and rba_set_rig_sensors with a sensor id, return RBA_ERR_UNSUPPORTED and change nothing. */
int32_t rba_set_camera_clusters(rba_handle* h, const int32_t* cluster_of_camera);
/* Reads back the clustering in use (cluster_of_camera [Nc]), the last solve's cluster blocks before their factorisation
 * (blocks: per cluster in id order a full row-major (9k) x (9k) float64 block, its cameras ascending: the Jacobi-scaled,
 * damped reduced camera matrix restricted to the cluster, the camera and pair priors included, the rows and columns of held
 * entries set to the identity) and a status per cluster (0 factorised, 1 a pivot was <= 0 or not finite and the cluster
 * fell back to its cameras' SCHUR_JACOBI blocks).  Any pointer may be NULL.  RBA_ERR_STATE: another preconditioner_type,
 * or blocks / status asked for before a solve with the current clustering. */
int32_t rba_get_cluster_preconditioner(rba_handle* h, int32_t* cluster_of_camera, double* blocks, int32_t* status);
/* LinearizationQR::right_multiply (linearization_qr.hpp:823-825): y = (Q2^T Jp)^T (Q2^T Jp) x + lambda x (+ A^T A x of the
 * camera priors and the pair priors, off-diagonal blocks included: the operator PCG applies) with the damping of the last rba_solve.  A debug accessor of the full operator: it ignores rba_set_camera_fixed. */
int32_t rba_right_multiply(rba_handle* h, const void* x, void* y);
/* LinearizationQR::back_substitute (linearization_qr.hpp:165-179) without the camera update */
int32_t rba_back_substitute_f32(rba_handle* h, const float* pose_inc, float* l_diff_out);
int32_t rba_back_substitute_f64(rba_handle* h, const double* pose_inc, double* l_diff_out);
/* One landmark block in the reference's storage layout, rows x cols row-major with
 * cols = 9n + pad + 4 (landmark_block_dynamic.hpp:56-66): rows 0..2 = Q1^T[Jp|Jl|r] (damped if damping is
 * active), rows 3..2n-1 = Q2^T Jp (Jl and r columns of these rows are reported as 0 / not stored),
 * rows 2n..2n+2 = damping rows.  `lm` is the landmark index in problem order (must be in this shard).
 * RBA_ERR_UNSUPPORTED with operator_form = 1 (no Q2 panels exist in that mode). */
int32_t rba_debug_get_block(rba_handle* h, int32_t lm, void* out, int32_t rows, int32_t cols,
                            void* jl_col_scale3_out);

/* ---- timing hooks for bench.py -------------------------------------------------------------- */

/* Runs `reps` back-to-back rcs_matvec launches (operator only, x = current p buffer) and returns the mean
 * device time per launch in seconds (CUDA events on the solver stream). */
int32_t rba_time_matvec(rba_handle* h, int32_t reps, double* seconds_per_launch);
/* CUDA-event stopwatch on the solver stream: start records an event, stop records a second one,
 * synchronises and returns the device time between them in seconds */
int32_t rba_timer_start(rba_handle* h);
int32_t rba_timer_stop(rba_handle* h, double* seconds);
/* the CUDA stream all work of this handle is enqueued on (as void* = cudaStream_t) */
void* rba_stream(rba_handle* h);
int32_t rba_synchronize(rba_handle* h);

/* ---- multi-GPU (landmarks sharded by index; cameras replicated; SURVEY 8e) ------------------ */

/* 128-byte NCCL unique id (ncclGetUniqueId); call on rank 0, broadcast by the host, pass to every rank */
int32_t rba_nccl_unique_id(void* out128);
/* create the communicator for this handle (opts.rank / opts.nranks); collective across ranks */
int32_t rba_comm_init(rba_handle* h, const void* unique_id128);
/* Optional (same box, NVLink/NVSwitch peers): fuse the per-PCG-iteration all-reduce of the operator output into the PCG
 * vector kernel over peer memory.  Every rank exports 128 bytes (two CUDA IPC handles), the host all-gathers them in
 * rank order and passes the nranks * 128 bytes to every rank.  Without it (or if peer mapping fails) NCCL is used. */
int32_t rba_ipc_export(rba_handle* h, void* out128);
int32_t rba_ipc_import(rba_handle* h, const void* all_handles /* nranks * 128 bytes */);

#ifdef __cplusplus
}
#endif
#endif /* ROOTBA_B200_H_ */
