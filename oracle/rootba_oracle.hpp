// ===========================================================================
// rootba_oracle.hpp -- CPU ORACLE (TEST INFRASTRUCTURE ONLY).
//
// A plain C++17 restatement (no Eigen / TBB / Sophus / basalt) of the
// arithmetic of the reference's square-root BA inner loop.  It exists only as
// the *checker* for the CUDA path (tests/, __graft_entry__.smoke(), and the
// cpu_baseline / --impl reference legs of bench.py).  Nothing under
// rootba_b200/ may include, link or call it.
//
// PARITY STATUS: "parity unpinned".  The reference cannot be built in this
// container (Eigen 3.4.0, TBB, Sophus, basalt-headers, glog, ... are absent and
// every external/ submodule directory is empty) and the reference ships no
// golden vectors for this path (its only fixture, data/rootba/test/*.txt, is an
// empty submodule).  The oracle is pinned only indirectly, by re-running the
// reference's own *property* tests on it (tests/test_oracle_*.py):
//   - analytic Jacobians vs central differences
//       (src/rootba/bal/bal_bundle_adjustment_helper.test.cpp:54-148)
//   - projection value formula (src/rootba/bal/snavely_projection.test.cpp:155-188)
//   - QR == Schur-complement equivalence of b, precond blocks, H*x, l_diff and
//     landmark updates at 1e-5 (f32) / 1e-12 (f64)
//       (src/rootba/qr/linearization_qr.test.cpp:120-222)
//   - implicit matvec vs explicit sparse Q2^T Jp
//       (src/rootba/qr/linearization_qr.test.cpp:63-110)
// and by an independent dense float64 numpy derivation of the whole LM inner step
// from the per-observation Jacobians (tests/test_oracle_dense_numpy.py).
// Third-party arithmetic restated from its published behaviour:
//   Eigen 3.4.0 (makeHouseholder / applyHouseholderOnTheLeft / JacobiRotation /
//   LLT), Sophus@d0b7315a (SO3::exp, SE3), basalt-headers@91293fa4
//   (BalCamera::project).
//
// All "ref:" citations are relative to src/rootba/ of the reference (NikolausDemmel/rootba @ d3900037).
// ===========================================================================
#pragma once

#include <algorithm>
#include <cassert>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <mutex>
#include <string>
#include <functional>
#include <vector>

#ifdef _OPENMP
#include <omp.h>
#endif

namespace orc {

constexpr int POSE_SIZE = 9;        // ref: qr/linearization_qr.hpp:58 (6 pose + 3 intrinsics)
constexpr int CAM_STATE_SIZE = 10;  // ref: bal/bal_problem.hpp:72 (quat xyzw, t, f, k1, k2)

// ref: Sophus Constants<Scalar>::epsilon / epsilonSqrt (SURVEY A10)
template <class S> inline S sophus_epsilon();
template <> inline double sophus_epsilon<double>() { return 1e-10; }
template <> inline float sophus_epsilon<float>() { return 1e-5f; }
template <class S> inline S sophus_epsilon_sqrt() { return std::sqrt(sophus_epsilon<S>()); }

enum RobustNorm { ROBUST_NONE = 0, ROBUST_HUBER = 1 };
enum PreconditionerType { PRECOND_JACOBI = 0, PRECOND_SCHUR_JACOBI = 1 };

// Subset of ref: bal/solver_options.hpp:46-284 that the QR path reads.
struct Options {
  int use_householder = 1;                 // use_householder_marginalization :258
  int use_valid_projections_only = 0;      // optimized_cost==ERROR -> false (:124, solver_options.cpp:41)
  int robust_norm = ROBUST_NONE;           // bal_residual_options.hpp:52
  double huber_parameter = 1.0;            // bal_residual_options.hpp:58
  double jacobi_scaling_epsilon = 0.0;     // :208 ; 0 -> Sophus epsilonSqrt (linearizor_base.cpp:72)
  int preconditioner_type = PRECOND_SCHUR_JACOBI;  // :217
  int min_linear_solver_iterations = 0;    // :180
  int max_linear_solver_iterations = 500;  // :184
  double eta = 0.1;                        // :189
  int staged_execution = 1;                // :262
  int reduction_alg = 1;                   // :266
  int max_num_iterations = 20;             // :141
  double initial_trust_region_radius = 1e4;  // :152
  double min_trust_region_radius = 1e-32;  // :157
  double max_trust_region_radius = 1e16;   // :163
  double min_relative_decrease = 0;        // bal/solver_options.hpp:146-148 (reference default 0; Ceres uses 1e-3)
  double function_tolerance = 1e-6;        // :238
  double initial_vee = 2.0;                // :274
  double vee_factor = 2.0;                 // :278
  int num_threads = 1;                     // :246 (0 = all)
  int optimized_cost = 0;                  // 0 ERROR, 1 ERROR_VALID, 2 ERROR_VALID_AVG (:100-126)
  int verbose = 0;
};

// ref: bal/residual_info.hpp:59-89
struct ResidualItem {
  int num_obs = 0;
  double error = 0;
  double residual_sum = 0;
  double error_avg() const { return num_obs > 0 ? error / num_obs : 0.0; }
};
struct ResidualInfo {
  ResidualItem all, valid;
  bool is_numerically_valid = true;
};

// ---------------------------------------------------------------------------
// small math helpers
// ---------------------------------------------------------------------------
template <class S>
inline void quat_to_rot(const S* q /*x,y,z,w*/, S R[9]) {
  // Eigen::Quaternion::toRotationMatrix
  const S x = q[0], y = q[1], z = q[2], w = q[3];
  const S tx = 2 * x, ty = 2 * y, tz = 2 * z;
  const S twx = tx * w, twy = ty * w, twz = tz * w;
  const S txx = tx * x, txy = ty * x, txz = tz * x;
  const S tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
  R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}

// Sophus SO3::exp (SURVEY A10) -> unit quaternion (x,y,z,w)
template <class S>
inline void so3_exp(const S* omega, S* q) {
  const S theta_sq = omega[0] * omega[0] + omega[1] * omega[1] + omega[2] * omega[2];
  S imag_factor, real_factor;
  if (theta_sq < sophus_epsilon<S>() * sophus_epsilon<S>()) {
    const S theta_po4 = theta_sq * theta_sq;
    imag_factor = S(0.5) - S(1.0 / 48.0) * theta_sq + S(1.0 / 3840.0) * theta_po4;
    real_factor = S(1) - S(1.0 / 8.0) * theta_sq + S(1.0 / 384.0) * theta_po4;
  } else {
    const S theta = std::sqrt(theta_sq);
    const S half_theta = S(0.5) * theta;
    imag_factor = std::sin(half_theta) / theta;
    real_factor = std::cos(half_theta);
  }
  q[0] = imag_factor * omega[0];
  q[1] = imag_factor * omega[1];
  q[2] = imag_factor * omega[2];
  q[3] = real_factor;
}

// Sophus SO3 group product a*b with first-order renormalisation (SURVEY A10)
template <class S>
inline void quat_mul_sophus(const S* a, const S* b, S* out) {
  S r[4];
  r[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  r[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  r[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  r[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  const S sq = r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3];
  if (sq != S(1)) {
    const S scale = S(2) / (S(1) + sq);
    for (int i = 0; i < 4; ++i) r[i] *= scale;
  }
  for (int i = 0; i < 4; ++i) out[i] = r[i];
}

// ref: bal/bal_problem.hpp:97-109  T_c_w <- se3_expd(inc) * T_c_w ; intr += inc
template <class S>
inline void camera_apply_inc(S* cam /*10*/, const S* inc /*9*/) {
  S qe[4];
  so3_exp(inc + 3, qe);
  S Re[9];
  quat_to_rot(qe, Re);
  const S t0 = cam[4], t1 = cam[5], t2 = cam[6];
  S qn[4];
  quat_mul_sophus(qe, cam, qn);
  cam[0] = qn[0]; cam[1] = qn[1]; cam[2] = qn[2]; cam[3] = qn[3];
  cam[4] = Re[0] * t0 + Re[1] * t1 + Re[2] * t2 + inc[0];
  cam[5] = Re[3] * t0 + Re[4] * t1 + Re[5] * t2 + inc[1];
  cam[6] = Re[6] * t0 + Re[7] * t1 + Re[8] * t2 + inc[2];
  cam[7] += inc[6]; cam[8] += inc[7]; cam[9] += inc[8];
}

// basalt::BalCamera::project (SURVEY A9).  p: camera-frame point (3).
template <class S>
inline bool bal_project(const S* p, const S* intr /*f,k1,k2*/, S* proj,
                        S* d_proj_d_p /*2x3 row-major or null*/,
                        S* d_proj_d_i /*2x3 row-major or null*/) {
  const S f = intr[0], k1 = intr[1], k2 = intr[2];
  const S x = p[0], y = p[1], z = p[2];
  const S mx = x / z, my = y / z;
  const S mx2 = mx * mx, my2 = my * my;
  const S r2 = mx2 + my2;
  const S r4 = r2 * r2;
  const S rp = S(1) + k1 * r2 + k2 * r4;
  proj[0] = f * mx * rp;
  proj[1] = f * my * rp;
  if (d_proj_d_p) {
    const S tmp = k1 + k2 * S(2) * r2;
    d_proj_d_p[0] = f * (rp + S(2) * mx2 * tmp) / z;
    d_proj_d_p[4] = f * (rp + S(2) * my2 * tmp) / z;
    d_proj_d_p[1] = d_proj_d_p[3] = S(2) * f * mx * my * tmp / z;
    d_proj_d_p[2] = -f * mx * (rp + S(2) * tmp * r2) / z;
    d_proj_d_p[5] = -f * my * (rp + S(2) * tmp * r2) / z;
  }
  if (d_proj_d_i) {
    d_proj_d_i[0] = mx * rp; d_proj_d_i[1] = f * mx * r2; d_proj_d_i[2] = f * mx * r4;
    d_proj_d_i[3] = my * rp; d_proj_d_i[4] = f * my * r2; d_proj_d_i[5] = f * my * r4;
  }
  return z >= sophus_epsilon_sqrt<S>();
}

// ref: bal/bal_bundle_adjustment_helper.cpp:112-149  linearize_point
// Jp 2x6, Ji 2x3, Jl 2x3 row-major (may be null all together).
template <class S>
inline bool linearize_point(const S* obs, const S* p_w, const S* cam /*10*/,
                            bool ignore_validity_check, S* res, S* Jp, S* Ji, S* Jl) {
  S R[9];
  quat_to_rot(cam, R);
  S pc[3];
  for (int r = 0; r < 3; ++r)
    pc[r] = R[3 * r + 0] * p_w[0] + R[3 * r + 1] * p_w[1] + R[3 * r + 2] * p_w[2] + cam[4 + r];
  S d[6];
  bool valid;
  if (Jp || Ji || Jl) valid = bal_project(pc, cam + 7, res, d, Ji);
  else valid = bal_project<S>(pc, cam + 7, res, nullptr, nullptr);
  res[0] -= obs[0];
  res[1] -= obs[1];
  if (!ignore_validity_check && !valid) return false;
  if (Jp) {
    for (int r = 0; r < 2; ++r) {
      const S d0 = d[3 * r], d1 = d[3 * r + 1], d2 = d[3 * r + 2];
      Jp[6 * r + 0] = d0; Jp[6 * r + 1] = d1; Jp[6 * r + 2] = d2;
      // d * (-hat(pc)); -hat = [[0,pz,-py],[-pz,0,px],[py,-px,0]]
      Jp[6 * r + 3] = -d1 * pc[2] + d2 * pc[1];
      Jp[6 * r + 4] = d0 * pc[2] - d2 * pc[0];
      Jp[6 * r + 5] = -d0 * pc[1] + d1 * pc[0];
    }
  }
  if (Jl) {
    for (int r = 0; r < 2; ++r)
      for (int c = 0; c < 3; ++c)
        Jl[3 * r + c] = d[3 * r] * R[c] + d[3 * r + 1] * R[3 + c] + d[3 * r + 2] * R[6 + c];
  }
  return valid;
}

// ref: bal/bal_bundle_adjustment_helper.cpp:43-66  compute_error_weight
template <class S>
inline void compute_error_weight(int robust_norm, S huber, S res_squared, S& error, S& weight) {
  if (robust_norm == ROBUST_HUBER) {
    const S thresh = huber;
    const S hw = res_squared < thresh * thresh ? S(1.0) : thresh / std::sqrt(res_squared);
    error = S(0.5) * (S(2) - hw) * hw * res_squared;
    weight = hw;
  } else {
    error = S(0.5) * res_squared;
    weight = S(1.0);
  }
}

// Eigen JacobiRotation (SURVEY A8)
template <class S>
struct Givens {
  S c = 1, s = 0;
  void make(S p, S q) {
    if (q == S(0)) { c = p < S(0) ? S(-1) : S(1); s = S(0); }
    else if (p == S(0)) { c = S(0); s = q < S(0) ? S(1) : S(-1); }
    else if (std::abs(p) > std::abs(q)) {
      S t = q / p; S u = std::sqrt(S(1) + t * t); if (p < S(0)) u = -u;
      c = S(1) / u; s = -t * c;
    } else {
      S t = p / q; S u = std::sqrt(S(1) + t * t); if (q < S(0)) u = -u;
      s = -S(1) / u; c = -t * s;
    }
  }
  Givens adjoint() const { Givens g; g.c = c; g.s = -s; return g; }
};
// M.applyOnTheLeft(p, q, j): x=row p, y=row q ; x' = c x + s y ; y' = -s x + c y
template <class S>
inline void apply_givens_rows(S* xrow, S* yrow, int ncols, const Givens<S>& j) {
  if (j.c == S(1) && j.s == S(0)) return;
  for (int i = 0; i < ncols; ++i) {
    const S xi = xrow[i], yi = yrow[i];
    xrow[i] = j.c * xi + j.s * yi;
    yrow[i] = -j.s * xi + j.c * yi;
  }
}

// ---------------------------------------------------------------------------
// Landmark block (ref: qr/impl/landmark_block_base.ipp, qr/landmark_block_dynamic.hpp)
// ---------------------------------------------------------------------------
template <class S>
struct LandmarkBlock {
  enum State { ALLOCATED, NUMERICAL_FAILURE, LINEARIZED, MARGINALIZED };
  int n = 0;                 // number of observations
  std::vector<int> pose_idx; // camera indices, ascending (std::map order)
  int64_t obs_begin = 0;     // first observation (global obs array)
  int lm_id = 0;
  int padding_idx = 0, padding_size = 0, lm_idx = 0, res_idx = 0, num_cols = 0, num_rows = 0;
  std::vector<S> storage;    // row-major num_rows x num_cols
  std::vector<Givens<S>> damping_rotations;
  S Jl_col_scale[3] = {1, 1, 1};
  State state = ALLOCATED;

  S& at(int r, int c) { return storage[(size_t)r * num_cols + c]; }
  const S& at(int r, int c) const { return storage[(size_t)r * num_cols + c]; }
  S* row(int r) { return storage.data() + (size_t)r * num_cols; }
  const S* row(int r) const { return storage.data() + (size_t)r * num_cols; }
  int num_Q2T_rows() const { return num_rows - 3; }  // ipp:292-296
  bool has_landmark_damping() const { return !damping_rotations.empty(); }

  // ref: qr/landmark_block_dynamic.hpp:49-69
  void allocate(int lm, int64_t obs0, const int* cams, int n_obs) {
    lm_id = lm; obs_begin = obs0; n = n_obs;
    pose_idx.assign(cams, cams + n_obs);
    padding_idx = n * POSE_SIZE;
    num_rows = n * 2 + 3;
    padding_size = 0;
    int pad = padding_idx % 4;
    if (pad != 0) padding_size = 4 - pad;
    lm_idx = padding_idx + padding_size;
    res_idx = lm_idx + 3;
    num_cols = res_idx + 1;
    storage.assign((size_t)num_rows * num_cols, S(0));
    damping_rotations.clear();
    state = ALLOCATED;
  }
};

// ---------------------------------------------------------------------------
// Problem + LinearizationQR + LinearizorQR (+ SC cross-check) in one object
// ---------------------------------------------------------------------------
template <class S>
struct Problem {
  // --- BalProblem state (ref: bal/bal_problem.hpp:61-234), SoA ---
  int nc = 0, nl = 0;
  int64_t nobs = 0;
  std::vector<S> cams;      // 10 * nc
  std::vector<S> lms;       // 3 * nl
  std::vector<int64_t> lm_off;  // nl + 1
  std::vector<int> obs_cam;     // nobs, ascending per landmark
  std::vector<S> obs_xy;        // 2 * nobs
  std::vector<S> cams_backup, lms_backup;

  Options opt;

  // --- LinearizationQR (ref: qr/linearization_qr.hpp:80-111, 828-840) ---
  std::vector<LandmarkBlock<S>> blocks;
  std::vector<int64_t> landmark_block_idx;  // prefix sum of num_Q2T_rows
  int64_t num_rows_Q2Tr = 0;
  S pose_damping_diagonal = 0, pose_damping_diagonal_sqrt = 0;
  std::vector<std::mutex> pose_mutex;

  // --- LinearizorQR state (ref: solver/linearizor_qr.hpp:73-84) ---
  std::vector<S> pose_jacobian_scaling;  // 9 * nc
  std::vector<S> precond_blocks;         // 81 * nc row-major 9x9 (IndexedBlocks)
  bool new_linearization_point = false;

  // timings / stats of the last calls (seconds)
  double t_stage1 = 0, t_stage2 = 0, t_precond = 0, t_pcg = 0, t_backsub = 0, t_update = 0, t_error = 0;
  int last_cg_iterations = 0;
  int last_cg_termination = 0;  // 0 no convergence, 1 success, 2 failure
  int64_t total_matvecs = 0;

  S jacobi_eps() const {  // ref: solver/linearizor_base.cpp:72-79
    return opt.jacobi_scaling_epsilon > 0 ? S(opt.jacobi_scaling_epsilon) : sophus_epsilon_sqrt<S>();
  }
  int threads() const {
#ifdef _OPENMP
    return opt.num_threads > 0 ? opt.num_threads : omp_get_max_threads();
#else
    return 1;
#endif
  }

  void init(int nc_, int nl_, const int64_t* off, const int* oc, const S* oxy, const S* c, const S* l) {
    nc = nc_; nl = nl_; nobs = off[nl_];
    lm_off.assign(off, off + nl + 1);
    obs_cam.assign(oc, oc + nobs);
    obs_xy.assign(oxy, oxy + 2 * nobs);
    cams.assign(c, c + (size_t)CAM_STATE_SIZE * nc);
    lms.assign(l, l + (size_t)3 * nl);
    cams_backup = cams; lms_backup = lms;
    allocate_blocks();
  }

  // ref: qr/linearization_qr.hpp:80-111
  void allocate_blocks() {
    blocks.resize(nl);
    landmark_block_idx.resize(nl);
    num_rows_Q2Tr = 0;
    for (int i = 0; i < nl; ++i) {
      const int n = (int)(lm_off[i + 1] - lm_off[i]);
      assert(n >= 2);  // ref: ipp:73-76 / qr/landmark_block.cpp:54
      blocks[i].allocate(i, lm_off[i], obs_cam.data() + lm_off[i], n);
      landmark_block_idx[i] = num_rows_Q2Tr;
      num_rows_Q2Tr += blocks[i].num_Q2T_rows();
    }
    std::vector<std::mutex>(nc).swap(pose_mutex);
    pose_jacobian_scaling.assign((size_t)POSE_SIZE * nc, S(1));
    precond_blocks.assign((size_t)81 * nc, S(0));
  }

  void backup() { cams_backup = cams; lms_backup = lms; }   // ref: bal/bal_problem.cpp:590-598
  void restore() { cams = cams_backup; lms = lms_backup; }  // ref: bal/bal_problem.cpp:600-608

  // ---------------- per-landmark operations (ref: ipp) ----------------

  // ref: ipp:88-147
  void linearize_landmark(LandmarkBlock<S>& lb) const {
    std::fill(lb.storage.begin(), lb.storage.end(), S(0));
    lb.damping_rotations.clear();
    bool numerically_valid = true;
    const S* p_w = lms.data() + 3 * (size_t)lb.lm_id;
    for (int i = 0; i < lb.n; ++i) {
      const int cam_idx = lb.pose_idx[i];
      const int obs_idx = i * 2;
      const int pose_col = i * POSE_SIZE;
      const S* obs = obs_xy.data() + 2 * (lb.obs_begin + i);
      S Jp[12], Ji[6], Jl[6], res[2];
      const bool valid = linearize_point(obs, p_w, cams.data() + (size_t)CAM_STATE_SIZE * cam_idx,
                                         true, res, Jp, Ji, Jl);
      if (!opt.use_valid_projections_only || valid) {
        bool fin = true;
        for (int k = 0; k < 12; ++k) fin = fin && std::isfinite(Jp[k]);
        for (int k = 0; k < 6; ++k) fin = fin && std::isfinite(Ji[k]) && std::isfinite(Jl[k]);
        fin = fin && std::isfinite(res[0]) && std::isfinite(res[1]);
        numerically_valid = numerically_valid && fin;
        const S res_squared = res[0] * res[0] + res[1] * res[1];
        S werr, weight;
        compute_error_weight<S>(opt.robust_norm, S(opt.huber_parameter), res_squared, werr, weight);
        const S sw = std::sqrt(weight);
        for (int r = 0; r < 2; ++r) {
          S* row = lb.row(obs_idx + r);
          for (int c = 0; c < 6; ++c) row[pose_col + c] = sw * Jp[6 * r + c];
          for (int c = 0; c < 3; ++c) row[pose_col + 6 + c] = sw * Ji[3 * r + c];
          for (int c = 0; c < 3; ++c) row[lb.lm_idx + c] = sw * Jl[3 * r + c];
          row[lb.res_idx] = sw * res[r];
        }
      }
    }
    lb.state = numerically_valid ? LandmarkBlock<S>::LINEARIZED : LandmarkBlock<S>::NUMERICAL_FAILURE;
  }

  // ref: ipp:493-518 (column squared norms over rows 0..2n-1, scatter by camera)
  static void add_Jp_diag2(const LandmarkBlock<S>& lb, S* res) {
    const int nr = lb.num_rows - 3;
    for (int i = 0; i < lb.n; ++i) {
      const int cam = lb.pose_idx[i];
      for (int c = 0; c < POSE_SIZE; ++c) {
        S acc = 0;
        for (int r = 0; r < nr; ++r) { const S v = lb.at(r, i * POSE_SIZE + c); acc += v * v; }
        res[(size_t)POSE_SIZE * cam + c] += acc;
      }
    }
  }

  // ref: ipp:554-569 (JACOBI: Jp_i^T Jp_i of the 2x9 block)
  static void add_Jp_T_Jp_blockdiag(const LandmarkBlock<S>& lb, S* blocks81) {
    for (int i = 0; i < lb.n; ++i) {
      const int cam = lb.pose_idx[i];
      S* B = blocks81 + (size_t)81 * cam;
      for (int a = 0; a < 9; ++a)
        for (int b = 0; b < 9; ++b)
          B[9 * a + b] += lb.at(2 * i, 9 * i + a) * lb.at(2 * i, 9 * i + b) +
                          lb.at(2 * i + 1, 9 * i + a) * lb.at(2 * i + 1, 9 * i + b);
    }
  }

  // ref: ipp:571-587
  void scale_Jl_cols(LandmarkBlock<S>& lb) const {
    const int nr = lb.num_rows - 3;
    for (int j = 0; j < 3; ++j) {
      S sq = 0;
      for (int r = 0; r < nr; ++r) { const S v = lb.at(r, lb.lm_idx + j); sq += v * v; }
      lb.Jl_col_scale[j] = S(1) / (jacobi_eps() + std::sqrt(sq));
    }
    for (int r = 0; r < nr; ++r)
      for (int j = 0; j < 3; ++j) lb.at(r, lb.lm_idx + j) *= lb.Jl_col_scale[j];
  }

  // ref: ipp:717-743 + Eigen makeHouseholder / applyHouseholderOnTheLeft (SURVEY A7)
  static void perform_qr_householder(LandmarkBlock<S>& lb) {
    const int num_cols = lb.num_cols, num_rows = lb.num_rows, lm_idx = lb.lm_idx;
    std::vector<S> essential(num_rows), tmp(num_cols);
    for (int k = 0; k < 3; ++k) {
      const int rem = num_rows - k - 3;
      // makeHouseholder on storage.col(lm_idx+k).segment(k, rem)
      S tailSq = 0;
      for (int r = 1; r < rem; ++r) { const S v = lb.at(k + r, lm_idx + k); tailSq += v * v; }
      const S c0 = lb.at(k, lm_idx + k);
      S tau, beta;
      if (tailSq <= std::numeric_limits<S>::min()) {
        tau = 0; beta = c0;
        for (int r = 1; r < rem; ++r) essential[r - 1] = 0;
      } else {
        beta = std::sqrt(c0 * c0 + tailSq);
        if (c0 >= S(0)) beta = -beta;
        for (int r = 1; r < rem; ++r) essential[r - 1] = lb.at(k + r, lm_idx + k) / (c0 - beta);
        tau = (beta - c0) / beta;
      }
      // applyHouseholderOnTheLeft on block(k, 0, rem, num_cols)
      if (rem == 1) {
        for (int c = 0; c < num_cols; ++c) lb.at(k, c) *= (S(1) - tau);
      } else if (tau != S(0)) {
        for (int c = 0; c < num_cols; ++c) {
          S t = 0;
          for (int r = 1; r < rem; ++r) t += essential[r - 1] * lb.at(k + r, c);
          tmp[c] = t + lb.at(k, c);
        }
        for (int c = 0; c < num_cols; ++c) lb.at(k, c) -= tau * tmp[c];
        for (int r = 1; r < rem; ++r) {
          const S te = tau * essential[r - 1];
          S* rowp = lb.row(k + r);
          for (int c = 0; c < num_cols; ++c) rowp[c] -= te * tmp[c];
        }
      }
    }
  }

  // ref: ipp:700-715
  static void perform_qr_givens(LandmarkBlock<S>& lb) {
    Givens<S> gr;
    for (int n = 0; n < 3; ++n) {
      for (int m = lb.num_rows - 4; m > n; --m) {
        gr.make(lb.at(m - 1, lb.lm_idx + n), lb.at(m, lb.lm_idx + n));
        apply_givens_rows(lb.row(m), lb.row(m - 1), lb.num_cols, gr);
      }
    }
  }

  // ref: ipp:149-163
  void perform_qr(LandmarkBlock<S>& lb) const {
    if (opt.use_householder) perform_qr_householder(lb);
    else perform_qr_givens(lb);
    lb.state = LandmarkBlock<S>::MARGINALIZED;
  }

  // ref: ipp:165-210
  static void set_landmark_damping(LandmarkBlock<S>& lb, S lambda) {
    const int lm_idx = lb.lm_idx, num_rows = lb.num_rows;
    if (lb.has_landmark_damping()) {
      for (int n = 2; n >= 0; --n)
        for (int m = n; m >= 0; --m) {
          apply_givens_rows(lb.row(num_rows - 3 + n - m), lb.row(n), lb.num_cols,
                            lb.damping_rotations.back().adjoint());
          lb.damping_rotations.pop_back();
        }
    }
    if (lambda == S(0)) {
      for (int d = 0; d < 3; ++d) lb.at(num_rows - 3 + d, lm_idx + d) = 0;
    } else {
      const S sl = std::sqrt(lambda);
      for (int d = 0; d < 3; ++d) lb.at(num_rows - 3 + d, lm_idx + d) = sl;
      for (int n = 0; n < 3; ++n)
        for (int m = 0; m <= n; ++m) {
          Givens<S> g;
          g.make(lb.at(n, lm_idx + n), lb.at(num_rows - 3 + n - m, lm_idx + n));
          lb.damping_rotations.push_back(g);
          apply_givens_rows(lb.row(num_rows - 3 + n - m), lb.row(n), lb.num_cols, g);
        }
    }
  }

  // ref: ipp:589-614
  static void scale_Jp_cols(LandmarkBlock<S>& lb, const S* jacobian_scaling) {
    const int nr = lb.num_rows - 3;
    for (int r = 0; r < nr; ++r) {
      S* rowp = lb.row(r);
      for (int i = 0; i < lb.n; ++i) {
        const S* sc = jacobian_scaling + (size_t)POSE_SIZE * lb.pose_idx[i];
        for (int c = 0; c < POSE_SIZE; ++c) rowp[i * POSE_SIZE + c] *= sc[c];
      }
      for (int c = 0; c < lb.padding_size; ++c) rowp[lb.padding_idx + c] *= S(0);
    }
  }

  // ref: ipp:520-552  (SCHUR_JACOBI block: B^T B over rows 3..num_rows-1)
  static void add_Q2TJp_T_Q2TJp_blockdiag(const LandmarkBlock<S>& lb, S* blocks81,
                                          std::vector<std::mutex>* mtx) {
    for (int i = 0; i < lb.n; ++i) {
      S tmp[81];
      for (int a = 0; a < 9; ++a)
        for (int b = 0; b < 9; ++b) {
          S acc = 0;
          for (int r = 3; r < lb.num_rows; ++r) acc += lb.at(r, 9 * i + a) * lb.at(r, 9 * i + b);
          tmp[9 * a + b] = acc;
        }
      const int cam = lb.pose_idx[i];
      S* B = blocks81 + (size_t)81 * cam;
      if (mtx) { std::scoped_lock lock((*mtx)[cam]); for (int k = 0; k < 81; ++k) B[k] += tmp[k]; }
      else for (int k = 0; k < 81; ++k) B[k] += tmp[k];
    }
  }

  // ref: ipp:443-466
  static void add_Q2TJp_T_Q2Tr(const LandmarkBlock<S>& lb, S* res, std::vector<std::mutex>* mtx) {
    const int ncol = lb.padding_idx;
    std::vector<S> xr(ncol, S(0));
    for (int r = 3; r < lb.num_rows; ++r) {
      const S rr = lb.at(r, lb.res_idx);
      const S* rowp = lb.row(r);
      for (int c = 0; c < ncol; ++c) xr[c] += rowp[c] * rr;
    }
    for (int i = 0; i < lb.n; ++i) {
      const int cam = lb.pose_idx[i];
      if (mtx) { std::scoped_lock lock((*mtx)[cam]); for (int c = 0; c < 9; ++c) res[(size_t)9 * cam + c] += xr[9 * i + c]; }
      else for (int c = 0; c < 9; ++c) res[(size_t)9 * cam + c] += xr[9 * i + c];
    }
  }

  // ref: ipp:400-441
  static void add_Q2TJp_T_Q2TJp_mult_x(const LandmarkBlock<S>& lb, S* res, const S* x_pose,
                                       std::vector<std::mutex>* mtx) {
    const int ncol = lb.padding_idx;
    S xr_stack[9 * 16];
    std::vector<S> xr_heap;
    S* xr = xr_stack;
    if (ncol > 9 * 16) { xr_heap.resize(ncol); xr = xr_heap.data(); }
    for (int i = 0; i < lb.n; ++i)
      for (int c = 0; c < 9; ++c) xr[9 * i + c] = x_pose[(size_t)9 * lb.pose_idx[i] + c];
    const int nr = lb.num_rows - 3;
    S tmp_stack[2 * 16];
    std::vector<S> tmp_heap;
    S* tmp = tmp_stack;
    if (nr > 32) { tmp_heap.resize(nr); tmp = tmp_heap.data(); }
    for (int r = 0; r < nr; ++r) {
      const S* rowp = lb.row(3 + r);
      S acc = 0;
      for (int c = 0; c < ncol; ++c) acc += rowp[c] * xr[c];
      tmp[r] = acc;
    }
    for (int c = 0; c < ncol; ++c) xr[c] = 0;
    for (int r = 0; r < nr; ++r) {
      const S* rowp = lb.row(3 + r);
      const S t = tmp[r];
      for (int c = 0; c < ncol; ++c) xr[c] += rowp[c] * t;
    }
    for (int i = 0; i < lb.n; ++i) {
      const int cam = lb.pose_idx[i];
      if (mtx) { std::scoped_lock lock((*mtx)[cam]); for (int c = 0; c < 9; ++c) res[(size_t)9 * cam + c] += xr[9 * i + c]; }
      else for (int c = 0; c < 9; ++c) res[(size_t)9 * cam + c] += xr[9 * i + c];
    }
  }

  // ref: ipp:212-284
  void back_substitute_block(LandmarkBlock<S>& lb, const S* pose_inc, S& l_diff, bool& fail) {
    const int ncol = lb.padding_idx, lm_idx = lb.lm_idx, res_idx = lb.res_idx, num_rows = lb.num_rows;
    std::vector<S> pr(ncol);
    for (int i = 0; i < lb.n; ++i)
      for (int c = 0; c < 9; ++c) pr[9 * i + c] = pose_inc[(size_t)9 * lb.pose_idx[i] + c];
    // rhs = Q1T_r + Q1T_Jp * pose_inc_reduced
    S rhs[3];
    for (int r = 0; r < 3; ++r) {
      S acc = 0;
      const S* rowp = lb.row(r);
      for (int c = 0; c < ncol; ++c) acc += rowp[c] * pr[c];
      rhs[r] = lb.at(r, res_idx) + acc;
    }
    // upper-triangular solve (Eigen triangularView<Upper>().solve)
    S sol[3];
    for (int r = 2; r >= 0; --r) {
      S acc = rhs[r];
      for (int c = r + 1; c < 3; ++c) acc -= lb.at(r, lm_idx + c) * sol[c];
      sol[r] = acc / lb.at(r, lm_idx + r);
    }
    S inc[3] = {-sol[0], -sol[1], -sol[2]};
    set_landmark_damping(lb, S(0));
    const int nr = num_rows - 3;
    std::vector<S> v(nr);
    for (int r = 0; r < nr; ++r) {
      S acc = 0;
      const S* rowp = lb.row(r);
      for (int c = 0; c < ncol; ++c) acc += rowp[c] * pr[c];
      v[r] = acc;
    }
    for (int r = 0; r < 3; ++r) {
      S acc = 0;
      for (int c = r; c < 3; ++c) acc += lb.at(r, lm_idx + c) * inc[c];
      v[r] += acc;
    }
    S acc = 0;
    for (int r = 0; r < nr; ++r) acc += v[r] * (S(0.5) * v[r] + lb.at(r, res_idx));
    l_diff -= acc;
    S* p_w = lms.data() + 3 * (size_t)lb.lm_id;
    if (!(std::isfinite(inc[0]) && std::isfinite(inc[1]) && std::isfinite(inc[2])) ||
        !(std::isfinite(p_w[0]) && std::isfinite(p_w[1]) && std::isfinite(p_w[2])))
      fail = true;  // reference: LOG(FATAL) ipp:266-279
    for (int d = 0; d < 3; ++d) p_w[d] += inc[d] * lb.Jl_col_scale[d];
  }

  // ---------------- LinearizationQR container ops ----------------

  void set_pose_damping(S lambda) {  // ref: qr/linearization_qr.hpp:138-143
    pose_damping_diagonal = lambda;
    pose_damping_diagonal_sqrt = std::sqrt(lambda);
  }
  bool has_pose_damping() const { return pose_damping_diagonal > 0; }

  // ref: qr/linearization_qr.hpp:634-712 ; returns false on numerical failure
  bool get_stage1(std::vector<S>& diag2, bool jacobi_blocks) {
    diag2.assign((size_t)9 * nc, S(0));
    if (jacobi_blocks) precond_blocks.assign((size_t)81 * nc, S(0));
    bool valid = true;
    const int T = threads();
    std::vector<std::vector<S>> d2(T), pb(T);
#pragma omp parallel num_threads(T)
    {
#ifdef _OPENMP
      const int tid = omp_get_thread_num();
#else
      const int tid = 0;
#endif
      d2[tid].assign((size_t)9 * nc, S(0));
      if (jacobi_blocks) pb[tid].assign((size_t)81 * nc, S(0));
      bool lvalid = true;
#pragma omp for schedule(dynamic, 256)
      for (int r = 0; r < nl; ++r) {
        auto& lb = blocks[r];
        linearize_landmark(lb);
        if (lb.state != LandmarkBlock<S>::NUMERICAL_FAILURE) {
          if (jacobi_blocks) add_Jp_T_Jp_blockdiag(lb, pb[tid].data());
          add_Jp_diag2(lb, d2[tid].data());
          scale_Jl_cols(lb);
          perform_qr(lb);
        } else {
          lvalid = false;
        }
      }
#pragma omp critical
      { valid = valid && lvalid; }
    }
    for (int t = 0; t < T; ++t) {
      for (size_t k = 0; k < diag2.size(); ++k) diag2[k] += d2[t][k];
      if (jacobi_blocks) for (size_t k = 0; k < precond_blocks.size(); ++k) precond_blocks[k] += pb[t][k];
    }
    return valid;
  }

  // ref: qr/linearization_qr.hpp:716-815 (stage2 per landmark: ipp:638-658)
  void get_stage2(S lambda, const S* jacobian_scaling, bool schur_jacobi_blocks, std::vector<S>& b) {
    b.assign((size_t)9 * nc, S(0));
    if (schur_jacobi_blocks) precond_blocks.assign((size_t)81 * nc, S(0));
    const int T = threads();
    std::vector<std::mutex>* mtx = T > 1 ? &pose_mutex : nullptr;
#pragma omp parallel for schedule(dynamic, 256) num_threads(T)
    for (int r = 0; r < nl; ++r) {
      auto& lb = blocks[r];
      if (jacobian_scaling) scale_Jp_cols(lb, jacobian_scaling);
      set_landmark_damping(lb, lambda);
      if (schur_jacobi_blocks) add_Q2TJp_T_Q2TJp_blockdiag(lb, precond_blocks.data(), mtx);
      add_Q2TJp_T_Q2Tr(lb, b.data(), mtx);
    }
    if (has_pose_damping() && schur_jacobi_blocks) {  // :796-802
      for (int c = 0; c < nc; ++c)
        for (int d = 0; d < 9; ++d) precond_blocks[(size_t)81 * c + 10 * d] += pose_damping_diagonal;
    }
  }

  // ref: qr/linearization_qr.hpp:406-429 (v3, per-camera mutex) / :294-334 (v0)
  void right_multiply(const S* x, S* y) {
    ++total_matvecs;
    const size_t N = (size_t)9 * nc;
    std::fill(y, y + N, S(0));
    const int T = threads();
    if (T == 1) {
      for (int r = 0; r < nl; ++r) add_Q2TJp_T_Q2TJp_mult_x(blocks[r], y, x, nullptr);
    } else if (opt.reduction_alg == 0) {
      std::vector<std::vector<S>> part(T);
#pragma omp parallel num_threads(T)
      {
#ifdef _OPENMP
        const int tid = omp_get_thread_num();
#else
        const int tid = 0;
#endif
        part[tid].assign(N, S(0));
#pragma omp for schedule(dynamic, 256)
        for (int r = 0; r < nl; ++r) add_Q2TJp_T_Q2TJp_mult_x(blocks[r], part[tid].data(), x, nullptr);
      }
      for (int t = 0; t < T; ++t) for (size_t k = 0; k < N; ++k) y[k] += part[t][k];
    } else {
#pragma omp parallel for schedule(dynamic, 256) num_threads(T)
      for (int r = 0; r < nl; ++r) add_Q2TJp_T_Q2TJp_mult_x(blocks[r], y, x, &pose_mutex);
    }
    if (has_pose_damping()) for (size_t k = 0; k < N; ++k) y[k] += x[k] * pose_damping_diagonal;
  }

  // ref: qr/linearization_qr.hpp:165-179
  S back_substitute(const S* pose_inc, bool& fail) {
    fail = false;
    const int T = threads();
    S total = 0;
    bool anyfail = false;
#pragma omp parallel num_threads(T)
    {
      S l = 0; bool f = false;
#pragma omp for schedule(dynamic, 256)
      for (int r = 0; r < nl; ++r) back_substitute_block(blocks[r], pose_inc, l, f);
#pragma omp critical
      { total += l; anyfail = anyfail || f; }
    }
    fail = anyfail;
    return total;
  }

  // ---------------- compute_error (ref: bal/bal_bundle_adjustment_helper.cpp:68-109) ----------------
  void compute_error(ResidualInfo& out) {
    auto t0 = std::chrono::high_resolution_clock::now();
    const bool ignore_validity_check = !opt.use_valid_projections_only;
    const int T = threads();
    ResidualInfo total;
#pragma omp parallel num_threads(T)
    {
      ResidualInfo acc;
#pragma omp for schedule(dynamic, 1024)
      for (int l = 0; l < nl; ++l) {
        for (int64_t o = lm_off[l]; o < lm_off[l + 1]; ++o) {
          S res[2];
          const bool pv = linearize_point<S>(obs_xy.data() + 2 * o, lms.data() + 3 * (size_t)l,
                                             cams.data() + (size_t)10 * obs_cam[o], ignore_validity_check,
                                             res, nullptr, nullptr, nullptr);
          const bool nv = std::isfinite(res[0]) && std::isfinite(res[1]);
          const S rsq = res[0] * res[0] + res[1] * res[1];
          S werr, w;
          compute_error_weight<S>(opt.robust_norm, S(opt.huber_parameter), rsq, werr, w);
          // ref: bal/residual_info.cpp:97-110 (accumulation in double)
          acc.is_numerically_valid = acc.is_numerically_valid && nv;
          ++acc.all.num_obs; acc.all.error += (double)werr; acc.all.residual_sum += (double)std::sqrt(rsq);
          if (pv) { ++acc.valid.num_obs; acc.valid.error += (double)werr; acc.valid.residual_sum += (double)std::sqrt(rsq); }
        }
      }
#pragma omp critical
      {
        total.all.num_obs += acc.all.num_obs; total.all.error += acc.all.error; total.all.residual_sum += acc.all.residual_sum;
        total.valid.num_obs += acc.valid.num_obs; total.valid.error += acc.valid.error; total.valid.residual_sum += acc.valid.residual_sum;
        total.is_numerically_valid = total.is_numerically_valid && acc.is_numerically_valid;
      }
    }
    out = total;
    t_error = std::chrono::duration<double>(std::chrono::high_resolution_clock::now() - t0).count();
  }

  // ---------------- BlockDiagonalPreconditioner (ref: cg/preconditioner.hpp:79-136) ----------------
  // inverse of (block + diag) via Cholesky of the upper triangle; returns false if not SPD
  static bool invert_block9(const S* in81, const S* diag9, S* out81) {
    S A[81];
    for (int r = 0; r < 9; ++r) for (int c = 0; c < 9; ++c) A[9 * r + c] = (c >= r) ? in81[9 * r + c] : in81[9 * c + r];
    if (diag9) for (int d = 0; d < 9; ++d) A[10 * d] += diag9[d];
    S L[81];
    std::fill(L, L + 81, S(0));
    bool ok = true;
    for (int j = 0; j < 9; ++j) {
      S s = A[10 * j];
      for (int k = 0; k < j; ++k) s -= L[9 * j + k] * L[9 * j + k];
      if (!(s > S(0))) ok = false;
      const S d = std::sqrt(s);
      L[10 * j] = d;
      for (int i = j + 1; i < 9; ++i) {
        S t = A[9 * j + i];
        for (int k = 0; k < j; ++k) t -= L[9 * i + k] * L[9 * j + k];
        L[9 * i + j] = t / d;
      }
    }
    for (int col = 0; col < 9; ++col) {
      S y[9];
      for (int i = 0; i < 9; ++i) {
        S t = (i == col) ? S(1) : S(0);
        for (int k = 0; k < i; ++k) t -= L[9 * i + k] * y[k];
        y[i] = t / L[10 * i];
      }
      for (int i = 8; i >= 0; --i) {
        S t = y[i];
        for (int k = i + 1; k < 9; ++k) t -= L[9 * k + i] * out81[9 * k + col];
        out81[9 * i + col] = t / L[10 * i];
      }
    }
    return ok;
  }

  // ---------------- LinearizorQR (ref: solver/linearizor_qr.cpp) ----------------

  // ref: solver/linearizor_qr.cpp:78-138 ; returns false on numerical failure (reference CHECK-aborts)
  bool linearize() {
    auto t0 = std::chrono::high_resolution_clock::now();
    const bool use_jacobi = opt.preconditioner_type == PRECOND_JACOBI;
    std::vector<S> scale2;
    bool ok;
    if (!opt.staged_execution) {
      // ref: :94-112 (four separate passes)
      ok = true;
      for (int r = 0; r < nl; ++r) { linearize_landmark(blocks[r]); ok = ok && blocks[r].state != LandmarkBlock<S>::NUMERICAL_FAILURE; }
      scale2.assign((size_t)9 * nc, S(0));
      if (ok) {
        for (int r = 0; r < nl; ++r) add_Jp_diag2(blocks[r], scale2.data());
        for (int r = 0; r < nl; ++r) scale_Jl_cols(blocks[r]);
        if (use_jacobi) { precond_blocks.assign((size_t)81 * nc, S(0)); for (int r = 0; r < nl; ++r) add_Jp_T_Jp_blockdiag(blocks[r], precond_blocks.data()); }
        for (int r = 0; r < nl; ++r) perform_qr(blocks[r]);
      }
    } else {
      ok = get_stage1(scale2, use_jacobi);
    }
    if (!ok) return false;
    const S eps = jacobi_eps();
    for (size_t k = 0; k < scale2.size(); ++k) pose_jacobian_scaling[k] = S(1) / (eps + std::sqrt(scale2[k]));
    new_linearization_point = true;
    t_stage1 = std::chrono::duration<double>(std::chrono::high_resolution_clock::now() - t0).count();
    return true;
  }

  // ref: cg/conjugate_gradient.hpp:113-298 driven by solver/linearizor_base.cpp:81-103
  // returns iterations ; termination in last_cg_termination
  std::function<void(const S*, S*)> op_override;  // Schur-complement solvers: H x through the SC landmark blocks
  int pcg(const std::vector<S>& bref, const std::vector<S>& inv_blocks, std::vector<S>& xref) {
    auto right_multiply = [&](const S* xin, S* yout) { if (op_override) op_override(xin, yout); else this->right_multiply(xin, yout); };
    const size_t N = (size_t)9 * nc;
    int num_iterations = 0;
    last_cg_termination = 0;
    auto dot = [&](const std::vector<S>& a, const std::vector<S>& b) { S s = 0; for (size_t k = 0; k < N; ++k) s += a[k] * b[k]; return s; };
    auto is_zero_or_infinity = [](double x) { return x == 0.0 || std::isinf(x); };
    const double norm_b = (double)std::sqrt(dot(bref, bref));
    if (norm_b == 0.0) { std::fill(xref.begin(), xref.end(), S(0)); last_cg_termination = 1; return 0; }
    std::vector<S> r(N), p(N), z(N), tmp(N), q(N);
    const double tol_r = -1.0 * norm_b;  // r_tolerance = -1 (linearizor_base.cpp:92)
    right_multiply(xref.data(), tmp.data());
    for (size_t k = 0; k < N; ++k) r[k] = bref[k] - tmp[k];
    double norm_r = (double)std::sqrt(dot(r, r));
    if (opt.min_linear_solver_iterations == 0 && norm_r <= tol_r) { last_cg_termination = 1; return 0; }
    double rho = 1.0;
    auto xdot_b_plus_r = [&]() { S s = 0; for (size_t k = 0; k < N; ++k) s += xref[k] * (bref[k] + r[k]); return s; };
    double q0 = -1.0 * (double)xdot_b_plus_r();
    for (num_iterations = 1;; ++num_iterations) {
      // solve_assign: 9x9 block gemv per camera (cg/preconditioner.hpp:122-136)
      for (int c = 0; c < nc; ++c) {
        const S* B = inv_blocks.data() + (size_t)81 * c;
        for (int i = 0; i < 9; ++i) {
          S acc = 0;
          for (int j = 0; j < 9; ++j) acc += B[9 * i + j] * r[(size_t)9 * c + j];
          z[(size_t)9 * c + i] = acc;
        }
      }
      const double last_rho = rho;
      rho = (double)dot(r, z);
      if (is_zero_or_infinity(rho)) { last_cg_termination = 2; break; }
      if (num_iterations == 1) {
        p = z;
      } else {
        const double beta = rho / last_rho;
        if (is_zero_or_infinity(beta)) { last_cg_termination = 2; break; }
        const S bs = (S)beta;
        for (size_t k = 0; k < N; ++k) p[k] = z[k] + bs * p[k];
      }
      right_multiply(p.data(), q.data());
      const double pq = (double)dot(p, q);
      if ((pq <= 0) || std::isinf(pq)) { last_cg_termination = 0; break; }
      const double alpha = rho / pq;
      if (std::isinf(alpha)) { last_cg_termination = 2; break; }
      const S as = (S)alpha;
      for (size_t k = 0; k < N; ++k) xref[k] = xref[k] + as * p[k];
      if (num_iterations % 10 == 0) {  // residual_reset_period = 10 (:87)
        right_multiply(xref.data(), tmp.data());
        for (size_t k = 0; k < N; ++k) r[k] = bref[k] - tmp[k];
      } else {
        for (size_t k = 0; k < N; ++k) r[k] = r[k] - as * q[k];
      }
      const double q1 = -1.0 * (double)xdot_b_plus_r();
      const double zeta = num_iterations * (q1 - q0) / q1;
      if (zeta < opt.eta && num_iterations >= opt.min_linear_solver_iterations) { last_cg_termination = 1; break; }
      q0 = q1;
      norm_r = (double)std::sqrt(dot(r, r));
      if (norm_r <= tol_r && num_iterations >= opt.min_linear_solver_iterations) { last_cg_termination = 1; break; }
      if (num_iterations >= opt.max_linear_solver_iterations) break;
    }
    for (size_t k = 0; k < N; ++k) xref[k] = -xref[k];  // linearizor_base.cpp:100
    return num_iterations;
  }

  // ref: solver/linearizor_qr.cpp:140-265 ; optional outputs for parity tests
  void solve(S lambda, std::vector<S>& inc, std::vector<S>* b_out = nullptr, std::vector<S>* inv_out = nullptr) {
    auto t0 = std::chrono::high_resolution_clock::now();
    const bool schur = opt.preconditioner_type == PRECOND_SCHUR_JACOBI;
    set_pose_damping(lambda);
    std::vector<S> b;
    if (!opt.staged_execution) {
      // ref: :166-187
      if (new_linearization_point) for (int r = 0; r < nl; ++r) scale_Jp_cols(blocks[r], pose_jacobian_scaling.data());
      for (int r = 0; r < nl; ++r) set_landmark_damping(blocks[r], lambda);
      if (schur) {
        precond_blocks.assign((size_t)81 * nc, S(0));
        for (int r = 0; r < nl; ++r) add_Q2TJp_T_Q2TJp_blockdiag(blocks[r], precond_blocks.data(), nullptr);
        if (has_pose_damping())  // qr/linearization_qr.hpp:555-559
          for (int c = 0; c < nc; ++c) for (int d = 0; d < 9; ++d) precond_blocks[(size_t)81 * c + 10 * d] += pose_damping_diagonal;
      }
      b.assign((size_t)9 * nc, S(0));
      for (int r = 0; r < nl; ++r) add_Q2TJp_T_Q2Tr(blocks[r], b.data(), nullptr);
    } else {
      get_stage2(lambda, new_linearization_point ? pose_jacobian_scaling.data() : nullptr, schur, b);
    }
    auto t1 = std::chrono::high_resolution_clock::now();
    t_stage2 = std::chrono::duration<double>(t1 - t0).count();
    // preconditioner (:203-245)
    std::vector<S> inv((size_t)81 * nc);
    if (!schur) {
      if (new_linearization_point) {
        // scale_jacobians: D B D (cg/block_sparse_matrix.hpp:89-100)
        for (int c = 0; c < nc; ++c) {
          S* B = precond_blocks.data() + (size_t)81 * c;
          const S* d = pose_jacobian_scaling.data() + (size_t)9 * c;
          for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) B[9 * i + j] = d[i] * B[9 * i + j] * d[j];
        }
      }
      S diag[9];
      for (int d = 0; d < 9; ++d) diag[d] = lambda;
#pragma omp parallel for num_threads(threads())
      for (int c = 0; c < nc; ++c) invert_block9(precond_blocks.data() + (size_t)81 * c, diag, inv.data() + (size_t)81 * c);
    } else {
#pragma omp parallel for num_threads(threads())
      for (int c = 0; c < nc; ++c) invert_block9(precond_blocks.data() + (size_t)81 * c, nullptr, inv.data() + (size_t)81 * c);
    }
    auto t2 = std::chrono::high_resolution_clock::now();
    t_precond = std::chrono::duration<double>(t2 - t1).count();
    inc.assign((size_t)9 * nc, S(0));
    last_cg_iterations = pcg(b, inv, inc);
    t_pcg = std::chrono::duration<double>(std::chrono::high_resolution_clock::now() - t2).count();
    new_linearization_point = false;
    if (b_out) *b_out = b;
    if (inv_out) *inv_out = inv;
  }

  // ref: solver/linearizor_qr.cpp:267-291
  S apply(std::vector<S>& inc) {
    auto t0 = std::chrono::high_resolution_clock::now();
    bool fail = false;
    S l_diff = back_substitute(inc.data(), fail);
    auto t1 = std::chrono::high_resolution_clock::now();
    t_backsub = std::chrono::duration<double>(t1 - t0).count();
    if (fail) l_diff = std::numeric_limits<S>::quiet_NaN();
    if (!std::isfinite(l_diff)) return std::numeric_limits<S>::quiet_NaN();
    for (size_t k = 0; k < inc.size(); ++k) inc[k] *= pose_jacobian_scaling[k];
    for (int c = 0; c < nc; ++c) camera_apply_inc(cams.data() + (size_t)10 * c, inc.data() + (size_t)9 * c);
    t_update = std::chrono::duration<double>(std::chrono::high_resolution_clock::now() - t1).count();
    return l_diff;
  }

  // ---------------- Schur-complement cross-check (ref: sc/landmark_block.hpp) ----------------
  // Independent formulation used by the reference's own tests to validate the QR path
  // (qr/linearization_qr.test.cpp:120-222).  Works on a fresh linearization at the current state.
  struct SCBlock { std::vector<S> Jp, Jl, r; S Jl_col_scale[3]; };  // Jp: n x (2x9), Jl: n x (2x3), r: n x 2

  void sc_linearize(std::vector<SCBlock>& sc, std::vector<S>& diag2) const {
    sc.resize(nl);
    diag2.assign((size_t)9 * nc, S(0));
    for (int l = 0; l < nl; ++l) {
      const int n = (int)(lm_off[l + 1] - lm_off[l]);
      auto& b = sc[l];
      b.Jp.assign((size_t)18 * n, 0); b.Jl.assign((size_t)6 * n, 0); b.r.assign((size_t)2 * n, 0);
      for (int i = 0; i < n; ++i) {
        const int64_t o = lm_off[l] + i;
        S Jp[12], Ji[6], Jl[6], res[2];
        const bool valid = linearize_point(obs_xy.data() + 2 * o, lms.data() + 3 * (size_t)l,
                                           cams.data() + (size_t)10 * obs_cam[o], true, res, Jp, Ji, Jl);
        if (!opt.use_valid_projections_only || valid) {
          const S rsq = res[0] * res[0] + res[1] * res[1];
          S werr, w;
          compute_error_weight<S>(opt.robust_norm, S(opt.huber_parameter), rsq, werr, w);
          const S sw = std::sqrt(w);
          for (int rr = 0; rr < 2; ++rr) {
            for (int c = 0; c < 6; ++c) b.Jp[18 * i + 9 * rr + c] = sw * Jp[6 * rr + c];
            for (int c = 0; c < 3; ++c) b.Jp[18 * i + 9 * rr + 6 + c] = sw * Ji[3 * rr + c];
            for (int c = 0; c < 3; ++c) b.Jl[6 * i + 3 * rr + c] = sw * Jl[3 * rr + c];
            b.r[2 * i + rr] = sw * res[rr];
          }
        }
        for (int c = 0; c < 9; ++c)  // sc/landmark_block.hpp:177-188
          diag2[(size_t)9 * obs_cam[o] + c] += b.Jp[18 * i + c] * b.Jp[18 * i + c] + b.Jp[18 * i + 9 + c] * b.Jp[18 * i + 9 + c];
      }
      // scale_Jl_cols (sc/landmark_block.hpp:190-201)
      for (int j = 0; j < 3; ++j) {
        S sq = 0;
        for (int k = 0; k < 2 * n; ++k) sq += b.Jl[3 * k + j] * b.Jl[3 * k + j];
        b.Jl_col_scale[j] = S(1) / (jacobi_eps() + std::sqrt(sq));
        for (int k = 0; k < 2 * n; ++k) b.Jl[3 * k + j] *= b.Jl_col_scale[j];
      }
    }
  }
  void sc_scale_Jp(std::vector<SCBlock>& sc, const S* scaling) const {  // sc/landmark_block.hpp:203-213
    for (int l = 0; l < nl; ++l) {
      const int n = (int)(lm_off[l + 1] - lm_off[l]);
      for (int i = 0; i < n; ++i) {
        const S* d = scaling + (size_t)9 * obs_cam[lm_off[l] + i];
        for (int rr = 0; rr < 2; ++rr) for (int c = 0; c < 9; ++c) sc[l].Jp[18 * i + 9 * rr + c] *= d[c];
      }
    }
  }
  static void inv3(const S* A, S* Ai) {
    const S a = A[0], b = A[1], c = A[2], d = A[3], e = A[4], f = A[5], g = A[6], h = A[7], i = A[8];
    const S det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
    const S id = S(1) / det;
    Ai[0] = (e * i - f * h) * id; Ai[1] = (c * h - b * i) * id; Ai[2] = (b * f - c * e) * id;
    Ai[3] = (f * g - d * i) * id; Ai[4] = (a * i - c * g) * id; Ai[5] = (c * d - a * f) * id;
    Ai[6] = (d * h - e * g) * id; Ai[7] = (b * g - a * h) * id; Ai[8] = (a * e - b * d) * id;
  }
  void sc_Hll_inv(const SCBlock& b, int n, S lambda, S* Hi) const {
    S H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int k = 0; k < 2 * n; ++k) for (int a = 0; a < 3; ++a) for (int c = 0; c < 3; ++c) H[3 * a + c] += b.Jl[3 * k + a] * b.Jl[3 * k + c];
    for (int d = 0; d < 3; ++d) H[4 * d] += lambda;
    inv3(H, Hi);
  }
  // b, diagonal blocks of H_pp (+pose damping), y = H_pp x  (sc/landmark_block.hpp:238-279)
  void sc_get_Hb(const std::vector<SCBlock>& sc, S lambda, S pose_damping, std::vector<S>& b,
                 std::vector<S>& diag_blocks, const S* x, std::vector<S>& y) const {
    b.assign((size_t)9 * nc, 0); diag_blocks.assign((size_t)81 * nc, 0); y.assign((size_t)9 * nc, 0);
    for (int l = 0; l < nl; ++l) {
      const int n = (int)(lm_off[l + 1] - lm_off[l]);
      const auto& B = sc[l];
      S Hi[9];
      sc_Hll_inv(B, n, lambda, Hi);
      S Jlr[3] = {0, 0, 0};
      for (int k = 0; k < 2 * n; ++k) for (int a = 0; a < 3; ++a) Jlr[a] += B.Jl[3 * k + a] * B.r[k];
      S Hbl[3];
      for (int a = 0; a < 3; ++a) Hbl[a] = Hi[3 * a] * Jlr[0] + Hi[3 * a + 1] * Jlr[1] + Hi[3 * a + 2] * Jlr[2];
      // s = sum_j Jl_j^T Jp_j x_j
      S s[3] = {0, 0, 0};
      std::vector<S> Jpx((size_t)2 * n);
      for (int j = 0; j < n; ++j) {
        const S* xj = x + (size_t)9 * obs_cam[lm_off[l] + j];
        for (int rr = 0; rr < 2; ++rr) {
          S acc = 0;
          for (int c = 0; c < 9; ++c) acc += B.Jp[18 * j + 9 * rr + c] * xj[c];
          Jpx[2 * j + rr] = acc;
          for (int a = 0; a < 3; ++a) s[a] += B.Jl[6 * j + 3 * rr + a] * acc;
        }
      }
      S His[3];
      for (int a = 0; a < 3; ++a) His[a] = Hi[3 * a] * s[0] + Hi[3 * a + 1] * s[1] + Hi[3 * a + 2] * s[2];
      for (int i = 0; i < n; ++i) {
        const int cam = obs_cam[lm_off[l] + i];
        // M = Jl_i Hi Jl_i^T (2x2)
        S JH[6];
        for (int rr = 0; rr < 2; ++rr) for (int a = 0; a < 3; ++a)
          JH[3 * rr + a] = B.Jl[6 * i + 3 * rr] * Hi[a] + B.Jl[6 * i + 3 * rr + 1] * Hi[3 + a] + B.Jl[6 * i + 3 * rr + 2] * Hi[6 + a];
        S M[4];
        for (int rr = 0; rr < 2; ++rr) for (int qq = 0; qq < 2; ++qq)
          M[2 * rr + qq] = JH[3 * rr] * B.Jl[6 * i + 3 * qq] + JH[3 * rr + 1] * B.Jl[6 * i + 3 * qq + 1] + JH[3 * rr + 2] * B.Jl[6 * i + 3 * qq + 2];
        S* D = diag_blocks.data() + (size_t)81 * cam;
        for (int a = 0; a < 9; ++a) for (int c = 0; c < 9; ++c) {
          const S ja0 = B.Jp[18 * i + a], ja1 = B.Jp[18 * i + 9 + a];
          const S jc0 = B.Jp[18 * i + c], jc1 = B.Jp[18 * i + 9 + c];
          D[9 * a + c] += ja0 * jc0 + ja1 * jc1 - (ja0 * (M[0] * jc0 + M[1] * jc1) + ja1 * (M[2] * jc0 + M[3] * jc1));
        }
        // b_i += Jp_i^T (r_i - Jl_i Hbl)
        S ri[2];
        for (int rr = 0; rr < 2; ++rr)
          ri[rr] = B.r[2 * i + rr] - (B.Jl[6 * i + 3 * rr] * Hbl[0] + B.Jl[6 * i + 3 * rr + 1] * Hbl[1] + B.Jl[6 * i + 3 * rr + 2] * Hbl[2]);
        for (int c = 0; c < 9; ++c) b[(size_t)9 * cam + c] += B.Jp[18 * i + c] * ri[0] + B.Jp[18 * i + 9 + c] * ri[1];
        // y_i += Jp_i^T (Jp_i x_i - Jl_i Hi s)
        S vi[2];
        for (int rr = 0; rr < 2; ++rr)
          vi[rr] = Jpx[2 * i + rr] - (B.Jl[6 * i + 3 * rr] * His[0] + B.Jl[6 * i + 3 * rr + 1] * His[1] + B.Jl[6 * i + 3 * rr + 2] * His[2]);
        for (int c = 0; c < 9; ++c) y[(size_t)9 * cam + c] += B.Jp[18 * i + c] * vi[0] + B.Jp[18 * i + 9 + c] * vi[1];
      }
    }
    if (pose_damping > 0) {  // sc/linearization_sc.hpp:342-346
      for (int c = 0; c < nc; ++c) for (int d = 0; d < 9; ++d) diag_blocks[(size_t)81 * c + 10 * d] += pose_damping;
      for (size_t k = 0; k < y.size(); ++k) y[k] += pose_damping * x[k];
    }
  }
  // sc/landmark_block.hpp:409-446 ; updates lms_out (copy of landmark positions)
  S sc_back_substitute(const std::vector<SCBlock>& sc, S lambda, const S* pose_inc, std::vector<S>& lms_out) const {
    lms_out = lms;
    S l_diff = 0;
    for (int l = 0; l < nl; ++l) {
      const int n = (int)(lm_off[l + 1] - lm_off[l]);
      const auto& B = sc[l];
      S H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, tmp[3] = {0, 0, 0};
      std::vector<S> J_inc((size_t)2 * n, S(0));
      for (int i = 0; i < n; ++i) {
        const S* pi = pose_inc + (size_t)9 * obs_cam[lm_off[l] + i];
        for (int rr = 0; rr < 2; ++rr) {
          S acc = 0;
          for (int c = 0; c < 9; ++c) acc += B.Jp[18 * i + 9 * rr + c] * pi[c];
          J_inc[2 * i + rr] += acc;
          for (int a = 0; a < 3; ++a) {
            tmp[a] += B.Jl[6 * i + 3 * rr + a] * (B.r[2 * i + rr] + acc);
            for (int c = 0; c < 3; ++c) H[3 * a + c] += B.Jl[6 * i + 3 * rr + a] * B.Jl[6 * i + 3 * rr + c];
          }
        }
      }
      for (int d = 0; d < 3; ++d) H[4 * d] += lambda;
      S Hi[9];
      inv3(H, Hi);
      S inc[3];
      for (int a = 0; a < 3; ++a) inc[a] = -(Hi[3 * a] * tmp[0] + Hi[3 * a + 1] * tmp[1] + Hi[3 * a + 2] * tmp[2]);
      S acc = 0;
      for (int k = 0; k < 2 * n; ++k) {
        const S ji = J_inc[k] + B.Jl[3 * k] * inc[0] + B.Jl[3 * k + 1] * inc[1] + B.Jl[3 * k + 2] * inc[2];
        acc += ji * (S(0.5) * ji + B.r[k]);
      }
      l_diff -= acc;
      for (int d = 0; d < 3; ++d) lms_out[3 * (size_t)l + d] += inc[d] * B.Jl_col_scale[d];
    }
    return l_diff;
  }

  // ---------------- LinearizorSC / LinearizorPowerSC (ref: solver/linearizor_sc.cpp, solver/linearizor_power_sc.cpp) -----------
  std::vector<SCBlock> scl;             // the linearisation of the SC solvers
  std::vector<S> sc_scaling;            // pose_jacobian_scaling_
  S sc_lambda = 0;
  int last_power_order = 0, last_power_termination = 0;
  // linearize(): linearize_problem + get_Jp_diag2 + scale_Jl_cols + Jacobi scaling (linearizor_sc.cpp:78-110); the pose
  // Jacobians are scaled here once (the reference does it in the first solve(), :128-131 -- same numbers)
  void sc_linearizor_linearize() {
    std::vector<S> d2;
    sc_linearize(scl, d2);
    sc_scaling.resize(d2.size());
    for (size_t k = 0; k < d2.size(); ++k) sc_scaling[k] = S(1) / (jacobi_eps() + std::sqrt(d2[k]));
    sc_scale_Jp(scl, sc_scaling.data());
  }
  // LinearizorSC::solve (linearizor_sc.cpp:112-204): H_pp, b_p (sc/linearization_sc.hpp get_Hb), SCHUR_JACOBI block
  // preconditioner from the diagonal blocks of H_pp, PCG (LinearizorBase::pcg)
  void sc_linearizor_solve(S lambda, std::vector<S>& inc, std::vector<S>* b_out = nullptr, std::vector<S>* inv_out = nullptr) {
    sc_lambda = lambda;
    const size_t N = (size_t)9 * nc;
    std::vector<S> b, diag, y, zero(N, S(0));
    sc_get_Hb(scl, lambda, lambda, b, diag, zero.data(), y);
    std::vector<S> inv((size_t)81 * nc);
    for (int c = 0; c < nc; ++c) invert_block9(diag.data() + (size_t)81 * c, nullptr, inv.data() + (size_t)81 * c);
    op_override = [&](const S* xin, S* yout) {
      std::vector<S> b2, d2, y2;
      sc_get_Hb(scl, lambda, lambda, b2, d2, xin, y2);
      std::copy(y2.begin(), y2.end(), yout);
    };
    inc.assign(N, S(0));
    last_cg_iterations = pcg(b, inv, inc);
    op_override = nullptr;
    if (b_out) *b_out = b;
    if (inv_out) *inv_out = inv;
  }
  // E_0 x = Jp^T Jl Hll^-1 Jl^T Jp x  (sc/linearization_power_sc.hpp:261-287)
  void sc_right_mul_e0(S lambda, const S* x, S* out) const {
    std::fill(out, out + (size_t)9 * nc, S(0));
    for (int l = 0; l < nl; ++l) {
      const int n = (int)(lm_off[l + 1] - lm_off[l]);
      const auto& B = scl[l];
      S Hi[9];
      sc_Hll_inv(B, n, lambda, Hi);
      S s[3] = {0, 0, 0};
      for (int j = 0; j < n; ++j) {
        const S* xj = x + (size_t)9 * obs_cam[lm_off[l] + j];
        for (int rr = 0; rr < 2; ++rr) {
          S acc = 0;
          for (int c = 0; c < 9; ++c) acc += B.Jp[18 * j + 9 * rr + c] * xj[c];
          for (int a = 0; a < 3; ++a) s[a] += B.Jl[6 * j + 3 * rr + a] * acc;
        }
      }
      S His[3];
      for (int a = 0; a < 3; ++a) His[a] = Hi[3 * a] * s[0] + Hi[3 * a + 1] * s[1] + Hi[3 * a + 2] * s[2];
      for (int i = 0; i < n; ++i) {
        S* o = out + (size_t)9 * obs_cam[lm_off[l] + i];
        for (int rr = 0; rr < 2; ++rr) {
          const S t = B.Jl[6 * i + 3 * rr] * His[0] + B.Jl[6 * i + 3 * rr + 1] * His[1] + B.Jl[6 * i + 3 * rr + 2] * His[2];
          for (int c = 0; c < 9; ++c) o[c] += B.Jp[18 * i + 9 * rr + c] * t;
        }
      }
    }
  }
  // LinearizorPowerSC::solve (linearizor_power_sc.cpp:112-167) = prepare_Hb + the power series of
  // LinearizationPowerSC::solve (sc/linearization_power_sc.hpp:92-160)
  void power_sc_linearizor_solve(S lambda, int power_order, S q_tolerance, std::vector<S>& accum, std::vector<S>* b_out = nullptr) {
    sc_lambda = lambda;
    const size_t N = (size_t)9 * nc;
    // prepare_Hb: b_p as in the SC solver; Hpp = sum Jp_i^T Jp_i (+ lambda) inverted per camera
    std::vector<S> b, diag, y, zero(N, S(0));
    sc_get_Hb(scl, lambda, S(0), b, diag, zero.data(), y);
    std::vector<S> Hpp((size_t)81 * nc, S(0)), Hinv((size_t)81 * nc);
    for (int l = 0; l < nl; ++l) {
      const int n = (int)(lm_off[l + 1] - lm_off[l]);
      for (int i = 0; i < n; ++i) {
        S* Dc = Hpp.data() + (size_t)81 * obs_cam[lm_off[l] + i];
        const S* J = scl[l].Jp.data() + 18 * i;
        for (int a = 0; a < 9; ++a) for (int c = 0; c < 9; ++c) Dc[9 * a + c] += J[a] * J[c] + J[9 + a] * J[9 + c];
      }
    }
    S dg[9];
    for (int d = 0; d < 9; ++d) dg[d] = lambda;
    for (int c = 0; c < nc; ++c) invert_block9(Hpp.data() + (size_t)81 * c, dg, Hinv.data() + (size_t)81 * c);
    auto mul_inv = [&](const std::vector<S>& v, std::vector<S>& out) {
      for (int c = 0; c < nc; ++c)
        for (int i = 0; i < 9; ++i) {
          S acc = 0;
          for (int j = 0; j < 9; ++j) acc += Hinv[(size_t)81 * c + 9 * i + j] * v[(size_t)9 * c + j];
          out[(size_t)9 * c + i] = acc;
        }
    };
    auto norm = [&](const std::vector<S>& v) { S sq = 0; for (S e : v) sq += e * e; return std::sqrt(sq); };
    std::vector<S> nb(N), tmp(N), e(N);
    for (size_t k = 0; k < N; ++k) nb[k] = -b[k];
    accum.assign(N, S(0));
    mul_inv(nb, accum);
    tmp = accum;
    last_power_termination = 0; last_power_order = power_order;
    for (int i = 1; i <= power_order; ++i) {
      sc_right_mul_e0(lambda, tmp.data(), e.data());
      mul_inv(e, tmp);
      for (size_t k = 0; k < N; ++k) accum[k] += tmp[k];
      if (q_tolerance > 0) {
        const S zeta = S(i) * norm(tmp) / norm(accum);
        if (zeta < q_tolerance) { last_power_termination = 1; last_power_order = i; break; }
      }
    }
    if (b_out) *b_out = b;
  }
  // LinearizorSC::apply / LinearizorPowerSC::apply (linearizor_sc.cpp:206-228): SC back-substitution + camera update
  S sc_linearizor_apply(std::vector<S>& inc) {
    std::vector<S> lms_new;
    const S l_diff = sc_back_substitute(scl, sc_lambda, inc.data(), lms_new);
    if (!std::isfinite(l_diff)) return std::numeric_limits<S>::quiet_NaN();
    lms = lms_new;
    for (size_t k = 0; k < inc.size(); ++k) inc[k] *= sc_scaling[k];
    for (int c = 0; c < nc; ++c) camera_apply_inc(cams.data() + (size_t)10 * c, inc.data() + (size_t)9 * c);
    return l_diff;
  }
};

// ---------------------------------------------------------------------------
// LM loop (ref: solver/bal_bundle_adjustment.cpp:249-544 optimize_lm_ours)
// ---------------------------------------------------------------------------
struct IterationLog {
  int iteration = 0;
  double cost = 0, cost_valid = 0;
  int num_obs_valid = 0;
  int step_is_valid = 0, step_is_successful = 0;
  double lambda = 0, trust_region_radius = 0, relative_decrease = 0, l_diff = 0;
  int cg_iterations = 0;
  double stage1_time = 0, stage2_time = 0, precond_time = 0, pcg_time = 0, backsub_time = 0, update_time = 0, error_time = 0, iteration_time = 0;
};

template <class S>
inline double cost_of(const ResidualInfo& ri, int optimized_cost) {
  switch (optimized_cost) {
    case 1: return ri.valid.error;
    case 2: return ri.valid.error_avg();
    default: return ri.all.error;
  }
}

// termination: 0 NO_CONVERGENCE, 1 CONVERGENCE
template <class S>
int optimize_lm(Problem<S>& P, std::vector<IterationLog>& log) {
  const Options& o = P.opt;
  const S min_lambda(1.0 / o.max_trust_region_radius);
  const S max_lambda(1.0 / o.min_trust_region_radius);
  const S vee_factor(o.vee_factor);
  const S initial_vee(o.initial_vee);
  const int max_lm_iter = o.max_num_iterations;
  S lambda(1.0 / o.initial_trust_region_radius);
  S lambda_vee(initial_vee);
  bool terminated = false;
  int termination = 0;
  log.clear();
  for (int it = 0; it <= max_lm_iter && !terminated;) {
    auto ti0 = std::chrono::high_resolution_clock::now();
    IterationLog L;
    L.iteration = it;
    ResidualInfo ri;
    P.compute_error(ri);
    L.error_time += P.t_error;
    if (!ri.is_numerically_valid) { return -1; }
    if (it == 0) {
      L.cost = ri.all.error; L.cost_valid = ri.valid.error; L.num_obs_valid = ri.valid.num_obs;
      L.trust_region_radius = 1 / (double)lambda; L.lambda = lambda;
      L.step_is_successful = 1; L.step_is_valid = 1;
      L.iteration_time = std::chrono::duration<double>(std::chrono::high_resolution_clock::now() - ti0).count();
      log.push_back(L);
      ++it;
      continue;
    }
    if (!P.linearize()) return -1;
    L.stage1_time = P.t_stage1;
    for (int j = 0; it <= max_lm_iter && !terminated; j++) {
      if (j > 0) {
        L = IterationLog();
        L.iteration = it;
        ti0 = std::chrono::high_resolution_clock::now();
      }
      std::vector<S> inc;
      P.solve(lambda, inc);
      L.stage2_time = P.t_stage2; L.precond_time = P.t_precond; L.pcg_time = P.t_pcg; L.cg_iterations = P.last_cg_iterations;
      L.lambda = lambda;
      bool inc_finite = true;
      for (S v : inc) inc_finite = inc_finite && std::isfinite(v);
      if (!inc_finite) {
        L.step_is_valid = 0; L.step_is_successful = 0;
        lambda = lambda_vee * lambda;
        lambda_vee *= vee_factor;
        L.trust_region_radius = 1 / (double)lambda;
        L.iteration_time = std::chrono::duration<double>(std::chrono::high_resolution_clock::now() - ti0).count();
        log.push_back(L);
        it++;
        if (lambda > max_lambda) { terminated = true; termination = 0; }
        continue;
      }
      P.backup();
      S l_diff = P.apply(inc);
      L.backsub_time = P.t_backsub; L.update_time = P.t_update;
      ResidualInfo ri2;
      P.compute_error(ri2);
      L.error_time += P.t_error;
      L.cost = ri2.all.error; L.cost_valid = ri2.valid.error; L.num_obs_valid = ri2.valid.num_obs;
      L.l_diff = l_diff;
      if (!std::isfinite(l_diff)) {
        L.step_is_valid = 0; L.step_is_successful = 0;
      } else if (!ri2.is_numerically_valid) {
        L.step_is_valid = 0; L.step_is_successful = 0;
      } else {
        S f_diff = S(cost_of<S>(ri, o.optimized_cost) - cost_of<S>(ri2, o.optimized_cost));
        if (o.optimized_cost == 2) l_diff /= ri.valid.num_obs;
        const S step_quality = f_diff / l_diff;
        L.relative_decrease = step_quality;
        L.step_is_valid = l_diff > 0;
        L.step_is_successful = L.step_is_valid && step_quality > o.min_relative_decrease;
      }
      if (L.step_is_successful) {
        lambda *= S(std::max(1.0 / 3, 1 - std::pow(2 * L.relative_decrease - 1, 3)));
        lambda = std::max(min_lambda, lambda);
        lambda_vee = initial_vee;
        L.trust_region_radius = 1 / (double)lambda;
        L.iteration_time = std::chrono::duration<double>(std::chrono::high_resolution_clock::now() - ti0).count();
        // function tolerance (ref: :174-201), cost_change vs previous log entry
        const double prev = o.optimized_cost == 0 ? log.back().cost : log.back().cost_valid;
        const double cur = o.optimized_cost == 0 ? L.cost : L.cost_valid;
        log.push_back(L);
        it++;
        if (std::abs(prev - cur) <= o.function_tolerance * cur) { terminated = true; termination = 1; }
        break;
      } else {
        lambda = lambda_vee * lambda;
        lambda_vee *= vee_factor;
        L.trust_region_radius = 1 / (double)lambda;
        L.iteration_time = std::chrono::duration<double>(std::chrono::high_resolution_clock::now() - ti0).count();
        log.push_back(L);
        P.restore();
        it++;
        if (lambda > max_lambda) { terminated = true; termination = 0; }
      }
    }
  }
  return termination;
}

// ---------------------------------------------------------------------------
// BAL text loader + normalisation (ref: bal/bal_problem.cpp:189-282, 428-469, 773-852)
// Always parsed / normalised in double, then cast (ref: :795-832).
// ---------------------------------------------------------------------------
struct BalData {
  int nc = 0, nl = 0;
  int64_t nobs = 0;
  std::vector<double> cams;  // 10*nc (quat xyzw, t, f, k1, k2)
  std::vector<double> lms;   // 3*nl
  std::vector<int64_t> lm_off;
  std::vector<int> obs_cam;
  std::vector<double> obs_xy;
};

inline double median_destructive(std::vector<double>& d) {  // ref: bal/bal_problem.cpp:116-122
  const size_t n = d.size();
  auto mid = d.begin() + n / 2;
  std::nth_element(d.begin(), mid, d.end());
  return *mid;
}

// returns 0 ok, <0 error
inline int load_bal(const char* path, BalData& D) {
  FILE* f = std::fopen(path, "r");
  if (!f) return -1;
  int nc, nl, nobs;
  if (std::fscanf(f, "%d %d %d", &nc, &nl, &nobs) != 3 || nc <= 0 || nl <= 0 || nobs <= 0) { std::fclose(f); return -2; }
  struct O { int cam; double x, y; };
  std::vector<std::vector<O>> per_lm(nl);
  for (int i = 0; i < nobs; ++i) {
    int c, l; double x, y;
    if (std::fscanf(f, "%d %d %lf %lf", &c, &l, &x, &y) != 4) { std::fclose(f); return -3; }
    if (c < 0 || c >= nc || l < 0 || l >= nl) { std::fclose(f); return -4; }
    per_lm[l].push_back({c, x, -y});  // invert y axis (:243)
  }
  D.nc = nc; D.nl = nl; D.nobs = nobs;
  D.cams.resize((size_t)10 * nc);
  for (int i = 0; i < nc; ++i) {
    double p[9];
    for (int k = 0; k < 9; ++k) if (std::fscanf(f, "%lf", &p[k]) != 1) { std::fclose(f); return -5; }
    double q[4];
    so3_exp<double>(p, q);
    // axis_inversion = SO3(diag(1,-1,-1)) = quaternion (x=1,y=0,z=0,w=0); T.so3 = axis_inversion * exp(r)
    const double ai[4] = {1, 0, 0, 0};
    double qn[4];
    quat_mul_sophus<double>(ai, q, qn);
    double* c = D.cams.data() + (size_t)10 * i;
    c[0] = qn[0]; c[1] = qn[1]; c[2] = qn[2]; c[3] = qn[3];
    c[4] = p[3]; c[5] = -p[4]; c[6] = -p[5];
    c[7] = p[6]; c[8] = p[7]; c[9] = p[8];
  }
  D.lms.resize((size_t)3 * nl);
  for (int i = 0; i < nl; ++i)
    for (int k = 0; k < 3; ++k) if (std::fscanf(f, "%lf", &D.lms[(size_t)3 * i + k]) != 1) { std::fclose(f); return -6; }
  std::fclose(f);
  D.lm_off.assign(nl + 1, 0);
  D.obs_cam.resize(nobs); D.obs_xy.resize((size_t)2 * nobs);
  int64_t k = 0;
  for (int l = 0; l < nl; ++l) {
    auto& v = per_lm[l];
    std::sort(v.begin(), v.end(), [](const O& a, const O& b) { return a.cam < b.cam; });  // std::map order
    for (size_t i = 1; i < v.size(); ++i) if (v[i].cam == v[i - 1].cam) return -7;  // duplicate (:229-230)
    D.lm_off[l] = k;
    for (auto& o : v) { D.obs_cam[k] = o.cam; D.obs_xy[2 * k] = o.x; D.obs_xy[2 * k + 1] = o.y; ++k; }
  }
  D.lm_off[nl] = k;
  return 0;
}

// Eigen::Quaternion(rotation matrix) as Sophus::SO3(R) uses it (Eigen/src/Geometry/Quaternion.h, quaternionbase_assign_impl:
// trace branch / largest-diagonal branch).  R row-major; q = (x, y, z, w).  Restated, unpinned like the rest of Appendix A.
inline void rot_to_quat(const double* R, double* q) {
  double t = R[0] + R[4] + R[8];
  if (t > 0) {
    t = std::sqrt(t + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (R[7] - R[5]) * t;
    q[1] = (R[2] - R[6]) * t;
    q[2] = (R[3] - R[1]) * t;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[4 * i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(R[4 * i] - R[4 * j] - R[4 * k] + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (R[3 * k + j] - R[3 * j + k]) * t;
    q[j] = (R[3 * j + i] + R[3 * i + j]) * t;
    q[k] = (R[3 * k + i] + R[3 * i + k]) * t;
  }
}

// ref: bal/bal_problem.cpp:284-404  load_bundler ("bundle.out" v0.3): one comment line, "num_cams num_points", per camera
// 15 values (f k1 k2, R row-major, t; f == 0 = uninitialised camera: skipped, later cameras move up), per point position (3),
// colour (3, ignored), view list: n, then n x (camera, feature key, x, y).  Same axis conventions as load_bal.
inline int load_bundler(const char* path, BalData& D) {
  FILE* f = std::fopen(path, "r");
  if (!f) return -1;
  char line[1000];
  bool first = true, done = false;
  while (!done && std::fgets(line, sizeof(line), f)) {  // readcommentline_or_throw (:76-107)
    const size_t len = std::strlen(line);
    if (len == 0 || (first && line[0] != '#')) { std::fclose(f); return -2; }
    first = false;
    done = line[len - 1] == '\n';
  }
  if (!done) { std::fclose(f); return -2; }
  int ncf, nl;
  if (std::fscanf(f, "%d %d", &ncf, &nl) != 2 || ncf <= 0 || nl <= 0) { std::fclose(f); return -2; }
  std::vector<int> cam_map(ncf, -1);
  D = BalData();
  for (int i = 0; i < ncf; ++i) {
    double p[15];
    for (double& v : p) if (std::fscanf(f, "%lf", &v) != 1) { std::fclose(f); return -5; }
    if (p[0] == 0) continue;
    cam_map[i] = D.nc++;
    double q[4], qn[4];
    rot_to_quat(p + 3, q);
    const double ai[4] = {1, 0, 0, 0};
    quat_mul_sophus<double>(ai, q, qn);
    const double c[10] = {qn[0], qn[1], qn[2], qn[3], p[12], -p[13], -p[14], p[0], p[1], p[2]};
    D.cams.insert(D.cams.end(), c, c + 10);
  }
  D.nl = nl;
  D.lms.resize((size_t)3 * nl);
  D.lm_off.assign(1, 0);
  struct O { int cam; double x, y; };
  std::vector<O> v;
  for (int l = 0; l < nl; ++l) {
    double col[3];
    int n;
    for (int k = 0; k < 3; ++k) if (std::fscanf(f, "%lf", &D.lms[(size_t)3 * l + k]) != 1) { std::fclose(f); return -6; }
    for (int k = 0; k < 3; ++k) if (std::fscanf(f, "%lf", &col[k]) != 1) { std::fclose(f); return -6; }
    if (std::fscanf(f, "%d", &n) != 1) { std::fclose(f); return -6; }
    v.clear();
    for (int j = 0; j < n; ++j) {
      int c, key; double x, y;
      if (std::fscanf(f, "%d %d %lf %lf", &c, &key, &x, &y) != 4) { std::fclose(f); return -3; }
      if (c >= 0 && c < ncf && cam_map[c] >= 0) v.push_back({cam_map[c], x, -y});
    }
    std::sort(v.begin(), v.end(), [](const O& a, const O& b) { return a.cam < b.cam; });
    for (size_t i = 1; i < v.size(); ++i) if (v[i].cam == v[i - 1].cam) { std::fclose(f); return -7; }
    for (auto& o : v) { D.obs_cam.push_back(o.cam); D.obs_xy.push_back(o.x); D.obs_xy.push_back(o.y); }
    D.lm_off.push_back((int64_t)D.obs_cam.size());
  }
  std::fclose(f);
  D.nobs = (int64_t)D.obs_cam.size();
  return 0;
}

// ref: bal/bal_problem.cpp:428-469
inline void normalize(BalData& D, double new_scale) {
  std::vector<double> tmp(D.nl);
  double median[3];
  for (int j = 0; j < 3; ++j) {
    for (int i = 0; i < D.nl; ++i) tmp[i] = D.lms[(size_t)3 * i + j];
    median[j] = median_destructive(tmp);
  }
  for (int i = 0; i < D.nl; ++i)
    tmp[i] = std::abs(D.lms[(size_t)3 * i] - median[0]) + std::abs(D.lms[(size_t)3 * i + 1] - median[1]) + std::abs(D.lms[(size_t)3 * i + 2] - median[2]);
  const double mad = median_destructive(tmp);
  const double scale = new_scale / mad;
  for (int i = 0; i < D.nl; ++i)
    for (int j = 0; j < 3; ++j) D.lms[(size_t)3 * i + j] = scale * (D.lms[(size_t)3 * i + j] - median[j]);
  for (int i = 0; i < D.nc; ++i) {
    double* c = D.cams.data() + (size_t)10 * i;
    double R[9];
    quat_to_rot<double>(c, R);
    // T_w_c translation = -R^T t ; center = scale * (center - median) ; t = -R center
    double ctr[3];
    for (int a = 0; a < 3; ++a) ctr[a] = -(R[a] * c[4] + R[3 + a] * c[5] + R[6 + a] * c[6]);
    for (int a = 0; a < 3; ++a) ctr[a] = scale * (ctr[a] - median[a]);
    for (int a = 0; a < 3; ++a) c[4 + a] = -(R[3 * a] * ctr[0] + R[3 * a + 1] * ctr[1] + R[3 * a + 2] * ctr[2]);
  }
}

// ref: bal/bal_problem.cpp:471-505  filter_obs: drop observations whose landmark lies closer than `threshold` in front of
// the camera (z of T_c_w * p_w), then drop landmarks left with fewer than 2 observations.  threshold <= 0: no-op.
inline void filter_obs(BalData& D, double threshold) {
  if (!(threshold > 0)) return;
  BalData R;
  R.nc = D.nc;
  R.cams = D.cams;
  R.lm_off.push_back(0);
  for (int l = 0; l < D.nl; ++l) {
    const double* p = D.lms.data() + 3 * (size_t)l;
    const size_t keep_from = R.obs_cam.size();
    for (int64_t k = D.lm_off[l]; k < D.lm_off[l + 1]; ++k) {
      const double* c = D.cams.data() + 10 * (size_t)D.obs_cam[k];
      double Rm[9];
      quat_to_rot(c, Rm);
      const double z = Rm[6] * p[0] + Rm[7] * p[1] + Rm[8] * p[2] + c[6];
      if (z < threshold) continue;
      R.obs_cam.push_back(D.obs_cam[k]);
      R.obs_xy.push_back(D.obs_xy[2 * k]);
      R.obs_xy.push_back(D.obs_xy[2 * k + 1]);
    }
    if (R.obs_cam.size() - keep_from >= 2) {
      R.lms.insert(R.lms.end(), p, p + 3);
      R.lm_off.push_back((int64_t)R.obs_cam.size());
    } else {
      R.obs_cam.resize(keep_from);
      R.obs_xy.resize(2 * keep_from);
    }
  }
  R.nl = (int)R.lm_off.size() - 1;
  R.nobs = (int64_t)R.obs_cam.size();
  D = std::move(R);
}

}  // namespace orc
