// Host-side mirror of the reference's solver seam on top of the C ABI (include/rootba_b200.h):
//   SolverOptions      <-> rootba::SolverOptions      (src/rootba/bal/solver_options.hpp:46-284, QR-relevant subset)
//   ResidualInfo       <-> rootba::ResidualInfo       (src/rootba/bal/residual_info.hpp:59-89)
//   LinearizorQR       <-> rootba::LinearizorQR       (src/rootba/solver/linearizor_qr.cpp:52-291) behind
//                          rootba::Linearizor         (src/rootba/solver/linearizor.hpp:47-83)
//   bundle_adjust_manual <-> optimize_lm_ours         (src/rootba/solver/bal_bundle_adjustment.cpp:249-544)
#pragma once

#include <chrono>
#include <cmath>
#include <cstdio>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/rootba_b200.h"
#include "bal_io_fast.hpp"
#include "bal_problem.hpp"

namespace rootba_b200 {

struct SolverOptions {
  enum class PreconditionerType { JACOBI = 0, SCHUR_JACOBI = 1, CLUSTER_JACOBI = 2 };  // solver_options.hpp:73-75
  enum class OptimizedCost { ERROR = 0, ERROR_VALID = 1, ERROR_VALID_AVG = 2 };
  enum class RobustNorm { NONE = 0, HUBER = 1 };
  OptimizedCost optimized_cost = OptimizedCost::ERROR;
  int max_num_iterations = 20;
  double min_relative_decrease = 0;  // solver_options.hpp:146-148
  double initial_trust_region_radius = 1e4;
  double min_trust_region_radius = 1e-32;
  double max_trust_region_radius = 1e16;
  int min_linear_solver_iterations = 0;
  int max_linear_solver_iterations = 500;
  double eta = 0.1;
  double jacobi_scaling_epsilon = 0.0;
  PreconditionerType preconditioner_type = PreconditionerType::SCHUR_JACOBI;
  double function_tolerance = 1e-6;
  bool use_double = true;
  bool use_householder_marginalization = true;
  double initial_vee = 2.0;
  double vee_factor = 2.0;
  RobustNorm robust_norm = RobustNorm::NONE;
  double huber_parameter = 1.0;
  int device = -1;
  enum class SolverType { SQUARE_ROOT = 0, SCHUR_COMPLEMENT = 1, POWER_SCHUR_COMPLEMENT = 2 };  // solver_options.hpp:63-76
  SolverType solver_type = SolverType::SQUARE_ROOT;
  int power_order = 20;   // :270
  enum class LinearSolverType { ITERATIVE_SCHUR = 0, DENSE_SCHUR = 1 };  // solver_options.hpp:77-80, 225-230
  LinearSolverType linear_solver_type = LinearSolverType::ITERATIVE_SCHUR;  // DENSE_SCHUR: exact steps (rba_solver_opts.linear_solver_type)
  int operator_form = 0;  // not in the reference: 0 = dense Q2 panels (reference algorithm), 1 = implicit (rba_solver_opts.operator_form)
  bool use_projection_validity_check() const { return optimized_cost != OptimizedCost::ERROR; }  // solver_options.cpp:41-51
};

struct ResidualItem { long long num_obs = 0; double error = 0, residual_sum = 0; double error_avg() const { return num_obs > 0 ? error / num_obs : 0.0; } };
struct ResidualInfo { ResidualItem all, valid; bool is_numerically_valid = true; };

struct IterationSummary {
  int iteration = 0;
  ResidualInfo cost;
  bool step_is_valid = false, step_is_successful = false;
  double trust_region_radius = 0, relative_decrease = 0;
  int linear_solver_iterations = 0;
  double stage1_time_in_seconds = 0, stage2_time_in_seconds = 0, compute_preconditioner_time_in_seconds = 0,
         solve_reduced_system_time_in_seconds = 0, back_substitution_time_in_seconds = 0, update_cameras_time_in_seconds = 0,
         residual_evaluation_time_in_seconds = 0;
  double iteration_time_in_seconds = 0, cumulative_time_in_seconds = 0;  // wall clock, like rootba::Timer (bal_bundle_adjustment.cpp:315-316)
};
struct SolverSummary {
  std::vector<IterationSummary> iterations;
  std::string termination_type = "NO_CONVERGENCE", message;
  int num_linear_solves = 0, num_residual_evaluations = 0, num_jacobian_evaluations = 0;
  double preprocessor_time_in_seconds = 0, minimizer_time_in_seconds = 0, total_time_in_seconds = 0;  // :286, :530-532
};

template <class S> struct Abi;
template <> struct Abi<float> {
  static int create(const rba_problem_view* p, const rba_solver_opts* o, rba_handle** h) { return rba_create_f32(p, o, h); }
  static int solve(rba_handle* h, float l, float* inc, rba_cg_summary* cg) { return rba_solve_f32(h, l, inc, cg); }
  static int apply(rba_handle* h, const float* inc, float* l) { return rba_apply_f32(h, inc, l); }
};
template <> struct Abi<double> {
  static int create(const rba_problem_view* p, const rba_solver_opts* o, rba_handle** h) { return rba_create_f64(p, o, h); }
  static int solve(rba_handle* h, double l, double* inc, rba_cg_summary* cg) { return rba_solve_f64(h, l, inc, cg); }
  static int apply(rba_handle* h, const double* inc, double* l) { return rba_apply_f64(h, inc, l); }
};

inline void check(int rc, bool allow_numerical_failure = false) {
  if (rc == RBA_OK || (allow_numerical_failure && rc == RBA_NUMERICAL_FAILURE)) return;
  throw std::runtime_error(std::string("rootba_b200: ") + rba_last_error());  // the reference CHECK-aborts here
}

// Problem: BalProblem<Scalar> (reference-style AoS + std::map) or BalProblemSoA<Scalar> (flat, from the parallel loader)
template <typename Scalar_, class Problem_ = BalProblem<Scalar_>>
class LinearizorQR {
 public:
  using Scalar = Scalar_;
  using Problem = Problem_;
  using VecX = std::vector<Scalar>;

  static std::unique_ptr<LinearizorQR> create(Problem& bal_problem, const SolverOptions& options, SolverSummary* summary = nullptr) {
    return std::unique_ptr<LinearizorQR>(new LinearizorQR(bal_problem, options, summary));
  }
  ~LinearizorQR() { if (h_) rba_destroy(h_); }

  void start_iteration(IterationSummary* it_summary = nullptr) { it_summary_ = it_summary; }
  void finish_iteration() {}

  void compute_error(ResidualInfo& ri) {
    rba_residual_info r;
    check(rba_compute_error(h_, &r));
    ri.all = {r.all_num_obs, r.all_error, r.all_residual_sum};
    ri.valid = {r.valid_num_obs, r.valid_error, r.valid_residual_sum};
    ri.is_numerically_valid = r.is_numerically_valid != 0;
    if (it_summary_) it_summary_->residual_evaluation_time_in_seconds += timings().residual_evaluation_time;
    if (summary_) summary_->num_residual_evaluations += 1;
  }
  void linearize() {
    check(rba_linearize(h_));  // numerical failure -> throw ("did not expect numerical failure during linearization")
    if (it_summary_) it_summary_->stage1_time_in_seconds = timings().stage1_time;
    if (summary_) summary_->num_jacobian_evaluations += 1;
  }
  VecX solve(Scalar lambda) {
    VecX inc((size_t)9 * bal_problem_.num_cameras());
    rba_cg_summary cg;
    check(Abi<Scalar>::solve(h_, lambda, inc.data(), &cg));
    if (it_summary_) {
      const auto t = timings();
      it_summary_->stage2_time_in_seconds = t.stage2_time;
      it_summary_->compute_preconditioner_time_in_seconds = t.compute_preconditioner_time;
      it_summary_->solve_reduced_system_time_in_seconds = t.solve_reduced_system_time;
      it_summary_->linear_solver_iterations = cg.num_iterations;
    }
    if (summary_) summary_->num_linear_solves += 1;
    return inc;
  }
  Scalar apply(VecX&& inc) {
    Scalar l_diff = 0;
    check(Abi<Scalar>::apply(h_, inc.data(), &l_diff), true);
    if (it_summary_) { const auto t = timings(); it_summary_->back_substitution_time_in_seconds = t.back_substitution_time; it_summary_->update_cameras_time_in_seconds = t.update_cameras_time; }
    return l_diff;
  }
  // BalProblem::backup / restore act on the device-resident state
  void backup() { check(rba_backup(h_)); }
  void restore() { check(rba_restore(h_)); }
  void download_state() {
    std::vector<Scalar> c, l;
    bal_problem_.export_state(c, l);
    check(rba_get_state(h_, c.data(), l.data()));
    bal_problem_.import_state(c, l);
  }
  rba_stage_timings timings() const { rba_stage_timings t; rba_get_timings(h_, &t); return t; }
  rba_workload_stats stats() const { rba_workload_stats s; rba_get_workload_stats(h_, &s); return s; }

 private:
  LinearizorQR(Problem& bp, const SolverOptions& o, SolverSummary* summary) : bal_problem_(bp), summary_(summary) {
    rba_solver_opts so;
    rba_default_solver_opts(&so);
    so.use_householder_marginalization = o.use_householder_marginalization;
    so.use_valid_projections_only = o.use_projection_validity_check();
    so.robust_norm = (int)o.robust_norm;
    so.huber_parameter = o.huber_parameter;
    so.jacobi_scaling_epsilon = o.jacobi_scaling_epsilon;
    so.preconditioner_type = (int)o.preconditioner_type;
    so.min_linear_solver_iterations = o.min_linear_solver_iterations;
    so.max_linear_solver_iterations = o.max_linear_solver_iterations;
    so.eta = o.eta;
    so.device = o.device;
    so.operator_form = o.operator_form;
    so.solver_type = (int)o.solver_type;  // Linearizor::create (linearizor.cpp:48-65): same entry points for the three solvers
    so.power_order = o.power_order;
    so.linear_solver_type = (int)o.linear_solver_type;
    bp.export_topology(lm_off_, obs_cam_, obs_xy_);
    rba_problem_view pv{bp.num_cameras(), bp.num_landmarks(), (int64_t)obs_cam_.size(), lm_off_.data(), obs_cam_.data(), obs_xy_.data()};
    check(Abi<Scalar>::create(&pv, &so, &h_));
    std::vector<Scalar> c, l;
    bp.export_state(c, l);
    check(rba_set_state(h_, c.data(), l.data()));
    if (!bp.camera_fixed.empty()) {
      if ((int)bp.camera_fixed.size() != bp.num_cameras()) throw std::runtime_error("camera_fixed must have one entry per camera");
      check(rba_set_camera_fixed(h_, bp.camera_fixed.data()));
    }
    if (!bp.intrinsics_group.empty()) {
      if ((int)bp.intrinsics_group.size() != bp.num_cameras()) throw std::runtime_error("intrinsics_group must have one entry per camera");
      check(rba_set_intrinsics_groups(h_, bp.intrinsics_group.data()));
    }
    if (!bp.camera_prior_mean.empty() || !bp.camera_prior_sqrt_info.empty()) {
      if (bp.camera_prior_mean.size() != (size_t)10 * bp.num_cameras() || bp.camera_prior_sqrt_info.size() != (size_t)81 * bp.num_cameras())
        throw std::runtime_error("camera priors must have 10 mean and 81 sqrt_info entries per camera");
      const VecX m(bp.camera_prior_mean.begin(), bp.camera_prior_mean.end());
      const VecX L(bp.camera_prior_sqrt_info.begin(), bp.camera_prior_sqrt_info.end());
      check(rba_set_camera_prior(h_, m.data(), L.data()));
    }
    if (!bp.camera_pair_prior_pairs.empty()) {
      const size_t np = bp.camera_pair_prior_pairs.size() / 2;
      if (bp.camera_pair_prior_pairs.size() != 2 * np || bp.camera_pair_prior_mean.size() != 7 * np ||
          bp.camera_pair_prior_sqrt_info.size() != 36 * np)
        throw std::runtime_error("pair priors must have 2 camera indices, 7 mean and 36 sqrt_info entries per pair");
      const VecX m(bp.camera_pair_prior_mean.begin(), bp.camera_pair_prior_mean.end());
      const VecX L(bp.camera_pair_prior_sqrt_info.begin(), bp.camera_pair_prior_sqrt_info.end());
      check(rba_set_camera_pair_prior(h_, (int32_t)np, bp.camera_pair_prior_pairs.data(), m.data(), L.data()));
    }
    if (!bp.landmark_prior_idx.empty()) {
      const size_t np = bp.landmark_prior_idx.size();
      if (bp.landmark_prior_mean.size() != 3 * np || bp.landmark_prior_sqrt_info.size() != 9 * np)
        throw std::runtime_error("landmark priors must have 3 mean and 9 sqrt_info entries per prior");
      const VecX m(bp.landmark_prior_mean.begin(), bp.landmark_prior_mean.end());
      const VecX L(bp.landmark_prior_sqrt_info.begin(), bp.landmark_prior_sqrt_info.end());
      check(rba_set_landmark_prior(h_, (int32_t)np, bp.landmark_prior_idx.data(), m.data(), L.data()));
    }
    if (!bp.obs_sqrt_info.empty()) {
      if ((int64_t)bp.obs_sqrt_info.size() != 4 * (int64_t)bp.num_observations())
        throw std::runtime_error("obs_sqrt_info must have 4 entries (a row-major 2x2) per observation");
      const VecX W(bp.obs_sqrt_info.begin(), bp.obs_sqrt_info.end());
      check(rba_set_observation_info(h_, W.data()));
    }
    if (!bp.obs_loss_kind.empty() || !bp.obs_loss_scale.empty()) {
      if ((int64_t)bp.obs_loss_kind.size() != (int64_t)bp.num_observations() || bp.obs_loss_scale.size() != bp.obs_loss_kind.size())
        throw std::runtime_error("obs_loss_kind and obs_loss_scale must have one entry per observation");
      const VecX a(bp.obs_loss_scale.begin(), bp.obs_loss_scale.end());
      check(rba_set_observation_loss(h_, bp.obs_loss_kind.data(), a.data()));
    }
    const struct { int32_t which; const std::vector<uint8_t>& kind; const std::vector<double>& scale; size_t num; const char* what; } prior_losses[] = {
        {RBA_PRIOR_CAMERA, bp.camera_prior_loss_kind, bp.camera_prior_loss_scale, (size_t)bp.num_cameras(), "camera_prior_loss"},
        {RBA_PRIOR_PAIR, bp.camera_pair_prior_loss_kind, bp.camera_pair_prior_loss_scale, bp.camera_pair_prior_pairs.size() / 2, "camera_pair_prior_loss"},
        {RBA_PRIOR_LANDMARK, bp.landmark_prior_loss_kind, bp.landmark_prior_loss_scale, bp.landmark_prior_idx.size(), "landmark_prior_loss"}};
    for (const auto& l : prior_losses) {
      if (l.kind.empty() && l.scale.empty()) continue;
      if (l.kind.size() != l.num || l.scale.size() != l.num)
        throw std::runtime_error(std::string(l.what) + "_kind and _scale must have one entry per prior of the kind");
      const VecX a(l.scale.begin(), l.scale.end());
      check(rba_set_prior_loss(h_, l.which, (int32_t)l.num, l.kind.data(), a.data()));
    }
  }
  Problem& bal_problem_;
  SolverSummary* summary_ = nullptr;
  IterationSummary* it_summary_ = nullptr;
  rba_handle* h_ = nullptr;
  std::vector<int64_t> lm_off_;
  std::vector<int32_t> obs_cam_;
  std::vector<Scalar> obs_xy_;
};

// optimize_lm_ours (bal_bundle_adjustment.cpp:249-544): the host-serial LM loop.  Generic over the Linearizor (anything
// with the members of rootba::Linearizor, solver/linearizor.hpp:56-82, plus backup / restore / download_state for the
// device-resident state): the GPU LinearizorQR in production, an oracle-backed one in tests/cpp/lm_loop_cpu.cpp.
template <typename Scalar, class Lin>
void optimize_lm(Lin& lin, const SolverOptions& o, SolverSummary& summary, bool quiet = false) {
  Lin* linearizor = &lin;
  using clock = std::chrono::steady_clock;
  const auto since = [](clock::time_point t) { return std::chrono::duration<double>(clock::now() - t).count(); };
  const auto t_total = clock::now();
  const Scalar min_lambda(1.0 / o.max_trust_region_radius), max_lambda(1.0 / o.min_trust_region_radius);
  const Scalar vee_factor(o.vee_factor), initial_vee(o.initial_vee);
  Scalar lambda(1.0 / o.initial_trust_region_radius), lambda_vee(initial_vee);
  auto t_iter = clock::now();
  const auto log_iteration = [&](IterationSummary& s) {  // finish_iteration (bal_bundle_adjustment.cpp:56-88)
    s.iteration_time_in_seconds = since(t_iter);
    s.cumulative_time_in_seconds = summary.preprocessor_time_in_seconds + since(t_total);
    t_iter = clock::now();
    summary.iterations.push_back(s);
  };
  auto cost_of = [&](const ResidualInfo& ri) {
    switch (o.optimized_cost) {
      case SolverOptions::OptimizedCost::ERROR: return ri.all.error;
      case SolverOptions::OptimizedCost::ERROR_VALID: return ri.valid.error;
      default: return ri.valid.error_avg();
    }
  };
  bool terminated = false;
  const int max_lm_iter = o.max_num_iterations;
  for (int it = 0; it <= max_lm_iter && !terminated;) {
    IterationSummary it_summary;
    it_summary.iteration = it;
    linearizor->start_iteration(&it_summary);
    ResidualInfo ri;
    linearizor->compute_error(ri);
    if (!quiet) std::printf("Iteration %d, error: %.4e (mean res: %.2f, num: %lld), error valid: %.4e (num: %lld)\n", it, ri.all.error,
                            ri.all.num_obs ? ri.all.residual_sum / ri.all.num_obs : 0.0, ri.all.num_obs, ri.valid.error, ri.valid.num_obs);
    if (!ri.is_numerically_valid) throw std::runtime_error("did not expect numerical failure during linearization");
    if (it == 0) {
      it_summary.cost = ri; it_summary.trust_region_radius = 1 / (double)lambda;
      it_summary.step_is_successful = it_summary.step_is_valid = true;
      log_iteration(it_summary);
      ++it;
      continue;
    }
    linearizor->linearize();
    if (!quiet) std::printf("\t[INFO] Stage 1 time %.6fs.\n", it_summary.stage1_time_in_seconds);
    for (int j = 0; it <= max_lm_iter && !terminated; ++j) {
      if (j > 0) { it_summary = IterationSummary(); it_summary.iteration = it; linearizor->start_iteration(&it_summary); }
      auto inc = linearizor->solve(lambda);
      if (!quiet) std::printf("\t[INFO] Stage 2 time %.6fs.\n\t[CG] iterations %d Time %.6fs.\n", it_summary.stage2_time_in_seconds,
                              it_summary.linear_solver_iterations, it_summary.solve_reduced_system_time_in_seconds);
      bool finite = true;
      for (Scalar v : inc) finite = finite && std::isfinite(v);
      if (!finite) {
        lambda = lambda_vee * lambda; lambda_vee *= vee_factor;
        it_summary.trust_region_radius = 1 / (double)lambda;
        log_iteration(it_summary);
        ++it;
        if (lambda > max_lambda) { terminated = true; summary.message = "Solver did not converge and reached maximum damping lambda"; }
        continue;
      }
      linearizor->backup();  // bal_problem.backup() (:401) acts on the device-resident state
      Scalar l_diff = linearizor->apply(std::move(inc));
      ResidualInfo ri2;
      linearizor->compute_error(ri2);
      it_summary.cost = ri2;
      if (!std::isfinite(l_diff) || !ri2.is_numerically_valid) {
        it_summary.step_is_valid = it_summary.step_is_successful = false;
      } else {
        Scalar f_diff = Scalar(cost_of(ri) - cost_of(ri2));
        if (o.optimized_cost == SolverOptions::OptimizedCost::ERROR_VALID_AVG) l_diff /= ri.valid.num_obs;
        const Scalar step_quality = f_diff / l_diff;
        if (!quiet) std::printf("\t[EVAL] f_diff %.4e l_diff %.4e step_quality %.4e\n", (double)f_diff, (double)l_diff, (double)step_quality);
        it_summary.relative_decrease = step_quality;
        it_summary.step_is_valid = l_diff > 0;
        it_summary.step_is_successful = it_summary.step_is_valid && step_quality > o.min_relative_decrease;
      }
      if (it_summary.step_is_successful) {
        if (!quiet) std::printf("\t[Success] error: %.4e, lambda: %.1e, cg_iter: %d\n", ri2.all.error, (double)lambda, it_summary.linear_solver_iterations);
        lambda *= Scalar(std::max(1.0 / 3, 1 - std::pow(2 * it_summary.relative_decrease - 1, 3)));
        lambda = std::max(min_lambda, lambda);
        lambda_vee = initial_vee;
        it_summary.trust_region_radius = 1 / (double)lambda;
        const ResidualInfo& prev = summary.iterations.back().cost;
        const bool use_all = o.optimized_cost == SolverOptions::OptimizedCost::ERROR;
        const double pc = use_all ? prev.all.error : prev.valid.error, cc = use_all ? ri2.all.error : ri2.valid.error;
        log_iteration(it_summary);
        ++it;
        if (std::abs(pc - cc) <= o.function_tolerance * cc) { terminated = true; summary.termination_type = "CONVERGENCE"; summary.message = "Function tolerance reached."; }
        break;
      } else {
        if (!quiet) std::printf("\t[%s] error: %.4e, lambda: %.1e, cg_iter: %d\n", it_summary.step_is_valid ? "Reject" : "Invalid", ri2.all.error, (double)lambda, it_summary.linear_solver_iterations);
        lambda = lambda_vee * lambda; lambda_vee *= vee_factor;
        it_summary.trust_region_radius = 1 / (double)lambda;
        log_iteration(it_summary);
        linearizor->restore();  // bal_problem.restore() (:509)
        ++it;
        if (lambda > max_lambda) { terminated = true; summary.message = "Solver did not converge and reached maximum damping lambda"; }
      }
    }
  }
  if (!terminated) summary.message = "Solver did not converge after maximum number of " + std::to_string(max_lm_iter) + " iterations";
  linearizor->download_state();
  summary.minimizer_time_in_seconds = since(t_total);
  summary.total_time_in_seconds = summary.preprocessor_time_in_seconds + summary.minimizer_time_in_seconds;
  if (!quiet) std::printf("%s: %s\n", summary.termination_type.c_str(), summary.message.c_str());
}

// rootba::bundle_adjust_manual (bal_bundle_adjustment.cpp:546-569): create the linearizor, run the LM loop
template <typename Scalar, class Problem>
void bundle_adjust_manual(Problem& bal_problem, const SolverOptions& o, SolverSummary* out = nullptr, bool quiet = false) {
  SolverSummary local;
  SolverSummary& summary = out ? *out : local;
  summary = SolverSummary();
  const auto t0 = std::chrono::steady_clock::now();
  auto linearizor = LinearizorQR<Scalar, Problem>::create(bal_problem, o, &summary);
  summary.preprocessor_time_in_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  optimize_lm<Scalar>(*linearizor, o, summary, quiet);
}

}  // namespace rootba_b200
