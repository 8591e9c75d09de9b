// bal_qr: square-root BA solver on a BAL file with the GPU linearizor (counterpart of src/app/bal_qr.cpp:44-115).
//   bal_qr --input <bal file> [--no-use-double] [--max-num-iterations N] [--preconditioner-type JACOBI|SCHUR_JACOBI]
//          [--residual-robust-norm NONE|HUBER] [--residual-huber-parameter X] [--no-normalize] [--dump-problem out.bin]
//          [--loader parallel|map] [--num-threads T] [--operator-form dense|implicit] [--init-depth-threshold Z]
//          [--fix-intrinsics] [--fix-cameras I,J,...] [--shared-intrinsics]
//   --loader parallel (default): mmap + multi-threaded parse into flat arrays (bal_io_fast.hpp);
//   --loader map: the reference-style fscanf + std::map loader (bal_problem.hpp).  Both give identical problems.
#include <chrono>
#include <cstring>
#include <fstream>
#include <iostream>

#include "ba_log.hpp"
#include "solver.hpp"

using namespace rootba_b200;

static double seconds_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// camera parameters held constant (rba_set_camera_fixed): --fix-intrinsics, --fix-cameras I,J,...
struct FixOptions {
  bool intrinsics = false;
  bool shared_intrinsics = false;  // every camera in one intrinsics group (rba_set_intrinsics_groups)
  std::vector<long long> cameras;  // indices into the loaded problem
};

// "I,J,..." -> indices; false on an empty or malformed list
static bool parse_camera_list(const std::string& v, std::vector<long long>& out) {
  size_t pos = 0;
  while (true) {
    const size_t end = v.find(',', pos);
    const std::string tok = v.substr(pos, end == std::string::npos ? std::string::npos : end - pos);
    if (tok.empty() || tok.find_first_not_of("0123456789") != std::string::npos || tok.size() > 12) return false;
    out.push_back(std::stoll(tok));
    if (end == std::string::npos) return true;
    pos = end + 1;
  }
}

template <class S, class Problem>
int solve_and_log(Problem& problem, const SolverOptions& o, const FixOptions& fix, const std::string& log_path, const std::string& input, double load_time);

template <class S>
int run(const std::string& input, bool normalize, const SolverOptions& o, const FixOptions& fix, const std::string& log_path, bool parallel_loader, int num_threads,
        double depth_thr) {
  const auto t0 = std::chrono::steady_clock::now();
  if (parallel_loader) {
    auto problem = load_normalized_bal_problem_parallel<S>(input, normalize, 100.0, num_threads, depth_thr);
    std::printf("Loaded BAL problem (%d cams, %d lms, %lld obs) from '%s' in %.3fs (parallel loader)\n", problem.num_cameras(),
                problem.num_landmarks(), (long long)problem.num_observations(), input.c_str(), seconds_since(t0));
    return solve_and_log<S>(problem, o, fix, log_path, input, seconds_since(t0));
  }
  auto problem = load_normalized_bal_problem<S>(input, normalize, 100.0, depth_thr);
  std::printf("Loaded BAL problem (%d cams, %d lms, %lld obs) from '%s' in %.3fs (map loader)\n", problem.num_cameras(),
              problem.num_landmarks(), (long long)problem.num_observations(), input.c_str(), seconds_since(t0));
  return solve_and_log<S>(problem, o, fix, log_path, input, seconds_since(t0));
}

template <class S, class Problem>
int solve_and_log(Problem& problem, const SolverOptions& o, const FixOptions& fix, const std::string& log_path, const std::string& input, double load_time) {
  if (fix.intrinsics || !fix.cameras.empty()) {
    problem.camera_fixed.assign((size_t)problem.num_cameras(), fix.intrinsics ? (uint8_t)RBA_FIX_INTRINSICS : (uint8_t)0);
    for (long long c : fix.cameras) {
      if (c >= problem.num_cameras()) {
        std::cerr << "--fix-cameras: camera " << c << " out of range (the loaded problem has " << problem.num_cameras() << " cameras)\n";
        return 2;
      }
      problem.camera_fixed[(size_t)c] = (uint8_t)RBA_FIX_ALL;
    }
  }
  if (fix.shared_intrinsics) problem.intrinsics_group.assign((size_t)problem.num_cameras(), 0);
  const DatasetSummary ds = summarize_problem<S>(problem, input);
  SolverSummary summary;
  bundle_adjust_manual<S>(problem, o, &summary);
  PipelineTimingSummary pt;
  pt.load_time = load_time;
  pt.optimize_time = summary.total_time_in_seconds;
  // ba_log.json in the reference's format (bal/ba_log.hpp:139-252, ba_log.cpp:62-150), see ba_log.hpp
  if (!write_ba_log(log_path, ds, pt, summary)) { std::cerr << "Could not save BA log to " << log_path << "\n"; return 1; }
  return 0;
}

// --selftest-log: the log writer on a fabricated 4-iteration summary (accepted, rejected, accepted) -- no GPU needed
static int selftest_log(const std::string& path) {
  SolverSummary s;
  s.termination_type = "CONVERGENCE";
  s.message = "Function tolerance reached.";
  const double costs[4] = {100.0, 40.0, 55.0, 39.99999};
  const bool ok[4] = {true, true, false, true};
  for (int i = 0; i < 4; ++i) {
    IterationSummary it;
    it.iteration = i;
    it.cost.all = {10, costs[i], 10 * std::sqrt(costs[i])};
    it.cost.valid = {9, 0.9 * costs[i], 9 * std::sqrt(costs[i])};
    it.step_is_valid = true;
    it.step_is_successful = ok[i];
    it.trust_region_radius = 1e4 * (i + 1);
    it.relative_decrease = i ? 0.5 : 0.0;
    it.linear_solver_iterations = 3 * i;
    it.stage1_time_in_seconds = i ? 0.001 : 0.0;
    it.stage2_time_in_seconds = 0.002 * i;
    it.solve_reduced_system_time_in_seconds = 0.01 * i;
    it.back_substitution_time_in_seconds = 0.0005 * i;
    it.iteration_time_in_seconds = 0.02;
    it.cumulative_time_in_seconds = 0.02 * (i + 1);
    s.iterations.push_back(it);
  }
  s.num_linear_solves = 3; s.num_residual_evaluations = 7; s.num_jacobian_evaluations = 2;
  s.total_time_in_seconds = 0.08; s.minimizer_time_in_seconds = 0.07; s.preprocessor_time_in_seconds = 0.01;
  BalProblemSoA<double> p;
  p.nc = 3; p.nl = 2;
  p.lm_off = {0, 2, 5}; p.obs_cam = {0, 1, 0, 1, 2}; p.obs_xy.assign(10, 0.0);
  const DatasetSummary ds = summarize_problem<double>(p, "selftest \"quoted\" path");
  PipelineTimingSummary pt;
  pt.load_time = 0.5; pt.optimize_time = 0.08;
  return write_ba_log(path, ds, pt, s) ? 0 : 1;
}

int main(int argc, char** argv) {
  std::string input, dump, log_path = "ba_log.json";
  bool use_double = true, normalize = true, parallel_loader = true;
  int num_threads = 0;
  double depth_thr = 0.0;  // BalDatasetOptions::init_depth_threshold (bal_dataset_options.hpp:82)
  SolverOptions o;
  FixOptions fix;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    auto next = [&]() -> std::string { if (i + 1 >= argc) { std::cerr << "missing value for " << a << "\n"; std::exit(2); } return argv[++i]; };
    if (a == "--input") input = next();
    else if (a == "--no-use-double") use_double = false;
    else if (a == "--use-double") use_double = true;
    else if (a == "--no-normalize") normalize = false;
    else if (a == "--max-num-iterations") o.max_num_iterations = std::stoi(next());
    else if (a == "--max-linear-solver-iterations") o.max_linear_solver_iterations = std::stoi(next());
    else if (a == "--eta") o.eta = std::stod(next());
    else if (a == "--function-tolerance") o.function_tolerance = std::stod(next());
    else if (a == "--preconditioner-type") {
      const std::string v = next();
      if (v == "JACOBI") o.preconditioner_type = SolverOptions::PreconditionerType::JACOBI;
      else if (v == "SCHUR_JACOBI") o.preconditioner_type = SolverOptions::PreconditionerType::SCHUR_JACOBI;
      else if (v == "CLUSTER_JACOBI") o.preconditioner_type = SolverOptions::PreconditionerType::CLUSTER_JACOBI;
      else { std::cerr << "--preconditioner-type JACOBI|SCHUR_JACOBI|CLUSTER_JACOBI\n"; return 2; }
    }
    else if (a == "--residual-robust-norm") { const std::string v = next(); o.robust_norm = v == "HUBER" ? SolverOptions::RobustNorm::HUBER : SolverOptions::RobustNorm::NONE; }
    else if (a == "--residual-huber-parameter") o.huber_parameter = std::stod(next());
    else if (a == "--optimized-cost") { const std::string v = next(); o.optimized_cost = v == "ERROR" ? SolverOptions::OptimizedCost::ERROR : v == "ERROR_VALID" ? SolverOptions::OptimizedCost::ERROR_VALID : SolverOptions::OptimizedCost::ERROR_VALID_AVG; }
    else if (a == "--operator-form") { const std::string v = next(); if (v != "dense" && v != "implicit") { std::cerr << "--operator-form dense|implicit\n"; return 2; } o.operator_form = v == "implicit"; }
    else if (a == "--solver-type") { const std::string v = next(); o.solver_type = v == "SCHUR_COMPLEMENT" ? SolverOptions::SolverType::SCHUR_COMPLEMENT : v == "POWER_SCHUR_COMPLEMENT" ? SolverOptions::SolverType::POWER_SCHUR_COMPLEMENT : SolverOptions::SolverType::SQUARE_ROOT; }
    else if (a == "--power-order") o.power_order = std::stoi(next());
    else if (a == "--linear-solver-type") {
      const std::string v = next();
      if (v != "ITERATIVE_SCHUR" && v != "DENSE_SCHUR") { std::cerr << "--linear-solver-type ITERATIVE_SCHUR|DENSE_SCHUR\n"; return 2; }
      o.linear_solver_type = v == "DENSE_SCHUR" ? SolverOptions::LinearSolverType::DENSE_SCHUR : SolverOptions::LinearSolverType::ITERATIVE_SCHUR;
    }
    else if (a == "--log-path") log_path = next();
    else if (a == "--loader") { const std::string v = next(); if (v != "parallel" && v != "map") { std::cerr << "--loader parallel|map\n"; return 2; } parallel_loader = v == "parallel"; }
    else if (a == "--num-threads") num_threads = std::stoi(next());
    else if (a == "--init-depth-threshold") depth_thr = std::stod(next());
    else if (a == "--dump-problem") dump = next();
    else if (a == "--fix-intrinsics") fix.intrinsics = true;
    else if (a == "--shared-intrinsics") fix.shared_intrinsics = true;
    else if (a == "--fix-cameras") {
      const std::string v = next();
      if (!parse_camera_list(v, fix.cameras)) { std::cerr << "--fix-cameras expects a comma-separated list of camera indices, got '" << v << "'\n"; return 2; }
    }
    else if (a == "--selftest-log") return selftest_log(next());
    else if (a == "--help" || a == "-h") {
      std::cout << "usage: bal_qr --input <bal file> [--no-use-double] [--max-num-iterations N] [--preconditioner-type JACOBI|SCHUR_JACOBI|CLUSTER_JACOBI] ...\n"
                   "  --linear-solver-type ITERATIVE_SCHUR|DENSE_SCHUR\n"
                   "                        the camera increment by truncated PCG (default) or exactly, by a dense Cholesky\n"
                   "                        factorisation of the reduced camera matrix\n"
                   "  --fix-intrinsics      hold f, k1, k2 of every camera constant\n"
                   "  --shared-intrinsics   every camera shares one f, k1, k2 (camera 0's at the start)\n"
                   "  --fix-cameras I,J,... hold every parameter of the listed cameras constant; indices refer to the loaded problem\n"
                   "                        (a Bundler file's cameras with focal length 0 are dropped by the loader first)\n";
      return 0;
    }
    else { std::cerr << "unknown option " << a << "\n"; return 2; }
  }
  if (input.empty()) { std::cerr << "--input is required\n"; return 2; }
  try {
    if (!dump.empty()) {  // loader check (host only, no GPU): normalised double arrays in SoA form
      std::vector<int64_t> off; std::vector<int32_t> oc; std::vector<double> xy, c, l;
      int nc = 0, nl = 0;
      const auto t0 = std::chrono::steady_clock::now();
      if (parallel_loader) {
        auto p = load_normalized_bal_problem_parallel<double>(input, normalize, 100.0, num_threads, depth_thr);
        std::printf("load time %.3fs (parallel loader)\n", seconds_since(t0));
        p.export_topology(off, oc, xy); p.export_state(c, l); nc = p.num_cameras(); nl = p.num_landmarks();
      } else {
        auto p = load_normalized_bal_problem<double>(input, normalize, 100.0, depth_thr);
        std::printf("load time %.3fs (map loader)\n", seconds_since(t0));
        p.export_topology(off, oc, xy); p.export_state(c, l); nc = p.num_cameras(); nl = p.num_landmarks();
      }
      std::ofstream f(dump, std::ios::binary);
      const int64_t hdr[3] = {nc, nl, (int64_t)oc.size()};
      f.write((const char*)hdr, sizeof(hdr));
      f.write((const char*)c.data(), c.size() * 8); f.write((const char*)l.data(), l.size() * 8);
      f.write((const char*)off.data(), off.size() * 8); f.write((const char*)oc.data(), oc.size() * 4); f.write((const char*)xy.data(), xy.size() * 8);
      return 0;
    }
    o.use_double = use_double;
    return use_double ? run<double>(input, normalize, o, fix, log_path, parallel_loader, num_threads, depth_thr)
                      : run<float>(input, normalize, o, fix, log_path, parallel_loader, num_threads, depth_thr);
  } catch (const std::exception& e) {
    std::cerr << "FATAL: " << e.what() << "\n";
    return 1;
  }
}
