// The C++ host's forwarding of the robust losses on the priors (ProblemPriors::*_prior_loss_*, LinearizorQR::create;
// DESIGN.md section 22), driven by test_gpu_prior_loss.py::test_cpp_host_forwards_the_prior_losses.
//
//   host_prior_loss DIR nc nl nobs npairs nlmp [short]
//
// reads the float64 problem and its priors and losses from the raw files of DIR, creates the handle through
// LinearizorQR<double, BalProblemSoA<double>>::create and prints the cost of rba_compute_error (%.17g).  `short` drops the
// last entry of the pair losses: the host must refuse it (exit code 3, the message on stdout).
#include <cstdio>
#include <fstream>
#include <iostream>
#include <string>

#include "bal_io_fast.hpp"
#include "solver.hpp"

using namespace rootba_b200;

template <class T>
static std::vector<T> read(const std::string& dir, const char* name, size_t n) {
  std::vector<T> v(n);
  std::ifstream f(dir + "/" + name, std::ios::binary);
  if (!f.read(reinterpret_cast<char*>(v.data()), (std::streamsize)(n * sizeof(T)))) throw std::runtime_error(std::string("cannot read ") + name);
  return v;
}

int main(int argc, char** argv) {
  if (argc < 7) { std::cerr << "usage: host_prior_loss DIR nc nl nobs npairs nlmp [short]\n"; return 2; }
  const std::string dir = argv[1];
  const size_t nc = std::stoul(argv[2]), nl = std::stoul(argv[3]), nobs = std::stoul(argv[4]), np = std::stoul(argv[5]),
               nm = std::stoul(argv[6]);
  BalProblemSoA<double> p;
  p.nc = (int)nc; p.nl = (int)nl;
  p.cams = read<double>(dir, "cams", 10 * nc); p.lms = read<double>(dir, "lms", 3 * nl);
  p.lm_off = read<int64_t>(dir, "lm_off", nl + 1); p.obs_cam = read<int32_t>(dir, "obs_cam", nobs);
  p.obs_xy = read<double>(dir, "obs_xy", 2 * nobs);
  p.camera_prior_mean = read<double>(dir, "cmean", 10 * nc); p.camera_prior_sqrt_info = read<double>(dir, "cL", 81 * nc);
  p.camera_pair_prior_pairs = read<int32_t>(dir, "pairs", 2 * np); p.camera_pair_prior_mean = read<double>(dir, "pmean", 7 * np);
  p.camera_pair_prior_sqrt_info = read<double>(dir, "pL", 36 * np);
  p.landmark_prior_idx = read<int32_t>(dir, "lidx", nm); p.landmark_prior_mean = read<double>(dir, "lmean", 3 * nm);
  p.landmark_prior_sqrt_info = read<double>(dir, "lL", 9 * nm);
  p.camera_prior_loss_kind = read<uint8_t>(dir, "ck", nc); p.camera_prior_loss_scale = read<double>(dir, "cs", nc);
  p.camera_pair_prior_loss_kind = read<uint8_t>(dir, "pk", np); p.camera_pair_prior_loss_scale = read<double>(dir, "ps", np);
  p.landmark_prior_loss_kind = read<uint8_t>(dir, "lk", nm); p.landmark_prior_loss_scale = read<double>(dir, "ls", nm);
  if (argc > 7 && std::string(argv[7]) == "short") p.camera_pair_prior_loss_kind.pop_back();
  SolverOptions o;
  try {
    auto lin = LinearizorQR<double, BalProblemSoA<double>>::create(p, o);
    ResidualInfo ri;
    lin->compute_error(ri);
    std::printf("%.17g\n", ri.all.error);
  } catch (const std::exception& e) {
    std::printf("%s\n", e.what());
    return 3;
  }
  return 0;
}
