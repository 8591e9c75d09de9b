// Parallel BAL text loader + flat (SoA) problem container for the GPU linearizor.
//
// Reference behaviour reproduced (src/rootba/bal/bal_problem.cpp:189-282 load_bal, :428-469 normalize,
// :773-852 load pipeline): whitespace-separated tokens "Nc Nl Nobs", then Nobs x (cam lm x y), then 9 values per
// camera (Rodrigues, t, f, k1, k2) and 3 per landmark; image y and the camera y/z axes are flipped; per landmark the
// observations end up in ascending camera order (the reference keeps them in a std::map, bal_problem.hpp:137);
// a duplicate (cam, lm) pair or a short / malformed file is fatal.  Values are parsed with std::from_chars, which is
// correctly rounded like glibc's fscanf("%lf"), so the result is bit-identical to the reference-style loader in
// bal_problem.hpp (tests/test_host_cpp.py compares the two byte by byte).
//
// What is different: the reference reads 29 M lines of Final-13682 with one fscanf per line into one std::map node per
// observation; here the file is read with one pread stream per thread, cut into one chunk per thread at token boundaries, tokens are counted
// (pass 1) and parsed in place (pass 2) straight into flat arrays, and the by-landmark CSR the C ABI wants
// (rba_problem_view) is built with a parallel counting sort.
#pragma once

#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <charconv>
#include <cmath>
#include <cstdint>
#include <chrono>
#include <functional>
#include <memory>
#include <stdexcept>
#include <string>
#include <random>
#include <thread>
#include <utility>
#include <vector>

namespace rootba_b200 {

namespace detail {

inline bool is_ws(char c) { return c == ' ' || c == '\n' || c == '\t' || c == '\r' || c == '\f' || c == '\v'; }

inline void parallel_for(int nthreads, const std::function<void(int)>& body) {
  if (nthreads <= 1) { body(0); return; }
  std::vector<std::thread> pool;
  pool.reserve(nthreads);
  for (int t = 0; t < nthreads; ++t) pool.emplace_back(body, t);
  for (auto& th : pool) th.join();
}

// Sophus SO3::exp and group product with renormalisation, as in bal_problem.hpp of this directory
inline void so3_exp(const double* w, double* q) {
  const double t2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  double im, re;
  if (t2 < 1e-20) { const double t4 = t2 * t2; im = 0.5 - t2 / 48.0 + t4 / 3840.0; re = 1.0 - t2 / 8.0 + t4 / 384.0; }
  else { const double t = std::sqrt(t2); im = std::sin(0.5 * t) / t; re = std::cos(0.5 * t); }
  q[0] = im * w[0]; q[1] = im * w[1]; q[2] = im * w[2]; q[3] = re;
}
inline void quat_mul(const double* a, const double* b, double* r) {
  r[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  r[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  r[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  r[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  const double sq = r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3];
  if (sq != 1.0) { const double s = 2.0 / (1.0 + sq); for (int i = 0; i < 4; ++i) r[i] *= s; }
}

// Eigen::Quaternion(rotation matrix) as Sophus::SO3(R) uses it: trace branch / largest-diagonal branch.
// R row-major, q = (x, y, z, w).
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

// autodetect_input_type (bal_problem.cpp:124-135): "bundle" in the file name -> bundler, else BAL (.cereal is not supported)
inline bool is_bundler_file(const std::string& path) {
  const size_t slash = path.find_last_of('/');
  return (slash == std::string::npos ? path : path.substr(slash + 1)).find("bundle") != std::string::npos;
}

// Whole file in memory, read with one pread stream per thread (parallel first touch; faster than faulting an mmap
// in page by page from the parsing threads).
struct FileBuffer {
  std::unique_ptr<char[]> buf;
  const char* data = nullptr;
  size_t size = 0;
  FileBuffer(const std::string& path, int nthreads) {
    const int fd = ::open(path.c_str(), O_RDONLY);
    if (fd < 0) throw std::runtime_error("Could not open '" + path + "'");
    struct stat st;
    if (::fstat(fd, &st) != 0 || st.st_size <= 0) { ::close(fd); throw std::runtime_error("Failed to parse '" + path + "'"); }
    size = (size_t)st.st_size;
    buf.reset(new char[size]);
    data = buf.get();
    const int nt = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::max(1, nthreads), size >> 20));
    std::atomic<int> err{0};
    parallel_for(nt, [&](int t) {
      size_t off = size / nt * t;
      const size_t end = t == nt - 1 ? size : size / nt * (t + 1);
      while (off < end) {
        const ssize_t r = ::pread(fd, buf.get() + off, end - off, (off_t)off);
        if (r <= 0) { err.store(1); return; }
        off += (size_t)r;
      }
    });
    ::close(fd);
    if (err.load()) throw std::runtime_error("Could not read '" + path + "'");
  }
};

}  // namespace detail

// Held cameras, priors and observation information of a problem (not in the reference), forwarded by LinearizorQR::create; an empty field = none.
// Both problem classes (BalProblemSoA, BalProblem) carry them.
struct ProblemPriors {
  std::vector<uint8_t> camera_fixed;               // [nc] RBA_FIX_* bits (rba_set_camera_fixed)
  std::vector<int32_t> intrinsics_group;           // [nc] group id, -1 = own intrinsics (rba_set_intrinsics_groups); empty = none
  // Gaussian camera priors (rba_set_camera_prior)
  std::vector<double> camera_prior_mean;           // [nc][10] qx,qy,qz,qw (R0), camera centre c0, f0, k1_0, k2_0
  std::vector<double> camera_prior_sqrt_info;      // [nc][81] row-major square-root information L
  // Relative pose priors between pairs of cameras (rba_set_camera_pair_prior)
  std::vector<int32_t> camera_pair_prior_pairs;    // [m][2] cameras (i, j)
  std::vector<double> camera_pair_prior_mean;      // [m][7] qx,qy,qz,qw (R0), t0 of T_i T_j^-1
  std::vector<double> camera_pair_prior_sqrt_info; // [m][36] row-major square-root information L
  // Gaussian priors on landmark positions (rba_set_landmark_prior)
  std::vector<int32_t> landmark_prior_idx;         // [m] landmark indices
  std::vector<double> landmark_prior_mean;         // [m][3] prior position x0
  std::vector<double> landmark_prior_sqrt_info;    // [m][9] row-major square-root information L
  // Square-root information of the observations (rba_set_observation_info)
  std::vector<double> obs_sqrt_info;               // [nobs][4] row-major 2x2 W in the order of the observations; 0 = switched off
  // Robust loss per observation (rba_set_observation_loss); both empty = the options' robust norm everywhere
  std::vector<uint8_t> obs_loss_kind;              // [nobs] RBA_LOSS_*
  std::vector<double> obs_loss_scale;              // [nobs] scale (inlier threshold in units of sigma; ignored for NONE)
  // Robust loss per prior (rba_set_prior_loss), one entry per camera / pair / landmark prior in the order above; both empty = NONE
  std::vector<uint8_t> camera_prior_loss_kind;     // [nc] RBA_LOSS_*
  std::vector<double> camera_prior_loss_scale;     // [nc] threshold on |L e|
  std::vector<uint8_t> camera_pair_prior_loss_kind;
  std::vector<double> camera_pair_prior_loss_scale;
  std::vector<uint8_t> landmark_prior_loss_kind;
  std::vector<double> landmark_prior_loss_scale;
};

// Flat mirror of rootba::BalProblem<Scalar> with the member surface LinearizorQR / bundle_adjust_manual need.
template <typename Scalar>
class BalProblemSoA : public ProblemPriors {
 public:
  static constexpr int CAM_STATE_SIZE = 10;  // bal_problem.hpp:72

  int nc = 0, nl = 0;
  std::vector<Scalar> cams;       // [nc][10]  T_c_w (quat xyzw, t) + (f, k1, k2)
  std::vector<Scalar> lms;        // [nl][3]
  std::vector<int64_t> lm_off;    // [nl + 1]
  std::vector<int32_t> obs_cam;   // ascending inside a landmark
  std::vector<Scalar> obs_xy;     // [nobs][2]

  int num_cameras() const { return nc; }
  int num_landmarks() const { return nl; }
  int64_t num_observations() const { return (int64_t)obs_cam.size(); }

  void export_topology(std::vector<int64_t>& off, std::vector<int32_t>& oc, std::vector<Scalar>& xy) const { off = lm_off; oc = obs_cam; xy = obs_xy; }
  void export_state(std::vector<Scalar>& c, std::vector<Scalar>& l) const { c = cams; l = lms; }
  void import_state(const std::vector<Scalar>& c, const std::vector<Scalar>& l) { cams = c; lms = l; }
  void backup() { cams_backup_ = cams; lms_backup_ = lms; }     // bal_problem.cpp:590-598
  void restore() { cams = cams_backup_; lms = lms_backup_; }    // bal_problem.cpp:600-608

  // ref: bal_problem.cpp:428-469 (same operation order as BalProblem::normalize in bal_problem.hpp)
  void normalize(double new_scale) {
    std::vector<Scalar> tmp(nl);
    Scalar median[3];
    for (int j = 0; j < 3; ++j) {
      for (int i = 0; i < nl; ++i) tmp[i] = lms[3 * (size_t)i + j];
      median[j] = median_destructive(tmp);
    }
    for (int i = 0; i < nl; ++i) {
      Scalar s = 0;
      for (int j = 0; j < 3; ++j) s += std::abs(lms[3 * (size_t)i + j] - median[j]);
      tmp[i] = s;
    }
    const Scalar mad = median_destructive(tmp);
    const Scalar scale = Scalar(new_scale) / mad;
    for (int i = 0; i < nl; ++i)
      for (int j = 0; j < 3; ++j) lms[3 * (size_t)i + j] = scale * (lms[3 * (size_t)i + j] - median[j]);
    for (int i = 0; i < nc; ++i) {
      Scalar* c = cams.data() + (size_t)CAM_STATE_SIZE * i;
      Scalar R[9];
      quat_to_rot(c, R);
      Scalar ctr[3];
      for (int a = 0; a < 3; ++a) ctr[a] = -(R[a] * c[4] + R[3 + a] * c[5] + R[6 + a] * c[6]);
      for (int a = 0; a < 3; ++a) ctr[a] = scale * (ctr[a] - median[a]);
      for (int a = 0; a < 3; ++a) c[4 + a] = -(R[3 * a] * ctr[0] + R[3 * a + 1] * ctr[1] + R[3 * a + 2] * ctr[2]);
    }
  }

  // ref: bal_problem.cpp:507-554 BalProblem::perturb (+ perturbation<T, N>, :105-114): camera centre in world coordinates
  // += N(0, translation_sigma), rotation <- exp(N(0, rotation_sigma)) * rotation, landmark += N(0, landmark_sigma); one
  // std::default_random_engine seeded with `seed` (seed < 0: std::random_device), a FRESH std::normal_distribution<double>
  // per 3-vector exactly like the reference -- with libstdc++ (what a GCC build of the reference links) the random stream
  // is therefore the reference's.  Runs in double before the cast to Scalar (bal_problem.cpp:820-826).
  void perturb(double rotation_sigma, double translation_sigma, double landmark_sigma, int seed) {
    static_assert(std::is_same<Scalar, double>::value, "perturb runs on the double problem, like the reference pipeline");
    std::default_random_engine eng = seed < 0 ? std::default_random_engine{std::random_device{}()}
                                              : std::default_random_engine{static_cast<std::default_random_engine::result_type>(seed)};
    auto perturbation = [&](double sigma, double* v) {
      std::normal_distribution<double> normal;
      for (int i = 0; i < 3; ++i) v[i] = 0.0 + normal(eng) * sigma;
    };
    if (rotation_sigma > 0 || translation_sigma > 0) {
      for (int i = 0; i < nc; ++i) {
        Scalar* c = cams.data() + (size_t)CAM_STATE_SIZE * i;
        if (translation_sigma > 0) {  // T_w_c.translation() += d ; T_c_w = T_w_c^-1  (rotation unchanged)
          Scalar R[9], ctr[3], d[3];
          quat_to_rot(c, R);
          for (int a = 0; a < 3; ++a) ctr[a] = -(R[a] * c[4] + R[3 + a] * c[5] + R[6 + a] * c[6]);
          perturbation(translation_sigma, d);
          for (int a = 0; a < 3; ++a) ctr[a] += d[a];
          for (int a = 0; a < 3; ++a) c[4 + a] = -(R[3 * a] * ctr[0] + R[3 * a + 1] * ctr[1] + R[3 * a + 2] * ctr[2]);
        }
        if (rotation_sigma > 0) {     // so3 <- exp(w) * so3 (translation unchanged, as the reference sets only .so3())
          double w[3], q[4], qn[4];
          perturbation(rotation_sigma, w);
          detail::so3_exp(w, q);
          detail::quat_mul(q, c, qn);
          for (int a = 0; a < 4; ++a) c[a] = qn[a];
        }
      }
    }
    if (landmark_sigma > 0)
      for (int i = 0; i < nl; ++i) {
        double d[3];
        perturbation(landmark_sigma, d);
        for (int a = 0; a < 3; ++a) lms[3 * (size_t)i + a] += d[a];
      }
  }

  // ref: bal_problem.cpp:471-505: drop observations with depth (z of T_c_w * p_w) below the threshold, then landmarks with
  // fewer than 2 observations left; threshold <= 0 is a no-op.  Same arithmetic as BalProblem::filter_obs (bal_problem.hpp).
  void filter_obs(double threshold) {
    if (!(threshold > 0)) return;
    std::vector<Scalar> nlms, nxy;
    std::vector<int64_t> noff(1, 0);
    std::vector<int32_t> ncam;
    for (int l = 0; l < nl; ++l) {
      const Scalar* p = lms.data() + 3 * (size_t)l;
      const size_t keep_from = ncam.size();
      for (int64_t k = lm_off[l]; k < lm_off[l + 1]; ++k) {
        const Scalar* c = cams.data() + (size_t)CAM_STATE_SIZE * obs_cam[k];
        Scalar R[9];
        quat_to_rot(c, R);
        const Scalar z = R[6] * p[0] + R[7] * p[1] + R[8] * p[2] + c[6];
        if (z < Scalar(threshold)) continue;
        ncam.push_back(obs_cam[k]);
        nxy.push_back(obs_xy[2 * k]);
        nxy.push_back(obs_xy[2 * k + 1]);
      }
      if (ncam.size() - keep_from >= 2) {
        nlms.insert(nlms.end(), p, p + 3);
        noff.push_back((int64_t)ncam.size());
      } else {
        ncam.resize(keep_from);
        nxy.resize(2 * keep_from);
      }
    }
    lms.swap(nlms); obs_xy.swap(nxy); lm_off.swap(noff); obs_cam.swap(ncam);
    nl = (int)lm_off.size() - 1;
  }

  template <typename Scalar2>
  BalProblemSoA<Scalar2> copy_cast() const {  // bal_problem.hpp:201-219
    BalProblemSoA<Scalar2> r;
    r.nc = nc; r.nl = nl;
    r.cams.assign(cams.begin(), cams.end());
    r.lms.assign(lms.begin(), lms.end());
    r.lm_off = lm_off; r.obs_cam = obs_cam;
    r.obs_xy.assign(obs_xy.begin(), obs_xy.end());
    return r;
  }

 private:
  static Scalar median_destructive(std::vector<Scalar>& d) {  // bal_problem.cpp:116-122
    auto mid = d.begin() + d.size() / 2;
    std::nth_element(d.begin(), mid, d.end());
    return *mid;
  }
  static void quat_to_rot(const Scalar* q, Scalar* R) {
    const Scalar x = q[0], y = q[1], z = q[2], w = q[3];
    const Scalar tx = 2 * x, ty = 2 * y, tz = 2 * z, twx = tx * w, twy = ty * w, twz = tz * w;
    const Scalar txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
  }
  std::vector<Scalar> cams_backup_, lms_backup_;
};

struct LoadTimings { double read = 0, count = 0, parse = 0, csr = 0; };  // seconds per phase

// ref: bal_problem.cpp:189-282, parallel.  nthreads <= 0: all hardware threads.
inline BalProblemSoA<double> load_bal_parallel(const std::string& path, int nthreads = 0, LoadTimings* timings = nullptr) {
  using detail::is_ws;
  using clock = std::chrono::steady_clock;
  const auto fail = [&](const char* why) -> void { throw std::runtime_error("Failed to parse '" + path + "' (" + why + ")"); };
  auto tp = clock::now();
  const auto lap = [&](double LoadTimings::*m) {
    const auto now = clock::now();
    if (timings) timings->*m += std::chrono::duration<double>(now - tp).count();
    tp = now;
  };
  if (nthreads <= 0) nthreads = (int)std::max(1u, std::thread::hardware_concurrency());
  detail::FileBuffer mf(path, nthreads);
  const char* d = mf.data;
  const size_t size = mf.size;
  nthreads = (int)std::min<size_t>(nthreads, std::max<size_t>(1, size >> 16));
  lap(&LoadTimings::read);

  // ---- header ----
  size_t pos = 0;
  long long hdr[3];
  for (long long& h : hdr) {
    while (pos < size && is_ws(d[pos])) ++pos;
    size_t e = pos;
    while (e < size && !is_ws(d[e])) ++e;
    const auto r = std::from_chars(d + pos, d + e, h);
    if (r.ec != std::errc() || r.ptr != d + e || h <= 0 || h > INT32_MAX) fail("header");
    pos = e;
  }
  const int nc = (int)hdr[0], nl = (int)hdr[1];
  const int64_t nobs = hdr[2];
  const int64_t n_obs_tok = 4 * nobs, n_cam_tok = 9LL * nc, n_tok = n_obs_tok + n_cam_tok + 3LL * nl;

  // ---- chunks at token boundaries ----
  std::vector<size_t> cut(nthreads + 1);
  for (int t = 0; t <= nthreads; ++t) {
    size_t b = t == nthreads ? size : pos + (size - pos) / nthreads * t;
    if (t > 0 && t < nthreads && b > pos && !is_ws(d[b - 1]))
      while (b < size && !is_ws(d[b])) ++b;  // do not start inside a token
    cut[t] = b;
  }
  // ---- pass 1: tokens per chunk ----
  std::vector<int64_t> tok0(nthreads + 1, 0);
  detail::parallel_for(nthreads, [&](int t) {
    int64_t cnt = 0;
    bool prev_ws = true;
    for (size_t i = cut[t]; i < cut[t + 1]; ++i) {
      const bool w = is_ws(d[i]);
      cnt += (prev_ws && !w);
      prev_ws = w;
    }
    tok0[t + 1] = cnt;
  });
  for (int t = 0; t < nthreads; ++t) tok0[t + 1] += tok0[t];
  if (tok0[nthreads] < n_tok) fail("file ends early");
  lap(&LoadTimings::count);

  // ---- pass 2: parse in place ----
  std::vector<int32_t> rec_cam((size_t)nobs), rec_lm((size_t)nobs);
  std::vector<double> rec_xy((size_t)2 * nobs), cam_raw((size_t)n_cam_tok);
  BalProblemSoA<double> out;
  out.nc = nc; out.nl = nl;
  out.lms.resize((size_t)3 * nl);
  std::vector<std::atomic<int32_t>> count((size_t)nl);
  for (auto& c : count) c.store(0, std::memory_order_relaxed);
  std::atomic<int> bad{0};
  detail::parallel_for(nthreads, [&](int t) {
    int64_t k = tok0[t];
    size_t i = cut[t];
    const size_t end = cut[t + 1];
    while (k < n_tok) {
      while (i < end && is_ws(d[i])) ++i;
      if (i >= end) break;
      size_t e = i;
      while (e < size && !is_ws(d[e])) ++e;
      const char* a = d + i;
      const char* b = d + e;
      if (k < n_obs_tok && (k & 3) < 2) {
        int v = -1;
        const auto r = std::from_chars(a, b, v);
        const int lim = (k & 3) == 0 ? nc : nl;
        if (r.ec != std::errc() || r.ptr != b || v < 0 || v >= lim) { bad.store(1); return; }
        if ((k & 3) == 0) rec_cam[(size_t)(k >> 2)] = v;
        else { rec_lm[(size_t)(k >> 2)] = v; count[v].fetch_add(1, std::memory_order_relaxed); }
      } else {
        if (*a == '+') ++a;  // from_chars does not take a leading plus sign, fscanf does
        double v = 0;
        const auto r = std::from_chars(a, b, v);
        if (r.ec != std::errc() || r.ptr != b) { bad.store(2); return; }
        if (k < n_obs_tok) rec_xy[(size_t)(2 * (k >> 2) + ((k & 3) - 2))] = (k & 3) == 3 ? -v : v;  // invert y axis (:243)
        else if (k < n_obs_tok + n_cam_tok) cam_raw[(size_t)(k - n_obs_tok)] = v;
        else out.lms[(size_t)(k - n_obs_tok - n_cam_tok)] = v;
      }
      ++k;
      i = e;
    }
  });
  if (bad.load()) fail(bad.load() == 1 ? "bad camera / landmark index" : "bad number");
  lap(&LoadTimings::parse);

  // ---- CSR by landmark, ascending camera inside a landmark ----
  out.lm_off.assign((size_t)nl + 1, 0);
  for (int l = 0; l < nl; ++l) out.lm_off[l + 1] = out.lm_off[l] + count[l].load(std::memory_order_relaxed);
  // BAL files normally list the observations landmark by landmark with ascending cameras: then the parsed records
  // already are the CSR (a strictly increasing (lm, cam) key also rules out duplicates).
  std::atomic<int> unsorted{0};
  detail::parallel_for(nthreads, [&](int t) {
    const int64_t r0 = std::max<int64_t>(1, nobs * t / nthreads), r1 = nobs * (t + 1) / nthreads;
    for (int64_t r = r0; r < r1; ++r) {
      const int32_t la = rec_lm[(size_t)(r - 1)], lb = rec_lm[(size_t)r];
      if (lb < la || (lb == la && rec_cam[(size_t)r] <= rec_cam[(size_t)(r - 1)])) { unsorted.store(1, std::memory_order_relaxed); return; }
    }
  });
  if (!unsorted.load()) {
    out.obs_cam = std::move(rec_cam);
    out.obs_xy = std::move(rec_xy);
  } else {
    out.obs_cam.resize((size_t)nobs);
    out.obs_xy.resize((size_t)2 * nobs);
    std::unique_ptr<int64_t[]> src(new int64_t[(size_t)nobs]);
    for (auto& c : count) c.store(0, std::memory_order_relaxed);
    detail::parallel_for(nthreads, [&](int t) {
      const int64_t r0 = nobs * t / nthreads, r1 = nobs * (t + 1) / nthreads;
      for (int64_t r = r0; r < r1; ++r) {
        const int l = rec_lm[(size_t)r];
        src[(size_t)(out.lm_off[l] + count[l].fetch_add(1, std::memory_order_relaxed))] = r;
      }
    });
    detail::parallel_for(nthreads, [&](int t) {
      const int l0 = (int)((int64_t)nl * t / nthreads), l1 = (int)((int64_t)nl * (t + 1) / nthreads);
      std::vector<std::pair<int32_t, int64_t>> seg;
      for (int l = l0; l < l1; ++l) {
        const int64_t b = out.lm_off[l], e = out.lm_off[l + 1];
        seg.clear();
        for (int64_t s = b; s < e; ++s) seg.emplace_back(rec_cam[(size_t)src[(size_t)s]], src[(size_t)s]);
        std::sort(seg.begin(), seg.end());
        for (int64_t s = b; s < e; ++s) {
          const auto& p = seg[(size_t)(s - b)];
          if (s > b && p.first == seg[(size_t)(s - b - 1)].first) { bad.store(3); return; }  // duplicate observation (:229-230)
          out.obs_cam[(size_t)s] = p.first;
          out.obs_xy[(size_t)(2 * s)] = rec_xy[(size_t)(2 * p.second)];
          out.obs_xy[(size_t)(2 * s + 1)] = rec_xy[(size_t)(2 * p.second + 1)];
        }
      }
    });
  }
  if (bad.load()) fail("duplicate observation");
  lap(&LoadTimings::csr);

  // ---- cameras: T_c_w.so3 = axis_inversion * exp(r), t = (t0, -t1, -t2)  (:247, 257-258) ----
  out.cams.resize((size_t)BalProblemSoA<double>::CAM_STATE_SIZE * nc);
  for (int i = 0; i < nc; ++i) {
    const double* p = cam_raw.data() + 9 * (size_t)i;
    double q[4], qn[4];
    detail::so3_exp(p, q);
    const double ai[4] = {1, 0, 0, 0};
    detail::quat_mul(ai, q, qn);
    double* c = out.cams.data() + 10 * (size_t)i;
    c[0] = qn[0]; c[1] = qn[1]; c[2] = qn[2]; c[3] = qn[3];
    c[4] = p[3]; c[5] = -p[4]; c[6] = -p[5];
    c[7] = p[6]; c[8] = p[7]; c[9] = p[8];
  }
  return out;
}

// ref: bal_problem.cpp:284-404  load_bundler ("bundle.out" v0.3).  View lists have variable length, so the token stream is
// walked once, sequentially, over the in-memory file (these files are small next to the BAL "final" problems).
inline BalProblemSoA<double> load_bundler_soa(const std::string& path, int nthreads = 0) {
  using detail::is_ws;
  const auto fail = [&](const char* why) -> void { throw std::runtime_error("Failed to parse '" + path + "' (" + why + ")"); };
  if (nthreads <= 0) nthreads = (int)std::max(1u, std::thread::hardware_concurrency());
  detail::FileBuffer fb(path, nthreads);
  const char* d = fb.data;
  const size_t size = fb.size;
  if (d[0] != '#') fail("expected a comment line");  // readcommentline_or_throw (:76-107)
  size_t pos = 0;
  while (pos < size && d[pos] != '\n') ++pos;
  if (pos >= size) fail("expected a comment line");
  ++pos;
  const auto token = [&](const char*& a, const char*& b) {
    while (pos < size && is_ws(d[pos])) ++pos;
    if (pos >= size) fail("file ends early");
    a = d + pos;
    while (pos < size && !is_ws(d[pos])) ++pos;
    b = d + pos;
  };
  const auto next_int = [&]() {
    const char *a, *b;
    token(a, b);
    long long v = 0;
    const auto r = std::from_chars(a, b, v);
    if (r.ec != std::errc() || r.ptr != b) fail("bad integer");
    return v;
  };
  const auto next_double = [&]() {
    const char *a, *b;
    token(a, b);
    if (*a == '+') ++a;
    double v = 0;
    const auto r = std::from_chars(a, b, v);
    if (r.ec != std::errc() || r.ptr != b) fail("bad number");
    return v;
  };
  const long long ncf = next_int(), nlf = next_int();
  if (ncf <= 0 || nlf <= 0 || ncf > INT32_MAX || nlf > INT32_MAX) fail("header");
  BalProblemSoA<double> out;
  std::vector<int> cam_map((size_t)ncf, -1);
  for (long long i = 0; i < ncf; ++i) {
    double p[15];
    for (double& v : p) v = next_double();
    if (p[0] == 0) continue;  // focal length 0: uninitialised camera (:323-326)
    cam_map[(size_t)i] = out.nc++;
    double q[4], qn[4];
    detail::rot_to_quat(p + 3, q);
    const double ai[4] = {1, 0, 0, 0};
    detail::quat_mul(ai, q, qn);
    const double c[10] = {qn[0], qn[1], qn[2], qn[3], p[12], -p[13], -p[14], p[0], p[1], p[2]};
    out.cams.insert(out.cams.end(), c, c + 10);
  }
  out.nl = (int)nlf;
  out.lms.resize((size_t)3 * nlf);
  out.lm_off.assign(1, 0);
  std::vector<std::pair<int32_t, std::array<double, 2>>> v;
  for (long long l = 0; l < nlf; ++l) {
    for (int k = 0; k < 3; ++k) out.lms[(size_t)(3 * l + k)] = next_double();
    for (int k = 0; k < 3; ++k) (void)next_double();  // colour
    const long long n = next_int();
    v.clear();
    for (long long j = 0; j < n; ++j) {
      const long long c = next_int();
      (void)next_int();  // feature key
      const double x = next_double(), y = next_double();
      if (c >= 0 && c < ncf && cam_map[(size_t)c] >= 0) v.push_back({cam_map[(size_t)c], {x, -y}});  // invert y axis (:390)
    }
    std::sort(v.begin(), v.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    for (size_t i = 0; i < v.size(); ++i) {
      if (i > 0 && v[i].first == v[i - 1].first) fail("duplicate observation");  // CHECK(inserted) (:377)
      out.obs_cam.push_back(v[i].first);
      out.obs_xy.push_back(v[i].second[0]);
      out.obs_xy.push_back(v[i].second[1]);
    }
    out.lm_off.push_back((int64_t)out.obs_cam.size());
  }
  return out;
}

// ref: bal_problem.cpp:773-852: load + normalise in double, then cast
template <class Scalar>
BalProblemSoA<Scalar> load_normalized_bal_problem_parallel(const std::string& path, bool normalize = true, double scale = 100.0,
                                                           int nthreads = 0, double init_depth_threshold = 0.0) {
  BalProblemSoA<double> p = detail::is_bundler_file(path) ? load_bundler_soa(path, nthreads) : load_bal_parallel(path, nthreads);
  if (normalize) p.normalize(scale);
  p.filter_obs(init_depth_threshold);  // (the reference perturbs between the two, bal_problem.cpp:818-824; no perturbation here)
  return p.template copy_cast<Scalar>();
}

}  // namespace rootba_b200
