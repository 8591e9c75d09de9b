// Host-side mirror of rootba::BalProblem<Scalar> (reference: src/rootba/bal/bal_problem.hpp:61-234,
// bal_problem.cpp:189-282 load_bal, :428-469 normalize, :773-852 load pipeline) without Eigen/Sophus.
// Same conventions after loading: camera looks along +z, image y down, camera state (qx,qy,qz,qw,t,f,k1,k2).
#pragma once

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "bal_io_fast.hpp"  // detail::rot_to_quat, detail::is_bundler_file

namespace rootba_b200 {

template <typename Scalar>
class BalProblem : public ProblemPriors {
 public:
  static constexpr int CAM_STATE_SIZE = 10;  // bal_problem.hpp:72
  using FrameIdx = int;                      // common_types.hpp:44-45

  struct Observation { std::array<Scalar, 2> pos; };
  struct Camera { std::array<Scalar, CAM_STATE_SIZE> params; };  // T_c_w (quat xyzw, t) + intrinsics (f, k1, k2)
  struct Landmark {
    std::array<Scalar, 3> p_w;
    std::map<FrameIdx, Observation> obs;  // ascending camera index, like the reference
  };

  BalProblem() = default;

  // ref: bal_problem.cpp:189-282
  void load_bal(const std::string& path) {
    FILE* f = std::fopen(path.c_str(), "r");
    if (!f) throw std::runtime_error("Could not open '" + path + "'");
    int nc, nl, nobs;
    if (std::fscanf(f, "%d %d %d", &nc, &nl, &nobs) != 3 || nc <= 0 || nl <= 0 || nobs <= 0) fail(f, path);
    cameras_.assign(nc, Camera());
    landmarks_.assign(nl, Landmark());
    for (int i = 0; i < nobs; ++i) {
      int c, l;
      double x, y;
      if (std::fscanf(f, "%d %d %lf %lf", &c, &l, &x, &y) != 4 || c < 0 || c >= nc || l < 0 || l >= nl) fail(f, path);
      auto ins = landmarks_[l].obs.emplace(c, Observation());
      if (!ins.second) fail(f, path);  // duplicate observation (:229-230)
      ins.first->second.pos = {Scalar(x), Scalar(-y)};  // invert y axis (:243)
    }
    for (int i = 0; i < nc; ++i) {
      double p[9];
      for (double& v : p)
        if (std::fscanf(f, "%lf", &v) != 1) fail(f, path);
      double q[4];
      so3_exp(p, q);
      // T_c_w.so3 = axis_inversion * exp(r), axis_inversion = rotation by pi about x = quaternion (1,0,0,0)  (:247,257-258)
      const double ai[4] = {1, 0, 0, 0};
      double qn[4];
      quat_mul(ai, q, qn);
      auto& c = cameras_[i].params;
      c = {Scalar(qn[0]), Scalar(qn[1]), Scalar(qn[2]), Scalar(qn[3]), Scalar(p[3]), Scalar(-p[4]), Scalar(-p[5]),
           Scalar(p[6]), Scalar(p[7]), Scalar(p[8])};
    }
    for (int i = 0; i < nl; ++i) {
      double p[3];
      for (double& v : p)
        if (std::fscanf(f, "%lf", &v) != 1) fail(f, path);
      landmarks_[i].p_w = {Scalar(p[0]), Scalar(p[1]), Scalar(p[2])};
    }
    std::fclose(f);
  }

  // ref: bal_problem.cpp:284-404, reference style: one fscanf per value, std::map per landmark
  void load_bundler(const std::string& path) {
    FILE* f = std::fopen(path.c_str(), "r");
    if (!f) throw std::runtime_error("Could not open '" + path + "'");
    char line[1000];
    bool first = true, done = false;
    while (!done && std::fgets(line, sizeof(line), f)) {  // readcommentline_or_throw (:76-107)
      const size_t len = std::strlen(line);
      if (len == 0 || (first && line[0] != '#')) fail(f, path);
      first = false;
      done = line[len - 1] == '\n';
    }
    int ncf, nl;
    if (!done || std::fscanf(f, "%d %d", &ncf, &nl) != 2 || ncf <= 0 || nl <= 0) fail(f, path);
    cameras_.clear();
    std::vector<int> cam_map(ncf, -1);
    for (int i = 0; i < ncf; ++i) {
      double p[15];
      for (double& v : p)
        if (std::fscanf(f, "%lf", &v) != 1) fail(f, path);
      if (p[0] == 0) continue;  // focal length 0: uninitialised camera
      cam_map[i] = (int)cameras_.size();
      double q[4], qn[4];
      detail::rot_to_quat(p + 3, q);
      const double ai[4] = {1, 0, 0, 0};
      quat_mul(ai, q, qn);
      Camera c;
      c.params = {Scalar(qn[0]), Scalar(qn[1]), Scalar(qn[2]), Scalar(qn[3]), Scalar(p[12]), Scalar(-p[13]), Scalar(-p[14]),
                  Scalar(p[0]), Scalar(p[1]), Scalar(p[2])};
      cameras_.push_back(c);
    }
    landmarks_.assign(nl, Landmark());
    for (int l = 0; l < nl; ++l) {
      double p[3], col[3];
      int n;
      for (double& v : p)
        if (std::fscanf(f, "%lf", &v) != 1) fail(f, path);
      for (double& v : col)
        if (std::fscanf(f, "%lf", &v) != 1) fail(f, path);
      if (std::fscanf(f, "%d", &n) != 1) fail(f, path);
      landmarks_[l].p_w = {Scalar(p[0]), Scalar(p[1]), Scalar(p[2])};
      for (int j = 0; j < n; ++j) {
        int c, key;
        double x, y;
        if (std::fscanf(f, "%d %d %lf %lf", &c, &key, &x, &y) != 4) fail(f, path);
        if (c < 0 || c >= ncf || cam_map[c] < 0) continue;
        auto ins = landmarks_[l].obs.emplace(cam_map[c], Observation());
        if (!ins.second) fail(f, path);
        ins.first->second.pos = {Scalar(x), Scalar(-y)};
      }
    }
    std::fclose(f);
  }

  // ref: bal_problem.cpp:428-469
  void normalize(double new_scale) {
    const int nl = num_landmarks();
    std::vector<Scalar> tmp(nl);
    Scalar median[3];
    for (int j = 0; j < 3; ++j) {
      for (int i = 0; i < nl; ++i) tmp[i] = landmarks_[i].p_w[j];
      median[j] = median_destructive(tmp);
    }
    for (int i = 0; i < nl; ++i) {
      Scalar s = 0;
      for (int j = 0; j < 3; ++j) s += std::abs(landmarks_[i].p_w[j] - median[j]);
      tmp[i] = s;
    }
    const Scalar mad = median_destructive(tmp);
    const Scalar scale = Scalar(new_scale) / mad;
    for (auto& lm : landmarks_)
      for (int j = 0; j < 3; ++j) lm.p_w[j] = scale * (lm.p_w[j] - median[j]);
    for (auto& cam : cameras_) {
      auto& c = cam.params;
      Scalar R[9];
      quat_to_rot(c.data(), R);
      Scalar ctr[3];
      for (int a = 0; a < 3; ++a) ctr[a] = -(R[a] * c[4] + R[3 + a] * c[5] + R[6 + a] * c[6]);
      for (int a = 0; a < 3; ++a) ctr[a] = scale * (ctr[a] - median[a]);
      for (int a = 0; a < 3; ++a) c[4 + a] = -(R[3 * a] * ctr[0] + R[3 * a + 1] * ctr[1] + R[3 * a + 2] * ctr[2]);
    }
  }

  // ref: bal_problem.cpp:471-505
  void filter_obs(double threshold) {
    if (!(threshold > 0)) return;
    for (auto& lm : landmarks_) {
      for (auto it = lm.obs.cbegin(); it != lm.obs.cend();) {
        const auto& c = cameras_.at(it->first).params;
        Scalar R[9];
        quat_to_rot(c.data(), R);
        const Scalar z = R[6] * lm.p_w[0] + R[7] * lm.p_w[1] + R[8] * lm.p_w[2] + c[6];
        if (z < Scalar(threshold)) it = lm.obs.erase(it);
        else ++it;
      }
    }
    std::vector<Landmark> kept;
    for (auto& lm : landmarks_)
      if (lm.obs.size() >= 2) kept.push_back(std::move(lm));
    landmarks_ = std::move(kept);
  }

  // ref: bal_problem.cpp:590-608
  void backup() { cameras_backup_ = cameras_; landmarks_backup_.resize(landmarks_.size()); for (size_t i = 0; i < landmarks_.size(); ++i) landmarks_backup_[i] = landmarks_[i].p_w; }
  void restore() { cameras_ = cameras_backup_; for (size_t i = 0; i < landmarks_.size(); ++i) landmarks_[i].p_w = landmarks_backup_[i]; }

  template <typename Scalar2>
  BalProblem<Scalar2> copy_cast() const {  // bal_problem.hpp:201-219
    BalProblem<Scalar2> r;
    r.cameras().resize(cameras_.size());
    r.landmarks().resize(landmarks_.size());
    for (size_t i = 0; i < cameras_.size(); ++i)
      for (int k = 0; k < CAM_STATE_SIZE; ++k) r.cameras()[i].params[k] = Scalar2(cameras_[i].params[k]);
    for (size_t i = 0; i < landmarks_.size(); ++i) {
      for (int k = 0; k < 3; ++k) r.landmarks()[i].p_w[k] = Scalar2(landmarks_[i].p_w[k]);
      for (const auto& [fid, o] : landmarks_[i].obs) r.landmarks()[i].obs[fid].pos = {Scalar2(o.pos[0]), Scalar2(o.pos[1])};
    }
    return r;
  }

  std::vector<Camera>& cameras() { return cameras_; }
  std::vector<Landmark>& landmarks() { return landmarks_; }
  const std::vector<Camera>& cameras() const { return cameras_; }
  const std::vector<Landmark>& landmarks() const { return landmarks_; }
  int num_cameras() const { return (int)cameras_.size(); }
  int num_landmarks() const { return (int)landmarks_.size(); }
  int64_t num_observations() const { int64_t n = 0; for (const auto& l : landmarks_) n += (int64_t)l.obs.size(); return n; }

  // SoA export for the C ABI (rba_problem_view) and state vectors
  void export_topology(std::vector<int64_t>& lm_off, std::vector<int32_t>& obs_cam, std::vector<Scalar>& obs_xy) const {
    lm_off.assign(landmarks_.size() + 1, 0);
    obs_cam.clear(); obs_xy.clear();
    for (size_t l = 0; l < landmarks_.size(); ++l) {
      lm_off[l] = (int64_t)obs_cam.size();
      for (const auto& [fid, o] : landmarks_[l].obs) { obs_cam.push_back(fid); obs_xy.push_back(o.pos[0]); obs_xy.push_back(o.pos[1]); }
    }
    lm_off[landmarks_.size()] = (int64_t)obs_cam.size();
  }
  void export_state(std::vector<Scalar>& cams, std::vector<Scalar>& lms) const {
    cams.resize((size_t)CAM_STATE_SIZE * cameras_.size()); lms.resize((size_t)3 * landmarks_.size());
    for (size_t i = 0; i < cameras_.size(); ++i) std::copy(cameras_[i].params.begin(), cameras_[i].params.end(), cams.begin() + CAM_STATE_SIZE * i);
    for (size_t i = 0; i < landmarks_.size(); ++i) std::copy(landmarks_[i].p_w.begin(), landmarks_[i].p_w.end(), lms.begin() + 3 * i);
  }
  void import_state(const std::vector<Scalar>& cams, const std::vector<Scalar>& lms) {
    for (size_t i = 0; i < cameras_.size(); ++i) std::copy(cams.begin() + CAM_STATE_SIZE * i, cams.begin() + CAM_STATE_SIZE * (i + 1), cameras_[i].params.begin());
    for (size_t i = 0; i < landmarks_.size(); ++i) std::copy(lms.begin() + 3 * i, lms.begin() + 3 * (i + 1), landmarks_[i].p_w.begin());
  }

 private:
  static void fail(FILE* f, const std::string& path) { std::fclose(f); throw std::runtime_error("Failed to parse '" + path + "'"); }
  static Scalar median_destructive(std::vector<Scalar>& d) {  // bal_problem.cpp:116-122
    auto mid = d.begin() + d.size() / 2;
    std::nth_element(d.begin(), mid, d.end());
    return *mid;
  }
  template <class T>
  static void quat_to_rot(const T* q, T* R) {
    const T x = q[0], y = q[1], z = q[2], w = q[3];
    const T tx = 2 * x, ty = 2 * y, tz = 2 * z, twx = tx * w, twy = ty * w, twz = tz * w;
    const T txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
  }
  static void so3_exp(const double* w, double* q) {  // Sophus SO3::exp
    const double t2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    double im, re;
    if (t2 < 1e-20) { const double t4 = t2 * t2; im = 0.5 - t2 / 48.0 + t4 / 3840.0; re = 1.0 - t2 / 8.0 + t4 / 384.0; }
    else { const double t = std::sqrt(t2); im = std::sin(0.5 * t) / t; re = std::cos(0.5 * t); }
    q[0] = im * w[0]; q[1] = im * w[1]; q[2] = im * w[2]; q[3] = re;
  }
  static void quat_mul(const double* a, const double* b, double* r) {  // Sophus SO3 product with renormalisation
    r[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    r[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    r[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    r[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
    const double sq = r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3];
    if (sq != 1.0) { const double s = 2.0 / (1.0 + sq); for (int i = 0; i < 4; ++i) r[i] *= s; }
  }

  std::vector<Camera> cameras_, cameras_backup_;
  std::vector<Landmark> landmarks_;
  std::vector<std::array<Scalar, 3>> landmarks_backup_;
};

// ref: bal_problem.cpp:773-852 load_normalized_bal_problem: always load + normalise in double, then cast
template <class Scalar>
BalProblem<Scalar> load_normalized_bal_problem(const std::string& path, bool normalize = true, double scale = 100.0,
                                              double init_depth_threshold = 0.0) {
  BalProblem<double> p;
  if (detail::is_bundler_file(path)) p.load_bundler(path);  // autodetect_input_type (bal_problem.cpp:124-135)
  else p.load_bal(path);
  if (normalize) p.normalize(scale);
  p.filter_obs(init_depth_threshold);
  return p.template copy_cast<Scalar>();
}

}  // namespace rootba_b200
