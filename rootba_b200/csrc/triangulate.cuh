// Triangulation and per-landmark refinement with the cameras held (rba_triangulate_landmarks, DESIGN.md section 25).
//
// One warp per requested landmark, lanes over its contiguous observation slots (slot0 .. slot0 + n - 1, lane i, i + 32, ...),
// every sum a warp_sum in that fixed order: the result of a landmark depends on its own track only, so it is bit-identical
// across calls, handles, solver configurations and shard counts.  Everything is float64 for either Scalar.
#pragma once

#include "covariance.cuh"

namespace rba {

constexpr int TRI_UNDISTORT_ITERS = 50;     // Newton iterations of the distortion inversion
constexpr double TRI_UNDISTORT_TOL = 1e-12; // converged when the Newton step is <= this * rho
constexpr double TRI_INFINITY = 1e-10;      // |X_h[3]| <= this * |X_h|: the linear estimate is at infinity
constexpr double TRI_LAMBDA0 = 1e-4;        // LM damping: start, bounds, factors
constexpr double TRI_LAMBDA_MIN = 1e-12, TRI_LAMBDA_MAX = 1e16;
constexpr double TRI_DAMP_FLOOR = 1e-12;    // the damping diagonal is max(H_kk, this * max_k H_kk)

struct TriItem {
  int lm;      // local landmark
  int sorted;  // its index in the length-sorted order (D.lmp_slot is indexed by it)
  int slot0;   // first observation slot
  int n;       // track length
};

struct TriOpts {
  int mode;
  int max_iterations;
  double min_angle;
  double ftol;
};

// The normalised image point m with obs / f = m (1 + k1 |m|^2 + k2 |m|^4): rho = |m| solves rho (1 + k1 rho^2 + k2 rho^4) = t,
// t = |obs / f|, by Newton from rho = t.  False (no usable ray) when the derivative 1 + 3 k1 rho^2 + 5 k2 rho^4 is <= 0 at an
// iterate (the final one included) or the iteration does not converge.
__device__ __forceinline__ bool tri_undistort(double u0, double u1, double k1, double k2, double& m0, double& m1) {
  const double t = sqrt(u0 * u0 + u1 * u1);
  if (t == 0.0) { m0 = 0.0; m1 = 0.0; return true; }
  double rho = t;
  bool conv = false;
  for (int it = 0; it <= TRI_UNDISTORT_ITERS; ++it) {
    const double r2 = rho * rho;
    const double g1 = 1.0 + k1 * r2 + k2 * r2 * r2;
    const double d = 1.0 + 3.0 * k1 * r2 + 5.0 * k2 * r2 * r2;
    if (!(d > 0.0)) return false;
    if (conv) { m0 = u0 / g1; m1 = u1 / g1; return true; }
    if (it == TRI_UNDISTORT_ITERS) return false;
    const double step = (rho * g1 - t) / d;
    rho -= step;
    if (!(rho > 0.0) || !isfinite(rho)) return false;
    conv = fabs(step) <= TRI_UNDISTORT_TOL * rho;
  }
  return false;
}

template <class S>
__device__ __forceinline__ void tri_load_cam(const DevPtrs<S>& D, int s, double (&cam)[10]) {
  const S* cp = D.cams + 10 * (size_t)D.slot_cam[s];
#pragma unroll
  for (int k = 0; k < 10; ++k) cam[k] = (double)cp[k];
}

// The landmark's share of the cost at X (rba_compute_error: valid_error with use_valid_projections_only, else all_error) and
// its IRLS normal equations h (00 01 02 11 12 22), g = sum w Jl^T r, the same in every lane.  Per slot, bit `vbit` of
// vb[s] is set to the projection validity at X (z >= eps_sqrt of S) and `lost` reports an observation in use that is valid
// under bit `cbit` and not at X.  A lane reads and writes only the bytes of its own slots.
template <class S>
__device__ __forceinline__ double tri_eval(const DevPtrs<S>& D, const KOpts& o, int s0, int n, int lp, const double* X,
                                          uint8_t* vb, int vbit, int cbit, double (&h)[6], double (&g)[3], bool& lost) {
  const int lane = threadIdx.x & 31;
  double c = 0.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) h[k] = 0.0;
  g[0] = g[1] = g[2] = 0.0;
  bool lo = false;
  for (int i = lane; i < n; i += 32) {
    const int s = s0 + i;
    const double obs[2] = {(double)D.slot_xy[2 * s], (double)D.slot_xy[2 * s + 1]};
    double cam[10];
    tri_load_cam(D, s, cam);
    double res[2], Jp[18], Jl[6];
    linearize_point<double, true>(obs, X, cam, res, Jp, Jl);
    const bool inuse = !(D.obs_W && whiten_observation<double, true>(D.obs_W, s, res, Jp, Jl));
    double R[9];
    quat_to_rot(cam, R);
    const double z = R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + cam[6];
    const bool valid = z >= (double)ST<S>::eps_sqrt();
    unsigned bits = vb[s];
    if (inuse && ((bits >> cbit) & 1u) && !valid) lo = true;
    bits = valid ? (bits | (1u << vbit)) : (bits & ~(1u << vbit));
    vb[s] = (uint8_t)bits;
    if (inuse && (valid || !o.use_valid_projections_only)) {
      const double rsq = res[0] * res[0] + res[1] * res[1];
      double err, w;
      if (D.obs_loss) slot_error_weight<true>(o, D.obs_loss, D.nslots, s, rsq, err, w);
      else error_weight(o, rsq, err, w);
      c += err;
      h[0] += w * (Jl[0] * Jl[0] + Jl[3] * Jl[3]);
      h[1] += w * (Jl[0] * Jl[1] + Jl[3] * Jl[4]);
      h[2] += w * (Jl[0] * Jl[2] + Jl[3] * Jl[5]);
      h[3] += w * (Jl[1] * Jl[1] + Jl[4] * Jl[4]);
      h[4] += w * (Jl[1] * Jl[2] + Jl[4] * Jl[5]);
      h[5] += w * (Jl[2] * Jl[2] + Jl[5] * Jl[5]);
#pragma unroll
      for (int k = 0; k < 3; ++k) g[k] += w * (Jl[k] * res[0] + Jl[3 + k] * res[1]);
    }
  }
  c = warp_sum(c);
#pragma unroll
  for (int k = 0; k < 6; ++k) h[k] = warp_sum(h[k]);
#pragma unroll
  for (int k = 0; k < 3; ++k) g[k] = warp_sum(g[k]);
  lost = __any_sync(0xffffffffu, lo);
  if (lp >= 0) {  // + the landmark prior (sections 17 and 22), the same operations in every lane
    double r[3], err, w = 1.0;
    const double sp = lmp_residual(D, lp, X, r);
    if (D.lmp_loss) lmp_loss(D, lp, sp, err, w);
    else err = 0.5 * sp;
    c += err;
    const S* Lp = D.lmp_Lu + 9 * (size_t)lp;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const double a0 = (double)Lp[3 * i], a1 = (double)Lp[3 * i + 1], a2 = (double)Lp[3 * i + 2];
      h[0] += w * a0 * a0; h[1] += w * a0 * a1; h[2] += w * a0 * a2;
      h[3] += w * a1 * a1; h[4] += w * a1 * a2; h[5] += w * a2 * a2;
      g[0] += w * a0 * r[i]; g[1] += w * a1 * r[i]; g[2] += w * a2 * r[i];
    }
  }
  return c;
}

// Solves (H + lambda diag(d)) x = -g by Cholesky; false when the damped matrix is not positive definite.
__device__ __forceinline__ bool tri_solve3(const double (&h)[6], const double (&g)[3], double lambda, double (&x)[3]) {
  const double dmax = fmax(h[0], fmax(h[3], h[5]));
  const double fl = TRI_DAMP_FLOOR * dmax;
  const double a00 = h[0] + lambda * fmax(h[0], fl), a11 = h[3] + lambda * fmax(h[3], fl), a22 = h[5] + lambda * fmax(h[5], fl);
  if (!(a00 > 0.0)) return false;
  const double l00 = sqrt(a00), l10 = h[1] / l00, l20 = h[2] / l00;
  const double d11 = a11 - l10 * l10;
  if (!(d11 > 0.0)) return false;
  const double l11 = sqrt(d11), l21 = (h[4] - l20 * l10) / l11;
  const double d22 = a22 - l20 * l20 - l21 * l21;
  if (!(d22 > 0.0)) return false;
  const double l22 = sqrt(d22);
  const double y0 = -g[0] / l00, y1 = (-g[1] - l10 * y0) / l11, y2 = (-g[2] - l20 * y0 - l21 * y1) / l22;
  x[2] = y2 / l22;
  x[1] = (y1 - l21 * x[2]) / l11;
  x[0] = (y0 - l10 * x[1] - l20 * x[2]) / l00;
  return isfinite(x[0]) && isfinite(x[1]) && isfinite(x[2]);
}

template <class S>
__device__ __forceinline__ void tri_round(double (&X)[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) X[k] = (double)(S)X[k];
}

// Warp per item (items in the length-sorted order, so the warps of one CTA see similar track lengths).  Scratch per slot:
// ray [nslots] the ray direction R^T (m, 1) and, in w, 1 = usable ray, 0 = not (written once, in pass 1); vb [nslots] bits
// 1 and 2 = projection validity at the current and at the candidate position of the refinement.  Outputs per item: status
// (RBA_TRI_* bits), angle, cost.
template <class S>
__global__ void __launch_bounds__(128) k_triangulate(DevPtrs<S> D, KOpts o, TriOpts t, const TriItem* __restrict__ items,
                                                     int nitems, double4* __restrict__ ray, uint8_t* __restrict__ vb,
                                                     uint8_t* __restrict__ status_out,
                                                     double* __restrict__ angle_out, double* __restrict__ cost_out) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int it = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); it < nitems; it += warps) {
    const TriItem item = items[it];
    const int s0 = item.slot0, n = item.n;
    const int lp = D.lmp_slot ? D.lmp_slot[item.sorted] : -1;
    double X[3] = {(double)D.lms[3 * item.lm], (double)D.lms[3 * item.lm + 1], (double)D.lms[3 * item.lm + 2]};
    unsigned status = 0;
    // 1. the usable rays and the sum of their centres
    int nr = 0;
    double cs[3] = {0.0, 0.0, 0.0};
    for (int i = lane; i < n; i += 32) {
      const int s = s0 + i;
      double cam[10];
      tri_load_cam(D, s, cam);
      bool use = cam[7] != 0.0;
      if (D.obs_W) {
        const S* W = D.obs_W + 4 * (size_t)s;
        use = use && !(W[0] == S(0) && W[1] == S(0) && W[2] == S(0) && W[3] == S(0));
      }
      double m0 = 0.0, m1 = 0.0;
      if (use) use = tri_undistort((double)D.slot_xy[2 * s] / cam[7], (double)D.slot_xy[2 * s + 1] / cam[7], cam[8], cam[9], m0, m1);
      double R[9];
      quat_to_rot(cam, R);
      double4 r;
      r.x = R[0] * m0 + R[3] * m1 + R[6];
      r.y = R[1] * m0 + R[4] * m1 + R[7];
      r.z = R[2] * m0 + R[5] * m1 + R[8];
      r.w = use ? 1.0 : 0.0;
      ray[s] = r;
      vb[s] = 0;
      if (use) {
        ++nr;
#pragma unroll
        for (int k = 0; k < 3; ++k) cs[k] -= R[k] * cam[4] + R[3 + k] * cam[5] + R[6 + k] * cam[6];
      }
    }
    nr = warp_sum(nr);
    __syncwarp();  // every lane's rays are visible to the warp
    // 2. the largest angle between two usable rays: row i by the whole warp, its pairs (i, j > i) split over the lanes, so
    //    every lane takes at most ceil((n - 1) / 32) pairs of a row
    double amax = 0.0;
    for (int i = 0; i < n - 1; ++i) {
      const double4 a = ray[s0 + i];
      if (a.w == 0.0) continue;
      for (int j = i + 1 + lane; j < n; j += 32) {
        const double4 b = ray[s0 + j];
        if (b.w == 0.0) continue;
        const double cx = a.y * b.z - a.z * b.y, cy = a.z * b.x - a.x * b.z, cz = a.x * b.y - a.y * b.x;
        amax = fmax(amax, atan2(sqrt(cx * cx + cy * cy + cz * cz), a.x * b.x + a.y * b.y + a.z * b.z));
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) amax = fmax(amax, __shfl_xor_sync(0xffffffffu, amax, off));
    if (nr < 2) status |= RBA_TRI_FEW_RAYS;
    else if (amax < t.min_angle) status |= RBA_TRI_SMALL_ANGLE;
    const bool rays_ok = status == 0;
    bool changed = false;
    // 3. LINEAR: the homogeneous midpoint estimate in centred, scaled coordinates
    if ((t.mode & RBA_TRIANGULATE_LINEAR) && rays_ok) {
#pragma unroll
      for (int k = 0; k < 3; ++k) cs[k] = warp_sum(cs[k]) / nr;
      double ss = 0.0;
      for (int i = lane; i < n; i += 32) {
        const int s = s0 + i;
        if (ray[s].w == 0.0) continue;
        double cam[10], R[9];
        tri_load_cam(D, s, cam);
        quat_to_rot(cam, R);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double ck = -(R[k] * cam[4] + R[3 + k] * cam[5] + R[6 + k] * cam[6]) - cs[k];
          ss += ck * ck;
        }
      }
      double sc = sqrt(warp_sum(ss) / nr);
      if (!(sc > 0.0)) sc = 1.0;
      double m[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};  // upper triangle of the 4x4 M, row by row
      for (int i = lane; i < n; i += 32) {
        const int s = s0 + i;
        const double4 d = ray[s];
        if (d.w == 0.0) continue;
        double cam[10], R[9];
        tri_load_cam(D, s, cam);
        quat_to_rot(cam, R);
        double B[12];  // [R | (R cbar + t) / sc], then (I - v v^T) B
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          B[4 * r] = R[3 * r]; B[4 * r + 1] = R[3 * r + 1]; B[4 * r + 2] = R[3 * r + 2];
          B[4 * r + 3] = (R[3 * r] * cs[0] + R[3 * r + 1] * cs[1] + R[3 * r + 2] * cs[2] + cam[4 + r]) / sc;
        }
        // d is the direction in the world frame; v = R d / |R d| the unit ray in the camera frame.  R of a quaternion that is
        // not exactly unit (a float32 state) is not exactly orthogonal, so R d is normalised itself: only for |v| = 1 is the
        // Gram matrix of (I - v v^T) B the M = B^T (I - v v^T) B of the midpoint estimate
        double v[3] = {R[0] * d.x + R[1] * d.y + R[2] * d.z, R[3] * d.x + R[4] * d.y + R[5] * d.z,
                       R[6] * d.x + R[7] * d.y + R[8] * d.z};
        const double vn = 1.0 / sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
#pragma unroll
        for (int r = 0; r < 3; ++r) v[r] *= vn;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const double p = v[0] * B[c] + v[1] * B[4 + c] + v[2] * B[8 + c];
#pragma unroll
          for (int r = 0; r < 3; ++r) B[4 * r + c] -= v[r] * p;
        }
        int k = 0;
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = a; b < 4; ++b) m[k++] += B[a] * B[b] + B[4 + a] * B[4 + b] + B[8 + a] * B[8 + b];
      }
#pragma unroll
      for (int k = 0; k < 10; ++k) m[k] = warp_sum(m[k]);
      double A[16] = {m[0], m[1], m[2], m[3], m[1], m[4], m[5], m[6], m[2], m[5], m[7], m[8], m[3], m[6], m[8], m[9]}, V[16];
      sym_eig<4>(A, V);
      double xh[4], emin = A[0];  // the eigenvector of the smallest eigenvalue (first of equal ones)
#pragma unroll
      for (int r = 0; r < 4; ++r) xh[r] = V[4 * r];
#pragma unroll
      for (int k = 1; k < 4; ++k)
        if (A[5 * k] < emin) {
          emin = A[5 * k];
#pragma unroll
          for (int r = 0; r < 4; ++r) xh[r] = V[4 * r + k];
        }
      const double xn = sqrt(xh[0] * xh[0] + xh[1] * xh[1] + xh[2] * xh[2] + xh[3] * xh[3]);
      if (!(fabs(xh[3]) > TRI_INFINITY * xn)) {
        status |= RBA_TRI_AT_INFINITY;
      } else {
        const double Y[3] = {cs[0] + sc * xh[0] / xh[3], cs[1] + sc * xh[1] / xh[3], cs[2] + sc * xh[2] / xh[3]};
        bool behind = false;
        for (int i = lane; i < n; i += 32) {
          const int s = s0 + i;
          if (ray[s].w == 0.0) continue;
          double cam[10], R[9];
          tri_load_cam(D, s, cam);
          quat_to_rot(cam, R);
          const double z = R[6] * Y[0] + R[7] * Y[1] + R[8] * Y[2] + cam[6];
          if (!(z >= (double)ST<S>::eps_sqrt())) behind = true;
        }
        if (__any_sync(0xffffffffu, behind)) {
          status |= RBA_TRI_BEHIND;
        } else {
#pragma unroll
          for (int k = 0; k < 3; ++k) X[k] = Y[k];
          tri_round<S>(X);
          changed = true;
        }
      }
    }
    // 4. REFINE: Levenberg-Marquardt on the landmark's own cost, cameras held
    double h[6], g[3];
    bool lost;
    int cur = 1;  // the bit of vb[s] holding the validity at X
    double cost = tri_eval(D, o, s0, n, lp, X, vb, cur, cur, h, g, lost);
    if ((t.mode & RBA_TRIANGULATE_REFINE) && (rays_ok || ((status & RBA_TRI_FEW_RAYS) && lp >= 0))) {
      const double c_start = cost;
      double Xb[3] = {X[0], X[1], X[2]}, lambda = TRI_LAMBDA0;
      int accepted = 0;
      bool conv = false;
      for (int k = 0; k < t.max_iterations && lambda <= TRI_LAMBDA_MAX; ++k) {
        if (g[0] == 0.0 && g[1] == 0.0 && g[2] == 0.0) { conv = true; break; }
        double dx[3];
        if (!tri_solve3(h, g, lambda, dx)) { lambda *= 10.0; continue; }
        const double Xn[3] = {Xb[0] + dx[0], Xb[1] + dx[1], Xb[2] + dx[2]};
        double hn[6], gn[3];
        const int nxt = 3 - cur;
        const double cn = tri_eval(D, o, s0, n, lp, Xn, vb, nxt, cur, hn, gn, lost);
        if (cn < cost && !lost) {
          conv = cost - cn <= t.ftol * cost;
          cost = cn; cur = nxt; ++accepted;
#pragma unroll
          for (int j = 0; j < 3; ++j) { Xb[j] = Xn[j]; g[j] = gn[j]; }
#pragma unroll
          for (int j = 0; j < 6; ++j) h[j] = hn[j];
          lambda = fmax(lambda * 0.1, TRI_LAMBDA_MIN);
          if (conv) break;
        } else {
          if (!lost && cn - cost <= t.ftol * cost) { conv = true; break; }  // no change the tolerance can tell apart
          lambda *= 10.0;
        }
      }
      if (conv) status |= RBA_TRI_CONVERGED;
      if (accepted > 0) {
        tri_round<S>(Xb);
        const double cr = tri_eval(D, o, s0, n, lp, Xb, vb, cur, cur, h, g, lost);
        if (cr < c_start) {
#pragma unroll
          for (int j = 0; j < 3; ++j) X[j] = Xb[j];
          cost = cr;
          changed = true;
          status |= RBA_TRI_REFINED;
        } else {
          cost = c_start;
        }
      }
    }
    if (changed) status |= RBA_TRI_WRITTEN;
    if (lane == 0) {
      if (changed)
#pragma unroll
        for (int k = 0; k < 3; ++k) D.lms[3 * item.lm + k] = (S)X[k];
      status_out[it] = (uint8_t)status;
      angle_out[it] = nr >= 2 ? amax : 0.0;
      cost_out[it] = cost;
    }
  }
}

}  // namespace rba
