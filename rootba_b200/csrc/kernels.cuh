// Hand-written sm_90a kernels of the square-root BA inner loop.  See DESIGN.md for the data layout,
// the algorithmic bytes of every kernel and the reference function each one replaces.
// "ref:" citations are relative to src/rootba/ of the reference (NikolausDemmel/rootba @ d3900037).
#pragma once

#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <cfloat>
#include <cmath>
#include <cstdint>

#include "layout.hpp"

namespace rba {

// ------------------------------------------------------------------------------------------------
// scalar traits
// ------------------------------------------------------------------------------------------------
template <class S> struct ST;
template <> struct ST<float> {
  using V2 = float2;
  using V4 = float4;
  __host__ __device__ static float eps_sqrt() { return 0.0031622776601683794f; }  // sqrt(1e-5), Sophus (A10)
  __host__ __device__ static float eps() { return 1e-5f; }
  __host__ __device__ static float tiny() { return FLT_MIN; }
};
template <> struct ST<double> {
  using V2 = double2;
  using V4 = double4;
  __host__ __device__ static double eps_sqrt() { return 1e-5; }
  __host__ __device__ static double eps() { return 1e-10; }
  __host__ __device__ static double tiny() { return DBL_MIN; }
};

__device__ __forceinline__ float2 mk2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ double2 mk2(double a, double b) { return make_double2(a, b); }

struct KOpts {
  int use_valid_projections_only;
  int robust_norm;
  double huber;
  double jacobi_eps;  // effective epsilon (already resolved)
  int write_panel;    // 0 with operator_form = implicit: the dense Q2 panels are neither stored nor read
};

// PCG scalars live on the device in double (ref: cg/conjugate_gradient.hpp:124-263 keeps them in double)
struct PcgState {
  double rho[2];
  double q0[2];
  double norm_b;
  double last_pq, last_alpha, last_zeta;
  int iter;
  int done;
  int term;    // 0 NO_CONVERGENCE, 1 SUCCESS, 2 FAILURE
  int reason;  // 0 max-iter, 1 zeta, 2 |b|=0, 3 rho, 4 beta, 5 indefinite pq, 6 alpha
};

constexpr int NPART = 64;  // blocks (= partial slots) of every vector kernel

template <class S>
struct DevPtrs {
  // state
  S* cams; S* lms;
  // topology
  const TileInfo* tiles; int ntiles;
  const int* sorted_lm;
  const int* slot_cam; const int* slot_lm; const S* slot_xy; int nslots;
  // linearization storage
  S* panel;      // Q2^T Jp panels, tile layout
  S* jp;         // [nslots][20] scaled, weighted pose Jacobian rows (2x9) + 2 pad   (16-byte aligned records)
  S* q1u;        // [nslots][28] undamped Q1^T Jp (3x9) + 1 pad
  S* q1d;        // [nslots][28] damped   Q1^T Jp (3x9) + 1 pad
  S* jl;         // [nslots][6]  scaled Jl (2x3)
  S* res;        // [nslots][2]  weighted residual
  S* lmk;        // [nsorted][24] Ru(6) q1r_u(3) Rd(6) q1r_d(3) Jl_col_scale(3) pad
  S* qtr;        // [nslots][2]  Q^T r of the landmark the slot belongs to: row rho of landmark (slot0) at qtr[2 slot0 + rho]
  S* dmp;        // [nslots][28] the 3 damping rows of the Q2 panel restricted to the 9 columns of the slot (3x9) + 1 pad
  S* blk0;       // [nslots][48] lambda-independent part of the slot's SCHUR_JACOBI block (45 upper entries) -- stage-1 scratch
  // camera vectors [9 nc]
  S* diag2; S* scaling; S* b; S* x; S* r; S* z; S* p; S* q; S* y; S* inc;
  S* blocks;     // [nc][81] preconditioner blocks (damping added)
  S* jblocks;    // [nc][81] JACOBI blocks (scaled, no damping)
  S* blocks0;    // [nc][81] lambda-independent part of the SCHUR_JACOBI blocks (rows 3..2n-1 of the Q2 panels; this shard)
  S* b0;         // [9 nc]   lambda-independent part of the gradient (this shard)
  S* inv;        // [nc][81] explicit inverses
  // scatter buffers
  S* yobs;       // [nyslots][9]
  S* partial;    // [max items][9]
  S* pblk;       // [csr_obs items][48] partial preconditioner blocks (45 used)
  int nc;
  const uint8_t* cam_fixed;  // [nc] RBA_FIX_* bits per camera (rba_set_camera_fixed), nullptr = every parameter free
  const S* prior_H;          // [nc][81] A^T A of the scaled camera priors (rba_set_camera_prior) and the pair priors' diagonal
                             //   blocks (rba_set_camera_pair_prior), nullptr = neither
  // pair priors (DESIGN.md section 15): camera-major CSR of the directed edges i -> j; pair_ov == nullptr = no pair priors
  const int* pair_ptr;       // [nc + 1]
  const int* pair_nbr;       // [edges] j
  const S* pair_O;           // [edges][36] O_ij = A_i^T A_j (pose 6x6, row-major), scaled
  S* pair_ov;                // [9 nc] sum_j O_ij v_j of the vector the next PCG / power-series vector step consumes
  // landmark priors (rba_set_landmark_prior, DESIGN.md section 17); lmp_slot == nullptr = none in this shard.  Only the
  // kernels' LMP instances read them.
  const int* lmp_slot;       // [nsorted] prior slot of each sorted landmark, -1 = no prior (and padding)
  const S* lmp_mean;         // [m][3] x0
  const S* lmp_L;            // [m][9] row-major square-root information L (unscaled)
  S* lmp_Lg;                 // [m][12] L diag(jls) (9, row-major) and g = L (x - x0) (3) of the last linearisation
  // observation information (rba_set_observation_info, DESIGN.md section 19); nullptr = none (identity everywhere) in this
  // shard.  Only the kernels' OBSW instances, k_obs_residuals and k_cov_landmark read it.
  const S* obs_W;            // [nslots][4] row-major 2x2 square-root information W of each slot (padding slots zero)
  // robust loss per observation (rba_set_observation_loss, DESIGN.md section 21); nullptr = the handle's robust_norm on every
  // observation of this shard.  Only the kernels' OBSL instances, k_obs_residuals and k_cov_landmark read it (slot_loss).
  const S* obs_loss;         // float: [nslots] {scale, uint32 kind}; double: [nslots] scale, then [nslots] uint8 kind (padding NONE)
  // robust losses on the landmark priors (rba_set_prior_loss, DESIGN.md section 22); lmp_loss == nullptr = none.  While they
  // are on, lmp_L is sqrt(w) L of the last linearisation; k_cov_landmark's LMPL instances re-weight the unweighted L here.
  const S* lmp_Lu;           // [m][9] the unweighted L
  const S* lmp_loss;         // the loss records of the lmp_n priors (slot_loss layout)
  int lmp_n;
};

// increment entries (tx,ty,tz, rx,ry,rz, f,k1,k2) held by a camera's RBA_FIX_* bits, as a 9-bit mask
__host__ __device__ __forceinline__ unsigned fixed_entry_mask(unsigned flags) {
  return ((flags & 1u) ? 0x3fu : 0u) | ((flags & 14u) << 5);
}

// ------------------------------------------------------------------------------------------------
// device math (same formulas and operation order as the oracle / reference)
// ------------------------------------------------------------------------------------------------
template <class S>
__device__ __forceinline__ void quat_to_rot(const S* q, S* R) {  // Eigen::Quaternion::toRotationMatrix
  const S x = q[0], y = q[1], z = q[2], w = q[3];
  const S tx = 2 * x, ty = 2 * y, tz = 2 * z;
  const S twx = tx * w, twy = ty * w, twz = tz * w;
  const S txx = tx * x, txy = ty * x, txz = tz * x;
  const S tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
  R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}

// ref: bal/bal_bundle_adjustment_helper.cpp:112-149 (linearize_point) + basalt BalCamera::project (A9)
// JAC=false: residual only.  Jp 2x9 (pose 6 + intrinsics 3) row-major, Jl 2x3.
template <class S, bool JAC>
__device__ __forceinline__ bool linearize_point(const S* obs, const S* pw, const S* cam, S* res, S* Jp9, S* Jl) {
  S R[9];
  quat_to_rot(cam, R);
  S pc[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) pc[r] = R[3 * r] * pw[0] + R[3 * r + 1] * pw[1] + R[3 * r + 2] * pw[2] + cam[4 + r];
  const S f = cam[7], k1 = cam[8], k2 = cam[9];
  const S z = pc[2];
  const S mx = pc[0] / z, my = pc[1] / z;
  const S mx2 = mx * mx, my2 = my * my;
  const S r2 = mx2 + my2;
  const S r4 = r2 * r2;
  const S rp = S(1) + k1 * r2 + k2 * r4;
  res[0] = f * mx * rp - obs[0];
  res[1] = f * my * rp - obs[1];
  if (JAC) {
    const S tmp = k1 + k2 * S(2) * r2;
    S d[6];
    d[0] = f * (rp + S(2) * mx2 * tmp) / z;
    d[4] = f * (rp + S(2) * my2 * tmp) / z;
    d[1] = d[3] = S(2) * f * mx * my * tmp / z;
    d[2] = -f * mx * (rp + S(2) * tmp * r2) / z;
    d[5] = -f * my * (rp + S(2) * tmp * r2) / z;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const S d0 = d[3 * r], d1 = d[3 * r + 1], d2 = d[3 * r + 2];
      Jp9[9 * r + 0] = d0; Jp9[9 * r + 1] = d1; Jp9[9 * r + 2] = d2;
      Jp9[9 * r + 3] = -d1 * pc[2] + d2 * pc[1];
      Jp9[9 * r + 4] = d0 * pc[2] - d2 * pc[0];
      Jp9[9 * r + 5] = -d0 * pc[1] + d1 * pc[0];
#pragma unroll
      for (int c = 0; c < 3; ++c) Jl[3 * r + c] = d0 * R[c] + d1 * R[3 + c] + d2 * R[6 + c];
    }
    Jp9[6] = mx * rp; Jp9[7] = f * mx * r2; Jp9[8] = f * mx * r4;
    Jp9[15] = my * rp; Jp9[16] = f * my * r2; Jp9[17] = f * my * r4;
  }
  return z >= ST<S>::eps_sqrt();
}

// ref: bal/bal_bundle_adjustment_helper.cpp:43-66
template <class S>
__device__ __forceinline__ void error_weight(const KOpts& o, S rsq, S& err, S& w) {
  if (o.robust_norm == 1) {
    const S th = (S)o.huber;
    const S hw = rsq < th * th ? S(1) : th / sqrt(rsq);
    err = S(0.5) * (S(2) - hw) * hw * rsq;
    w = hw;
  } else {
    err = S(0.5) * rsq;
    w = S(1);
  }
}

// Observation information (DESIGN.md section 19): res <- W res and, with JAC, the two rows of Jp and Jl <- W [row 0; row 1],
// W = obs_W[slot] (row-major 2x2, stored in SW, applied in S).  Returns W == 0, the observation is switched off: then res,
// Jp and Jl are set to zero whatever they held (a projection that is not finite must not survive as 0 * NaN).
template <class S, bool JAC, class SW>
__device__ __forceinline__ bool whiten_observation(const SW* __restrict__ obs_W, size_t slot, S* res, S* Jp, S* Jl) {
  S W[4];
  if constexpr (sizeof(SW) == 4) {
    const float4 v = *reinterpret_cast<const float4*>(obs_W + 4 * slot);
    W[0] = (S)v.x; W[1] = (S)v.y; W[2] = (S)v.z; W[3] = (S)v.w;
  } else {
    const double2 a = *reinterpret_cast<const double2*>(obs_W + 4 * slot), b = *reinterpret_cast<const double2*>(obs_W + 4 * slot + 2);
    W[0] = (S)a.x; W[1] = (S)a.y; W[2] = (S)b.x; W[3] = (S)b.y;
  }
  const bool off = W[0] == S(0) && W[1] == S(0) && W[2] == S(0) && W[3] == S(0);
  const S r0 = res[0], r1 = res[1];
  res[0] = off ? S(0) : W[0] * r0 + W[1] * r1;
  res[1] = off ? S(0) : W[2] * r0 + W[3] * r1;
  if (JAC) {
#pragma unroll
    for (int c = 0; c < 9; ++c) {
      const S a = Jp[c], b = Jp[9 + c];
      Jp[c] = off ? S(0) : W[0] * a + W[1] * b;
      Jp[9 + c] = off ? S(0) : W[2] * a + W[3] * b;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const S a = Jl[c], b = Jl[3 + c];
      Jl[c] = off ? S(0) : W[0] * a + W[1] * b;
      Jl[3 + c] = off ? S(0) : W[2] * a + W[3] * b;
    }
  }
  return off;
}

// Robust loss of one observation (DESIGN.md section 21), kind = RBA_LOSS_* (0 NONE, 1 HUBER, 2 CAUCHY, 3 SOFT_L1, 4 TUKEY),
// a the scale (inlier threshold in units of sigma), s = |W r|^2, u = s / a^2.  err = rho(s) / 2 and w = rho'(s), each rho
// normalised to rho(s) ~ s, w -> 1 as s -> 0.  Any other kind is NONE.
//   HUBER    w = 1 if s < a^2, else a / sqrt(s); err = 1/2 (2 - w) w s: error_weight's arithmetic with th = a
//   CAUCHY   rho = a^2 log1p(u);  w = 1 / (1 + u) = a^2 / (a^2 + s)
//   SOFT_L1  rho = 2 a^2 (sqrt(1 + u) - 1) = 2 s / (sqrt(1 + u) + 1);  w = 1 / sqrt(1 + u) = a / sqrt(a^2 + s)
//   TUKEY    rho = (a^2 / 3) (1 - (1 - u)^3) = (a^2 / 3) u (3 - 3u + u^2) for u < 1, else a^2 / 3;  w = (1 - u)^2, else 0,
//            1 - u = (a^2 - s) / a^2
// w of every kind takes one square root and one division, like error_weight (each correctly rounded, so HUBER gives
// error_weight's values bit for bit): the float32 Householder linearisation has no registers for more.  The divisions of
// err are dead code in the kernels that need w only.
template <class S>
__device__ __forceinline__ void observation_loss(unsigned kind, S a, S s, S& err, S& w) {
  const S a2 = a * a;
  const bool hub = kind == 1, cau = kind == 2, tuk = kind == 4;
  const S t = sqrt(hub ? s : a2 + s);                                           // HUBER sqrt(s), SOFT_L1 sqrt(a^2 + s)
  const S q = (cau ? a2 : tuk ? a2 - s : a) / (cau ? a2 + s : tuk ? a2 : t);  // w of HUBER beyond a, CAUCHY, SOFT_L1; 1 - u of TUKEY
  if (hub) {
    w = s < a2 ? S(1) : q;
    err = S(0.5) * (S(2) - w) * w * s;
  } else if (cau) {
    w = q;
    err = S(0.5) * a2 * log1p(s / a2);
  } else if (kind == 3) {
    w = q;
    err = a * s / (t + a);  // s / (sqrt(1 + u) + 1)
  } else if (tuk) {
    const S u = s / a2, c = a2 * S(1.0 / 6.0);
    w = s < a2 ? q * q : S(0);
    err = s < a2 ? c * (u * (S(3) - S(3) * u + u * u)) : c;
  } else {
    w = S(1);
    err = S(0.5) * s;
  }
}

// The loss of a slot from the records of rba_set_observation_loss: float one 8-byte {scale, uint32 kind} per slot (one load),
// double the scales [nslots] followed by one uint8 kind per slot.
template <class SL>
__device__ __forceinline__ void slot_loss(const SL* __restrict__ loss, int nslots, size_t slot, unsigned& kind, SL& a) {
  if constexpr (sizeof(SL) == 4) {
    const uint2 v = *reinterpret_cast<const uint2*>(loss + 2 * slot);
    a = __uint_as_float(v.x);
    kind = v.y;
  } else {
    a = loss[slot];
    kind = reinterpret_cast<const uint8_t*>(loss + nslots)[slot];
  }
}

// err and w of a slot at s = |W r|^2: OBSL the slot's own loss (evaluated in S), else the handle's (error_weight)
template <bool OBSL, class S, class SL>
__device__ __forceinline__ void slot_error_weight(const KOpts& o, const SL* __restrict__ loss, int nslots, size_t slot, S s,
                                                  S& err, S& w) {
  if constexpr (OBSL) {
    unsigned kind;
    SL a;
    slot_loss(loss, nslots, slot, kind, a);
    observation_loss<S>(kind, (S)a, s, err, w);
  } else {
    error_weight(o, s, err, w);
  }
}

template <class T>
__device__ __forceinline__ T group_sum(T v, int G) {
  for (int o = G >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <class T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ bool finite_s(float v) { return isfinite(v); }
__device__ __forceinline__ bool finite_s(double v) { return isfinite(v); }

// block-wide sum of K doubles per thread -> out[blockIdx.x*K + k] (thread 0); blockDim multiple of 32, <= 1024
template <int K>
__device__ __forceinline__ void block_sum_store(double (&v)[K], double* out) {
  __shared__ double sm[32][K];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = warp_sum(v[k]);
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < K; ++k) sm[w][k] = v[k];
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double s = 0;
      for (int i = 0; i < nw; ++i) s += sm[i][k];
      out[blockIdx.x * K + k] = s;
    }
  }
  __syncthreads();
}

// sum of n <= 1024 partial doubles in a fixed order, result broadcast to every thread of the block
__device__ __forceinline__ double block_sum_partials(const double* part, int n, int stride, int off) {
  __shared__ double bs_sm[32];
  __shared__ double bs_total;
  double v = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) v += part[i * stride + off];
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (lane == 0) bs_sm[w] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0;
    for (int i = 0; i < nw; ++i) s += bs_sm[i];
    bs_total = s;
  }
  __syncthreads();
  const double r = bs_total;
  __syncthreads();
  return r;
}

// ------------------------------------------------------------------------------------------------
// K0  error  (ref: bal/bal_bundle_adjustment_helper.cpp:68-109, residual_info.cpp:97-110)
//     thread per observation slot; accumulation in double; out partials [gridDim][6]
//     OBSW (observation information, DESIGN.md section 19): the residual is W r; a switched-off observation (W == 0) counts
//     in "all" only and its projection is not checked for finiteness.
//     OBSL (observation losses, DESIGN.md section 21): err from the slot's own loss (observation_loss) instead of error_weight.
// ------------------------------------------------------------------------------------------------
template <class S, bool OBSW = false, bool OBSL = false>
__global__ void __launch_bounds__(256) k_error(DevPtrs<S> D, KOpts o, double* partials, int* bad_flag) {
  double acc[6] = {0, 0, 0, 0, 0, 0};  // all: n, err, res ; valid: n, err, res
  bool bad = false;
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < D.nslots; s += gridDim.x * blockDim.x) {
    const int lm = D.slot_lm[s];
    if (lm < 0) continue;
    S obs[2] = {D.slot_xy[2 * s], D.slot_xy[2 * s + 1]};
    S pw[3] = {D.lms[3 * lm], D.lms[3 * lm + 1], D.lms[3 * lm + 2]};
    S cam[10];
    const S* cp = D.cams + 10 * (size_t)D.slot_cam[s];
#pragma unroll
    for (int k = 0; k < 10; ++k) cam[k] = cp[k];
    S res[2];
    bool pv = linearize_point<S, false>(obs, pw, cam, res, nullptr, nullptr);
    if constexpr (OBSW) pv = !whiten_observation<S, false>(D.obs_W, s, res, nullptr, nullptr) && pv;
    if (!(finite_s(res[0]) && finite_s(res[1]))) bad = true;
    const S rsq = res[0] * res[0] + res[1] * res[1];
    S err, w;
    slot_error_weight<OBSL>(o, D.obs_loss, D.nslots, s, rsq, err, w);
    const double rn = (double)sqrt(rsq);
    acc[0] += 1.0; acc[1] += (double)err; acc[2] += rn;
    // ref: with the validity check enabled linearize_point returns false for invalid projections and they
    // count only in "all"; with it disabled the return value is still the projection validity.
    if (pv) { acc[3] += 1.0; acc[4] += (double)err; acc[5] += rn; }
  }
  if (bad) atomicOr(bad_flag, 1);
  block_sum_store<6>(acc, partials);
}

// rba_get_observation_residuals: k_error per slot without the reduction.  res [nslots][2] = W r (r without observation
// information), hw [nslots] = the robust weight on |W r|^2 (the slot's own loss while D.obs_loss is set, else error_weight),
// flags [nslots]: bit 0 = projection valid, bit 1 = in use (W != 0).  Padding slots are not written.
template <class S>
__global__ void __launch_bounds__(256) k_obs_residuals(DevPtrs<S> D, KOpts o, S* __restrict__ res_out, S* __restrict__ hw_out,
                                                       uint8_t* __restrict__ flags_out) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= D.nslots) return;
  const int lm = D.slot_lm[s];
  if (lm < 0) return;
  S obs[2] = {D.slot_xy[2 * s], D.slot_xy[2 * s + 1]};
  S pw[3] = {D.lms[3 * lm], D.lms[3 * lm + 1], D.lms[3 * lm + 2]};
  S cam[10];
  const S* cp = D.cams + 10 * (size_t)D.slot_cam[s];
#pragma unroll
  for (int k = 0; k < 10; ++k) cam[k] = cp[k];
  S res[2];
  const bool pv = linearize_point<S, false>(obs, pw, cam, res, nullptr, nullptr);
  const bool off = D.obs_W && whiten_observation<S, false>(D.obs_W, s, res, nullptr, nullptr);
  S err, w;
  if (D.obs_loss) slot_error_weight<true>(o, D.obs_loss, D.nslots, s, res[0] * res[0] + res[1] * res[1], err, w);
  else error_weight(o, res[0] * res[0] + res[1] * res[1], err, w);
  res_out[2 * (size_t)s] = res[0];
  res_out[2 * (size_t)s + 1] = res[1];
  hw_out[s] = w;
  flags_out[s] = (uint8_t)((pv ? 1 : 0) | (off ? 0 : 2));
}

// sums [n][K] double partials -> out[K]   (single block)
template <int K>
__global__ void k_sum_partials(const double* part, int n, double* out) {
  for (int k = 0; k < K; ++k) {
    const double s = block_sum_partials(part, n, K, k);
    if (threadIdx.x == 0) out[k] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// K1a  squared column norms of sqrt(w) * Jp per observation  (ref: qr/impl/landmark_block_base.ipp:493-518)
//      thread per slot -> yobs[slot][9]; reduced per camera by k_cam_reduce (deterministic)
//      OBSW (observation information, DESIGN.md section 19): the norms of sqrt(w) * W Jp, w from |W r|^2
//      OBSL (observation losses, DESIGN.md section 21): w from the slot's own loss
// ------------------------------------------------------------------------------------------------
template <class S, bool OBSW = false, bool OBSL = false>
__global__ void __launch_bounds__(256) k_jp_norms(DevPtrs<S> D, KOpts o, int* bad_flag) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < D.nslots; s += gridDim.x * blockDim.x) {
    const int lm = D.slot_lm[s];
    if (lm < 0) continue;
    S obs[2] = {D.slot_xy[2 * s], D.slot_xy[2 * s + 1]};
    S pw[3] = {D.lms[3 * lm], D.lms[3 * lm + 1], D.lms[3 * lm + 2]};
    S cam[10];
    const S* cp = D.cams + 10 * (size_t)D.slot_cam[s];
#pragma unroll
    for (int k = 0; k < 10; ++k) cam[k] = cp[k];
    S res[2], Jp[18], Jl[6];
    const bool valid = linearize_point<S, true>(obs, pw, cam, res, Jp, Jl);
    if constexpr (OBSW) whiten_observation<S, true>(D.obs_W, s, res, Jp, Jl);
    S out[9];
    if (!o.use_valid_projections_only || valid) {
      bool fin = finite_s(res[0]) && finite_s(res[1]);
#pragma unroll
      for (int k = 0; k < 18; ++k) fin = fin && finite_s(Jp[k]);
#pragma unroll
      for (int k = 0; k < 6; ++k) fin = fin && finite_s(Jl[k]);
      if (!fin) atomicOr(bad_flag, 1);
      S err, w;
      slot_error_weight<OBSL>(o, D.obs_loss, D.nslots, s, res[0] * res[0] + res[1] * res[1], err, w);
      const S sw = sqrt(w);
#pragma unroll
      for (int c = 0; c < 9; ++c) {
        const S a = sw * Jp[c], b = sw * Jp[9 + c];
        out[c] = a * a + b * b;
      }
    } else {
#pragma unroll
      for (int c = 0; c < 9; ++c) out[c] = 0;
    }
#pragma unroll
    for (int c = 0; c < 9; ++c) D.yobs[9 * (size_t)s + c] = out[c];
  }
}

constexpr int MAX_PEERS = 8;

// Peer-memory exchange (multi-GPU, one box): every rank owns ONE cudaMalloc region that the other ranks map through
// CUDA IPC.  All exchanges are PUSH based: a rank stores its contribution straight into slot [parity][own rank] of every
// peer's staging area (posted NVLink writes, they overlap the producing kernel), the next kernel in the stream publishes
// a sequence number into every peer's flag with st.release.sys, waits for the peers' numbers in its OWN memory
// (ld.acquire.sys on local memory) and sums the staged contributions in rank order -- bit-identical on every rank, no
// remote load on the critical path.  Double buffering by the parity of the sequence number makes buffer reuse safe: a
// rank can only push number s + 2 after it has seen every peer's flag s + 1, which a peer publishes after it has
// finished reading number s.
// region layout (bytes):   [0, 64) int yflag[2][8] | [64, 128) int cflag[2][8] | [128, 192) int sflag[2][8]
//                          [256, 2304) 8-byte sstage[2][8][16] | off_y: S ystage[2][nranks][9 nc] | off_c: S cstage[2][nranks][cmax]
struct PeerComm {
  int nranks, rank;
  char* base[MAX_PEERS];   // base of rank r's region (own entry: local pointer)
  long long off_y, off_c;  // byte offsets of the staging areas
  long long cmax;          // elements per (parity, rank) slot of cstage
  int* dead;               // device flag of THIS rank: set when an exchange timed out; every later exchange fails at once
};
constexpr int PEER_SMALL_MAX = 16;
__device__ __forceinline__ int* peer_flag(const PeerComm& pc, int dest, int family, int par, int src) {
  return reinterpret_cast<int*>(pc.base[dest] + 64 * family) + par * MAX_PEERS + src;
}
template <class S>
__device__ __forceinline__ S* peer_ystage(const PeerComm& pc, int dest, int par, int src, int nc) {
  return reinterpret_cast<S*>(pc.base[dest] + pc.off_y) + ((size_t)par * pc.nranks + src) * 9 * (size_t)nc;
}
template <class T>
__device__ __forceinline__ T* peer_cstage(const PeerComm& pc, int dest, int par, int src) {
  return reinterpret_cast<T*>(pc.base[dest] + pc.off_c) + ((size_t)par * pc.nranks + src) * (size_t)pc.cmax;
}
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(int* p, int v) {
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// wait until the local flag of (family, parity, src) has reached seq; false after ~2 s (a peer died) or when an earlier
// exchange of this rank has already failed (sticky: a dead peer costs one timeout, not one per kernel)
__device__ __forceinline__ bool peer_wait(const PeerComm& pc, int family, int par, int src, int seq) {
  const int* f = peer_flag(pc, pc.rank, family, par, src);
  if (*reinterpret_cast<volatile int*>(pc.dead)) return false;
  long long spins = 0;
  while (ld_acquire_sys(f) - seq < 0)
    if (++spins > (1LL << 22)) { *reinterpret_cast<volatile int*>(pc.dead) = 1; return false; }
  return true;
}

// Generic vector all-reduce over peer memory, two kernels so that the kernel boundary is the grid-wide "all my stores are
// issued" point: k_peer_push stores this rank's vector into every peer's cstage[parity][rank], k_peer_sum publishes the
// sequence number, waits for the peers' and writes the rank-ordered sum.  Grids are <= the SM count (co-resident: a
// spinning block can never starve an unscheduled one).
template <class T>
__global__ void __launch_bounds__(256) k_peer_push(PeerComm pc, const T* __restrict__ src, long long count, int par) {
  for (int d = 0; d < pc.nranks; ++d) {
    T* dst = peer_cstage<T>(pc, d, par, pc.rank);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i];
  }
}
template <class T>
__global__ void __launch_bounds__(256) k_peer_sum(PeerComm pc, T* __restrict__ dst, long long count, int par, int seq, int* fail_flag) {
  __shared__ int ok;
  if (threadIdx.x == 0) ok = 1;
  if (blockIdx.x == 0 && threadIdx.x < pc.nranks) { __threadfence_system(); st_release_sys(peer_flag(pc, threadIdx.x, 1, par, pc.rank), seq); }
  __syncthreads();
  if (threadIdx.x < pc.nranks && !peer_wait(pc, 1, par, threadIdx.x, seq)) ok = 0;
  __syncthreads();
  if (!ok) { if (threadIdx.x == 0) atomicOr(fail_flag, 2); return; }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    T sacc = 0;
    for (int r = 0; r < pc.nranks; ++r) sacc += __ldcg(peer_cstage<T>(pc, pc.rank, par, r) + i);
    dst[i] = sacc;
  }
}
// <= 16 scalars (nd doubles + nf int flags) in ONE single-block kernel: stage, fence, publish, wait, sum.
__global__ void __launch_bounds__(64) k_peer_small(PeerComm pc, double* vals, int nd, int* flags, int nf, int par, int seq, int* fail_flag) {
  __shared__ int ok;
  const int t = threadIdx.x, n = nd + nf;
  if (t == 0) ok = 1;
  if (t < n) {
    const double v = t < nd ? vals[t] : (double)flags[t - nd];
    for (int d = 0; d < pc.nranks; ++d)
      reinterpret_cast<double*>(pc.base[d] + 256)[((size_t)par * MAX_PEERS + pc.rank) * PEER_SMALL_MAX + t] = v;
    __threadfence_system();
  }
  __syncthreads();
  if (t < pc.nranks) st_release_sys(peer_flag(pc, t, 2, par, pc.rank), seq);
  if (t < pc.nranks && !peer_wait(pc, 2, par, t, seq)) ok = 0;
  __syncthreads();
  if (!ok) { if (t == 0) atomicOr(fail_flag, 2); return; }
  if (t < n) {
    double sacc = 0;
    for (int r = 0; r < pc.nranks; ++r)
      sacc += __ldcg(reinterpret_cast<const double*>(pc.base[pc.rank] + 256) + ((size_t)par * MAX_PEERS + r) * PEER_SMALL_MAX + t);
    if (t < nd) vals[t] = sacc; else flags[t - nd] = (int)sacc;
  }
}

// ------------------------------------------------------------------------------------------------
// deterministic scatter, phase 2: per-camera segmented sum of 9-vectors
//   warp per ReduceItem (segment of a camera's slot list) -> partial[item][9]
// ------------------------------------------------------------------------------------------------
// one warp reduces one ReduceItem (<= SEG_LEN slots).  Lane (s, c) = (lane / 9, lane % 9), s < 3, reads component c of
// slot 3t + s: the 9 scalars of a slot are one 36-byte run, so a warp-wide load touches 3 slots = 3..6 sectors instead
// of 32.  The slot indices are first staged in shared memory with coalesced loads (one round trip), then the value loads
// are issued 16 deep, so an item costs ~1 + SEG_LEN/48 round trips instead of 2 * SEG_LEN/32.
template <class S>
__device__ __forceinline__ void cam_stage_indices(const int* __restrict__ slots, const ReduceItem& I, int lane, int* sidx) {
  const int cnt = I.end - I.begin;
#pragma unroll
  for (int t = 0; t < (SEG_LEN + 31) / 32; ++t) {
    const int e = lane + 32 * t;
    if (e < cnt) sidx[e] = __ldg(slots + I.begin + e);
  }
  __syncwarp();
}
template <class S>
__device__ __forceinline__ void cam_sum_staged(const S* __restrict__ src, const ReduceItem& I, int lane, S* __restrict__ out9,
                                               const int* sidx) {
  const int cnt = I.end - I.begin;
  const int s3 = lane / 9, c = lane - 9 * s3;
  const bool on = lane < 27;
  S acc = 0;
  constexpr int DEPTH = 16;  // value loads in flight per lane; 3 * DEPTH slots per round
  for (int base = 0; base < cnt; base += 3 * DEPTH) {
    S v[DEPTH];
#pragma unroll
    for (int t = 0; t < DEPTH; ++t) {
      const int e = base + 3 * t + s3;
      v[t] = (on && e < cnt) ? src[9 * (size_t)sidx[e] + c] : S(0);
    }
#pragma unroll
    for (int t = 0; t < DEPTH; ++t) acc += v[t];
  }
  __syncwarp();
  // lanes c, c + 9, c + 18 hold the three partial sums of component c
  const S a1 = __shfl_sync(0xffffffffu, acc, (lane + 9) & 31);
  const S a2 = __shfl_sync(0xffffffffu, acc, (lane + 18) & 31);
  if (lane < 9) out9[lane] = acc + a1 + a2;
}
template <class S>
__device__ __forceinline__ void cam_reduce_item(const S* __restrict__ src, const int* __restrict__ slots, const ReduceItem& I,
                                                int lane, S* __restrict__ out9, int* sidx /* [SEG_LEN] per warp */) {
  cam_stage_indices<S>(slots, I, lane, sidx);
  cam_sum_staged(src, I, lane, out9, sidx);
}

template <class S>
__global__ void __launch_bounds__(256) k_cam_reduce(const S* __restrict__ src, const int* __restrict__ slots,
                                                     const ReduceItem* __restrict__ items, int nitems,
                                                     S* __restrict__ partial, const int* done, int pdl) {
  // `done` is written only by the PCG vector kernel BEFORE the operator kernel this one depends on: it is final here
  if (done && *reinterpret_cast<const volatile int*>(done)) return;
  __shared__ int sidx_all[8][SEG_LEN];
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  // the slot indices are constant: stage the first item's before the grid dependency is awaited
  const int it0 = blockIdx.x * wpb + (threadIdx.x >> 5);
  if (it0 < nitems) cam_stage_indices<S>(slots, items[it0], lane, sidx_all[threadIdx.x >> 5]);
  if (pdl) {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  }
  for (int it = it0; it < nitems; it += gridDim.x * wpb) {
    const ReduceItem I = items[it];
    if (it != it0) cam_stage_indices<S>(slots, I, lane, sidx_all[threadIdx.x >> 5]);
    cam_sum_staged(src, I, lane, partial + 9 * (size_t)it, sidx_all[threadIdx.x >> 5]);
  }
}

// Same, and the warp that completes the LAST segment of a camera (arrival counter) adds the camera's segment sums in
// their fixed order and writes y[cam][9]: the result is complete when the kernel ends, deterministic, and needs no
// second kernel.  cam_cnt must be zero on entry and is left zero.
template <class S, bool PEERS>
__global__ void __launch_bounds__(256) k_cam_reduce_final(const S* __restrict__ src, const int* __restrict__ slots,
                                                           const ReduceItem* __restrict__ items, int nitems,
                                                           const int* __restrict__ cam_item_ptr, S* __restrict__ partial,
                                                           int* cam_cnt, S* __restrict__ y, const int* done, int pdl,
                                                           PeerComm pc, int seq, int nc) {
  __shared__ int sidx_all[8][SEG_LEN];
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  if (done && *reinterpret_cast<const volatile int*>(done)) return;  // monotonic flag, see k_matvec_small_tma
  // the slot indices are constant: stage the first item's before the grid dependency is awaited
  const int it0 = blockIdx.x * wpb + (threadIdx.x >> 5);
  if (it0 < nitems) cam_stage_indices<S>(slots, items[it0], lane, sidx_all[threadIdx.x >> 5]);
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  if (done && *done) return;
  if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  for (int it = it0; it < nitems; it += gridDim.x * wpb) {
    const ReduceItem I = items[it];
    if (it != it0) cam_stage_indices<S>(slots, I, lane, sidx_all[threadIdx.x >> 5]);
    cam_sum_staged(src, I, lane, partial + 9 * (size_t)it, sidx_all[threadIdx.x >> 5]);
    const int i0 = cam_item_ptr[I.cam], i1 = cam_item_ptr[I.cam + 1];
    // the camera's sum goes to y, or (several shards, peer exchange) into slot [parity][own rank] of EVERY rank's staging
    // area; cameras without observations in this shard are never written and stay zero there
    auto emit = [&](S v) {
      if constexpr (PEERS) {
        for (int d = 0; d < pc.nranks; ++d) peer_ystage<S>(pc, d, seq & 1, pc.rank, nc)[9 * (size_t)I.cam + lane] = v;
      } else {
        y[9 * (size_t)I.cam + lane] = v;
      }
    };
    if (i1 - i0 == 1) {
      if (lane < 9) emit(partial[9 * (size_t)it + lane]);
      continue;
    }
    __threadfence();
    int last = 0;
    if (lane == 0) last = (atomicAdd(cam_cnt + I.cam, 1) == i1 - i0 - 1) ? 1 : 0;
    last = __shfl_sync(0xffffffffu, last, 0);
    if (last) {
      __threadfence();
      if (lane < 9) {
        S sacc = 0;
        for (int q = i0; q < i1; ++q) sacc += __ldcg(partial + 9 * (size_t)q + lane);
        emit(sacc);
      }
      if (lane == 0) cam_cnt[I.cam] = 0;
    }
  }
}

// ref: solver/linearizor_qr.cpp:130-132
template <class S>
__global__ void k_scaling(const S* diag2, S* scaling, int n, S eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) scaling[i] = S(1) / (eps + sqrt(diag2[i]));
}


// ---- warp-cooperative copies between a tile's contiguous global region and scratch (16-byte vectors) ----
template <class S>
__device__ __forceinline__ void warp_copy_in(S* __restrict__ dst, const S* __restrict__ src, int count, int lane) {
  using V4 = typename ST<S>::V4;
  constexpr int VW = 16 / sizeof(S) >= 4 ? 4 : 2;  // scalars per 16-byte (f32) / 32-byte (f64 double4 is 32 B: use 2)
  if (sizeof(S) == 4) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int e = lane; e < count / 4; e += 32) d4[e] = __ldg(s4 + e);
  } else {
    const double2* s2 = reinterpret_cast<const double2*>(src);
    double2* d2 = reinterpret_cast<double2*>(dst);
    for (int e = lane; e < count / 2; e += 32) d2[e] = __ldg(s2 + e);
  }
  (void)VW;
}
template <class S>
__device__ __forceinline__ void warp_copy_out(S* __restrict__ dst, const S* __restrict__ src, int count, int lane) {
  if (sizeof(S) == 4) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int e = lane; e < count / 4; e += 32) d4[e] = s4[e];
  } else {
    const double2* s2 = reinterpret_cast<const double2*>(src);
    double2* d2 = reinterpret_cast<double2*>(dst);
    for (int e = lane; e < count / 2; e += 32) d2[e] = s2[e];
  }
}

// ---- per-lane loads/stores of 16-byte aligned per-observation records (N scalars, N % 4 == 0) ----
template <class S, int N>
__device__ __forceinline__ void load_rec(const S* __restrict__ src, S (&v)[N]) {
  if (sizeof(S) == 4) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
#pragma unroll
    for (int q = 0; q < N / 4; ++q) { const float4 t = __ldg(s4 + q); v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w; }
  } else {
    const double2* s2 = reinterpret_cast<const double2*>(src);
#pragma unroll
    for (int q = 0; q < N / 2; ++q) { const double2 t = __ldg(s2 + q); v[2 * q] = t.x; v[2 * q + 1] = t.y; }
  }
}
template <class S, int N>
__device__ __forceinline__ void store_rec(S* __restrict__ dst, const S (&v)[N]) {
  if (sizeof(S) == 4) {
    float4* d4 = reinterpret_cast<float4*>(dst);
#pragma unroll
    for (int q = 0; q < N / 4; ++q) d4[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  } else {
    double2* d2 = reinterpret_cast<double2*>(dst);
#pragma unroll
    for (int q = 0; q < N / 2; ++q) d2[q] = make_double2(v[2 * q], v[2 * q + 1]);
  }
}

// scratch of a tile kernel: shared memory when the tile fits, else a per-warp slice of a global buffer
template <class S>
struct Scratch {
  S* gbase;          // global scratch (may be null when every tile fits in shared memory)
  long long gstride; // scalars per warp
  int smem_cap;      // scalars of shared memory per warp
};
template <class S>
__device__ __forceinline__ S* scratch_ptr(const Scratch<S>& sc, S* smem_warp, int need) {
  if (need <= sc.smem_cap) return smem_warp;
  const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  return sc.gbase + w * sc.gstride;
}

// Order in which the persistent warps of a tile kernel take their tiles: position k * (number of warps) + w holds the
// k-th tile of warp w, dealt longest-processing-time-first on the host (a warp's list ends at the first -1).  order ==
// nullptr: plain round-robin over the tiles.
struct TileOrder {
  const int* order;
  int count;
};
__device__ __forceinline__ int tile_at(const TileOrder& to, int idx, int ntiles) {
  if (!to.order) return idx < ntiles ? idx : -1;
  return idx < to.count ? __ldg(to.order + idx) : -1;
}

template <class S>
struct Rot { S c, s; };

template <class S>
__device__ __forceinline__ Rot<S> make_givens(S p, S q) {  // Eigen JacobiRotation::makeGivens (SURVEY A8)
  Rot<S> g;
  if (q == S(0)) { g.c = p < S(0) ? S(-1) : S(1); g.s = 0; }
  else if (p == S(0)) { g.c = 0; g.s = q < S(0) ? S(1) : S(-1); }
  else if (fabs(p) > fabs(q)) {
    const S t = q / p; S u = sqrt(S(1) + t * t); if (p < S(0)) u = -u;
    g.c = S(1) / u; g.s = -t * g.c;
  } else {
    const S t = p / q; S u = sqrt(S(1) + t * t); if (q < S(0)) u = -u;
    g.s = -S(1) / u; g.c = -t * g.s;
  }
  return g;
}
// applyOnTheLeft(p=damping row, q=row n): x' = c x + s y ; y' = -s x + c y
template <class S>
__device__ __forceinline__ void rot_apply(const Rot<S>& g, S& x, S& y) {
  const S xi = x, yi = y;
  x = g.c * xi + g.s * yi;
  y = -g.s * xi + g.c * yi;
}

// ------------------------------------------------------------------------------------------------
// K1b  linearize + Jl scaling + Householder QR of the 3 landmark columns + write marginalised panel
//   ref: ipp:88-147 (linearize_landmark), :571-587 (scale_Jl_cols), :717-743 (perform_qr_householder),
//        Eigen makeHouseholder/applyHouseholderOnTheLeft (SURVEY A7), pose-Jacobian scaling ipp:589-614
//        folded in (the scaling vector is known before this kernel runs, see DESIGN.md).
//   One warp per tile; group of G lanes per landmark.  The three reflectors are generated exactly like
//   Eigen does on the 2n x 4 matrix [Jl | r] (shuffle reductions inside the group) and applied to the
//   block-diagonal Jp through their compact-WY form, one output element = 3 FMAs, written straight into
//   the coalesced panel layout.
// ------------------------------------------------------------------------------------------------
//   LMP (landmark priors, DESIGN.md section 17): the prior's squared column norms |L col c|^2 join the landmark's column
//   norms behind jls (the scaling of the whole Jacobian), and lane 0 of the group writes L diag(jls) and g = L (x - x0).
//   OBSW (observation information, DESIGN.md section 19): the rows of an observation are sqrt(w) W [Jp | Jl | r], w from
//   |W r|^2; W == 0 gives the all-zero record of a dropped projection.
//   OBSL (observation losses, DESIGN.md section 21): w from the slot's own loss; w == 0 (TUKEY beyond its scale) gives rows
//   of zeros.
template <class S, bool GIVENS, bool LMP = false, bool OBSW = false, bool OBSL = false>
__global__ void __launch_bounds__(128) k_linearize_qr(DevPtrs<S> D, KOpts o, Scratch<S> sc, int* bad_flag, TileOrder to) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using V2 = typename ST<S>::V2;
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  S* ws_smem = reinterpret_cast<S*>(smem_raw) + (size_t)wib * sc.smem_cap;
  const S eps = (S)o.jacobi_eps;
  for (int idx = blockIdx.x * (blockDim.x >> 5) + wib;; idx += gridDim.x * (blockDim.x >> 5)) {
    const int t = tile_at(to, idx, D.ntiles);
    if (t < 0) break;
    const TileInfo T = D.tiles[t];
    const int n = T.n, G = T.G, KP = T.KP;
    const int g = lane / G, j = lane - g * G;
    const bool active = g < T.nvalid;
    const int Wn = (32 / G) * n;
    S* ws = scratch_ptr(sc, ws_smem, Wn * 60 + 64);
    const int GS = 32 * n + 1;        // per-landmark scratch stride, odd => group-broadcast reads hit distinct banks
    S* sJ = ws + (size_t)g * GS;      // [n][26]: jp row0 (9) | jp row1 (9) | jl row0 (3) | jl row1 (3) | r (2)
    S* sV = sJ + 26 * n;              // [2n][3] Householder vectors
    S* sQ = ws + (((size_t)(32 / G) * GS + 3) & ~(size_t)3);  // [W*n][28] staging of the undamped Q1^T Jp rows
    const int slot0 = T.slot_base + g * n;
    const int sidx = T.lm_base + g;
    S pw[3] = {0, 0, 0};
    if (active) {
      const int lm = D.sorted_lm[sidx];
      pw[0] = D.lms[3 * lm]; pw[1] = D.lms[3 * lm + 1]; pw[2] = D.lms[3 * lm + 2];
    }
    __syncwarp();
    // ---- a. Jacobians of the observations (ref: ipp:106-140) ----
    for (int i = j; i < n; i += G) {
      S* e = sJ + 26 * i;
      bool wrote = false;
      if (active) {
        const int s = slot0 + i;
        const int cam_i = D.slot_cam[s];
        S obs[2] = {D.slot_xy[2 * s], D.slot_xy[2 * s + 1]};
        S cam[10];
        const S* cp = D.cams + 10 * (size_t)cam_i;
#pragma unroll
        for (int k = 0; k < 10; ++k) cam[k] = cp[k];
        S res[2], Jp[18], Jl[6];
        const bool valid = linearize_point<S, true>(obs, pw, cam, res, Jp, Jl);
        if constexpr (OBSW) whiten_observation<S, true>(D.obs_W, s, res, Jp, Jl);
        if (!o.use_valid_projections_only || valid) {
          bool fin = finite_s(res[0]) && finite_s(res[1]);
#pragma unroll
          for (int k = 0; k < 18; ++k) fin = fin && finite_s(Jp[k]);
#pragma unroll
          for (int k = 0; k < 6; ++k) fin = fin && finite_s(Jl[k]);
          if (!fin) atomicOr(bad_flag, 1);
          S err, w;
          if constexpr (OBSL) {
            // the unweighted rows first, so that the registers of Jp and Jl are free while the slot's loss is evaluated (the
            // compiler barrier keeps them from being forwarded), then weighted in place with the arithmetic below
#pragma unroll
            for (int c = 0; c < 18; ++c) e[c] = Jp[c];
#pragma unroll
            for (int c = 0; c < 6; ++c) e[18 + c] = Jl[c];
            asm volatile("" ::: "memory");
            slot_error_weight<true>(o, D.obs_loss, D.nslots, s, res[0] * res[0] + res[1] * res[1], err, w);
            const S sw = sqrt(w);
            const S* sc = D.scaling + 9 * (size_t)cam_i;
#pragma unroll
            for (int c = 0; c < 9; ++c) {
              const S d = sc[c];
              e[c] = (sw * e[c]) * d;
              e[9 + c] = (sw * e[9 + c]) * d;
            }
#pragma unroll
            for (int c = 0; c < 6; ++c) e[18 + c] = sw * e[18 + c];
            e[24] = sw * res[0];
            e[25] = sw * res[1];
          } else {
            error_weight(o, res[0] * res[0] + res[1] * res[1], err, w);
            const S sw = sqrt(w);
            const S* sc = D.scaling + 9 * (size_t)cam_i;
#pragma unroll
            for (int c = 0; c < 9; ++c) {
              const S d = sc[c];
              e[c] = (sw * Jp[c]) * d;
              e[9 + c] = (sw * Jp[9 + c]) * d;
            }
#pragma unroll
            for (int c = 0; c < 6; ++c) e[18 + c] = sw * Jl[c];
            e[24] = sw * res[0];
            e[25] = sw * res[1];
          }
          wrote = true;
        }
      }
      if (!wrote)
#pragma unroll
        for (int c = 0; c < 26; ++c) e[c] = 0;
    }
    __syncwarp();
    // ---- b. scale_Jl_cols (ref: ipp:571-587) ----
    S cs[3] = {0, 0, 0};
    for (int i = j; i < n; i += G) {
      const S* e = sJ + 26 * i + 18;
#pragma unroll
      for (int c = 0; c < 3; ++c) cs[c] += e[c] * e[c] + e[3 + c] * e[3 + c];
    }
    S jls[3];
    S lpn[3] = {0, 0, 0};
    if constexpr (LMP) {
      const int lp = active ? D.lmp_slot[sidx] : -1;
      if (lp >= 0) {
        const S* Lp = D.lmp_L + 9 * (size_t)lp;
#pragma unroll
        for (int c = 0; c < 3; ++c) lpn[c] = Lp[c] * Lp[c] + Lp[3 + c] * Lp[3 + c] + Lp[6 + c] * Lp[6 + c];
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      cs[c] = group_sum(cs[c], G);
      if constexpr (LMP) cs[c] += lpn[c];
      jls[c] = S(1) / (eps + sqrt(cs[c]));
    }
    for (int i = j; i < n; i += G) {
      S* e = sJ + 26 * i + 18;
#pragma unroll
      for (int c = 0; c < 3; ++c) { e[c] *= jls[c]; e[3 + c] *= jls[c]; }
    }
    __syncwarp();
    // ---- write the per-observation records (scaled Jp, scaled Jl, weighted residual), coalesced per landmark ----
    for (int g2 = 0; g2 < T.nvalid; ++g2) {
      const S* src = ws + (size_t)g2 * GS;
      const size_t sb = (size_t)(T.slot_base + g2 * n);
      S* jo = D.jp + 20 * sb;
      for (int e = lane; e < n * 20; e += 32) {
        const int i2 = e / 20, k = e - 20 * i2;
        jo[e] = k < 18 ? src[26 * i2 + k] : S(0);
      }
      S* lo = D.jl + 6 * sb;
      for (int e = lane; e < n * 6; e += 32) {
        const int i2 = e / 6, k = e - 6 * i2;
        lo[e] = src[26 * i2 + 18 + k];
      }
      S* ro = D.res + 2 * sb;
      for (int e = lane; e < n * 2; e += 32) ro[e] = src[26 * (e >> 1) + 24 + (e & 1)];
    }
    __syncwarp();
    // ---- c. Householder QR of A = [Jl | r] (2n x 4), rows rho = 2i + parity ----
#define A_AT(rho, c) sJ[26 * ((rho) >> 1) + ((c) < 3 ? 18 + 3 * ((rho)&1) + (c) : 24 + ((rho)&1))]
    S tau[3] = {0, 0, 0};
    const int nrows = 2 * n;
    if constexpr (GIVENS) {
      // perform_qr_givens (ref: ipp:700-715): for column k the adjacent-row rotations (m-1, m), m = 2n-1 .. k+1, are a
      // sequential chain (each uses the entry the previous one produced): one lane per landmark runs it on the 2n x 4
      // matrix and keeps every (c, s): c in sV[3m + k], s in the entry A(m, k) the rotation has just annihilated.
      // (The reference rotates full rows, i.e. also the ~0 leftovers in columns < k; nothing downstream reads them.)
      if (j == 0) {
#pragma unroll 1
        for (int k = 0; k < 3; ++k) {
#pragma unroll 1
          for (int m = nrows - 1; m > k; --m) {
            const Rot<S> gr = make_givens(A_AT(m - 1, k), A_AT(m, k));
            for (int c = k; c < 4; ++c) {
              S x = A_AT(m, c), y = A_AT(m - 1, c);
              rot_apply(gr, x, y);  // applyOnTheLeft(m, m-1, gr)
              A_AT(m, c) = x; A_AT(m - 1, c) = y;
            }
            sV[3 * m + k] = gr.c;
            A_AT(m, k) = gr.s;
          }
        }
      }
      __syncwarp();
    }
#pragma unroll 1
    for (int k = 0; k < (GIVENS ? 0 : 3); ++k) {
      S ts = 0;
      for (int rho = j; rho < nrows; rho += G)
        if (rho > k) { const S v = A_AT(rho, k); ts += v * v; }
      ts = group_sum(ts, G);
      const S c0 = A_AT(k, k);
      S beta, tk, den;
      const bool degenerate = ts <= ST<S>::tiny();
      if (degenerate) { tk = 0; beta = c0; den = S(1); }
      else {
        beta = sqrt(c0 * c0 + ts);
        if (c0 >= S(0)) beta = -beta;
        den = c0 - beta;
        tk = (beta - c0) / beta;
      }
      tau[k] = tk;
      // tmp_c = essential^T bottom + row k   for the remaining columns
      S tmp[3] = {0, 0, 0};
      for (int rho = j; rho < nrows; rho += G) {
        if (rho > k) {
          const S v = degenerate ? S(0) : A_AT(rho, k) / den;
#pragma unroll
          for (int c = 1; c <= 3; ++c) if (k + c <= 3) tmp[c - 1] += v * A_AT(rho, k + c);
        }
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) tmp[c] = group_sum(tmp[c], G);
#pragma unroll
      for (int c = 1; c <= 3; ++c) if (k + c <= 3) tmp[c - 1] += A_AT(k, k + c);
      __syncwarp();
      for (int rho = j; rho < nrows; rho += G) {
        S v;
        if (rho < k) v = 0;
        else if (rho == k) {
          v = 1;
          A_AT(k, k) = beta;
          if (tk != S(0))
#pragma unroll
            for (int c = 1; c <= 3; ++c) if (k + c <= 3) A_AT(k, k + c) -= tk * tmp[c - 1];
        } else {
          v = degenerate ? S(0) : A_AT(rho, k) / den;
          if (tk != S(0)) {
            const S te = tk * v;
#pragma unroll
            for (int c = 1; c <= 3; ++c) if (k + c <= 3) A_AT(rho, k + c) -= te * tmp[c - 1];
          }
        }
        sV[3 * rho + k] = v;
      }
      __syncwarp();
    }
    S g10 = 0, g20 = 0, g21 = 0;
    if constexpr (!GIVENS) {
      for (int rho = j; rho < nrows; rho += G) {
        const S v0 = sV[3 * rho], v1 = sV[3 * rho + 1], v2 = sV[3 * rho + 2];
        g10 += v1 * v0; g20 += v2 * v0; g21 += v2 * v1;
      }
      g10 = group_sum(g10, G); g20 = group_sum(g20, G); g21 = group_sum(g21, G);
    }
    if (active && j == 0) {
      S* lk = D.lmk + 24 * (size_t)sidx;
      lk[0] = A_AT(0, 0); lk[1] = A_AT(0, 1); lk[2] = A_AT(0, 2);
      lk[3] = A_AT(1, 1); lk[4] = A_AT(1, 2); lk[5] = A_AT(2, 2);
      lk[6] = A_AT(0, 3); lk[7] = A_AT(1, 3); lk[8] = A_AT(2, 3);
      lk[18] = jls[0]; lk[19] = jls[1]; lk[20] = jls[2];
      if constexpr (LMP) {
        const int lp = D.lmp_slot[sidx];  // (slot and position re-read here: keeping them live from stage a spills)
        if (lp >= 0) {
          const S* Lp = D.lmp_L + 9 * (size_t)lp;
          const S* m = D.lmp_mean + 3 * (size_t)lp;
          const S* x = D.lms + 3 * (size_t)D.sorted_lm[sidx];
          const S e0 = x[0] - m[0], e1 = x[1] - m[1], e2 = x[2] - m[2];
          S* out = D.lmp_Lg + 12 * (size_t)lp;
#pragma unroll
          for (int r = 0; r < 3; ++r) {
#pragma unroll
            for (int c = 0; c < 3; ++c) out[3 * r + c] = Lp[3 * r + c] * jls[c];
            out[9 + r] = Lp[3 * r] * e0 + Lp[3 * r + 1] * e1 + Lp[3 * r + 2] * e2;
          }
        }
      }
    }
    // Q^T r (rows 0..2 = Q1^T r, rows 3..2n-1 = Q2^T r: the residual column of the marginalised block, ipp:443-466)
    if (active)
      for (int rho = j; rho < nrows; rho += G) D.qtr[2 * (size_t)slot0 + rho] = A_AT(rho, 3);
    // ---- d. apply Q^T = H2 H1 H0 to the block-diagonal Jp (compact WY) and write q1u + panel ----
    V2* ptile = reinterpret_cast<V2*>(D.panel + T.panel_off);
    const int ncols = 9 * n;
    if constexpr (GIVENS) {
      // Each panel column is an independent 2n-vector (non-zero in rows 2i, 2i+1 only) that goes through the same three
      // rotation chains.  Chain k at rotation m needs row m-1 as left by chain k-1, which chain k-1 finishes one step
      // later, so one descending sweep runs the three chains with a lag of one row each:
      //   step t: chain 0 does rotation t, chain 1 rotation t+1, chain 2 rotation t+2 (= final row t+2).
      const int R = nrows - 1;
#pragma unroll 1
      for (int k = 0; k < KP; ++k) {
        const int c0 = 2 * j + 2 * G * k;
        S a0[2], a1[2], cur0[2], cur1[2] = {0, 0}, cur2[2] = {0, 0};
        int r2i[2], oi[2], op[2];
        bool vc[2];
#pragma unroll
        for (int v = 0; v < 2; ++v) {
          const int c = c0 + v;
          vc[v] = c < ncols;
          const int i = vc[v] ? c / 9 : 0;
          const int p = vc[v] ? c - 9 * i : 0;
          oi[v] = i; op[v] = p; r2i[v] = 2 * i;
          a0[v] = vc[v] ? sJ[26 * i + p] : S(0);
          a1[v] = vc[v] ? sJ[26 * i + 9 + p] : S(0);
          cur0[v] = (R == r2i[v] + 1) ? a1[v] : S(0);
        }
        V2* pk = ptile + (size_t)k * 32 + lane;
#pragma unroll 1
        for (int t = R; t >= 1; --t) {
          const Rot<S> g0{sV[3 * t], A_AT(t, 0)};
          S o0[2], o1[2] = {0, 0};
#pragma unroll
          for (int v = 0; v < 2; ++v) {
            S y = (t - 1 == r2i[v]) ? a0[v] : ((t - 1 == r2i[v] + 1) ? a1[v] : S(0));
            o0[v] = cur0[v];
            rot_apply(g0, o0[v], y);
            cur0[v] = y;
          }
          if (t == R) {
            cur1[0] = o0[0]; cur1[1] = o0[1];
            continue;
          }
          const Rot<S> g1{sV[3 * (t + 1) + 1], A_AT(t + 1, 1)};
#pragma unroll
          for (int v = 0; v < 2; ++v) {
            S y = o0[v];
            o1[v] = cur1[v];
            rot_apply(g1, o1[v], y);
            cur1[v] = y;
          }
          if (t == R - 1) {
            cur2[0] = o1[0]; cur2[1] = o1[1];
            continue;
          }
          const Rot<S> g2{sV[3 * (t + 2) + 2], A_AT(t + 2, 2)};
          S f[2];
#pragma unroll
          for (int v = 0; v < 2; ++v) {
            S y = o1[v];
            f[v] = cur2[v];
            rot_apply(g2, f[v], y);
            cur2[v] = y;
          }
          if (active && o.write_panel) pk[(size_t)(t + 2 - 3) * KP * 32] = mk2(vc[0] ? f[0] : S(0), vc[1] ? f[1] : S(0));
        }
#pragma unroll
        for (int v = 0; v < 2; ++v)
          if (vc[v]) {
            S* q = sQ + 28 * (g * n + oi[v]) + op[v];
            q[0] = cur0[v]; q[9] = cur1[v]; q[18] = cur2[v];
          }
      }
    }
#pragma unroll 1
    for (int k = 0; k < (GIVENS ? 0 : KP); ++k) {
      const int c0 = 2 * j + 2 * G * k;
      S a0[2], a1[2], w0[2], w1[2], w2[2];
      int r2i[2], oi[2], op[2];
      bool vc[2];
#pragma unroll
      for (int v = 0; v < 2; ++v) {
        const int c = c0 + v;
        vc[v] = c < ncols;
        const int i = vc[v] ? c / 9 : 0;
        const int p = vc[v] ? c - 9 * i : 0;
        oi[v] = i; op[v] = p; r2i[v] = 2 * i;
        a0[v] = vc[v] ? sJ[26 * i + p] : S(0);
        a1[v] = vc[v] ? sJ[26 * i + 9 + p] : S(0);
        const S* va = sV + 3 * (2 * i);
        const S z0 = va[0] * a0[v] + va[3] * a1[v];
        const S z1 = va[1] * a0[v] + va[4] * a1[v];
        const S z2 = va[2] * a0[v] + va[5] * a1[v];
        w0[v] = tau[0] * z0;
        w1[v] = tau[1] * (z1 - g10 * w0[v]);
        w2[v] = tau[2] * (z2 - g20 * w0[v] - g21 * w1[v]);
      }
      // rows 0..2 = Q1^T Jp (undamped) -> staging
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const S v0 = sV[3 * r], v1 = sV[3 * r + 1], v2 = sV[3 * r + 2];
#pragma unroll
        for (int v = 0; v < 2; ++v) {
          const S sel = (r == r2i[v]) ? a0[v] : ((r == r2i[v] + 1) ? a1[v] : S(0));
          if (vc[v]) sQ[28 * (g * n + oi[v]) + 9 * r + op[v]] = sel - (w0[v] * v0 + w1[v] * v1 + w2[v] * v2);
        }
      }
      // rows 3..2n-1 = Q2^T Jp: out = -V[r] . w ; the two rows that carry the original Jacobian entries are patched below
      if (active && o.write_panel) {
        V2* pk = ptile + (size_t)k * 32 + lane;
        const S nw00 = vc[0] ? -w0[0] : S(0), nw01 = vc[0] ? -w1[0] : S(0), nw02 = vc[0] ? -w2[0] : S(0);
        const S nw10 = vc[1] ? -w0[1] : S(0), nw11 = vc[1] ? -w1[1] : S(0), nw12 = vc[1] ? -w2[1] : S(0);
        const S* vp = sV + 9;
#pragma unroll 4
        for (int r = 3; r < nrows; ++r, vp += 3) {
          const S v0 = vp[0], v1 = vp[1], v2 = vp[2];
          pk[(size_t)(r - 3) * KP * 32] = mk2(nw00 * v0 + nw01 * v1 + nw02 * v2, nw10 * v0 + nw11 * v1 + nw12 * v2);
        }
        // patch: rows 2i and 2i+1 of each column also carry a0 / a1 (same lane re-writes its own element)
#pragma unroll
        for (int v = 0; v < 2; ++v) {
          if (!vc[v]) continue;
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const int r = r2i[v] + q;
            if (r >= 3) {
              const S* vq = sV + 3 * r;
              const S val = (q == 0 ? a0[v] : a1[v]) - (w0[v] * vq[0] + w1[v] * vq[1] + w2[v] * vq[2]);
              S* dst = reinterpret_cast<S*>(pk + (size_t)(r - 3) * KP * 32) + v;
              *dst = val;
            }
          }
        }
      }
    }
#undef A_AT
    for (int e = lane; e < Wn; e += 32) sQ[28 * e + 27] = 0;  // pad
    __syncwarp();
    warp_copy_out(D.q1u + 28 * (size_t)T.slot_base, sQ, T.nvalid * n * 28, lane);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// K2  stage 2: Givens landmark damping, RCS gradient (ref: ipp:638-658 = :165-210, :443-466)
//   The 6 rotations only mix the 3 Q1 rows with the 3 damping rows, so each panel column is an
//   independent 6-vector: q1d and the 3 damping rows are recomputed from the undamped q1u (instead of
//   un-doing the previous rotations, ipp:175-186).  The gradient uses orthogonality of [Q1d; P]:
//   P^T (Q2^T r) = Jp^T r - Q1d^T (Q1^T r)_d.
// ------------------------------------------------------------------------------------------------

// scratch scalars per warp for a tile (host mirrors this in Solver::init)
__host__ __device__ inline int stage2_need(int n, int G, int KP) {
  const int W = 32 / G, Wn = W * n;
  const int CS = (2 * G * KP) | 1;
  return 3 * W * CS + Wn * 9 + W * 20 + 8;
}

// One warp per tile, one lane per observation: the 112-byte q1u / q1d and 80-byte jp records are moved with
// 16-byte vector accesses straight from / to registers; only the 3 damping rows (which must land in the
// column-interleaved panel layout) and the gradient are staged through shared memory for coalesced stores.
// PANEL = true (default, the reference's arithmetic): the gradient is P^T (Q2^T r) (ipp:443-466) and the SCHUR_JACOBI
// blocks are B^T B of the panel columns (ipp:520-552).  Panel rows 3..2n-1 do not depend on lambda, so their
// contribution (b0, blocks0) is accumulated once per linearisation by k_panel_grad_blocks; this kernel adds the part of
// the three damping rows: yobs[slot] = sum_d D_d (Q^T r)_{damping row d}, and keeps the rows' 3x9 entries per slot (dmp)
// for the block kernel.  PANEL = false (no panels stored: operator_form = implicit): the orthogonality identities
//   P^T (Q2^T r) = Jp^T r - Q1d^T (Q1^T r)_d ,  B^T B = Jp^T Jp - Q1d^T Q1d   (they cancel: float64 recommended).
// The landmark prior's 3 rows [L~ | 0 | g] and the 3 damping rows [sqrt(lambda) I | 0 | 0] have no camera columns, so a QR
// of the 6x3 [L~; sqrt(lambda) I] with the residual [g; 0] compresses them into 3 rows [C | 0 | c], C upper triangular
// (DESIGN.md section 17).  Givens rotations in Eigen's convention, as the damping rotations; a zero column (rank-deficient
// L, and lambda = 0) only meets rotations with c = +-1, s = 0.  The residual left in rows 3..5 does not depend on the
// step and is dropped.
template <class S>
__device__ __forceinline__ void lm_prior_compress(const S* __restrict__ Lg, S sl, S (&C)[3][3], S (&c)[3]) {
  S M[6][4];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { M[r][k] = Lg[3 * r + k]; M[3 + r][k] = r == k ? sl : S(0); }
    M[r][3] = Lg[9 + r];
    M[3 + r][3] = 0;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int m = k + 1; m < 6; ++m) {
      const Rot<S> gq = make_givens(M[k][k], M[m][k]);
#pragma unroll
      for (int cc = k; cc < 4; ++cc) rot_apply(gq, M[m][cc], M[k][cc]);
    }
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int k = 0; k < 3; ++k) C[r][k] = k >= r ? M[r][k] : S(0);
    c[r] = M[r][3];
  }
}

// LMP (landmark priors): a landmark with a prior starts its 6 rotations from Dw = C, dr = c (lm_prior_compress) instead
// of sqrt(lambda) I, 0, also at lambda = 0; every other landmark, and every per-observation step, is unchanged.
template <class S, bool PANEL, bool LMP = false>
__global__ void __launch_bounds__(128) k_stage2(DevPtrs<S> D, S lambda, Scratch<S> sc, int write_panel) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using V2 = typename ST<S>::V2;
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  S* ws_smem = reinterpret_cast<S*>(smem_raw) + (size_t)wib * sc.smem_cap;
  for (int t = blockIdx.x * (blockDim.x >> 5) + wib; t < D.ntiles; t += gridDim.x * (blockDim.x >> 5)) {
    const TileInfo T = D.tiles[t];
    const int n = T.n, G = T.G, KP = T.KP, W = 32 / G, Wn = W * n;
    const int ncols = 9 * n;
    const int CS = (2 * G * KP) | 1;
    const int g = lane / G, j = lane - g * G;
    const bool active = g < T.nvalid;
    S* ws = scratch_ptr(sc, ws_smem, stage2_need(n, G, KP));
    S* sD = ws;                      // [3][W][CS] damping rows in (landmark, column) order
    S* sG = sD + 3 * W * CS;         // [Wn][9]    gradient contribution per observation
    S* sRot = sG + Wn * 9;           // [W][20]    6 rotations (c,s) + damped Q1^T r (3) + residual entries of the damping rows (3)
    // ---- rotations of landmark `lane` (ref: ipp:188-209), Eigen makeGivens / applyOnTheLeft ----
    if (lane < T.nvalid) {
      S* lk = D.lmk + 24 * (size_t)(T.lm_base + lane);
      S Rw[3][3] = {{lk[0], lk[1], lk[2]}, {0, lk[3], lk[4]}, {0, 0, lk[5]}};
      S Dw[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
      S rr[3] = {lk[6], lk[7], lk[8]}, dr[3] = {0, 0, 0};
      S* ro = sRot + 20 * lane;
      int lp = -1;
      if constexpr (LMP) lp = D.lmp_slot[T.lm_base + lane];
      if (lambda == S(0) && lp < 0) {
#pragma unroll
        for (int q = 0; q < 6; ++q) { ro[2 * q] = 1; ro[2 * q + 1] = 0; }
      } else {
        const S sl = sqrt(lambda);
        if (LMP && lp >= 0) lm_prior_compress(D.lmp_Lg + 12 * (size_t)lp, sl, Dw, dr);
        else { Dw[0][0] = sl; Dw[1][1] = sl; Dw[2][2] = sl; }
        int q = 0;
#pragma unroll
        for (int nn = 0; nn < 3; ++nn)
#pragma unroll
          for (int m = 0; m <= nn; ++m) {
            const int d = nn - m;
            const Rot<S> gq = make_givens(Rw[nn][nn], Dw[d][nn]);
            ro[2 * q] = gq.c; ro[2 * q + 1] = gq.s;
            ++q;
#pragma unroll
            for (int c = 0; c < 3; ++c) rot_apply(gq, Dw[d][c], Rw[nn][c]);
            rot_apply(gq, dr[d], rr[nn]);
          }
      }
      ro[12] = rr[0]; ro[13] = rr[1]; ro[14] = rr[2];
      ro[15] = dr[0]; ro[16] = dr[1]; ro[17] = dr[2];
      lk[9] = Rw[0][0]; lk[10] = Rw[0][1]; lk[11] = Rw[0][2]; lk[12] = Rw[1][1]; lk[13] = Rw[1][2]; lk[14] = Rw[2][2];
      lk[15] = rr[0]; lk[16] = rr[1]; lk[17] = rr[2];
    }
    __syncwarp();
    // ---- one observation per lane and step: q1d, damping-row entries, gradient ----
    if (active) {
      Rot<S> rot[6];
      const S* ro = sRot + 20 * g;
#pragma unroll
      for (int q = 0; q < 6; ++q) { rot[q].c = ro[2 * q]; rot[q].s = ro[2 * q + 1]; }
      const S rr0 = ro[12], rr1 = ro[13], rr2 = ro[14];
      const S dr0 = ro[15], dr1 = ro[16], dr2 = ro[17];
      for (int i = j; i < n; i += G) {
        const size_t sl = (size_t)(T.slot_base + g * n + i);
        S q[28], jp[PANEL ? 4 : 20], dm[PANEL ? 28 : 4];
        load_rec<S, 28>(D.q1u + 28 * sl, q);
        S r0 = 0, r1 = 0;
        if constexpr (!PANEL) {
          load_rec<S, 20>(D.jp + 20 * sl, jp);
          r0 = D.res[2 * sl]; r1 = D.res[2 * sl + 1];
        }
        S* d0 = sD + (0 * W + g) * CS + 9 * i;
        S* d1 = sD + (1 * W + g) * CS + 9 * i;
        S* d2 = sD + (2 * W + g) * CS + 9 * i;
        S* go = sG + 9 * (g * n + i);
#pragma unroll
        for (int p = 0; p < 9; ++p) {
          S qv[3] = {q[p], q[9 + p], q[18 + p]}, dv[3] = {0, 0, 0};
          int qi = 0;
#pragma unroll
          for (int nn = 0; nn < 3; ++nn)
#pragma unroll
            for (int m = 0; m <= nn; ++m) rot_apply(rot[qi++], dv[nn - m], qv[nn]);
          q[p] = qv[0]; q[9 + p] = qv[1]; q[18 + p] = qv[2];
          d0[p] = dv[0]; d1[p] = dv[1]; d2[p] = dv[2];
          if constexpr (PANEL) {
            // damping-row part of P^T (Q2^T r) (ipp:443-466); rows 3..2n-1 are in b0
            dm[p] = dv[0]; dm[9 + p] = dv[1]; dm[18 + p] = dv[2];
            go[p] = dv[0] * dr0 + dv[1] * dr1 + dv[2] * dr2;
          } else {
            // gradient of the reduced system: b_c = jp_c^T r_i - q1d_c^T (Q1^T r)_d
            go[p] = jp[p] * r0 + jp[9 + p] * r1 - (qv[0] * rr0 + qv[1] * rr1 + qv[2] * rr2);
          }
        }
        q[27] = 0;
        store_rec<S, 28>(D.q1d + 28 * sl, q);
        if constexpr (PANEL) {
          dm[27] = 0;
          store_rec<S, 28>(D.dmp + 28 * sl, dm);
        }
      }
    }
    __syncwarp();
    // ---- coalesced stores: gradient (observation-major), damping rows (panel layout) ----
    {
      const int nsl = T.nvalid * n;
      for (int e = lane; e < nsl * 9; e += 32) D.yobs[9 * (size_t)T.slot_base + e] = sG[e];
      if constexpr (!PANEL) {
        // the dmp records, kept here only for the assembly of S (allocated when the handle may build it): from the rows in
        // shared memory, the same values as the panel rows below
        if (D.dmp)
          for (int e = lane; e < nsl * 28; e += 32) {
            const int sl = e / 28, k = e - 28 * sl, gg = sl / n, d = k / 9;
            D.dmp[28 * (size_t)T.slot_base + e] = k < 27 ? sD[(d * W + gg) * CS + 9 * (sl - gg * n) + (k - 9 * d)] : S(0);
          }
      }
      if (active && write_panel) {
        V2* ptile = reinterpret_cast<V2*>(D.panel + T.panel_off) + (size_t)(2 * n - 3) * KP * 32 + lane;
        for (int k = 0; k < KP; ++k) {
          const int c = 2 * j + 2 * G * k;
#pragma unroll
          for (int d = 0; d < 3; ++d) {
            const S* row = sD + (d * W + g) * CS;
            ptile[((size_t)d * KP + k) * 32] = mk2(c < ncols ? row[c] : S(0), c + 1 < ncols ? row[c + 1] : S(0));
          }
        }
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// K2sc  stage 2 of the Schur-complement solvers (solver_type = SCHUR_COMPLEMENT / POWER_SCHUR_COMPLEMENT; SURVEY 8f row 3)
//   ref: sc/landmark_block.hpp:215-279 (set_landmark_damping, Hll^-1, add_Hb), solver/linearizor_sc.cpp:112-204.
//   The landmark is eliminated through the NORMAL equations instead of QR: Hll = Jl^T Jl + lambda I (3x3), factorised
//   Hll = R^T R (Cholesky, R upper).  Everything downstream is then the SAME data as the QR path with the implicit
//   operator, because Hll^-1 = R^-1 R^-T:
//       q1d_i := R^-T Jl_i^T Jp_i   (3x9)        =>  sum_i q1d_i^T (sum_j q1d_j x_j) = Jp^T Jl Hll^-1 Jl^T Jp x  (E_0 x)
//       rr    := R^-T Jl^T r                      =>  b_i = Jp_i^T r_i - q1d_i^T rr = Jp_i^T (r_i - Jl_i Hll^-1 Jl^T r)
//       landmark increment = -R^-1 (rr + sum_i q1d_i dp_i) = -Hll^-1 Jl^T (r + Jp dp)
//   so the reduced operator (k_matvec_implicit*), the SCHUR_JACOBI blocks (k_precond_partial<1>), PCG and the
//   back-substitution kernel are shared with the square-root solver; only this kernel differs -- and with it the
//   numerics: the condition number of the landmark block is squared, which is what the QR solver avoids.
//   One warp per tile, G lanes per landmark, lane per observation.
// ------------------------------------------------------------------------------------------------
//   LMP (landmark priors, DESIGN.md section 17): Hll += L~^T L~ and Jl^T r += L~^T g of the landmark's prior.
template <class S, bool LMP = false>
__global__ void __launch_bounds__(128) k_sc_stage2(DevPtrs<S> D, S lambda) {
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int t = blockIdx.x * (blockDim.x >> 5) + wib; t < D.ntiles; t += gridDim.x * (blockDim.x >> 5)) {
    const TileInfo T = D.tiles[t];
    const int n = T.n, G = T.G;
    const int g = lane / G, j = lane - g * G;
    const bool active = g < T.nvalid;
    const size_t slot0 = (size_t)(T.slot_base + g * n);
    S h[6] = {0, 0, 0, 0, 0, 0}, gv[3] = {0, 0, 0};
    if (active) {
      for (int i = j; i < n; i += G) {
        const S* jl = D.jl + 6 * (slot0 + i);
        const S r0 = D.res[2 * (slot0 + i)], r1 = D.res[2 * (slot0 + i) + 1];
        const S a0 = jl[0], a1 = jl[1], a2 = jl[2], b0 = jl[3], b1 = jl[4], b2 = jl[5];
        h[0] += a0 * a0 + b0 * b0; h[1] += a0 * a1 + b0 * b1; h[2] += a0 * a2 + b0 * b2;
        h[3] += a1 * a1 + b1 * b1; h[4] += a1 * a2 + b1 * b2; h[5] += a2 * a2 + b2 * b2;
        gv[0] += a0 * r0 + b0 * r1; gv[1] += a1 * r0 + b1 * r1; gv[2] += a2 * r0 + b2 * r1;
      }
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) h[k] = group_sum(h[k], G);
#pragma unroll
    for (int k = 0; k < 3; ++k) gv[k] = group_sum(gv[k], G);
    if constexpr (LMP) {
      const int lp = D.lmp_slot[T.lm_base + g];
      if (lp >= 0) {
        const S* pg = D.lmp_Lg + 12 * (size_t)lp;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const S a0 = pg[3 * r], a1 = pg[3 * r + 1], a2 = pg[3 * r + 2], gr = pg[9 + r];
          h[0] += a0 * a0; h[1] += a0 * a1; h[2] += a0 * a2; h[3] += a1 * a1; h[4] += a1 * a2; h[5] += a2 * a2;
          gv[0] += a0 * gr; gv[1] += a1 * gr; gv[2] += a2 * gr;
        }
      }
    }
    h[0] += lambda; h[3] += lambda; h[5] += lambda;  // landmark damping: Hll = Jl^T Jl + lambda I (sc/landmark_block.hpp:244-247)
    // Cholesky Hll = R^T R.  A block that is singular in working precision (one valid observation, lam below the resolution
    // of its diagonal) gives a NaN pivot; it reaches b, PCG and the l_diff of rba_apply, which reports it (as the reference,
    // whose Hll.inverse() feeds inf / NaN into CG), so no flag is raised here.
    const S r00 = sqrt(h[0]);
    const S r01 = h[1] / r00, r02 = h[2] / r00;
    const S r11 = sqrt(h[3] - r01 * r01);
    const S r12 = (h[4] - r01 * r02) / r11;
    const S r22 = sqrt(h[5] - r02 * r02 - r12 * r12);
    const S rr0 = gv[0] / r00;
    const S rr1 = (gv[1] - r01 * rr0) / r11;
    const S rr2 = (gv[2] - r02 * rr0 - r12 * rr1) / r22;
    if (active && j == 0) {
      S* lk = D.lmk + 24 * (size_t)(T.lm_base + g);
      lk[9] = r00; lk[10] = r01; lk[11] = r02; lk[12] = r11; lk[13] = r12; lk[14] = r22;
      lk[15] = rr0; lk[16] = rr1; lk[17] = rr2;
    }
    if (active) {
      for (int i = j; i < n; i += G) {
        const size_t sl = slot0 + i;
        S jp[20], q[28];
        load_rec<S, 20>(D.jp + 20 * sl, jp);
        const S* jl = D.jl + 6 * sl;
        const S a0 = jl[0], a1 = jl[1], a2 = jl[2], b0 = jl[3], b1 = jl[4], b2 = jl[5];
        const S r0 = D.res[2 * sl], r1 = D.res[2 * sl + 1];
        S* go = D.yobs + 9 * sl;
#pragma unroll
        for (int p = 0; p < 9; ++p) {
          const S t0 = a0 * jp[p] + b0 * jp[9 + p], t1 = a1 * jp[p] + b1 * jp[9 + p], t2 = a2 * jp[p] + b2 * jp[9 + p];
          const S c0 = t0 / r00;
          const S c1 = (t1 - r01 * c0) / r11;
          const S c2 = (t2 - r02 * c0 - r12 * c1) / r22;
          q[p] = c0; q[9 + p] = c1; q[18 + p] = c2;
          go[p] = jp[p] * r0 + jp[9 + p] * r1 - (c0 * rr0 + c1 * rr1 + c2 * rr2);
        }
        q[27] = 0;
        store_rec<S, 28>(D.q1d + 28 * sl, q);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// K4i  the same operator in implicit form (opt-in: rba_solver_opts.operator_form = 1; SURVEY 8d last remark)
//   [Q1d; P] is an orthogonal transform of [Jp; 0], so  P^T P = Jp^T Jp - Q1d^T Q1d  (the identity k_stage2 and
//   k_precond_partial already use) and, per landmark with observations i,
//       u   = sum_i Q1d_i x_i                      (3-vector;  x_i = the 9 entries of the camera of observation i)
//       y_i = Jp_i^T (Jp_i x_i) - Q1d_i^T u
//   The kernel reads the 80-byte jp and 112-byte q1d records (192 n bytes per landmark in f32) instead of the dense
//   18 n^2 s panel.  It is the Schur-complement product in disguise: the subtraction cancels, so in float32 it gives up
//   the numerical advantage that is the point of the square-root formulation -- hence opt-in, default stays the
//   reference's dense Q2 panel product (ref: ipp:400-441).
//   One warp per tile, one lane per observation (as k_stage2); writes yobs[slot][9], reduced per camera by
//   k_cam_reduce_final over the observation CSR.
// ------------------------------------------------------------------------------------------------
template <class S>
__global__ void __launch_bounds__(128) k_matvec_implicit(DevPtrs<S> D, int tile_begin, const S* __restrict__ xvec, const int* done, int pdl,
                                                          int e0_only = 0) {
  if (done && *reinterpret_cast<const volatile int*>(done)) return;  // monotonic flag, see k_matvec_small_tma
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  if (done && *done) return;
  if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int t = tile_begin + blockIdx.x * (blockDim.x >> 5) + wib; t < D.ntiles; t += gridDim.x * (blockDim.x >> 5)) {
    const TileInfo T = D.tiles[t];
    const int n = T.n, G = T.G;
    const int g = lane / G, j = lane - g * G;
    const bool active = g < T.nvalid;
    const size_t sl0 = (size_t)(T.slot_base + g * n);
    S u0 = 0, u1 = 0, u2 = 0;
    if (active) {
      for (int i = j; i < n; i += G) {
        const size_t sl = sl0 + i;
        S q[28];
        load_rec<S, 28>(D.q1d + 28 * sl, q);
        const S* xc = xvec + 9 * (size_t)D.slot_cam[sl];
#pragma unroll
        for (int p = 0; p < 9; ++p) {
          const S xv = xc[p];
          u0 += q[p] * xv; u1 += q[9 + p] * xv; u2 += q[18 + p] * xv;
        }
      }
    }
    u0 = group_sum(u0, G); u1 = group_sum(u1, G); u2 = group_sum(u2, G);
    if (active) {
      for (int i = j; i < n; i += G) {
        const size_t sl = sl0 + i;
        S q[28], jp[20];
        load_rec<S, 28>(D.q1d + 28 * sl, q);
        load_rec<S, 20>(D.jp + 20 * sl, jp);
        const S* xc = xvec + 9 * (size_t)D.slot_cam[sl];
        S t0 = 0, t1 = 0;
#pragma unroll
        for (int p = 0; p < 9; ++p) {
          const S xv = xc[p];
          t0 += jp[p] * xv; t1 += jp[9 + p] * xv;
        }
        S* yo = D.yobs + 9 * sl;
#pragma unroll
        // e0_only (Power-SC): y_i = Q1d_i^T u = (Jp^T Jl Hll^-1 Jl^T Jp x)_i alone (sc/linearization_power_sc.hpp:261-287)
        for (int p = 0; p < 9; ++p) {
          const S e0 = q[p] * u0 + q[9 + p] * u1 + q[18 + p] * u2;
          yo[p] = e0_only ? e0 : (jp[p] * t0 + jp[9 + p] * t1) - e0;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// K3a  block-Jacobi preconditioner blocks, camera-major (ref: ipp:520-552 SCHUR_JACOBI, :554-569 JACOBI)
//   (Q2^T Jp)_i^T (Q2^T Jp)_i = Jp_i^T Jp_i - (Q1d^T Jp)_i^T (Q1d^T Jp)_i  (Q orthogonal, Givens on 6 rows)
//   thread per ReduceItem chunk of <= 32 observations ... here: one thread per (item, 8-slot subchunk) would
//   be finer; we use thread per item-of-32 built on the host (pb_items).
// ------------------------------------------------------------------------------------------------
// MODE 0: JACOBI  sum Jp_i^T Jp_i                                         (ipp:554-569)
// MODE 1: SCHUR_JACOBI through the orthogonality identity  Jp^T Jp - Q1d^T Q1d  (operator_form = implicit only)
// MODE 2: SCHUR_JACOBI, part of the 3 damping rows  sum_d D_d^T D_d  from the dmp records   (ipp:520-552, rows 2n..2n+2)
// MODE 3: SCHUR_JACOBI, lambda-independent part: sum of the per-slot blk0 records written by k_panel_grad_blocks
template <class S, int MODE>
__global__ void __launch_bounds__(128) k_precond_partial(const S* __restrict__ recA, const S* __restrict__ recB,
                                                          const int* __restrict__ slots, const ReduceItem* __restrict__ items,
                                                          int nitems, S* __restrict__ pblk) {
  const int it = blockIdx.x * blockDim.x + threadIdx.x;
  if (it >= nitems) return;
  const ReduceItem I = items[it];
  S acc[45];
#pragma unroll
  for (int k = 0; k < 45; ++k) acc[k] = 0;
  for (int e = I.begin; e < I.end; ++e) {
    const size_t sl = (size_t)slots[e];
    if constexpr (MODE == 3) {
      S v[48];
      load_rec<S, 48>(recA + 48 * sl, v);
#pragma unroll
      for (int k = 0; k < 45; ++k) acc[k] += v[k];
    } else if constexpr (MODE == 2) {
      S v[28];
      load_rec<S, 28>(recA + 28 * sl, v);
      int k = 0;
#pragma unroll
      for (int a = 0; a < 9; ++a)
#pragma unroll
        for (int b = a; b < 9; ++b) acc[k++] += v[a] * v[b] + v[9 + a] * v[9 + b] + v[18 + a] * v[18 + b];
    } else {
      S v[20], w[MODE == 1 ? 28 : 4];
      load_rec<S, 20>(recA + 20 * sl, v);
      if constexpr (MODE == 1) load_rec<S, 28>(recB + 28 * sl, w);
      int k = 0;
#pragma unroll
      for (int a = 0; a < 9; ++a)
#pragma unroll
        for (int b = a; b < 9; ++b) {
          S sacc = v[a] * v[b] + v[9 + a] * v[9 + b];
          if constexpr (MODE == 1) sacc -= w[a] * w[b] + w[9 + a] * w[9 + b] + w[18 + a] * w[18 + b];
          acc[k++] += sacc;
        }
    }
  }
  S* o = pblk + 48 * (size_t)it;
#pragma unroll
  for (int k = 0; k < 45; ++k) o[k] = acc[k];
}

// blocks[cam][81] = (addend[cam][81] +) sum of partial upper triangles (symmetrised)
template <class S>
__global__ void k_precond_final(const S* __restrict__ pblk, const int* __restrict__ cam_item_ptr, int nc,
                                const S* __restrict__ addend, S* __restrict__ blocks) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 45 * nc) return;
  const int cam = i / 45, k = i - 45 * cam;
  S s = 0;
  for (int it = cam_item_ptr[cam]; it < cam_item_ptr[cam + 1]; ++it) s += pblk[48 * (size_t)it + k];
  int a = 0, rem = k;
  while (rem >= 9 - a) { rem -= 9 - a; ++a; }
  const int b = a + rem;
  if (addend) s += addend[81 * (size_t)cam + 9 * a + b];
  blocks[81 * (size_t)cam + 9 * a + b] = s;
  blocks[81 * (size_t)cam + 9 * b + a] = s;
}

// ------------------------------------------------------------------------------------------------
// K2p  lambda-independent part of the RCS gradient and of the SCHUR_JACOBI blocks from the stored Q2 panels, once per
//      linearisation:  per observation slot i of a landmark, with B = panel rows 3..2n-1 restricted to the slot's 9 columns
//      and t = (Q2^T r) rows 3..2n-1:   blk0[slot] = B^T B (45 upper entries),   yobs[slot] = B^T t.
//   ref: ipp:520-552 (add_Q2TJp_T_Q2TJp_blockdiag), ipp:443-466 (add_Q2TJp_T_Q2Tr).  Sums of squares: no cancellation,
//   positive semi-definite by construction -- the float32 robustness the square-root formulation is about.
//   Warp per tile, lane per observation (32 observations per pass); a row of the tile is covered exactly once by the
//   lanes' 5 two-scalar loads each (L1 merges the sectors shared by neighbouring observations).
// ------------------------------------------------------------------------------------------------
template <class S>
__global__ void __launch_bounds__(128) k_panel_grad_blocks(DevPtrs<S> D, int want_blocks, TileOrder to) {
  using V2 = typename ST<S>::V2;
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int idx = blockIdx.x * (blockDim.x >> 5) + wib;; idx += gridDim.x * (blockDim.x >> 5)) {
    const int t = tile_at(to, idx, D.ntiles);
    if (t < 0) break;
    const TileInfo T = D.tiles[t];
    const int n = T.n, G = T.G, KP = T.KP;
    const int lg = 31 - __clz(G);
    const int nobs = T.nvalid * n;
    const int nrows = 2 * n - 3;
    const V2* __restrict__ ptile = reinterpret_cast<const V2*>(D.panel + T.panel_off);
    const size_t rstride = (size_t)KP * 32;
    for (int e = lane; e < nobs; e += 32) {
      const int g = e / n, i = e - g * n;
      const int c0 = 9 * i;
      const bool odd = c0 & 1;
      const int p0 = c0 >> 1;
      int off[5];
#pragma unroll
      for (int q = 0; q < 5; ++q) {
        const int p = p0 + q;
        off[q] = (p >> lg) * 32 + g * G + (p & (G - 1));
      }
      const S* __restrict__ tq = D.qtr + 2 * (size_t)(T.slot_base + g * n) + 3;
      S acc[45], gacc[9];
#pragma unroll
      for (int k = 0; k < 45; ++k) acc[k] = 0;
#pragma unroll
      for (int k = 0; k < 9; ++k) gacc[k] = 0;
#pragma unroll 2
      for (int r = 0; r < nrows; ++r) {
        const V2* pr = ptile + (size_t)r * rstride;
        V2 a[5];
#pragma unroll
        for (int q = 0; q < 5; ++q) a[q] = __ldg(pr + off[q]);
        const S tr = __ldg(tq + r);
        const S el[10] = {a[0].x, a[0].y, a[1].x, a[1].y, a[2].x, a[2].y, a[3].x, a[3].y, a[4].x, a[4].y};
        S v[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) v[k] = odd ? el[k + 1] : el[k];
#pragma unroll
        for (int k = 0; k < 9; ++k) gacc[k] += v[k] * tr;
        if (want_blocks) {
          int k = 0;
#pragma unroll
          for (int x = 0; x < 9; ++x)
#pragma unroll
            for (int y = x; y < 9; ++y) acc[k++] += v[x] * v[y];
        }
      }
      const size_t sl = (size_t)(T.slot_base + e);
#pragma unroll
      for (int k = 0; k < 9; ++k) D.yobs[9 * sl + k] = gacc[k];
      if (want_blocks) {
        S o[48];
#pragma unroll
        for (int k = 0; k < 45; ++k) o[k] = acc[k];
        o[45] = o[46] = o[47] = 0;
        store_rec<S, 48>(D.blk0 + 48 * sl, o);
      }
    }
  }
}

// K3b  (blocks + lambda I) -> explicit inverse via Cholesky (ref: cg/preconditioner.hpp:79-120; pose damping
//      linearization_qr.hpp:796-802 / linearizor_qr.cpp:228-232).  thread per camera.
//      Camera with fixed parameters (cam_fixed): the fixed rows and columns of the damped block become the identity before
//      the Cholesky and are zeroed in the inverse, and the fixed entries of b (final here) are zeroed.  The result is the
//      inverse of the free sub-block: z = M^-1 r then has exactly zero fixed entries whatever r holds there, which keeps PCG
//      and the power series on the restricted system (DESIGN.md, "Fixed camera parameters").
//      Camera priors (DESIGN.md section 14): prior_H (the SCHUR_JACOBI blocks; the JACOBI blocks hold it since the
//      linearisation) is added to the block and prior_g to b (already summed over the shards), both before the masking.
template <class S>
__global__ void __launch_bounds__(64) k_precond_invert(const S* __restrict__ src, S lambda, int nc,
                                                        S* __restrict__ blocks_out, S* __restrict__ inv,
                                                        const uint8_t* __restrict__ cam_fixed, S* __restrict__ b,
                                                        const S* __restrict__ prior_H = nullptr, const S* __restrict__ prior_g = nullptr) {
  const int cam = blockIdx.x * blockDim.x + threadIdx.x;
  if (cam >= nc) return;
  const unsigned fm = cam_fixed ? fixed_entry_mask(cam_fixed[cam]) : 0u;
  // everything is fully unrolled so that the 9x9 block lives in registers (no local-memory round trips)
  S A[9][9];
#pragma unroll
  for (int r = 0; r < 9; ++r)
#pragma unroll
    for (int c = 0; c < 9; ++c) A[r][c] = src[81 * (size_t)cam + 9 * r + c];
  if (prior_H)
#pragma unroll
    for (int r = 0; r < 9; ++r)
#pragma unroll
      for (int c = 0; c < 9; ++c) A[r][c] += prior_H[81 * (size_t)cam + 9 * r + c];
  if (prior_g)
#pragma unroll
    for (int d = 0; d < 9; ++d) b[9 * (size_t)cam + d] += prior_g[9 * (size_t)cam + d];
#pragma unroll
  for (int d = 0; d < 9; ++d) A[d][d] += lambda;
  if (blocks_out)
#pragma unroll
    for (int r = 0; r < 9; ++r)
#pragma unroll
      for (int c = 0; c < 9; ++c) blocks_out[81 * (size_t)cam + 9 * r + c] = A[r][c];
  if (fm) {
#pragma unroll
    for (int r = 0; r < 9; ++r)
#pragma unroll
      for (int c = 0; c < 9; ++c)
        if (((fm >> r) | (fm >> c)) & 1u) A[r][c] = (r == c) ? S(1) : S(0);
#pragma unroll
    for (int d = 0; d < 9; ++d)
      if ((fm >> d) & 1u) b[9 * (size_t)cam + d] = S(0);
  }
  // in-place Cholesky of the upper-stored symmetric block: lower factor L in A[i][j], i >= j
  // (selfadjointView<Upper>().llt(), ref: cg/preconditioner.hpp:107-113)
#pragma unroll
  for (int jj = 0; jj < 9; ++jj) {
    S sdiag = A[jj][jj];
#pragma unroll
    for (int k = 0; k < jj; ++k) sdiag -= A[jj][k] * A[jj][k];
    const S d = sqrt(sdiag);
    A[jj][jj] = d;
#pragma unroll
    for (int i = jj + 1; i < 9; ++i) {
      S t = A[jj][i];  // upper entry (jj, i) of the symmetric input
#pragma unroll
      for (int k = 0; k < jj; ++k) t -= A[i][k] * A[jj][k];
      A[i][jj] = t / d;
    }
  }
  // Li = L^-1 (lower triangular), stored in the strict upper part + a separate diagonal
  S Li[9][9];
#pragma unroll
  for (int c = 0; c < 9; ++c) {
#pragma unroll
    for (int r = 0; r < 9; ++r) {
      if (r < c) Li[r][c] = 0;
      else {
        S t = (r == c) ? S(1) : S(0);
#pragma unroll
        for (int k = 0; k < 9; ++k) if (k >= c && k < r) t -= A[r][k] * Li[k][c];
        Li[r][c] = t / A[r][r];
      }
    }
  }
  // A fixed entry d has an identity row and column in the block, so column d of Li is the unit vector e_d and row d of Li
  // is zero off the diagonal.  Zeroing Li[d][d] therefore zeroes row and column d of the inverse exactly and leaves the free
  // entries (the inverse of the free sub-block) unchanged.
  if (fm)
#pragma unroll
    for (int d = 0; d < 9; ++d)
      if ((fm >> d) & 1u) Li[d][d] = S(0);
  // inverse = Li^T Li
  S* out = inv + 81 * (size_t)cam;
#pragma unroll
  for (int r = 0; r < 9; ++r)
#pragma unroll
    for (int c = r; c < 9; ++c) {
      S t = 0;
#pragma unroll
      for (int k = 0; k < 9; ++k) if (k >= c) t += Li[k][r] * Li[k][c];
      out[9 * r + c] = t;
      out[9 * c + r] = t;
    }
}

// ------------------------------------------------------------------------------------------------
// K4  rcs_matvec: y_obs = P^T (P x_red) per landmark, P = dense Q2^T Jp panel (2n x 9n)
//   ref: qr/impl/landmark_block_base.ipp:400-441 under qr/linearization_qr.hpp:406-429
//   Warp per MatvecItem; lanes own panel columns; the panel is streamed exactly once with coalesced
//   2-scalar vector loads; row dot products are reduced with log2(G) shuffles; x is gathered and y is
//   written through a per-warp shared-memory transpose so that both are coalesced.
// ------------------------------------------------------------------------------------------------
// Gather x_red of the W landmarks of a tile into shared memory (xs[g][c], row stride CS, padding zeroed).
// All index loads are issued before the first dependent x load, and all x loads before the first store, so a
// tile costs two memory round trips instead of 2 * (columns / 32).
template <class S, int KP>
__device__ __forceinline__ void gather_x(const DevPtrs<S>& D, const TileInfo& T, int lane, S* xs,
                                         const S* __restrict__ xvec, int CS) {
  constexpr int NT = 2 * KP;  // W * ncols <= 64 * KP
  const int n = T.n, W = 32 / T.G, ncols = 9 * n;
  const int total = T.nvalid * ncols;
  for (int e = lane; e < W * CS; e += 32) xs[e] = 0;
  int off[NT], dst[NT];
  {
    int g2 = 0, c = lane;
    while (c >= ncols) { c -= ncols; ++g2; }
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const int e = lane + 32 * t;
      const bool ok = e < total;
      const int i = c / 9, p = c - 9 * i;
      off[t] = ok ? D.slot_cam[T.slot_base + g2 * n + i] * 9 + p : -1;
      dst[t] = g2 * CS + c;
      c += 32;
      while (c >= ncols) { c -= ncols; ++g2; }
    }
  }
  S val[NT];
#pragma unroll
  for (int t = 0; t < NT; ++t) val[t] = off[t] >= 0 ? xvec[off[t]] : S(0);
  __syncwarp();
#pragma unroll
  for (int t = 0; t < NT; ++t) if (off[t] >= 0) xs[dst[t]] = val[t];
  __syncwarp();
}

template <class S, int KP>
__device__ __forceinline__ void matvec_item(const DevPtrs<S>& D, const MatvecItem& it, const TileInfo& T, int lane,
                                            S* xs, const S* __restrict__ xvec) {
  using V2 = typename ST<S>::V2;
  const int n = T.n, G = T.G;
  const int g = lane / G, j = lane - g * G;
  const int ncols = 9 * n;
  const int CS = (2 * G * KP) | 1;
  // zero padding columns, gather x_red of the W landmarks (coalesced runs of 9)
  gather_x<S, KP>(D, T, lane, xs, xvec, CS);
  V2 xv[KP], yv[KP];
#pragma unroll
  for (int k = 0; k < KP; ++k) {
    const int c = 2 * j + 2 * G * k;
    xv[k] = mk2(xs[g * CS + c], xs[g * CS + c + 1]);
    yv[k] = mk2(S(0), S(0));
  }
  __syncwarp();
  const V2* __restrict__ prow = reinterpret_cast<const V2*>(D.panel + T.panel_off) + (size_t)it.row0 * KP * 32 + lane;
  const int nrows = it.nrows;
#pragma unroll 2
  for (int r = 0; r < nrows; ++r) {
    V2 v[KP];
#pragma unroll
    for (int k = 0; k < KP; ++k) v[k] = __ldg(prow + (size_t)(r * KP + k) * 32);
    S d = 0;
#pragma unroll
    for (int k = 0; k < KP; ++k) d += v[k].x * xv[k].x + v[k].y * xv[k].y;
    d = group_sum(d, G);
#pragma unroll
    for (int k = 0; k < KP; ++k) { yv[k].x += d * v[k].x; yv[k].y += d * v[k].y; }
  }
#pragma unroll
  for (int k = 0; k < KP; ++k) {
    const int c = 2 * j + 2 * G * k;
    xs[g * CS + c] = yv[k].x;
    xs[g * CS + c + 1] = yv[k].y;
  }
  __syncwarp();
  {
    int g2 = 0, c = lane;
    while (c >= ncols) { c -= ncols; ++g2; }
    while (g2 < T.nvalid) {
      D.yobs[9 * (size_t)(it.yslot_base + g2 * n) + c] = xs[g2 * CS + c];
      c += 32;
      while (c >= ncols) { c -= ncols; ++g2; }
    }
  }
  __syncwarp();
}

// generic variant for very long tracks (KP beyond the register-resident classes): x and y live in shared memory
template <class S>
__device__ __forceinline__ void matvec_item_generic(const DevPtrs<S>& D, const MatvecItem& it, const TileInfo& T,
                                                    int lane, S* xs, const S* __restrict__ xvec) {
  using V2 = typename ST<S>::V2;
  const int n = T.n, KP = T.KP;  // G == 32, W == 1
  const int ncols = 9 * n, CP = 64 * KP;
  S* ys = xs + CP;
  for (int c = lane; c < CP; c += 32) {
    S v = 0;
    if (c < ncols) {
      const int i = c / 9, p = c - 9 * i;
      v = xvec[9 * (size_t)D.slot_cam[T.slot_base + i] + p];
    }
    xs[c] = v;
    ys[c] = 0;
  }
  __syncwarp();
  const V2* __restrict__ prow = reinterpret_cast<const V2*>(D.panel + T.panel_off) + (size_t)it.row0 * KP * 32 + lane;
  for (int r = 0; r < it.nrows; ++r) {
    S d = 0;
    for (int k = 0; k < KP; ++k) {
      const V2 v = __ldg(prow + (size_t)(r * KP + k) * 32);
      const int c = 2 * lane + 64 * k;
      d += v.x * xs[c] + v.y * xs[c + 1];
    }
    d = warp_sum(d);
    for (int k = 0; k < KP; ++k) {
      const V2 v = __ldg(prow + (size_t)(r * KP + k) * 32);  // second touch hits L1/L2
      const int c = 2 * lane + 64 * k;
      ys[c] += d * v.x;
      ys[c + 1] += d * v.y;
    }
  }
  __syncwarp();
  for (int c = lane; c < ncols; c += 32) D.yobs[9 * (size_t)it.yslot_base + c] = ys[c];
  __syncwarp();
}

// ---- TMA (cp.async.bulk) + mbarrier helpers: 1-D bulk global->shared copies, SASS UBLKCP -------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// The panels are read exactly once per matvec and are larger than L2: stream them with an evict-first L2 policy so that
// the camera vectors, the index arrays and the per-observation y buffer stay L2 resident.
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// The assembled S is smaller than L2 and read again by every PCG iteration after the switch: keep it there.
__device__ __forceinline__ uint64_t l2_evict_last_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  const uint32_t a = smem_u32(bar);
  do {
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(ok)
                 : "r"(a), "r"(parity)
                 : "memory");
  } while (!ok);
}

// Producer cursor of the per-warp panel stream: the MatvecItems of a warp are consumed in order and every item
// is one CONTIGUOUS chunk of HBM (nrows x KP x 64 scalars), cut into stages of <= STAGE_BYTES whole rows.
template <class S>
struct PanelStream {
  const S* src;          // next global address to fetch
  int rows_left;         // rows of the current producer item not yet requested
  int row_scalars;       // KP * 64
  int rows_per_stage;
  int next_item;         // next item index of this warp's sequence to open
  unsigned issued;       // stages issued so far
  uint64_t policy;       // L2 cache policy of the bulk copies
};

template <class S, int NS, int STAGE_BYTES>
__device__ __forceinline__ bool stream_produce(PanelStream<S>& ps, const DevPtrs<S>& D, const MatvecItem* __restrict__ items,
                                               int item_end, int item_stride, unsigned char* ring, uint64_t* bars, int lane) {
  if (ps.rows_left == 0) {
    if (ps.next_item >= item_end) return false;
    const MatvecItem it = items[ps.next_item];
    if (it.nrows == 0) { ps.next_item = item_end; return false; }  // padding of the host's dealing: end of this warp's list
    const TileInfo T = D.tiles[it.tile];
    ps.row_scalars = T.KP * 64;
    ps.src = D.panel + T.panel_off + (size_t)it.row0 * ps.row_scalars;
    ps.rows_left = it.nrows;
    ps.rows_per_stage = max(1, STAGE_BYTES / (int)(ps.row_scalars * sizeof(S)));
    ps.next_item += item_stride;
  }
  const int rows = min(ps.rows_per_stage, ps.rows_left);
  const uint32_t bytes = (uint32_t)(rows * ps.row_scalars * sizeof(S));
  const unsigned slot = ps.issued % NS;
  if (lane == 0) {
    mbar_expect_tx(&bars[slot], bytes);
    bulk_g2s(ring + (size_t)slot * STAGE_BYTES, ps.src, bytes, &bars[slot], ps.policy);
  }
  ps.src += (size_t)rows * ps.row_scalars;
  ps.rows_left -= rows;
  ++ps.issued;
  return true;
}

// predicated butterfly inside a group of G lanes (G uniform in the warp): no loop, no divergent branch
template <class T>
__device__ __forceinline__ T group_sum_p(T v, int G) {
  T t;
  t = __shfl_xor_sync(0xffffffffu, v, 16); if (G > 16) v += t;
  t = __shfl_xor_sync(0xffffffffu, v, 8);  if (G > 8) v += t;
  t = __shfl_xor_sync(0xffffffffu, v, 4);  if (G > 4) v += t;
  t = __shfl_xor_sync(0xffffffffu, v, 2);  if (G > 2) v += t;
  t = __shfl_xor_sync(0xffffffffu, v, 1);  if (G > 1) v += t;
  return v;
}

// one item, rows streamed through the shared-memory ring filled by TMA bulk copies.
// Every lane gathers x for the 2*KP columns it owns straight from the (L1/L2 resident) camera vector and
// writes its y entries straight to the per-observation buffer: no transposition, no per-item barrier.
template <class S, int KP, int NS, int STAGE_BYTES>
__device__ __forceinline__ void matvec_item_tma(const DevPtrs<S>& D, const MatvecItem& it, const TileInfo& T, int lane,
                                                const S* __restrict__ xvec, PanelStream<S>& ps, unsigned& consumed,
                                                const MatvecItem* __restrict__ items, int item_end, int item_stride,
                                                unsigned char* ring, uint64_t* bars) {
  using V2 = typename ST<S>::V2;
  const int n = T.n, G = T.G;
  const int g = lane / G, j = lane - g * G;
  const int ncols = 9 * n;
  const bool active = g < T.nvalid;
  const int slot0 = T.slot_base + g * n;
  // ---- gather: offsets first (index loads), then the x loads ----
  int off0[KP], off1[KP];
  {
    const int step = 2 * G;
    const int di = step / 9, dp = step - 9 * di;
    int c = 2 * j;
    int i = c / 9, p = c - 9 * i;
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      const bool v0 = active && c < ncols, v1 = active && (c + 1) < ncols;
      const int i1 = (p == 8) ? i + 1 : i, p1 = (p == 8) ? 0 : p + 1;
      const int cam0 = v0 ? __ldg(D.slot_cam + slot0 + i) : 0;
      const int cam1 = v1 ? __ldg(D.slot_cam + slot0 + i1) : 0;
      off0[k] = v0 ? 9 * cam0 + p : -1;
      off1[k] = v1 ? 9 * cam1 + p1 : -1;
      c += step; i += di; p += dp;
      if (p >= 9) { p -= 9; ++i; }
    }
  }
  V2 xv[KP], yv[KP];
#pragma unroll
  for (int k = 0; k < KP; ++k) {
    xv[k] = mk2(off0[k] >= 0 ? __ldg(xvec + off0[k]) : S(0), off1[k] >= 0 ? __ldg(xvec + off1[k]) : S(0));
    yv[k] = mk2(S(0), S(0));
  }
  // ---- rows from the ring ----
  int rows_left = it.nrows;
  constexpr int RPS = (STAGE_BYTES / (int)(KP * 64 * sizeof(S))) > 0 ? (STAGE_BYTES / (int)(KP * 64 * sizeof(S))) : 1;
  while (rows_left > 0) {
    const unsigned slot = consumed % NS;
    mbar_wait(&bars[slot], (consumed / NS) & 1u);
    const int rows = min(RPS, rows_left);
    const V2* st = reinterpret_cast<const V2*>(ring + (size_t)slot * STAGE_BYTES) + lane;
    // one row per step: 96 registers and 20 warps per SM measured equal or better than two rows per step (146 registers)
    for (int r = 0; r < rows; ++r) {
      V2 va[KP];
#pragma unroll
      for (int k = 0; k < KP; ++k) va[k] = st[(r * KP + k) * 32];
      S da0 = 0, da1 = 0;
#pragma unroll
      for (int k = 0; k < KP; ++k) { da0 = fma(va[k].x, xv[k].x, da0); da1 = fma(va[k].y, xv[k].y, da1); }
      S da = group_sum_p(da0 + da1, G);
#pragma unroll
      for (int k = 0; k < KP; ++k) { yv[k].x = fma(da, va[k].x, yv[k].x); yv[k].y = fma(da, va[k].y, yv[k].y); }
    }
    __syncwarp();  // every lane is done reading the stage before it is handed back to the TMA engine
    ++consumed;
    rows_left -= rows;
    stream_produce<S, NS, STAGE_BYTES>(ps, D, items, item_end, item_stride, ring, bars, lane);
  }
  // ---- y: each lane writes the columns it owns (contiguous inside a group) ----
  if (active) {
    S* yo = D.yobs + 9 * (size_t)(it.yslot_base + g * n);
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      const int c = 2 * j + 2 * G * k;
      if (c < ncols) yo[c] = yv[k].x;
      if (c + 1 < ncols) yo[c + 1] = yv[k].y;
    }
  }
}

// K4 (TMA variant): persistent warps, each streams the panels of its items through a private NS-stage
// shared-memory ring (cp.async.bulk + mbarrier complete_tx), so the bytes in flight per SM are set by the
// ring size (WARPS * NS * STAGE_BYTES) instead of by registers.
// Minimum resident CTAs: 5 for float32 (the shared-memory limit), 2 for float64 (register-limited).
template <class S, int WARPS, int NS, int STAGE_BYTES>
__global__ void __launch_bounds__(WARPS * 32, sizeof(S) == 4 ? 5 : 2) k_matvec_small_tma(DevPtrs<S> D, const MatvecItem* __restrict__ items,
                                                                  int item_begin, int item_end,
                                                                  const S* __restrict__ xvec, const int* done, int pdl) {
  extern __shared__ __align__(128) unsigned char smem_tma[];
  __shared__ __align__(8) uint64_t bars_all[WARPS][NS];
  // `done` only ever goes 0 -> 1 inside one solve: if it is already set we may leave before the grid dependency is
  // resolved (a stale 0 is harmless, the flag is read again after griddepcontrol.wait)
  if (done && *reinterpret_cast<const volatile int*>(done)) return;
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* ring = smem_tma + (size_t)wib * NS * STAGE_BYTES;
  uint64_t* bars = bars_all[wib];
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < NS; ++s) mbar_init(&bars[s], 1);
    mbar_fence_init();
  }
  __syncwarp();
  const int stride = gridDim.x * WARPS;
  const int first = item_begin + blockIdx.x * WARPS + wib;
  PanelStream<S> ps;
  ps.src = nullptr; ps.rows_left = 0; ps.row_scalars = 0; ps.rows_per_stage = 1; ps.next_item = first; ps.issued = 0; ps.policy = l2_evict_first_policy();
  unsigned consumed = 0;
  // the panel stream does not depend on the previous kernel (the panels are constant during PCG): prime the ring first,
  // then wait for the grid dependency (programmatic dependent launch), then read x / the done flag
#pragma unroll 1
  for (int s = 0; s < NS; ++s)
    if (!stream_produce<S, NS, STAGE_BYTES>(ps, D, items, item_end, stride, ring, bars, lane)) break;
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  if (done && *done) {
    // drain the bulk copies already in flight before the CTA may exit
    for (unsigned s = 0; s < ps.issued; ++s) mbar_wait(&bars[s % NS], (s / NS) & 1u);
    return;
  }
  if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  for (int q = first; q < item_end; q += stride) {
    const MatvecItem it = items[q];
    if (it.nrows == 0) break;  // padding: end of this warp's list
    const TileInfo T = D.tiles[it.tile];
    switch (T.KP) {
      case 5: matvec_item_tma<S, 5, NS, STAGE_BYTES>(D, it, T, lane, xvec, ps, consumed, items, item_end, stride, ring, bars); break;
      case 6: matvec_item_tma<S, 6, NS, STAGE_BYTES>(D, it, T, lane, xvec, ps, consumed, items, item_end, stride, ring, bars); break;
      case 7: matvec_item_tma<S, 7, NS, STAGE_BYTES>(D, it, T, lane, xvec, ps, consumed, items, item_end, stride, ring, bars); break;
      case 8: matvec_item_tma<S, 8, NS, STAGE_BYTES>(D, it, T, lane, xvec, ps, consumed, items, item_end, stride, ring, bars); break;
      case 9: matvec_item_tma<S, 9, NS, STAGE_BYTES>(D, it, T, lane, xvec, ps, consumed, items, item_end, stride, ring, bars); break;
      default: break;
    }
  }
}

// K4i, streamed: same arithmetic as k_matvec_implicit for the tiles [0, tile_end) whose W * n <= MAXSLOTS slots.
// A tile's q1d and jp records are two contiguous chunks of HBM: lane 0 brings them into a per-warp 2-stage shared-memory
// ring with two cp.async.bulk copies (mbarrier complete_tx), the next-but-one tile is requested as soon as a stage has
// been consumed, and every lane then reads its own 112 / 80-byte records with 16-byte LDS (stride 28 words: conflict
// free per quarter warp) instead of 12 uncoalesced 16-byte global loads per observation.  The per-observation results
// leave through shared memory as one contiguous run per tile.  The records are constant during PCG, so the first two
// tiles are requested before griddepcontrol.wait.
template <class S>
__device__ __forceinline__ void lds_rec28(const S* src, S (&v)[28]) {
  if (sizeof(S) == 4) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
#pragma unroll
    for (int q = 0; q < 7; ++q) { const float4 t = s4[q]; v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w; }
  } else {
    const double2* s2 = reinterpret_cast<const double2*>(src);
#pragma unroll
    for (int q = 0; q < 14; ++q) { const double2 t = s2[q]; v[2 * q] = t.x; v[2 * q + 1] = t.y; }
  }
}
template <class S>
__device__ __forceinline__ void lds_rec20(const S* src, S (&v)[20]) {
  if (sizeof(S) == 4) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
#pragma unroll
    for (int q = 0; q < 5; ++q) { const float4 t = s4[q]; v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w; }
  } else {
    const double2* s2 = reinterpret_cast<const double2*>(src);
#pragma unroll
    for (int q = 0; q < 10; ++q) { const double2 t = s2[q]; v[2 * q] = t.x; v[2 * q + 1] = t.y; }
  }
}

// MAXSLOTS <= 64: a lane owns at most two observations (A: i = j, B: i = j + G).
template <class S, int WARPS, int MAXSLOTS, int NS>
__global__ void __launch_bounds__(WARPS * 32) k_matvec_implicit_tma(DevPtrs<S> D, int tile_end, const S* __restrict__ xvec,
                                                                     const int* done, int pdl, int e0_only = 0) {
  static_assert(MAXSLOTS <= 64, "two observations per lane");
  extern __shared__ __align__(128) unsigned char smem_imp[];
  __shared__ __align__(8) uint64_t bars_all[WARPS][NS];
  if (done && *reinterpret_cast<const volatile int*>(done)) return;  // monotonic flag, see k_matvec_small_tma
  constexpr int QBYTES = MAXSLOTS * 28 * (int)sizeof(S), JBYTES = MAXSLOTS * 20 * (int)sizeof(S);
  constexpr int STAGE = QBYTES + JBYTES;
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* base = smem_imp + (size_t)wib * NS * STAGE;
  uint64_t* bars = bars_all[wib];
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < NS; ++s) mbar_init(&bars[s], 1);
    mbar_fence_init();
  }
  __syncwarp();
  const uint64_t policy = l2_evict_first_policy();
  const int stride = gridDim.x * WARPS;
  const int first = blockIdx.x * WARPS + wib;
  auto produce = [&](int t, int s) {
    if (lane == 0) {
      const TileInfo T = D.tiles[t];
      const uint32_t wn = (uint32_t)((32 / T.G) * T.n);
      const uint32_t qb = wn * 28u * (uint32_t)sizeof(S), jb = wn * 20u * (uint32_t)sizeof(S);
      mbar_expect_tx(&bars[s], qb + jb);
      bulk_g2s(base + (size_t)s * STAGE, D.q1d + 28 * (size_t)T.slot_base, qb, &bars[s], policy);
      bulk_g2s(base + (size_t)s * STAGE + QBYTES, D.jp + 20 * (size_t)T.slot_base, jb, &bars[s], policy);
    }
  };
  // the records are constant during PCG: request the first NS tiles before the grid dependency is awaited
  int issued = 0;
  for (int t = first; t < tile_end && issued < NS; t += stride) produce(t, issued++);
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  if (done && *done) {
    for (int s = 0; s < issued; ++s) mbar_wait(&bars[s], 0);  // drain the copies in flight before the CTA may exit
    return;
  }
  if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // x of the two observations of a lane is gathered one tile ahead (index loads at the top of the previous iteration,
  // value loads after its first pass), so the dependent slot_cam -> x round trips overlap compute
  S x0[9], x1[9];
  int cn0 = 0, cn1 = 0;
  bool hn0 = false, hn1 = false;
  TileInfo Tn = D.tiles[min(first, tile_end - 1)];
  auto next_indices = [&](const TileInfo& T2, bool valid) {
    const int g2 = lane / T2.G, j2 = lane - g2 * T2.G;
    const bool act = valid && g2 < T2.nvalid;
    hn0 = act && j2 < T2.n; hn1 = act && j2 + T2.G < T2.n;
    cn0 = hn0 ? __ldg(D.slot_cam + T2.slot_base + g2 * T2.n + j2) : 0;
    cn1 = hn1 ? __ldg(D.slot_cam + T2.slot_base + g2 * T2.n + j2 + T2.G) : 0;
  };
  auto next_values = [&]() {
#pragma unroll
    for (int p = 0; p < 9; ++p) {
      x0[p] = hn0 ? __ldg(xvec + 9 * (size_t)cn0 + p) : S(0);
      x1[p] = hn1 ? __ldg(xvec + 9 * (size_t)cn1 + p) : S(0);
    }
  };
  next_indices(Tn, first < tile_end);
  next_values();
  int k = 0;
  for (int t = first; t < tile_end; t += stride, ++k) {
    const int s = k % NS;
    const TileInfo T = Tn;
    const int n = T.n, G = T.G;
    const int g = lane / G, j = lane - g * G;
    const bool hasA = hn0, hasB = hn1;
    const int eA = g * n + j, eB = eA + G;
    S xa[9], xb[9];
#pragma unroll
    for (int p = 0; p < 9; ++p) { xa[p] = x0[p]; xb[p] = x1[p]; }
    const bool more = t + stride < tile_end;
    if (more) Tn = D.tiles[t + stride];
    next_indices(Tn, more);
    mbar_wait(&bars[s], (uint32_t)((k / NS) & 1));
    S* sq = reinterpret_cast<S*>(base + (size_t)s * STAGE);
    const S* sj = reinterpret_cast<const S*>(base + (size_t)s * STAGE + QBYTES);
    // ---- pass 1: u = sum_i Q1d_i x_i over the landmark ----
    S u0 = 0, u1 = 0, u2 = 0;
    {
      S q[28];
      if (hasA) {
        lds_rec28<S>(sq + 28 * eA, q);
#pragma unroll
        for (int p = 0; p < 9; ++p) { u0 += q[p] * xa[p]; u1 += q[9 + p] * xa[p]; u2 += q[18 + p] * xa[p]; }
      }
      if (hasB) {
        lds_rec28<S>(sq + 28 * eB, q);
#pragma unroll
        for (int p = 0; p < 9; ++p) { u0 += q[p] * xb[p]; u1 += q[9 + p] * xb[p]; u2 += q[18 + p] * xb[p]; }
      }
    }
    u0 = group_sum_p(u0, G); u1 = group_sum_p(u1, G); u2 = group_sum_p(u2, G);
    next_values();  // the index loads issued at the top have landed by now
    // ---- pass 2: y_i = Jp_i^T (Jp_i x_i) - Q1d_i^T u, kept in registers until every lane is done with the records ----
    S ya[9], yb[9];
    {
      S q[28], jp[20];
      if (hasA) {
        lds_rec28<S>(sq + 28 * eA, q);
        lds_rec20<S>(sj + 20 * eA, jp);
        S t0 = 0, t1 = 0;
#pragma unroll
        for (int p = 0; p < 9; ++p) { t0 += jp[p] * xa[p]; t1 += jp[9 + p] * xa[p]; }
#pragma unroll
        for (int p = 0; p < 9; ++p) {
          const S e0 = q[p] * u0 + q[9 + p] * u1 + q[18 + p] * u2;
          ya[p] = e0_only ? e0 : (jp[p] * t0 + jp[9 + p] * t1) - e0;
        }
      }
      if (hasB) {
        lds_rec28<S>(sq + 28 * eB, q);
        lds_rec20<S>(sj + 20 * eB, jp);
        S t0 = 0, t1 = 0;
#pragma unroll
        for (int p = 0; p < 9; ++p) { t0 += jp[p] * xb[p]; t1 += jp[9 + p] * xb[p]; }
#pragma unroll
        for (int p = 0; p < 9; ++p) {
          const S e0 = q[p] * u0 + q[9 + p] * u1 + q[18 + p] * u2;
          yb[p] = e0_only ? e0 : (jp[p] * t0 + jp[9 + p] * t1) - e0;
        }
      }
    }
    __syncwarp();
    // the q1d records of this stage are dead: reuse their space to turn the per-lane results into one contiguous run
    if (hasA) {
#pragma unroll
      for (int p = 0; p < 9; ++p) sq[9 * eA + p] = ya[p];
    }
    if (hasB) {
#pragma unroll
      for (int p = 0; p < 9; ++p) sq[9 * eB + p] = yb[p];
    }
    __syncwarp();
    {
      const int cnt = T.nvalid * n * 9;
      S* yg = D.yobs + 9 * (size_t)T.slot_base;
      for (int e = lane; e < cnt; e += 32) yg[e] = sq[e];
    }
    __syncwarp();
    // this stage is free again: request the tile NS steps ahead into it
    if (t + NS * stride < tile_end) produce(t + NS * stride, s);
  }
}

template <class S, int WARPS, int KPMAX>
__global__ void __launch_bounds__(WARPS * 32) k_matvec_large(DevPtrs<S> D, const MatvecItem* __restrict__ items,
                                                              int item_begin, int item_end, int scratch_per_warp,
                                                              const S* __restrict__ xvec, const int* done) {
  if (done && *done) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  S* xs = reinterpret_cast<S*>(smem_raw) + (size_t)wib * scratch_per_warp;
  for (int q = item_begin + blockIdx.x * WARPS + wib; q < item_end; q += gridDim.x * WARPS) {
    const MatvecItem it = items[q];
    const TileInfo T = D.tiles[it.tile];
    if (T.KP == 10) matvec_item<S, 10>(D, it, T, lane, xs, xvec);
    else if (KPMAX >= 12 && T.KP == 12) matvec_item<S, (KPMAX >= 12 ? 12 : 10)>(D, it, T, lane, xs, xvec);
    else if (KPMAX >= 14 && T.KP == 14) matvec_item<S, (KPMAX >= 14 ? 14 : 10)>(D, it, T, lane, xs, xvec);
    else if (KPMAX >= 16 && T.KP == 16) matvec_item<S, (KPMAX >= 16 ? 16 : 10)>(D, it, T, lane, xs, xvec);
    else matvec_item_generic<S>(D, it, T, lane, xs, xvec);
  }
}

// ------------------------------------------------------------------------------------------------
// PCG vector kernels (ref: cg/conjugate_gradient.hpp:113-298, cg/preconditioner.hpp:122-136)
//   all launched with exactly NPART blocks of 128 threads; thread per camera (9-vectors);
//   partial sums per block in double, combined in a fixed order by the consumer kernel.
// ------------------------------------------------------------------------------------------------
// sum_j O_ij v_j of the pair priors (DESIGN.md section 15), entry e = 9 i + a of the camera vector (zero on the intrinsic
// rows a >= 6), edges in list order
template <class S>
__device__ __forceinline__ S pair_ov_entry(const DevPtrs<S>& D, const S* __restrict__ v, int e) {
  const int cam = e / 9, a = e - 9 * cam;
  S s = 0;
  if (a < 6)
    for (int q = D.pair_ptr[cam], q1 = D.pair_ptr[cam + 1]; q < q1; ++q) {
      const S* O = D.pair_O + 36 * (size_t)q + 6 * a;
      const S* vj = v + 9 * (size_t)D.pair_nbr[q];
#pragma unroll
      for (int k = 0; k < 6; ++k) s += O[k] * vj[k];
    }
  return s;
}

// out = y + lambda v (+ A^T A v of the camera priors) (+ sum_j O_ij v_j of the pair priors), y = the camera-reduced
// operator output [9 nc]; out may be y.
// The operator of rba_right_multiply: the same order of operations as P1 of k_pcg_vec.
template <class S>
__global__ void __launch_bounds__(128) k_pcg_q(DevPtrs<S> D, const S* yfull, const S* __restrict__ vec, S* out, S lambda) {
  for (int cam = blockIdx.x * blockDim.x + threadIdx.x; cam < D.nc; cam += gridDim.x * blockDim.x) {
    S yv[9];
#pragma unroll
    for (int c = 0; c < 9; ++c) yv[c] = yfull[9 * (size_t)cam + c];
#pragma unroll
    for (int c = 0; c < 9; ++c) {
      const S pv = vec[9 * (size_t)cam + c];
      S qv = yv[c] + lambda * pv;
      if (D.prior_H) {  // + A^T A v of the camera prior, in the order of k_pcg_vec<S, true>
        const S* hr = D.prior_H + 81 * (size_t)cam + 9 * c;
        S h = 0;
#pragma unroll
        for (int k = 0; k < 9; ++k) h += hr[k] * vec[9 * (size_t)cam + k];
        qv += h;
      }
      if (D.pair_ov) qv += pair_ov_entry(D, vec, 9 * cam + c);  // the value k_pair_ov gives k_pcg_vec<S, true, true>
      out[9 * (size_t)cam + c] = qv;
    }
  }
}

// out = per-camera sum of the segment partials (+ addend)
template <class S>
__global__ void k_cam_final9(const S* __restrict__ partial, const int* __restrict__ cam_item_ptr, int nc,
                             S* __restrict__ out, const S* __restrict__ addend = nullptr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 9 * nc) return;
  const int cam = i / 9, c = i - 9 * cam;
  S s = 0;
  for (int it = cam_item_ptr[cam]; it < cam_item_ptr[cam + 1]; ++it) s += partial[9 * (size_t)it + c];
  if (addend) s += addend[i];
  out[i] = s;
}

// ------------------------------------------------------------------------------------------------
// PCG vector step on ONE thread-block cluster (hardware cluster barriers instead of kernel boundaries):
//   P1  q = y + lambda * v, partial v.q                       (v = p, or x in the residual-refresh half step)
//   P2  alpha = rho / p.q ; x += alpha p ; r -= alpha q ; z = M^-1 r ; partial r.z and x.(b + r)
//   P3  Nash-Sofer test zeta = i (Q_i - Q_{i-1}) / Q_i < eta ; rho, beta ; p = z + beta p   (next iteration's p)
// ref: cg/conjugate_gradient.hpp:161-295 ; scalars in double, vectors in Scalar, alpha/beta narrowed to Scalar.
// mode 0 regular iteration, 1 refresh first half (stop after x += alpha p), 2 refresh second half (v = x,
// r = b - H x), 3 initialisation (x = 0, r = b, z, rho, p = z).
// y = D.y holds the camera-reduced (and, with several shards, all-reduced) operator output.
// Cameras are dealt to the CTAs in contiguous ranges; thread t of a CTA owns elements e0 + t + k * blockDim.  Everything
// that does not depend on the operator output (x, r, p, b and the 9-float row of M^-1) is fetched before the grid
// dependency is awaited and stays in registers across the phases (EPT elements per thread); the new residual of a
// camera is exchanged through shared memory.  Larger problems loop over rounds and re-read from global memory.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_nctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
// store a double into the same shared-memory variable of CTA `rank` of the cluster (distributed shared memory)
__device__ __forceinline__ void st_dsmem_f64(const double* local, uint32_t rank, double v) {
  uint32_t ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"((uint32_t)__cvta_generic_to_shared(local)), "r"(rank));
  asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(ra), "d"(v) : "memory");
}
constexpr int CL_MAX = 16;  // largest cluster of the PCG vector kernel
// Cluster-wide sums without global memory: every CTA block-reduces NV doubles per thread and stores its totals into slot
// [k0 + v][own rank] of EVERY CTA's `cl` array through distributed shared memory; after the next cluster barrier
// cluster_total() adds the per-CTA totals in rank order (bit-identical in every CTA).
template <int NV>
__device__ __forceinline__ void cluster_publish(double (&v)[NV], double (*cl)[CL_MAX], int k0) {
  __shared__ double red[32][NV];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < NV; ++k) v[k] = warp_sum(v[k]);
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < NV; ++k) red[w][k] = v[k];
  __syncthreads();
  const uint32_t me = cluster_ctarank(), nr = cluster_nctarank();
  if (threadIdx.x < nr) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      double s = 0;
      for (int q = 0; q < nw; ++q) s += red[q][k];
      st_dsmem_f64(&cl[k0 + k][me], threadIdx.x, s);
    }
  }
  __syncthreads();  // red may be reused by the next publish
}
__device__ __forceinline__ double cluster_total(double (*cl)[CL_MAX], int k) {
  const uint32_t nr = cluster_nctarank();
  double s = 0;
  for (uint32_t r = 0; r < nr; ++r) s += cl[k][r];
  return s;
}

constexpr int VEC_THREADS = 512;
constexpr int VEC_EPT = 2;

template <class S>
__device__ __forceinline__ S ld_volatile(const S* p) { return *reinterpret_cast<const volatile S*>(p); }

// Progress of the PCG loop in host-mapped pinned memory: prog[0] = last completed iteration, prog[1] = 1 once the solve has
// ended.  The host reads it without any stream operation to decide how far ahead it may enqueue (Solver::solve_enqueue).
__device__ __forceinline__ void pcg_publish_progress(int* prog, int iter, int done) {
  if (!prog) return;
  *reinterpret_cast<volatile int*>(prog) = iter;
  if (done) {
    __threadfence_system();
    *reinterpret_cast<volatile int*>(prog + 1) = 1;
  }
}


// One CTA per SM (the grid is one cluster): the minimum of 1 block lets ptxas use up to 128 registers, where its sm_90
// default caps the kernel at 64 and spills the register-resident vectors.
// PRIOR (D.prior_H set, DESIGN.md section 14): P1 adds the camera-prior term, q = y + lambda v + A^T A v.  The rows of A^T A
// are fetched with the M^-1 rows, ahead of the grid dependency; the 9 entries of v of a camera are exchanged through shared
// memory like r for z = M^-1 r.  PRIOR = false is the kernel without priors, unchanged.
// PAIR (D.pair_ov set, DESIGN.md section 15; implies PRIOR, whose A^T A holds the pair priors' diagonal blocks): P1 also adds
// sum_j O_ij v_j, which k_pair_ov, the kernel this one depends on, has written to D.pair_ov.
template <class S, bool PRIOR = false, bool PAIR = false>
__global__ void __launch_bounds__(VEC_THREADS, 1) k_pcg_vec(DevPtrs<S> D, PcgState* st, S lambda, int i, int mode,
                                                         double eta, int min_it, int is_last, int pdl, PeerComm pc, int seq,
                                                         const int* __restrict__ cam_item_ptr, int* prog) {
  static_assert(PRIOR || !PAIR, "the pair priors' diagonal blocks are in prior_H");
  __shared__ S sr[VEC_THREADS * VEC_EPT + 16];
  __shared__ int peer_fail;
  __shared__ double cl_go;          // multi-GPU: CTA 0's verdict on the peer exchange (distributed shared memory)
  __shared__ double cl[4][CL_MAX];  // per-CTA totals of p.q | r.z | x.(b + r) | r.r, exchanged through distributed shared memory
  const int tid = threadIdx.x;
  const int cams_per_block = (D.nc + gridDim.x - 1) / gridDim.x;
  const int cam0 = min(D.nc, (int)blockIdx.x * cams_per_block);
  const int cam1 = min(D.nc, cam0 + cams_per_block);
  const int e0 = 9 * cam0, ne = 9 * (cam1 - cam0);
  const bool cached = ne <= VEC_THREADS * VEC_EPT;
  const int cur = i & 1, nxt = cur ^ 1;
  if (*reinterpret_cast<const volatile int*>(&st->done)) return;  // monotonic flag, see k_matvec_small_tma
  // ---- prefetch of everything that does not depend on the previous kernel of this iteration ----
  S xv[VEC_EPT], rv[VEC_EPT], pv[VEC_EPT], bv[VEC_EPT], qv[VEC_EPT], zv[VEC_EPT], inv[VEC_EPT][9];
  S hrow[PRIOR ? VEC_EPT : 1][9];  // rows of the camera prior's A^T A (PRIOR only)
  if (cached) {
#pragma unroll
    for (int k = 0; k < VEC_EPT; ++k) {
      const int l = tid + k * VEC_THREADS;
      const bool on = l < ne;
      const int e = e0 + (on ? l : 0);
      xv[k] = on ? D.x[e] : S(0); rv[k] = on ? D.r[e] : S(0); pv[k] = on ? D.p[e] : S(0); bv[k] = on ? D.b[e] : S(0);
      const S* row = D.inv + 9 * (size_t)e;  // inv[cam][a][:] = 9 consecutive scalars at 81 cam + 9 a = 9 e
#pragma unroll
      for (int c = 0; c < 9; ++c) inv[k][c] = on ? row[c] : S(0);
      if constexpr (PRIOR) {
        const S* hr = D.prior_H + 9 * (size_t)e;  // same layout as inv
#pragma unroll
        for (int c = 0; c < 9; ++c) hrow[k][c] = on ? hr[c] : S(0);
      }
      qv[k] = 0; zv[k] = 0;
    }
  }
  // one GPU: the operator's per-camera sums arrive as per-segment partial sums (k_cam_reduce); the segment range of every
  // element's camera is constant and fetched here, ahead of the grid dependency
  int pi0[VEC_EPT], pi1[VEC_EPT];
#pragma unroll
  for (int k = 0; k < VEC_EPT; ++k) {
    const int l = tid + k * VEC_THREADS;
    const bool on = cached && cam_item_ptr && l < ne;
    const int cam = (e0 + (on ? l : 0)) / 9;
    pi0[k] = on ? __ldg(cam_item_ptr + cam) : 0;
    pi1[k] = on ? __ldg(cam_item_ptr + cam + 1) : 0;
  }
  // scalars of the previous vector step: that kernel completed before the operator kernel this launch depends on, so
  // they (and the `done` flag read above) are final already
  const double rho_cur = st->rho[cur], q0_cur = st->q0[cur];
  // every CTA of the cluster runs (and stays) before the first distributed-shared-memory store.  A CTA that left above
  // does not hold the others up (the barrier waits for non-exited threads only), and in that case every CTA leaves
  // before it stores anything: the flag is final
  cluster_sync_all();
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  double alpha = 0;
  const bool peers = pc.nranks > 1 && mode != 3;
  const int par = seq & 1;
  if (peers) {
    // The producing kernel (k_cam_reduce_final) has pushed this rank's partial y into every peer's staging area and has
    // completed.  CTA 0 publishes the sequence number to every rank and waits for the peers' numbers in LOCAL memory;
    // its verdict reaches the other CTAs through distributed shared memory, so that the whole cluster takes the same path.
    if (cluster_ctarank() == 0) {
      if (tid == 0) peer_fail = 0;
      __syncthreads();
      if (tid < pc.nranks) {
        __threadfence_system();
        st_release_sys(peer_flag(pc, tid, 0, par, pc.rank), seq);
        if (!peer_wait(pc, 0, par, tid, seq)) peer_fail = 1;
      }
      __syncthreads();
      if (tid < (int)cluster_nctarank()) st_dsmem_f64(&cl_go, tid, peer_fail ? -1.0 : 1.0);
    }
    cluster_sync_all();
    if (cl_go < 0) {  // uniform over the cluster: a peer never published (dead rank); the solve is reported as FAILURE
      if (blockIdx.x == 0 && tid == 0) { st->done = 1; st->term = 2; st->reason = 99; st->iter = i; pcg_publish_progress(prog, i, 1); }
      return;
    }
  }
  const S* ys = peers ? peer_ystage<S>(pc, pc.rank, par, 0, D.nc) : nullptr;
  const size_t ystride = (size_t)9 * D.nc;
  auto load_y = [&](int e) -> S {
    if (!peers && cam_item_ptr) {  // segment sums in their fixed order, like k_cam_reduce_final's last arriver
      const int cam = e / 9, c = e - 9 * cam;
      S sacc = 0;
      for (int q = __ldg(cam_item_ptr + cam), q1 = __ldg(cam_item_ptr + cam + 1); q < q1; ++q) sacc += __ldcg(D.partial + 9 * (size_t)q + c);
      return sacc;
    }
    if (!peers) return __ldcg(D.y + e);
    S sacc = 0;  // rank order: bit-identical on every rank; __ldcg: the slots are written by remote stores, L1 may be stale
#pragma unroll
    for (int r = 0; r < MAX_PEERS; ++r)
      if (r < pc.nranks) sacc += __ldcg(ys + r * ystride + e);
    return sacc;
  };
  if (mode != 3) {
    // ---- P1 ----
    double acc = 0;
    if (cached) {
      if constexpr (PRIOR) {  // v of every camera of this CTA to shared memory (sr is free until P2a)
#pragma unroll
        for (int k = 0; k < VEC_EPT; ++k) {
          const int l = tid + k * VEC_THREADS;
          if (l < ne) sr[l] = (mode == 2) ? xv[k] : pv[k];
        }
        __syncthreads();
      }
#pragma unroll
      for (int k = 0; k < VEC_EPT; ++k) {
        const int l = tid + k * VEC_THREADS;
        if (l < ne) {
          const S vv = (mode == 2) ? xv[k] : pv[k];
          S yk;
          if (!peers && cam_item_ptr) {
            const int c = (e0 + l) % 9;
            yk = 0;
            for (int q = pi0[k]; q < pi1[k]; ++q) yk += __ldcg(D.partial + 9 * (size_t)q + c);
          } else yk = load_y(e0 + l);
          qv[k] = yk + lambda * vv;
          if constexpr (PRIOR) {
            const S* vc = sr + 9 * (l / 9);
            S h = 0;
#pragma unroll
            for (int c = 0; c < 9; ++c) h += hrow[k][c] * vc[c];
            qv[k] += h;
          }
          if constexpr (PAIR) qv[k] += __ldcg(D.pair_ov + e0 + l);
          acc += (double)(vv * qv[k]);
        }
      }
    } else {
      const S* vec = (mode == 2) ? D.x : D.p;
      for (int l = tid; l < ne; l += VEC_THREADS) {
        const S vv = vec[e0 + l];
        S q = load_y(e0 + l) + lambda * vv;
        if constexpr (PRIOR) {
          const S* hr = D.prior_H + 9 * (size_t)(e0 + l);
          const S* vc = vec + 9 * (size_t)((e0 + l) / 9);
          S h = 0;
#pragma unroll
          for (int c = 0; c < 9; ++c) h += hr[c] * vc[c];
          q += h;
        }
        if constexpr (PAIR) q += __ldcg(D.pair_ov + e0 + l);
        D.q[e0 + l] = q;
        acc += (double)(vv * q);
      }
    }
    { double a1[1] = {acc}; cluster_publish<1>(a1, cl, 0); }
    cluster_sync_all();
  }
  // ---- P2 ----
  if (mode == 0 || mode == 1) {
    const double pq = cluster_total(cl, 0);
    bool fail = false;
    int term = 0, reason = 0;
    if (pq <= 0 || isinf(pq)) { fail = true; term = 0; reason = 5; }
    else {
      alpha = rho_cur / pq;
      if (isinf(alpha)) { fail = true; term = 2; reason = 6; }
    }
    if (fail) {  // uniform across the cluster: nobody reaches the next barrier
      for (int l = tid; l < ne; l += VEC_THREADS) D.inc[e0 + l] = -D.x[e0 + l];
      if (blockIdx.x == 0 && tid == 0) { st->done = 1; st->term = term; st->reason = reason; st->last_pq = pq; st->iter = i; pcg_publish_progress(prog, i, 1); }
      return;
    }
    if (blockIdx.x == 0 && tid == 0) { st->last_pq = pq; st->last_alpha = alpha; }
  }
  const S as = (S)alpha;
  if (mode == 1) {
    if (cached) {
#pragma unroll
      for (int k = 0; k < VEC_EPT; ++k) { const int l = tid + k * VEC_THREADS; if (l < ne) D.x[e0 + l] = xv[k] + as * pv[k]; }
    } else {
      for (int l = tid; l < ne; l += VEC_THREADS) D.x[e0 + l] = D.x[e0 + l] + as * D.p[e0 + l];
    }
    return;
  }
  double rz = 0, xbr = 0, bb = 0;
  if (cached) {
    // P2a: x and r in registers, new residual to shared memory
#pragma unroll
    for (int k = 0; k < VEC_EPT; ++k) {
      const int l = tid + k * VEC_THREADS;
      if (l < ne) {
        if (mode == 0) { xv[k] = xv[k] + as * pv[k]; rv[k] = rv[k] - as * qv[k]; }
        else if (mode == 2) { rv[k] = bv[k] - qv[k]; }
        else { xv[k] = 0; rv[k] = bv[k]; }
        sr[l] = rv[k];
      }
    }
    __syncthreads();
    // P2b: z = M^-1 r (ref: cg/preconditioner.hpp:122-136) and the dot products
#pragma unroll
    for (int k = 0; k < VEC_EPT; ++k) {
      const int l = tid + k * VEC_THREADS;
      if (l < ne) {
        const S* rc = sr + 9 * (l / 9);
        S z = 0;
#pragma unroll
        for (int c = 0; c < 9; ++c) z += inv[k][c] * rc[c];
        zv[k] = z;
        rz += (double)(rv[k] * z);
        xbr += (double)(xv[k] * (bv[k] + rv[k]));
        bb += (double)(rv[k] * rv[k]);
        D.x[e0 + l] = xv[k];
        D.r[e0 + l] = rv[k];
      }
    }
  } else {
    for (int l = tid; l < ne; l += VEC_THREADS) {
      const int e = e0 + l;
      S r2;
      if (mode == 0) { D.x[e] = D.x[e] + as * D.p[e]; r2 = D.r[e] - as * D.q[e]; }
      else if (mode == 2) { r2 = D.b[e] - D.q[e]; }
      else { D.x[e] = 0; r2 = D.b[e]; }
      D.r[e] = r2;
    }
    __syncthreads();
    for (int l = tid; l < ne; l += VEC_THREADS) {
      const int e = e0 + l;
      const int cam = e / 9;
      const S* row = D.inv + 9 * (size_t)e;
      const S* rc = D.r + 9 * (size_t)cam;
      S z = 0;
#pragma unroll
      for (int c = 0; c < 9; ++c) z += row[c] * rc[c];
      D.z[e] = z;
      const S r2 = D.r[e];
      rz += (double)(r2 * z);
      xbr += (double)(D.x[e] * (D.b[e] + r2));
      bb += (double)(r2 * r2);
    }
  }
  { double a3[3] = {rz, xbr, bb}; cluster_publish<3>(a3, cl, 1); }
  cluster_sync_all();
  // ---- P3 ----
  const double rho_new = cluster_total(cl, 1);
  int done = 0, term = 0, reason = 0;
  double q1 = 0, zeta = 0, beta = 0, norm_b = 0;
  if (mode == 3) {
    norm_b = sqrt(cluster_total(cl, 3));
    if (norm_b == 0.0) { done = 1; term = 1; reason = 2; }
  } else {
    const double xbr_t = cluster_total(cl, 2);
    q1 = -xbr_t;
    zeta = (double)i * (q1 - q0_cur) / q1;
    if (zeta < eta && i >= min_it) { done = 1; term = 1; reason = 1; }
  }
  if (!done) {
    if (rho_new == 0.0 || isinf(rho_new)) { done = 1; term = 2; reason = 3; }
    else if (mode != 3) {
      beta = rho_new / rho_cur;
      if (beta == 0.0 || isinf(beta)) { done = 1; term = 2; reason = 4; }
    }
  }
  const S bs = (S)beta;
  if (cached) {
#pragma unroll
    for (int k = 0; k < VEC_EPT; ++k) {
      const int l = tid + k * VEC_THREADS;
      if (l < ne) {
        if (!done && !is_last) D.p[e0 + l] = (mode == 3) ? zv[k] : zv[k] + bs * pv[k];
        if (done || is_last) D.inc[e0 + l] = -xv[k];
      }
    }
  } else {
    for (int l = tid; l < ne; l += VEC_THREADS) {
      const int e = e0 + l;
      if (!done && !is_last) D.p[e] = (mode == 3) ? D.z[e] : D.z[e] + bs * D.p[e];
      if (done || is_last) D.inc[e] = -D.x[e];
    }
  }
  if (blockIdx.x == 0 && tid == 0) {
    st->rho[nxt] = rho_new;  // iteration i+1 reads slot (i+1)&1
    st->q0[nxt] = (mode == 3) ? 0.0 : q1;
    st->last_zeta = zeta;
    st->iter = i;
    if (mode == 3) { st->norm_b = norm_b; st->term = 0; st->reason = 0; }
    if (done) { st->done = 1; st->term = term; st->reason = reason; }
    pcg_publish_progress(prog, i, done || is_last);
  }
}

// ------------------------------------------------------------------------------------------------
// Power-series solve of the reduced camera system (solver_type = POWER_SCHUR_COMPLEMENT, "PoBA"):
//   ref: sc/linearization_power_sc.hpp:130-160:  accum = Hpp^-1 (-b); tmp = accum;
//        for i = 1..power_order: tmp = Hpp^-1 (E_0 tmp); accum += tmp; stop when i |tmp| / |accum| < eta.
//   One 16-CTA cluster like k_pcg_vec: i == 0 initialises, i >= 1 consumes y = E_0 p (camera-reduced by the previous
//   kernel).  D.p = tmp, D.x = accum, D.inv = Hpp^-1 (block-diagonal, damped), D.inc = the result (already the increment:
//   H inc = -b).  Norms are accumulated in double.
//   PAIR (pair priors, DESIGN.md section 15): the series runs on Hpp^-1 (E_0 - O), tmp = Hpp^-1 ((E_0 - O) tmp), with
//   O tmp = D.pair_ov written by k_pair_ov, the kernel this one depends on (Hpp holds the pairs' diagonal blocks).
// ------------------------------------------------------------------------------------------------
template <class S, bool PAIR = false>
__global__ void __launch_bounds__(VEC_THREADS) k_power_vec(DevPtrs<S> D, PcgState* st, int i, double eta, int is_last, int pdl) {
  __shared__ double cl[4][CL_MAX];
  const int tid = threadIdx.x;
  const int cams_per_block = (D.nc + gridDim.x - 1) / gridDim.x;
  const int cam0 = min(D.nc, (int)blockIdx.x * cams_per_block);
  const int cam1 = min(D.nc, cam0 + cams_per_block);
  const int e0 = 9 * cam0, ne = 9 * (cam1 - cam0);
  if (*reinterpret_cast<const volatile int*>(&st->done)) return;
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  if (st->done) return;
  if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  cluster_sync_all();
  double tt = 0, aa = 0;
  for (int l = tid; l < ne; l += VEC_THREADS) {
    const int e = e0 + l;
    const int cam = e / 9;
    const S* row = D.inv + 9 * (size_t)e;
    const S* v = (i == 0 ? D.b : D.y) + 9 * (size_t)cam;
    S z = 0;
    if constexpr (PAIR) {
      if (i != 0) {
        const S* ov = D.pair_ov + 9 * (size_t)cam;
#pragma unroll
        for (int c = 0; c < 9; ++c) z += row[c] * (__ldcg(v + c) - __ldcg(ov + c));
      } else {
#pragma unroll
        for (int c = 0; c < 9; ++c) z += row[c] * __ldcg(v + c);
      }
    } else {
#pragma unroll
      for (int c = 0; c < 9; ++c) z += row[c] * __ldcg(v + c);
    }
    if (i == 0) z = -z;
    const S acc = (i == 0) ? z : D.x[e] + z;
    D.x[e] = acc;
    D.p[e] = z;
    if (is_last || i == 0) D.inc[e] = acc;  // refreshed below on convergence
    tt += (double)z * (double)z;
    aa += (double)acc * (double)acc;
  }
  { double a2[2] = {tt, aa}; cluster_publish<2>(a2, cl, 0); }
  cluster_sync_all();
  const double tn = cluster_total(cl, 0), an = cluster_total(cl, 1);
  int done = 0, term = 0;
  double zeta = 0;
  if (i >= 1) {
    zeta = (double)i * sqrt(tn) / sqrt(an);
    if (eta > 0 && zeta < eta) { done = 1; term = 1; }
  }
  if (!isfinite(an)) { done = 1; term = 2; }
  if (done && !is_last && i != 0)
    for (int l = tid; l < ne; l += VEC_THREADS) D.inc[e0 + l] = D.x[e0 + l];
  if (blockIdx.x == 0 && tid == 0) {
    st->iter = i; st->last_zeta = zeta;
    if (done) { st->done = 1; st->term = term; st->reason = term == 1 ? 1 : 3; }
    else if (is_last) { st->term = 0; st->reason = 0; }
  }
}

// ------------------------------------------------------------------------------------------------
// K6  back-substitution (ref: ipp:212-284).  Model-cost change evaluated in the un-rotated basis:
//     Q^T (Jp dp + Jl inc) has the same norm / inner product with Q^T r as (Jp dp + Jl inc) with r.
// ------------------------------------------------------------------------------------------------
// One warp per tile, one lane per observation, no shared memory: every record is one or a few 16-byte loads.
// Pass 1 (q1d, dp) gives s_m and the landmark increment, pass 2 (jp, jl, r, dp) the model cost change.
// LMP (landmark priors, DESIGN.md section 17): l_diff also loses (L~ d)^T (1/2 L~ d + g) of each prior landmark, into this
// shard's partial (the term is landmark-owned: it is counted once by the sum over the shards).
template <class S, bool LMP = false>
__global__ void __launch_bounds__(128) k_back_substitute(DevPtrs<S> D, const S* __restrict__ pose_inc,
                                                          double* partials, int* bad_flag) {
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double ld[1] = {0};
  for (int t = blockIdx.x * (blockDim.x >> 5) + wib; t < D.ntiles; t += gridDim.x * (blockDim.x >> 5)) {
    const TileInfo T = D.tiles[t];
    const int n = T.n, G = T.G;
    const int g = lane / G, j = lane - g * G;
    const bool active = g < T.nvalid;
    const int sidx = T.lm_base + g;
    const size_t slot0 = (size_t)(T.slot_base + g * n);
    // ---- pass 1: s_m = sum_c q1d[m][c] dp[c]   (ref: ipp:233-239) ----
    S sm[3] = {0, 0, 0};
    if (active) {
#pragma unroll 2
      for (int i = j; i < n; i += G) {
        const size_t sl = slot0 + i;
        const S* dp = pose_inc + 9 * (size_t)__ldg(D.slot_cam + sl);
        S q[28];
        load_rec<S, 28>(D.q1d + 28 * sl, q);
#pragma unroll
        for (int c = 0; c < 9; ++c) {
          const S d = __ldg(dp + c);
          sm[0] += q[c] * d; sm[1] += q[9 + c] * d; sm[2] += q[18 + c] * d;
        }
      }
    }
#pragma unroll
    for (int m = 0; m < 3; ++m) sm[m] = group_sum(sm[m], G);
    S inc[3] = {0, 0, 0}, jls[3] = {0, 0, 0};
    if (active) {
      const S* lk = D.lmk + 24 * (size_t)sidx;
      const S rhs0 = lk[15] + sm[0], rhs1 = lk[16] + sm[1], rhs2 = lk[17] + sm[2];
      // upper-triangular solve with the damped R (Eigen triangularView<Upper>().solve)
      const S s2 = rhs2 / lk[14];
      const S s1 = (rhs1 - lk[13] * s2) / lk[12];
      const S s0 = (rhs0 - lk[10] * s1 - lk[11] * s2) / lk[9];
      inc[0] = -s0; inc[1] = -s1; inc[2] = -s2;
      jls[0] = lk[18]; jls[1] = lk[19]; jls[2] = lk[20];
    }
    // ---- pass 2: model cost change in the un-rotated basis (ref: ipp:255-262, see header comment) ----
    S lpart = 0;
    if (active) {
#pragma unroll 2
      for (int i = j; i < n; i += G) {
        const size_t sl = slot0 + i;
        const S* dp = pose_inc + 9 * (size_t)__ldg(D.slot_cam + sl);
        S jp[20], dv[9];
        load_rec<S, 20>(D.jp + 20 * sl, jp);
#pragma unroll
        for (int c = 0; c < 9; ++c) dv[c] = __ldg(dp + c);
        const S* jl = D.jl + 6 * sl;
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          S ji = 0;
#pragma unroll
          for (int c = 0; c < 9; ++c) ji += jp[9 * rr + c] * dv[c];
          ji += jl[3 * rr] * inc[0] + jl[3 * rr + 1] * inc[1] + jl[3 * rr + 2] * inc[2];
          lpart += ji * (S(0.5) * ji + D.res[2 * sl + rr]);
        }
      }
    }
    lpart = group_sum(lpart, G);
    if (active && j == 0) {
      if constexpr (LMP) {
        const int lp = D.lmp_slot[sidx];
        if (lp >= 0) {
          const S* pg = D.lmp_Lg + 12 * (size_t)lp;
#pragma unroll
          for (int r = 0; r < 3; ++r) {
            const S u = pg[3 * r] * inc[0] + pg[3 * r + 1] * inc[1] + pg[3 * r + 2] * inc[2];
            lpart += u * (S(0.5) * u + pg[9 + r]);
          }
        }
      }
      ld[0] -= (double)lpart;
      const int lm = D.sorted_lm[sidx];
      S* pw = D.lms + 3 * (size_t)lm;
      const bool ok = finite_s(inc[0]) && finite_s(inc[1]) && finite_s(inc[2]) && finite_s(pw[0]) && finite_s(pw[1]) && finite_s(pw[2]);
      if (!ok) atomicOr(bad_flag, 1);
#pragma unroll
      for (int d = 0; d < 3; ++d) pw[d] += inc[d] * jls[d];
    }
  }
  block_sum_store<1>(ld, partials);
}

// ------------------------------------------------------------------------------------------------
// K7  camera update (ref: solver/linearizor_qr.cpp:279-287, bal/bal_problem.hpp:97-109, Sophus se3_expd / SO3::exp)
// ------------------------------------------------------------------------------------------------
template <class S>
__global__ void k_camera_update(DevPtrs<S> D, const S* __restrict__ inc) {
  const int cam = blockIdx.x * blockDim.x + threadIdx.x;
  if (cam >= D.nc) return;
  S v[9];
#pragma unroll
  for (int c = 0; c < 9; ++c) v[c] = inc[9 * (size_t)cam + c] * D.scaling[9 * (size_t)cam + c];
  S* cm = D.cams + 10 * (size_t)cam;
  // SO3::exp (SURVEY A10)
  const S th2 = v[3] * v[3] + v[4] * v[4] + v[5] * v[5];
  S imag, real;
  if (th2 < ST<S>::eps() * ST<S>::eps()) {
    const S th4 = th2 * th2;
    imag = S(0.5) - S(1.0 / 48.0) * th2 + S(1.0 / 3840.0) * th4;
    real = S(1) - S(1.0 / 8.0) * th2 + S(1.0 / 384.0) * th4;
  } else {
    const S th = sqrt(th2);
    const S half = S(0.5) * th;
    imag = sin(half) / th;
    real = cos(half);
  }
  const S qe[4] = {imag * v[3], imag * v[4], imag * v[5], real};
  S Re[9];
  quat_to_rot(qe, Re);
  const S t0 = cm[4], t1 = cm[5], t2 = cm[6];
  const S a0 = qe[0], a1 = qe[1], a2 = qe[2], a3 = qe[3];
  const S b0 = cm[0], b1 = cm[1], b2 = cm[2], b3 = cm[3];
  S rq[4];
  rq[3] = a3 * b3 - a0 * b0 - a1 * b1 - a2 * b2;
  rq[0] = a3 * b0 + a0 * b3 + a1 * b2 - a2 * b1;
  rq[1] = a3 * b1 + a1 * b3 + a2 * b0 - a0 * b2;
  rq[2] = a3 * b2 + a2 * b3 + a0 * b1 - a1 * b0;
  const S sq = rq[0] * rq[0] + rq[1] * rq[1] + rq[2] * rq[2] + rq[3] * rq[3];
  if (sq != S(1)) {
    const S sc = S(2) / (S(1) + sq);
#pragma unroll
    for (int k = 0; k < 4; ++k) rq[k] *= sc;
  }
  // fixed parameters are not written: the quaternion product with exp(0) renormalises when |q|^2 != 1 and could change
  // the last bit, so a zero increment alone would not keep them constant
  const unsigned f = D.cam_fixed ? D.cam_fixed[cam] : 0u;
  if (!(f & 1u)) {
    cm[0] = rq[0]; cm[1] = rq[1]; cm[2] = rq[2]; cm[3] = rq[3];
    cm[4] = Re[0] * t0 + Re[1] * t1 + Re[2] * t2 + v[0];
    cm[5] = Re[3] * t0 + Re[4] * t1 + Re[5] * t2 + v[1];
    cm[6] = Re[6] * t0 + Re[7] * t1 + Re[8] * t2 + v[2];
  }
  if (!(f & 2u)) cm[7] += v[6];
  if (!(f & 4u)) cm[8] += v[7];
  if (!(f & 8u)) cm[9] += v[8];
}

// zero the increment entries of fixed camera parameters (a host increment given to rba_apply / rba_back_substitute), so that
// the back-substitution and l_diff see the increment the cameras receive.  Thread per entry.
template <class S>
__global__ void k_mask_fixed_inc(S* __restrict__ inc, const uint8_t* __restrict__ cam_fixed, int nc) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= 9 * nc) return;
  if ((fixed_entry_mask(cam_fixed[e / 9]) >> (e % 9)) & 1u) inc[e] = S(0);
}

// ------------------------------------------------------------------------------------------------
// K8  Gaussian camera priors (rba_set_camera_prior, DESIGN.md section 14).  Per camera the residual
//       e = (c - c0, Log(R R0^T), f - f0, k1 - k1_0, k2 - k2_0),   c = -R^T t the camera centre,
//     the cost 1/2 |L e|^2 and, for the increment (v, w, df, dk1, dk2) of k_camera_update (R' = Exp(w) R, t' = Exp(w) t + v),
//       de/dv = -R^T (rows 0..2),  dLog/dw = J_l^-1(Log(R R0^T)) (rows 3..5),  identity on the intrinsics (rows 6..8).
//     mean [nc][10] (qx,qy,qz,qw of R0, c0, f0, k1_0, k2_0; unit quaternion), sqrt_info [nc][81] row-major L.
// ------------------------------------------------------------------------------------------------
// SO(3) helpers of both prior kinds (absolute and pair priors).
// phi = Log(a (x) conj(m)) for unit quaternions a, m (xyzw, Hamilton product), the angle in [0, pi] (the product is
// flipped to w >= 0)
template <class S>
__device__ __forceinline__ void so3_log_rel(const S a0, const S a1, const S a2, const S a3, const S* __restrict__ m, S* phi) {
  const S b0 = -m[0], b1 = -m[1], b2 = -m[2], b3 = m[3];
  S w = a3 * b3 - a0 * b0 - a1 * b1 - a2 * b2;
  S v0 = a3 * b0 + a0 * b3 + a1 * b2 - a2 * b1;
  S v1 = a3 * b1 + a1 * b3 + a2 * b0 - a0 * b2;
  S v2 = a3 * b2 + a2 * b3 + a0 * b1 - a1 * b0;
  if (w < S(0)) { w = -w; v0 = -v0; v1 = -v1; v2 = -v2; }
  const S n2 = v0 * v0 + v1 * v1 + v2 * v2;
  const S n = sqrt(n2);
  // theta / n with theta = 2 atan2(n, w); series 2/w (1 - n^2 / (3 w^2)) where n is tiny against w
  const S fac = (n < ST<S>::eps_sqrt() * w) ? S(2) / w * (S(1) - n2 / (S(3) * w * w)) : S(2) * atan2(n, w) / n;
  phi[0] = fac * v0; phi[1] = fac * v1; phi[2] = fac * v2;
}
// J_l^-1(phi) (row-major 3x3) = I - 1/2 [phi]x + a [phi]x^2,  a = 1/th^2 - cot(th/2) / (2 th)  (series 1/12 + th^2/720 + th^4/30240)
template <class S>
__device__ __forceinline__ void so3_jl_inv(const S* phi, S* Jinv) {
  const S p0 = phi[0], p1 = phi[1], p2 = phi[2];
  const S th2 = p0 * p0 + p1 * p1 + p2 * p2;
  S a;
  if (th2 < S(1e-4)) a = S(1.0 / 12.0) + th2 * (S(1.0 / 720.0) + th2 * S(1.0 / 30240.0));
  else {
    const S th = sqrt(th2), h = S(0.5) * th;
    a = S(1) / th2 - cos(h) / (S(2) * th * sin(h));
  }
  // [phi]x^2 = phi phi^T - th^2 I
  Jinv[0] = S(1) + a * (p0 * p0 - th2); Jinv[1] = S(0.5) * p2 + a * p0 * p1;       Jinv[2] = -S(0.5) * p1 + a * p0 * p2;
  Jinv[3] = -S(0.5) * p2 + a * p1 * p0; Jinv[4] = S(1) + a * (p1 * p1 - th2);       Jinv[5] = S(0.5) * p0 + a * p1 * p2;
  Jinv[6] = S(0.5) * p1 + a * p2 * p0;  Jinv[7] = -S(0.5) * p0 + a * p2 * p1;       Jinv[8] = S(1) + a * (p2 * p2 - th2);
}

// e of one camera; with JAC also J_l^-1 (row-major 3x3) and R (row-major 3x3)
template <class S, bool JAC>
__device__ __forceinline__ void prior_residual(const S* __restrict__ cam, const S* __restrict__ mean, S* e, S* Jinv, S* R) {
  S Rl[9];
  S* Rm = JAC ? R : Rl;
  quat_to_rot(cam, Rm);
  const S t0 = cam[4], t1 = cam[5], t2 = cam[6];
#pragma unroll
  for (int k = 0; k < 3; ++k) e[k] = -(Rm[k] * t0 + Rm[3 + k] * t1 + Rm[6 + k] * t2) - mean[4 + k];
  so3_log_rel(cam[0], cam[1], cam[2], cam[3], mean, e + 3);  // Log(R R0^T)
  e[6] = cam[7] - mean[7]; e[7] = cam[8] - mean[8]; e[8] = cam[9] - mean[9];
  if (JAC) so3_jl_inv(e + 3, Jinv);
}

// row of L de/d(inc) for the row l [9] of L: L (-R^T) on v, L J_l^-1 on w, L itself on the intrinsics
template <class S>
__device__ __forceinline__ void prior_jac_row(const S* l, const S* R, const S* Jinv, S* row) {
#pragma unroll
  for (int j = 0; j < 3; ++j) row[j] = -(l[0] * R[3 * j] + l[1] * R[3 * j + 1] + l[2] * R[3 * j + 2]);
#pragma unroll
  for (int j = 0; j < 3; ++j) row[3 + j] = l[3] * Jinv[j] + l[4] * Jinv[3 + j] + l[5] * Jinv[6 + j];
#pragma unroll
  for (int j = 6; j < 9; ++j) row[j] = l[j];
}

// The per-item terms of the one-block kernels k_prior_cost and k_prior_ldiff, one struct per prior kind (item = camera,
// pair or landmark prior).  rows_of(p, f) calls f(i, (L e)_i) row by row (k_prior_residuals reads them), sq_norm(p) =
// |L e|^2 of item p, model_change(inc, p) = (A d)^T (1/2 A d + r) for its part d of the increment; each kind keeps its own
// summation order.
template <class S>
struct CameraPrior {
  using Scalar = S;
  static constexpr int NR = 9;  // rows of L e; L is NR x NR
  const S* cams;
  const S* mean;  // [nc][10]
  const S* L;     // [nc][81]
  const S* A;     // [nc][81]
  const S* r;     // [nc][9]
  // f(i, (L e)_i) for the rows i of item cam in order
  template <class F>
  __device__ void rows_of(int cam, F f) const {
    S e[9];
    prior_residual<S, false>(cams + 10 * (size_t)cam, mean + 10 * (size_t)cam, e, nullptr, nullptr);
    const S* Lc = L + 81 * (size_t)cam;
    for (int i = 0; i < 9; ++i) {
      S ri = 0;
#pragma unroll
      for (int k = 0; k < 9; ++k) ri += Lc[9 * i + k] * e[k];
      f(i, ri);
    }
  }
  __device__ S sq_norm(int cam) const {
    S c2 = 0;
    rows_of(cam, [&](int, S ri) { c2 += ri * ri; });
    return c2;
  }
  __device__ S model_change(const S* inc, int cam) const {
    S d[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) d[j] = inc[9 * (size_t)cam + j];
    const S* Ac = A + 81 * (size_t)cam;
    S lp = 0;
    for (int i = 0; i < 9; ++i) {
      S u = 0;
#pragma unroll
      for (int j = 0; j < 9; ++j) u += Ac[9 * i + j] * d[j];
      lp += u * (S(0.5) * u + r[9 * (size_t)cam + i]);
    }
    return lp;
  }
};

// once per linearisation, after the cross-shard sum of diag2 and before k_scaling: the unscaled prior Jacobian
// J = L de/d(inc) -> A [nc][81], r = L e -> pr [nc][9], and its squared column norms added to diag2 (the Jacobi scaling is
// that of the whole Jacobian).  Thread per camera; identical on every shard (the prior data and the cameras are replicated).
template <class S>
__global__ void k_prior_linearize(const S* __restrict__ cams, const S* __restrict__ mean, const S* __restrict__ Lsq, int nc,
                                  S* __restrict__ diag2, S* __restrict__ A, S* __restrict__ pr) {
  const int cam = blockIdx.x * blockDim.x + threadIdx.x;
  if (cam >= nc) return;
  S e[9], Jinv[9], R[9];
  prior_residual<S, true>(cams + 10 * (size_t)cam, mean + 10 * (size_t)cam, e, Jinv, R);
  const S* Lc = Lsq + 81 * (size_t)cam;
  S* Ac = A + 81 * (size_t)cam;
  S cn[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) cn[j] = 0;
  for (int i = 0; i < 9; ++i) {
    S l[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) l[k] = Lc[9 * i + k];
    S row[9], ri = 0;
#pragma unroll
    for (int k = 0; k < 9; ++k) ri += l[k] * e[k];
    prior_jac_row(l, R, Jinv, row);
#pragma unroll
    for (int j = 0; j < 9; ++j) { Ac[9 * i + j] = row[j]; cn[j] += row[j] * row[j]; }
    pr[9 * (size_t)cam + i] = ri;
  }
#pragma unroll
  for (int j = 0; j < 9; ++j) diag2[9 * (size_t)cam + j] += cn[j];
}

// after k_scaling (and after the JACOBI blocks are built): A <- J diag(s) in place, H = A^T A, g = A^T r, and H added to the
// JACOBI blocks when they exist (jblocks != nullptr; they are the Hpp of Power-SC).  Thread per camera.
template <class S>
__global__ void k_prior_scale(S* __restrict__ A, const S* __restrict__ pr, const S* __restrict__ scaling, int nc,
                              S* __restrict__ H, S* __restrict__ g, S* __restrict__ jblocks) {
  const int cam = blockIdx.x * blockDim.x + threadIdx.x;
  if (cam >= nc) return;
  S s[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) s[j] = scaling[9 * (size_t)cam + j];
  S* Ac = A + 81 * (size_t)cam;
  for (int i = 0; i < 9; ++i)
#pragma unroll
    for (int j = 0; j < 9; ++j) Ac[9 * i + j] *= s[j];
  for (int a = 0; a < 9; ++a) {
    S ga = 0;
    for (int i = 0; i < 9; ++i) ga += Ac[9 * i + a] * pr[9 * (size_t)cam + i];
    g[9 * (size_t)cam + a] = ga;
    for (int b = 0; b < 9; ++b) {
      S h = 0;
      for (int i = 0; i < 9; ++i) h += Ac[9 * i + a] * Ac[9 * i + b];
      H[81 * (size_t)cam + 9 * a + b] = h;
      if (jblocks) jblocks[81 * (size_t)cam + 9 * a + b] += h;
    }
  }
}

// sum over the cameras of one double per camera, in a fixed order, added to out[0] (and out[1] when two are given).
// One block: every entry point calls it after the cross-shard sum, so the prior term is added once and identically on every shard.
__device__ __forceinline__ double prior_block_sum(double v) {
  __shared__ double sh[32];
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += sh[w];
  return s;  // valid in thread 0
}

// cost sum_p 1/2 |L_p e_p|^2 of the n items of one prior kind K at the current parameters, added to the all / valid errors
// (red[1], red[4]); a non-finite sum sets the numerical-failure flag.  One block.
template <class K>
__global__ void k_prior_cost(K k, int n, double* red, int* bad_flag) {
  double acc = 0;
  for (int p = threadIdx.x; p < n; p += blockDim.x) acc += 0.5 * (double)k.sq_norm(p);
  const double s = prior_block_sum(acc);
  if (threadIdx.x == 0) {
    red[1] += s;
    red[4] += s;
    if (!isfinite(s)) *bad_flag = 1;
  }
}

// prior part of the model cost change: l_diff -= sum_p (A d)^T (1/2 A d + r) over the n items of one prior kind K for the
// (masked, scaled) increment d, added to red[0] (the back-substitution's l_diff, already summed over the shards).  One block.
template <class K>
__global__ void k_prior_ldiff(K k, const typename K::Scalar* __restrict__ inc, int n, double* red) {
  double acc = 0;
  for (int p = threadIdx.x; p < n; p += blockDim.x) acc -= (double)k.model_change(inc, p);
  const double s = prior_block_sum(acc);
  if (threadIdx.x == 0) red[0] += s;
}

// Landmark priors (DESIGN.md section 17): e_p = x_p - x0_p of this shard's priors (lm = local landmark of each).  Their cost
// is added BEFORE the sum over the shards: the term is landmark-owned, so each shard adds its own priors and the sum counts
// each once.  Their share of l_diff is computed per landmark in k_back_substitute.
template <class S>
struct LandmarkPrior {
  using Scalar = S;
  static constexpr int NR = 3;
  const S* lms;
  const int* lm;   // [m]
  const S* mean;   // [m][3]
  const S* L;      // [m][9]
  template <class F>
  __device__ void rows_of(int p, F f) const {
    const S* x = lms + 3 * (size_t)lm[p];
    const S* x0 = mean + 3 * (size_t)p;
    const S e0 = x[0] - x0[0], e1 = x[1] - x0[1], e2 = x[2] - x0[2];
    const S* Lp = L + 9 * (size_t)p;
#pragma unroll
    for (int r = 0; r < 3; ++r) f(r, Lp[3 * r] * e0 + Lp[3 * r + 1] * e1 + Lp[3 * r + 2] * e2);
  }
  __device__ S sq_norm(int p) const {
    S c2 = 0;
    rows_of(p, [&](int, S v) { c2 += v * v; });
    return c2;
  }
};

// Robust losses on the priors (rba_set_prior_loss, DESIGN.md section 22).  Prior kind K with one loss record per item
// (slot_loss layout over its n items) and the loss function of the observations, observation_loss, on s = |L e|^2:
// sq_norm(p) = rho(s), which k_prior_cost halves into the cost rho(s)/2; loss_of gives err = rho(s)/2 and w = rho'(s).
template <class K>
struct RobustPrior {
  using Scalar = typename K::Scalar;
  K k;
  const Scalar* loss;
  int n;
  __device__ void loss_of(int p, Scalar s, Scalar& err, Scalar& w) const {
    unsigned kind;
    Scalar a;
    slot_loss(loss, n, (size_t)p, kind, a);
    observation_loss<Scalar>(kind, a, s, err, w);
  }
  __device__ Scalar sq_norm(int p) const {
    Scalar err, w;
    loss_of(p, k.sq_norm(p), err, w);
    return Scalar(2) * err;
  }
};

// Once per linearisation, before the kernels that read L (k_prior_linearize, k_pair_linearize, the LMP instances of
// k_linearize_qr): Lw = sqrt(w) L per item, w at the linearisation point.  Everything the solve derives from a prior is
// linear in L, so its rows become sqrt(w) L de/d(inc) and sqrt(w) L e.  NONE gives w = 1 and Lw = L bit for bit; TUKEY
// beyond its scale w = 0 and all-zero rows.  Thread per item.
template <class K>
__global__ void k_prior_weight(RobustPrior<K> rk, typename K::Scalar* __restrict__ Lw) {
  using S = typename K::Scalar;
  constexpr int NL = K::NR * K::NR;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= rk.n) return;
  S err, w;
  rk.loss_of(p, rk.k.sq_norm(p), err, w);
  const S sw = sqrt(w);
  const S* Lp = rk.k.L + NL * (size_t)p;
  S* out = Lw + NL * (size_t)p;
  for (int i = 0; i < NL; ++i) out[i] = sw * Lp[i];
}

// rba_get_prior_residuals: per item at the current state res [NR] = L e (unweighted L) and w = rho'(|L e|^2) of its loss
// (loss == nullptr: every item NONE, w = 1).  Thread per item.
template <class K>
__global__ void k_prior_residuals(K k, const typename K::Scalar* __restrict__ loss, int n, typename K::Scalar* __restrict__ res,
                                  typename K::Scalar* __restrict__ wout) {
  using S = typename K::Scalar;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  S s = 0;
  k.rows_of(p, [&](int i, S ri) { res[K::NR * (size_t)p + i] = ri; s += ri * ri; });
  S w = S(1);
  if (loss) {
    S err;
    RobustPrior<K>{k, loss, n}.loss_of(p, s, err, w);
  }
  wout[p] = w;
}

// ------------------------------------------------------------------------------------------------
// K9  Relative pose priors between two cameras (rba_set_camera_pair_prior, DESIGN.md section 15).  Pair p = (i, j) with the
//     measured relative pose Z = (R0, t0) of T_i T_j^-1 and the 6x6 square-root information L:
//       e_t = t_i - R_i R_j^T t_j - t0,   e_r = Log(R_i R_j^T R0^T),   cost 1/2 |L (e_t, e_r)|^2.
//     For the increment of k_camera_update, with M = R_i R_j^T, t_rel = t_i - M t_j, phi = e_r:
//       de_t/dv_i = I,  de_t/dw_i = -[t_rel]x,  de_t/dv_j = -M,  de_t/dw_j = 0,
//       de_r/dw_i = J_l^-1(phi),  de_r/dw_j = -J_l^-1(phi) M,  de_r/dv = 0;  zero intrinsic columns.
//     pairs [m][2], mean [m][7] (qx,qy,qz,qw of R0, t0; unit quaternion), sqrt_info [m][36] row-major L.
//     A [m][2][36]: the pose blocks A_i, A_j (6x6, row-major) of L de/d(inc), unscaled after k_pair_linearize and scaled
//     after k_pair_scale; pr [m][6] = L e.  Incident pair sides are listed camera-major (ptr [nc + 1], item = 2 p + side,
//     ascending p within a camera), which is also the CSR of the directed edges i -> j of the off-diagonal blocks O_ij.
// ------------------------------------------------------------------------------------------------
// e [6] of one pair; M = R_i R_j^T and t_rel (needed by e); with JAC also J_l^-1(phi) and JM = J_l^-1(phi) M
template <class S, bool JAC>
__device__ __forceinline__ void pair_residual(const S* __restrict__ ci, const S* __restrict__ cj, const S* __restrict__ mean,
                                              S* e, S* M, S* tr, S* Jinv, S* JM) {
  S Ri[9], Rj[9];
  quat_to_rot(ci, Ri);
  quat_to_rot(cj, Rj);
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) M[3 * a + b] = Ri[3 * a] * Rj[3 * b] + Ri[3 * a + 1] * Rj[3 * b + 1] + Ri[3 * a + 2] * Rj[3 * b + 2];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    tr[a] = ci[4 + a] - (M[3 * a] * cj[4] + M[3 * a + 1] * cj[5] + M[3 * a + 2] * cj[6]);
    e[a] = tr[a] - mean[4 + a];
  }
  // q_i (x) conj(q_j) is the quaternion of M; phi = Log(M R0^T)
  const S a0 = ci[0], a1 = ci[1], a2 = ci[2], a3 = ci[3];
  const S b0 = -cj[0], b1 = -cj[1], b2 = -cj[2], b3 = cj[3];
  const S w = a3 * b3 - a0 * b0 - a1 * b1 - a2 * b2;
  const S x = a3 * b0 + a0 * b3 + a1 * b2 - a2 * b1;
  const S y = a3 * b1 + a1 * b3 + a2 * b0 - a0 * b2;
  const S z = a3 * b2 + a2 * b3 + a0 * b1 - a1 * b0;
  so3_log_rel(x, y, z, w, mean, e + 3);
  if (JAC) {
    so3_jl_inv(e + 3, Jinv);
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) JM[3 * a + b] = Jinv[3 * a] * M[b] + Jinv[3 * a + 1] * M[3 + b] + Jinv[3 * a + 2] * M[6 + b];
  }
}

// rows of A_i = L de/d(inc_i) and A_j = L de/d(inc_j) for the row l [6] of L:
//   A_i row (l_t, l_t (-[t_rel]x) + l_r J_l^-1),  A_j row (-l_t M, -l_r J_l^-1 M)
template <class S>
__device__ __forceinline__ void pair_jac_rows(const S* l, const S* M, const S* tr, const S* Jinv, const S* JM, S* ri, S* rj) {
#pragma unroll
  for (int j = 0; j < 3; ++j) ri[j] = l[j];
  ri[3] = -l[1] * tr[2] + l[2] * tr[1] + l[3] * Jinv[0] + l[4] * Jinv[3] + l[5] * Jinv[6];
  ri[4] = l[0] * tr[2] - l[2] * tr[0] + l[3] * Jinv[1] + l[4] * Jinv[4] + l[5] * Jinv[7];
  ri[5] = -l[0] * tr[1] + l[1] * tr[0] + l[3] * Jinv[2] + l[4] * Jinv[5] + l[5] * Jinv[8];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    rj[j] = -(l[0] * M[j] + l[1] * M[3 + j] + l[2] * M[6 + j]);
    rj[3 + j] = -(l[3] * JM[j] + l[4] * JM[3 + j] + l[5] * JM[6 + j]);
  }
}

// the pair priors' terms of k_prior_cost and k_prior_ldiff (A d = A_i d_i + A_j d_j)
template <class S>
struct PairPrior {
  using Scalar = S;
  static constexpr int NR = 6;
  const S* cams;
  const int* pairs;  // [m][2]
  const S* mean;     // [m][7]
  const S* L;        // [m][36]
  const S* A;        // [m][2][36]
  const S* r;        // [m][6]
  template <class F>
  __device__ void rows_of(int p, F f) const {
    S e[6], M[9], tr[3];
    pair_residual<S, false>(cams + 10 * (size_t)pairs[2 * p], cams + 10 * (size_t)pairs[2 * p + 1], mean + 7 * (size_t)p, e, M, tr,
                            nullptr, nullptr);
    const S* Lp = L + 36 * (size_t)p;
    for (int i = 0; i < 6; ++i) {
      S ri = 0;
#pragma unroll
      for (int k = 0; k < 6; ++k) ri += Lp[6 * i + k] * e[k];
      f(i, ri);
    }
  }
  __device__ S sq_norm(int p) const {
    S c2 = 0;
    rows_of(p, [&](int, S ri) { c2 += ri * ri; });
    return c2;
  }
  __device__ S model_change(const S* inc, int p) const {
    S di[6], dj[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) { di[j] = inc[9 * (size_t)pairs[2 * p] + j]; dj[j] = inc[9 * (size_t)pairs[2 * p + 1] + j]; }
    const S* Ai = A + 72 * (size_t)p;
    S lp = 0;
    for (int i = 0; i < 6; ++i) {
      S u = 0;
#pragma unroll
      for (int j = 0; j < 6; ++j) u += Ai[6 * i + j] * di[j] + Ai[36 + 6 * i + j] * dj[j];
      lp += u * (S(0.5) * u + r[6 * (size_t)p + i]);
    }
    return lp;
  }
};

// once per linearisation, after the cross-shard sum of diag2 (and the absolute priors) and before k_scaling: the unscaled
// pose blocks A_i = L de/d(inc_i), A_j = L de/d(inc_j) and r = L e.  Thread per pair; identical on every shard.
template <class S>
__global__ void k_pair_linearize(const S* __restrict__ cams, const int* __restrict__ pairs, const S* __restrict__ mean,
                                 const S* __restrict__ Lsq, int m, S* __restrict__ A, S* __restrict__ pr) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m) return;
  S e[6], M[9], tr[3], Jinv[9], JM[9];
  pair_residual<S, true>(cams + 10 * (size_t)pairs[2 * p], cams + 10 * (size_t)pairs[2 * p + 1], mean + 7 * (size_t)p, e, M, tr, Jinv, JM);
  const S* Lp = Lsq + 36 * (size_t)p;
  S* Ai = A + 72 * (size_t)p;
  S* Aj = Ai + 36;
  for (int i = 0; i < 6; ++i) {
    S l[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) l[k] = Lp[6 * i + k];
    S ri = 0;
#pragma unroll
    for (int k = 0; k < 6; ++k) ri += l[k] * e[k];
    pr[6 * (size_t)p + i] = ri;
    pair_jac_rows(l, M, tr, Jinv, JM, Ai + 6 * i, Aj + 6 * i);
  }
}

// squared column norms of the incident pair blocks added to diag2 (the Jacobi scaling of the whole Jacobian).  Thread per
// camera over its incident sides in list order: no atomics, bit-identical on every run and shard.
template <class S>
__global__ void k_pair_diag2(const S* __restrict__ A, const int* __restrict__ ptr, const int* __restrict__ item, int nc,
                             S* __restrict__ diag2) {
  const int cam = blockIdx.x * blockDim.x + threadIdx.x;
  if (cam >= nc) return;
  S cn[6];
#pragma unroll
  for (int j = 0; j < 6; ++j) cn[j] = 0;
  for (int q = ptr[cam]; q < ptr[cam + 1]; ++q) {
    const S* As = A + 36 * (size_t)item[q];
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int j = 0; j < 6; ++j) cn[j] += As[6 * i + j] * As[6 * i + j];
  }
#pragma unroll
  for (int j = 0; j < 6; ++j) diag2[9 * (size_t)cam + j] += cn[j];
}

// after k_scaling: A_s <- A_s diag(s of its camera), in place.  Thread per pair.
template <class S>
__global__ void k_pair_scale(S* __restrict__ A, const int* __restrict__ pairs, const S* __restrict__ scaling, int m) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m) return;
  for (int s = 0; s < 2; ++s) {
    const S* sc = scaling + 9 * (size_t)pairs[2 * p + s];
    S* As = A + 72 * (size_t)p + 36 * s;
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int j = 0; j < 6; ++j) As[6 * i + j] *= sc[j];
  }
}

// after k_pair_scale (and k_prior_scale): per camera the sum over its incident sides of A_s^T A_s into H [nc][81] and of
// A_s^T r into g [9 nc] (added to the absolute priors' H, g when `accumulate`, else written with zero intrinsic rows and
// columns), A_s^T A_s also into the JACOBI blocks when they exist, and O_ij = A_s^T A_other of every directed edge.
// Thread per camera, sides in list order.
template <class S>
__global__ void k_pair_accum(const S* __restrict__ A, const S* __restrict__ pr, const int* __restrict__ ptr,
                             const int* __restrict__ item, int nc, int accumulate, S* __restrict__ H, S* __restrict__ g,
                             S* __restrict__ jblocks, S* __restrict__ O) {
  const int cam = blockIdx.x * blockDim.x + threadIdx.x;
  if (cam >= nc) return;
  const int q0 = ptr[cam], q1 = ptr[cam + 1];
  S* Hc = H + 81 * (size_t)cam;
  for (int a = 0; a < 6; ++a) {
    S hrow[6], ga = 0;
#pragma unroll
    for (int b = 0; b < 6; ++b) hrow[b] = 0;
    for (int q = q0; q < q1; ++q) {
      const int it = item[q];
      const S* As = A + 36 * (size_t)it;
      const S* Ao = A + 36 * (size_t)(it ^ 1);
      const S* rp = pr + 6 * (size_t)(it >> 1);
      S orow[6];
#pragma unroll
      for (int b = 0; b < 6; ++b) orow[b] = 0;
      for (int i = 0; i < 6; ++i) {
        const S ai = As[6 * i + a];
        ga += ai * rp[i];
#pragma unroll
        for (int b = 0; b < 6; ++b) { hrow[b] += ai * As[6 * i + b]; orow[b] += ai * Ao[6 * i + b]; }
      }
#pragma unroll
      for (int b = 0; b < 6; ++b) O[36 * (size_t)q + 6 * a + b] = orow[b];
    }
    g[9 * (size_t)cam + a] = (accumulate ? g[9 * (size_t)cam + a] : S(0)) + ga;
#pragma unroll
    for (int b = 0; b < 6; ++b) {
      Hc[9 * a + b] = (accumulate ? Hc[9 * a + b] : S(0)) + hrow[b];
      if (jblocks) jblocks[81 * (size_t)cam + 9 * a + b] += hrow[b];
    }
  }
  if (!accumulate) {
    for (int k = 0; k < 81; ++k)
      if (k / 9 >= 6 || k % 9 >= 6) Hc[k] = 0;
    for (int a = 6; a < 9; ++a) g[9 * (size_t)cam + a] = 0;
  }
}

// Per PCG iteration (and power-series term), just ahead of the vector step: D.pair_ov = sum_j O_ij v_j for the vector v the
// step is about to consume.  A kernel of its own: the vector step reads other cameras' v here, and computing the product in
// a separate grid keeps it complete before any CTA of the vector step overwrites D.p or D.x.  Launched dependent on its
// predecessor; its own wait keeps the dependency chain transitive for the vector step, which waits for this grid.
template <class S>
__global__ void __launch_bounds__(256) k_pair_ov(DevPtrs<S> D, const PcgState* st, const S* __restrict__ v) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (*reinterpret_cast<const volatile int*>(&st->done)) return;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < 9 * D.nc; e += gridDim.x * blockDim.x) D.pair_ov[e] = pair_ov_entry(D, v, e);
}

}  // namespace rba
