// Resection and per-camera (per-rig) refinement with the landmarks held (rba_resect_cameras, DESIGN.md section 26).
//
// One CTA per unit: a free camera, or a rig of >= 2 cameras whose free pose is its lead's.  The threads stride over the
// unit's observation slots member by member (csr_obs), and every sum is a fixed-order block reduction (per-thread partial
// sums in shared memory, then the threads in order): a unit's result depends on its own observations and the call's starting state only, so it is
// bit-identical across calls, subsets and solver configurations.  Everything is float64 for either Scalar.  The small dense
// work (the 12x12 eigenproblem of the linear estimate, the <= 9x9 Cholesky of the refinement) runs on thread 0 out of
// shared memory.
#pragma once

#include "rigs.cuh"
#include "triangulate.cuh"

namespace rba {

constexpr int RES_THREADS = 64;
constexpr int RES_ACC = 61;            // doubles per thread of the shared accumulators (>= 60, odd against bank conflicts)
constexpr int RES_MIN_POINTS = 3;       // usable points below which a unit without a prior is left untouched
constexpr int RES_MIN_LINEAR = 6;       // usable points the linear estimate needs in its member
constexpr double RES_PLANAR = 1e-3;     // smallest / largest principal standard deviation of the points below this: DEGENERATE
constexpr double RES_SINGULAR = 1e-10;  // |det A| <= this |A|_F^3: DEGENERATE
constexpr int RES_MX = 43;              // doubles per member of the per-call table: M_j (7), A_j (36)

struct ResItem {
  int m0, nm;     // members mem[m0 .. m0 + nm), ascending camera index
  int lead;       // the camera holding the unit's pose
  unsigned free;  // fixed_entry_mask layout: the free entries of the lead's increment
};
struct ResMember {
  int cam;
  int begin, end;  // its observations csr_obs.slots[begin .. end)
};
struct ResOpts {
  int mode;
  int max_iterations;
  double ftol;
};
// The inputs besides DevPtrs, all read only.  cp_L == nullptr: no camera priors; pp_ptr == nullptr: no pair priors; a loss
// pointer nullptr: that kind has no losses.  R.lead == nullptr: no rigs; Z.home == nullptr: no sensors.
template <class S>
struct ResTerms {
  const S* snap;    // [nc][10] the cameras at the call's start
  const int* slots;  // csr_obs.slots
  RigView<S> R;
  SensorView<S> Z;
  const S* cp_mean; const S* cp_L; const S* cp_loss;
  const int* pp_ij; const S* pp_mean; const S* pp_L; const S* pp_loss; const int* pp_ptr; const int* pp_item; int pp_n;
};

// entry (a, b), a <= b, of the upper triangle of a symmetric 9x9 matrix stored row by row
__host__ __device__ __forceinline__ int res_hidx(int a, int b) { return a * 9 - a * (a - 1) / 2 + (b - a); }

// Every thread accumulates into its own row acc[threadIdx.x] of shared memory (registers cannot hold the 55 and 60 sums
// next to the Jacobians without spilling).  out[k] (k < K, shared) = the sum of column k over the threads in order.  Every
// thread returns after out is complete.
__device__ __forceinline__ void res_block_sum(int K, double (*acc)[RES_ACC], double* out) {
  __syncthreads();
  if ((int)threadIdx.x < K) {
    double s = 0.0;
    for (int i = 0; i < (int)blockDim.x; ++i) s += acc[i][threadIdx.x];
    out[threadIdx.x] = s;
  }
  __syncthreads();
}
__device__ __forceinline__ void res_zero(double* a, int K) {
  for (int k = 0; k < K; ++k) a[k] = 0.0;
}

// the unit quaternion (x, y, z, w) of a rotation matrix (row-major), by the largest of the four candidate pivots
__device__ __forceinline__ void res_rot_to_quat(const double* R, double* q) {
  const double tr = R[0] + R[4] + R[8];
  if (tr >= R[0] && tr >= R[4] && tr >= R[8]) {
    const double s = 2.0 * sqrt(1.0 + tr);
    q[3] = 0.25 * s; q[0] = (R[7] - R[5]) / s; q[1] = (R[2] - R[6]) / s; q[2] = (R[3] - R[1]) / s;
  } else if (R[0] >= R[4] && R[0] >= R[8]) {
    const double s = 2.0 * sqrt(1.0 + R[0] - R[4] - R[8]);
    q[0] = 0.25 * s; q[3] = (R[7] - R[5]) / s; q[1] = (R[1] + R[3]) / s; q[2] = (R[2] + R[6]) / s;
  } else if (R[4] >= R[8]) {
    const double s = 2.0 * sqrt(1.0 + R[4] - R[0] - R[8]);
    q[1] = 0.25 * s; q[3] = (R[2] - R[6]) / s; q[0] = (R[1] + R[3]) / s; q[2] = (R[5] + R[7]) / s;
  } else {
    const double s = 2.0 * sqrt(1.0 + R[8] - R[0] - R[4]);
    q[2] = 0.25 * s; q[3] = (R[3] - R[1]) / s; q[0] = (R[2] + R[6]) / s; q[1] = (R[5] + R[7]) / s;
  }
}

// The camera of member `cam` for the lead camera lc [10]: mode 0 the stored camera (snapshot); 1 M_j lc as it would be
// stored (rounded to S); 2 M_j lc in double.  The lead itself is lc; a member keeps its own intrinsics.
template <class S>
__device__ __forceinline__ void res_member(const ResTerms<S>& T, int cam, int lead, const double* m, const double* lc, int mode,
                                           double (&c)[10]) {
  if (mode == 0) {
#pragma unroll
    for (int k = 0; k < 10; ++k) c[k] = (double)T.snap[10 * (size_t)cam + k];
    return;
  }
  if (cam == lead) {
#pragma unroll
    for (int k = 0; k < 10; ++k) c[k] = lc[k];
    return;
  }
  double w[20];
#pragma unroll
  for (int k = 0; k < 10; ++k) w[k] = lc[k];
  retie_pose<double>(w, 1, 0, m);
#pragma unroll
  for (int k = 0; k < 7; ++k) c[k] = mode == 1 ? (double)(S)w[10 + k] : w[10 + k];
#pragma unroll
  for (int k = 7; k < 10; ++k) c[k] = (double)T.snap[10 * (size_t)cam + k];
}

// out [9] += the lead's row of a member's row: the pose part through A_j (A == nullptr: the identity), the intrinsics as they are
__device__ __forceinline__ void res_map_row(const double* row, int n, const double* A, double (&out)[9]) {
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    double v = 0.0;
    if (A) {
#pragma unroll
      for (int i = 0; i < 6; ++i) v += row[i] * A[6 * i + k];
    } else {
      v = row[k];
    }
    out[k] += v;
  }
  if (n == 9)
#pragma unroll
    for (int k = 6; k < 9; ++k) out[k] += row[k];
}

// acc [45 upper H | 9 g | cost] += w j^T j, w j^T r for one row j [9] of the lead's Jacobian
__device__ __forceinline__ void res_add_row(double* acc, const double (&j)[9], double r, double w) {
#pragma unroll
  for (int a = 0; a < 9; ++a) {
#pragma unroll
    for (int b = a; b < 9; ++b) acc[res_hidx(a, b)] += w * j[a] * j[b];
    acc[45 + a] += w * j[a] * r;
  }
}

// The camera prior of member `cam` at its camera c (sections 14 and 22) into acc, rows through A
template <class S>
__device__ __forceinline__ void res_camera_prior(const DevPtrs<S>& D, const ResTerms<S>& T, int cam, const double* c, const double* A,
                                                 double* acc) {
  const S* Lc = T.cp_L + 81 * (size_t)cam;
  double mean[10], e[9], Jinv[9], R[9];
#pragma unroll
  for (int k = 0; k < 10; ++k) mean[k] = (double)T.cp_mean[10 * (size_t)cam + k];
  prior_residual<double, true>(c, mean, e, Jinv, R);
  double sp = 0.0;
  bool any = false;
  for (int i = 0; i < 9; ++i) {
    double ri = 0.0;
#pragma unroll
    for (int k = 0; k < 9; ++k) { ri += (double)Lc[9 * i + k] * e[k]; any = any || Lc[9 * i + k] != S(0); }
    sp += ri * ri;
  }
  if (!any) return;
  double err = 0.5 * sp, w = 1.0;
  if (T.cp_loss) {
    unsigned kind;
    S a;
    slot_loss(T.cp_loss, D.nc, (size_t)cam, kind, a);
    observation_loss<double>(kind, (double)a, sp, err, w);
  }
  acc[54] += err;
  for (int i = 0; i < 9; ++i) {
    double l[9], row[9], ri = 0.0, j[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 9; ++k) { l[k] = (double)Lc[9 * i + k]; ri += l[k] * e[k]; }
    prior_jac_row(l, R, Jinv, row);
    res_map_row(row, 9, A, j);
    res_add_row(acc, j, ri, w);
  }
}

// The pair prior of the incident side `side_item` (2 p + side) of member `cam` at its camera c (sections 15 and 22) into acc.
// The other endpoint is read from the snapshot unless it is a member of the same unit: then both move, and the pair is
// counted from its first camera only.
template <class S>
__device__ __forceinline__ void res_pair_prior(const DevPtrs<S>& D, const ResTerms<S>& T, const ResItem& it, const ResMember* mem,
                                               const double* mx, const double* lc, int mode, const double* c,
                                               const double* A, int side_item, double* acc) {
  const int p = side_item >> 1, side = side_item & 1;
  const int ci = T.pp_ij[2 * p], cj = T.pp_ij[2 * p + 1];
  const int other = side ? ci : cj;
  int qo = -1;
  if (it.nm > 1 && T.R.lead[other] == it.lead)
    for (int q = 0; q < it.nm; ++q)
      if (mem[it.m0 + q].cam == other) qo = q;
  if (qo >= 0 && side == 1) return;
  double co[10];
  const double* Ao = nullptr;
  if (qo >= 0) {
    const double* m = mx + RES_MX * (size_t)(it.m0 + qo);
    res_member(T, other, it.lead, m, lc, mode, co);
    Ao = m + 7;
  } else {
#pragma unroll
    for (int k = 0; k < 10; ++k) co[k] = (double)T.snap[10 * (size_t)other + k];
  }
  const double* cI = side ? co : c;
  const double* cJ = side ? c : co;
  double mean[7], e[6], M[9], tr[3], Jinv[9], JM[9];
#pragma unroll
  for (int k = 0; k < 7; ++k) mean[k] = (double)T.pp_mean[7 * (size_t)p + k];
  pair_residual<double, true>(cI, cJ, mean, e, M, tr, Jinv, JM);
  const S* Lp = T.pp_L + 36 * (size_t)p;
  double sp = 0.0;
  for (int i = 0; i < 6; ++i) {
    double ri = 0.0;
#pragma unroll
    for (int k = 0; k < 6; ++k) ri += (double)Lp[6 * i + k] * e[k];
    sp += ri * ri;
  }
  double err = 0.5 * sp, w = 1.0;
  if (T.pp_loss) {
    unsigned kind;
    S a;
    slot_loss(T.pp_loss, T.pp_n, (size_t)p, kind, a);
    observation_loss<double>(kind, (double)a, sp, err, w);
  }
  acc[54] += err;
  const double* AI = side ? Ao : A;
  const double* AJ = side ? A : Ao;
  const bool inI = side == 1 ? qo >= 0 : true, inJ = side == 0 ? qo >= 0 : true;
  for (int i = 0; i < 6; ++i) {
    double l[6], ri = 0.0, rI[6], rJ[6], j[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 6; ++k) { l[k] = (double)Lp[6 * i + k]; ri += l[k] * e[k]; }
    pair_jac_rows(l, M, tr, Jinv, JM, rI, rJ);
    if (inI) res_map_row(rI, 6, AI, j);
    if (inJ) res_map_row(rJ, 6, AJ, j);
    res_add_row(acc, j, ri, w);
  }
}

// The unit's share of the cost (rba_compute_error) with its lead at lc (mode as res_member) and the IRLS normal equations of
// the lead's increment: out [45 upper H | 9 g | cost] in shared memory.  Per slot, bit `vbit` of vb[s] is set to the
// projection validity (z >= eps_sqrt of S), and the return value `lost` reports an observation in use that is valid under
// bit `cbit` and not now.  s_mc [10] is the shared camera of the member in hand.
template <class S>
__device__ double res_eval(const DevPtrs<S>& D, const KOpts& o, const ResTerms<S>& T, const ResItem& it, const ResMember* mem,
                           const double* mx, const double* lc, int mode, uint8_t* vb, int vbit, int cbit, double* s_mc,
                           double (*sacc)[RES_ACC], double* out, bool& lost) {
  double* acc = sacc[threadIdx.x];
  res_zero(acc, 55);
  bool lo = false;
  for (int q = 0; q < it.nm; ++q) {
    const ResMember mb = mem[it.m0 + q];
    const double* m = mx + RES_MX * (size_t)(it.m0 + q);
    if (threadIdx.x == 0) {
      double c[10];
      res_member(T, mb.cam, it.lead, m, lc, mode, c);
#pragma unroll
      for (int k = 0; k < 10; ++k) s_mc[k] = c[k];
    }
    __syncthreads();
    const double* A = it.nm > 1 ? m + 7 : nullptr;
    const int nr = it.nm > 1 ? 6 : 9;
    for (int e = mb.begin + threadIdx.x; e < mb.end; e += blockDim.x) {
      const int s = T.slots[e];
      const int l = D.slot_lm[s];
      const double obs[2] = {(double)D.slot_xy[2 * s], (double)D.slot_xy[2 * s + 1]};
      const double X[3] = {(double)D.lms[3 * (size_t)l], (double)D.lms[3 * (size_t)l + 1], (double)D.lms[3 * (size_t)l + 2]};
      double res[2], Jp[18], Jl[6];
      linearize_point<double, true>(obs, X, s_mc, res, Jp, Jl);
      const bool inuse = !(D.obs_W && whiten_observation<double, true>(D.obs_W, s, res, Jp, Jl));
      double R[9];
      quat_to_rot(s_mc, R);
      const double z = R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + s_mc[6];
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
        acc[54] += err;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          double j[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
          res_map_row(Jp + 9 * r, nr, A, j);
          res_add_row(acc, j, res[r], w);
        }
      }
    }
    if (T.cp_L && (int)threadIdx.x == q % (int)blockDim.x) res_camera_prior(D, T, mb.cam, s_mc, A, acc);
    if (T.pp_ptr)
      for (int e = T.pp_ptr[mb.cam] + threadIdx.x; e < T.pp_ptr[mb.cam + 1]; e += blockDim.x)
        res_pair_prior(D, T, it, mem, mx, lc, mode, s_mc, A, T.pp_item[e], acc);
    __syncthreads();  // s_mc is the next member's from here
  }
  lost = __syncthreads_or(lo) != 0;
  res_block_sum(55, sacc, out);
  return out[54];
}

// An observation slot of camera c is a usable point: in use (W != 0), f != 0 and its distortion inverts (section 25); m the
// normalised image point
template <class S>
__device__ __forceinline__ bool res_usable(const DevPtrs<S>& D, int s, const double* c, double& m0, double& m1) {
  if (c[7] == 0.0) return false;
  if (D.obs_W) {
    const S* W = D.obs_W + 4 * (size_t)s;
    if (W[0] == S(0) && W[1] == S(0) && W[2] == S(0) && W[3] == S(0)) return false;
  }
  return tri_undistort((double)D.slot_xy[2 * s] / c[7], (double)D.slot_xy[2 * s + 1] / c[7], c[8], c[9], m0, m1);
}

// (H + lambda diag(d)) x = -g over the free entries by Cholesky on L [81] (shared), d the damping diagonal of section 25;
// false when the damped matrix is not positive definite.  x is 0 on the held entries.  One thread.
__device__ __forceinline__ bool res_solve(const double* h, const double* g, unsigned free, double lambda, double* L, double (&x)[9]) {
  int idx[9], n = 0;
  double dmax = 0.0;
  for (int k = 0; k < 9; ++k)
    if ((free >> k) & 1u) { idx[n++] = k; dmax = fmax(dmax, h[res_hidx(k, k)]); }
  const double fl = TRI_DAMP_FLOOR * dmax;
  for (int a = 0; a < n; ++a)
    for (int b = 0; b <= a; ++b) {
      double v = h[res_hidx(idx[b], idx[a])];
      if (a == b) v += lambda * fmax(v, fl);
      for (int k = 0; k < b; ++k) v -= L[9 * a + k] * L[9 * b + k];
      if (a == b) {
        if (!(v > 0.0)) return false;
        L[9 * a + a] = sqrt(v);
      } else {
        L[9 * a + b] = v / L[9 * b + b];
      }
    }
  double y[9];
  for (int a = 0; a < n; ++a) {
    double v = -g[idx[a]];
    for (int k = 0; k < a; ++k) v -= L[9 * a + k] * y[k];
    y[a] = v / L[9 * a + a];
  }
  for (int a = n - 1; a >= 0; --a) {
    double v = y[a];
    for (int k = a + 1; k < n; ++k) v -= L[9 * k + a] * y[k];
    y[a] = v / L[9 * a + a];
  }
  bool ok = true;
  for (int k = 0; k < 9; ++k) x[k] = 0.0;
  for (int a = 0; a < n; ++a) { x[idx[a]] = y[a]; ok = ok && isfinite(y[a]); }
  return ok;
}

// The lead camera after the increment dx (v, w, df, dk1, dk2) in double: R' = Exp(w) R, t' = Exp(w) t + v (the state's
// left increment), the quaternion normalised.  A zero pose increment (a held pose) keeps the pose bit for bit: the
// normalisation alone could change the last bits of a quaternion that is not exactly unit.
__device__ __forceinline__ void res_apply(const double* c, const double (&dx)[9], double* out) {
  for (int k = 0; k < 3; ++k) out[7 + k] = c[7 + k] + dx[6 + k];
  if (dx[0] == 0.0 && dx[1] == 0.0 && dx[2] == 0.0 && dx[3] == 0.0 && dx[4] == 0.0 && dx[5] == 0.0) {
    for (int k = 0; k < 7; ++k) out[k] = c[k];
    return;
  }
  const double th2 = dx[3] * dx[3] + dx[4] * dx[4] + dx[5] * dx[5];
  double imag, real;
  if (th2 < ST<double>::eps() * ST<double>::eps()) {
    imag = 0.5 - th2 / 48.0;
    real = 1.0 - th2 / 8.0;
  } else {
    const double th = sqrt(th2);
    imag = sin(0.5 * th) / th;
    real = cos(0.5 * th);
  }
  const double qe[7] = {imag * dx[3], imag * dx[4], imag * dx[5], real, 0.0, 0.0, 0.0};
  double p[7];
  pose_mul(qe, c, p);  // Exp(w) T: rotation Exp(w) R, translation Exp(w) t
  const double n = 1.0 / sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2] + p[3] * p[3]);
  for (int k = 0; k < 4; ++k) out[k] = p[k] * n;
  for (int k = 0; k < 3; ++k) out[4 + k] = p[4 + k] + dx[k];
}

template <class S>
__device__ __forceinline__ void res_round(double* c) {
  for (int k = 0; k < 10; ++k) c[k] = (double)(S)c[k];
}

// Block per unit (units in decreasing observation count).  Scratch: mx [members][RES_MX] M_j and A_j of every member
// (written here, first), vb [nslots] bits 1 and 2 = projection validity at the current and at the candidate pose of the
// refinement.  Outputs per unit: status (RBA_RES_* bits), usable points, cost.
template <class S>
__global__ void __launch_bounds__(RES_THREADS) k_resect(DevPtrs<S> D, KOpts o, ResOpts t, ResTerms<S> T,
                                                        const ResItem* __restrict__ items, const ResMember* __restrict__ mem,
                                                        double* __restrict__ mx, uint8_t* __restrict__ vb,
                                                        uint8_t* __restrict__ status_out, int* __restrict__ points_out,
                                                        double* __restrict__ cost_out) {
  __shared__ double sacc[RES_THREADS][RES_ACC];
  __shared__ double s_sum[2][64];           // the normal equations and cost of the current and of the candidate pose
  __shared__ double s_cam[3][10];           // the lead camera: stored, current iterate, candidate
  __shared__ double s_mc[10];
  __shared__ double s_E[144], s_V[144];     // the 12x12 eigenproblem; s_E[0..80] also the Cholesky factor
  __shared__ double s_pose[12];             // the linear estimate of the estimating member: R (9), t (3)
  __shared__ double s_mm[64];               // the distinct entries of the DLT's M
  __shared__ int s_flag;
  const ResItem it = items[blockIdx.x];
  const int tid = threadIdx.x;
  unsigned status = 0;
  // 0. M_j and A_j of every member at the call's start: the identity for the lead, sensor_map for a sensor camera, else the
  //    held M_j of section 23
  for (int q = tid; q < it.nm; q += blockDim.x) {
    const int cam = mem[it.m0 + q].cam;
    double m[7] = {0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0}, A[36];
    if (cam != it.lead) {
      if (T.Z.home && T.Z.home[cam] >= 0) sensor_map(T.snap, T.R, T.Z, cam, m);
      else
        for (int k = 0; k < 7; ++k) m[k] = T.R.M[7 * (size_t)cam + k];
    }
    rig_adjoint(m, A);
    double* out = mx + RES_MX * (size_t)(it.m0 + q);
    for (int k = 0; k < 7; ++k) out[k] = m[k];
    for (int k = 0; k < 36; ++k) out[7 + k] = A[k];
  }
  if (tid == 0)
    for (int k = 0; k < 10; ++k) s_cam[0][k] = (double)T.snap[10 * (size_t)it.lead + k];
  // 1. usable points per member, the estimating member (most points, ties to the lowest index), the validity bits cleared,
  //    and whether the unit carries a camera or pair prior
  int pts = 0, best = -1, nbest = 0;
  for (int q = 0; q < it.nm; ++q) {
    const ResMember mb = mem[it.m0 + q];
    double c[10];
    for (int k = 0; k < 10; ++k) c[k] = (double)T.snap[10 * (size_t)mb.cam + k];
    int cnt = 0;
    for (int b = mb.begin; b < mb.end; b += blockDim.x) {
      bool use = false;
      if (b + tid < mb.end) {
        const int s = T.slots[b + tid];
        vb[s] = 0;
        double m0, m1;
        use = res_usable(D, s, c, m0, m1);
      }
      cnt += __syncthreads_count(use);
    }
    pts += cnt;
    if (cnt > nbest) { nbest = cnt; best = q; }
  }
  bool pri = false;
  for (int q = tid; q < it.nm; q += blockDim.x) {
    const int cam = mem[it.m0 + q].cam;
    if (T.pp_ptr && T.pp_ptr[cam + 1] > T.pp_ptr[cam]) pri = true;
    if (T.cp_L)
      for (int k = 0; k < 81; ++k) pri = pri || T.cp_L[81 * (size_t)cam + k] != S(0);
  }
  pri = __syncthreads_or(pri) != 0;
  const bool pose_free = (it.free & 0x3fu) != 0;
  bool untouched = false;
  if (it.free == 0) { status |= RBA_RES_HELD; untouched = true; }
  else if (pts < RES_MIN_POINTS) { status |= RBA_RES_FEW_POINTS; untouched = !pri; }
  bool changed = false;
  // 2. LINEAR: the DLT of the estimating member on unit rays in normalised world coordinates
  if ((t.mode & RBA_RESECT_LINEAR) && pose_free && !untouched) {
    if (nbest < RES_MIN_LINEAR) {
      status |= RBA_RES_DEGENERATE;
    } else {
      const ResMember mb = mem[it.m0 + best];
      const double* mj = mx + RES_MX * (size_t)(it.m0 + best);
      double c[10];
      for (int k = 0; k < 10; ++k) c[k] = (double)T.snap[10 * (size_t)mb.cam + k];
      // the mean, then the centred scatter of the usable points
      double* sx = sacc[tid];
      res_zero(sx, 3);
      for (int e = mb.begin + tid; e < mb.end; e += blockDim.x) {
        const int s = T.slots[e];
        double m0, m1;
        if (!res_usable(D, s, c, m0, m1)) continue;
        const int l = D.slot_lm[s];
        for (int k = 0; k < 3; ++k) sx[k] += (double)D.lms[3 * (size_t)l + k];
      }
      res_block_sum(3, sacc, s_E);
      const double xb[3] = {s_E[0] / nbest, s_E[1] / nbest, s_E[2] / nbest};
      double* sc = sacc[tid];  // 00 01 02 11 12 22
      res_zero(sc, 6);
      for (int e = mb.begin + tid; e < mb.end; e += blockDim.x) {
        const int s = T.slots[e];
        double m0, m1;
        if (!res_usable(D, s, c, m0, m1)) continue;
        const int l = D.slot_lm[s];
        double d[3];
        for (int k = 0; k < 3; ++k) d[k] = (double)D.lms[3 * (size_t)l + k] - xb[k];
        sc[0] += d[0] * d[0]; sc[1] += d[0] * d[1]; sc[2] += d[0] * d[2];
        sc[3] += d[1] * d[1]; sc[4] += d[1] * d[2]; sc[5] += d[2] * d[2];
      }
      res_block_sum(6, sacc, s_E + 8);
      double sx_s = sqrt((s_E[8] + s_E[11] + s_E[13]) / nbest);
      if (!(sx_s > 0.0)) sx_s = 1.0;
      // M = sum G^T (I - v v^T) G = sum (I - v v^T) (x) X~ X~^T: per block (a <= b) of the 3x3 the 10 entries (i <= j) of
      // c_ab X~ X~^T
      double* mm = sacc[tid];
      res_zero(mm, 60);
      for (int e = mb.begin + tid; e < mb.end; e += blockDim.x) {
        const int s = T.slots[e];
        double m0, m1;
        if (!res_usable(D, s, c, m0, m1)) continue;
        const int l = D.slot_lm[s];
        double xt[4] = {0.0, 0.0, 0.0, 1.0};
        for (int k = 0; k < 3; ++k) xt[k] = ((double)D.lms[3 * (size_t)l + k] - xb[k]) / sx_s;
        const double vn = 1.0 / sqrt(m0 * m0 + m1 * m1 + 1.0);
        const double v[3] = {m0 * vn, m1 * vn, vn};
        int pb = 0;
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int b = a; b < 3; ++b, ++pb) {
            const double cab = (a == b ? 1.0 : 0.0) - v[a] * v[b];
            int k = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
              for (int j = i; j < 4; ++j, ++k) mm[10 * pb + k] += cab * xt[i] * xt[j];
          }
      }
      res_block_sum(60, sacc, s_mm);
      if (tid == 0) {
        s_flag = 0;
        // planarity: the principal variances of the centred points
        double C[9] = {s_E[8], s_E[9], s_E[10], s_E[9], s_E[11], s_E[12], s_E[10], s_E[12], s_E[13]}, CV[9];
        sym_eig<3>(C, CV);
        const double vmin = fmin(C[0], fmin(C[4], C[8])), vmax = fmax(C[0], fmax(C[4], C[8]));
        if (!(vmin >= RES_PLANAR * RES_PLANAR * vmax)) s_flag = 1;
        if (!s_flag) {
          for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) {
              const int lo = a < b ? a : b, hi = a < b ? b : a;
              const int pb = lo * 3 - lo * (lo - 1) / 2 + (hi - lo);
              for (int i = 0; i < 4; ++i)
                for (int j = 0; j < 4; ++j) {
                  const int li = i < j ? i : j, hj = i < j ? j : i;
                  s_E[12 * (4 * a + i) + 4 * b + j] = s_mm[10 * pb + li * 4 - li * (li - 1) / 2 + (hj - li)];
                }
            }
          sym_eig<12>(s_E, s_V);
          int kmin = 0;
          for (int k = 1; k < 12; ++k)
            if (s_E[13 * k] < s_E[13 * kmin]) kmin = k;
          double P[12];
          for (int r = 0; r < 12; ++r) P[r] = s_V[12 * r + kmin];
          double A[9] = {P[0], P[1], P[2], P[4], P[5], P[6], P[8], P[9], P[10]}, b[3] = {P[3], P[7], P[11]};
          double det = A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
          if (det < 0.0) {
            for (int k = 0; k < 9; ++k) A[k] = -A[k];
            for (int k = 0; k < 3; ++k) b[k] = -b[k];
            det = -det;
          }
          double fro = 0.0;
          for (int k = 0; k < 9; ++k) fro += A[k] * A[k];
          fro = sqrt(fro);
          if (!(det > RES_SINGULAR * fro * fro * fro)) {
            s_flag = 1;
          } else {
            // R = A (A^T A)^-1/2, sigma the mean singular value of A
            double G[9], GV[9];
            for (int a = 0; a < 3; ++a)
              for (int bb = 0; bb < 3; ++bb) G[3 * a + bb] = A[a] * A[bb] + A[3 + a] * A[3 + bb] + A[6 + a] * A[6 + bb];
            sym_eig<3>(G, GV);
            const double sv[3] = {sqrt(G[0]), sqrt(G[4]), sqrt(G[8])};
            const double sig = (sv[0] + sv[1] + sv[2]) / 3.0;
            double Gi[9];  // (A^T A)^-1/2 = V diag(1 / sv) V^T
            for (int a = 0; a < 3; ++a)
              for (int bb = 0; bb < 3; ++bb)
                Gi[3 * a + bb] = GV[3 * a] * GV[3 * bb] / sv[0] + GV[3 * a + 1] * GV[3 * bb + 1] / sv[1] + GV[3 * a + 2] * GV[3 * bb + 2] / sv[2];
            for (int a = 0; a < 3; ++a)
              for (int bb = 0; bb < 3; ++bb) s_pose[3 * a + bb] = A[3 * a] * Gi[bb] + A[3 * a + 1] * Gi[3 + bb] + A[3 * a + 2] * Gi[6 + bb];
            for (int a = 0; a < 3; ++a)
              s_pose[9 + a] = sx_s * b[a] / sig - (s_pose[3 * a] * xb[0] + s_pose[3 * a + 1] * xb[1] + s_pose[3 * a + 2] * xb[2]);
            if (!(isfinite(sig) && sig > 0.0)) s_flag = 1;
          }
        }
      }
      __syncthreads();
      if (s_flag) {
        status |= RBA_RES_DEGENERATE;
      } else {
        // BEHIND: more than half of the member's usable points at depth < eps_sqrt of S under the estimate
        int nb = 0;
        for (int b0 = mb.begin; b0 < mb.end; b0 += blockDim.x) {
          bool behind = false;
          if (b0 + tid < mb.end) {
            const int s = T.slots[b0 + tid];
            double m0, m1;
            if (res_usable(D, s, c, m0, m1)) {
              const int l = D.slot_lm[s];
              const double X[3] = {(double)D.lms[3 * (size_t)l], (double)D.lms[3 * (size_t)l + 1], (double)D.lms[3 * (size_t)l + 2]};
              const double z = s_pose[6] * X[0] + s_pose[7] * X[1] + s_pose[8] * X[2] + s_pose[11];
              behind = !(z >= (double)ST<S>::eps_sqrt());
            }
          }
          nb += __syncthreads_count(behind);
        }
        if (2 * nb > nbest) {
          status |= RBA_RES_BEHIND;
        } else {
          if (tid == 0) {  // the lead's pose M_j^-1 T_j, rounded to S
            double tj[7], mi[7], lp[7];
            res_rot_to_quat(s_pose, tj);
            for (int k = 0; k < 3; ++k) tj[4 + k] = s_pose[9 + k];
            pose_inv(mj, mi);
            pose_mul(mi, tj, lp);
            const double n = 1.0 / sqrt(lp[0] * lp[0] + lp[1] * lp[1] + lp[2] * lp[2] + lp[3] * lp[3]);
            for (int k = 0; k < 4; ++k) s_cam[0][k] = lp[k] * n;
            for (int k = 0; k < 3; ++k) s_cam[0][4 + k] = lp[4 + k];
            res_round<S>(s_cam[0]);
          }
          changed = true;
        }
      }
    }
    __syncthreads();
  }
  // 3. REFINE: Levenberg-Marquardt on the unit's own cost, landmarks held
  bool lost;
  int cur = 1;  // the bit of vb[s] holding the validity at the current pose
  __syncthreads();
  double cost = res_eval(D, o, T, it, mem, mx, s_cam[0], changed ? 1 : 0, vb, cur, cur, s_mc, sacc, s_sum[0], lost);
  if ((t.mode & RBA_RESECT_REFINE) && !untouched) {
    const double c_start = cost;
    double* hc = s_sum[0];
    double* hn = s_sum[1];
    double* xc = s_cam[1];
    double* xn = s_cam[2];
    if (tid == 0)
      for (int k = 0; k < 10; ++k) xc[k] = s_cam[0][k];
    double lambda = TRI_LAMBDA0;
    int accepted = 0;
    bool conv = false;
    for (int k = 0; k < t.max_iterations && lambda <= TRI_LAMBDA_MAX; ++k) {
      __syncthreads();  // the last iteration's shared state is complete and read
      bool gz = true;
      for (int j = 0; j < 9; ++j)
        if (((it.free >> j) & 1u) && hc[45 + j] != 0.0) gz = false;
      if (gz) { conv = true; break; }
      if (tid == 0) {
        double dx[9];
        s_flag = res_solve(hc, hc + 45, it.free, lambda, s_E, dx);
        if (s_flag) res_apply(xc, dx, xn);
      }
      __syncthreads();
      if (!s_flag) { lambda *= 10.0; continue; }
      const int nxt = 3 - cur;
      const double cn = res_eval(D, o, T, it, mem, mx, xn, 2, vb, nxt, cur, s_mc, sacc, hn, lost);
      if (cn < cost && !lost) {
        conv = cost - cn <= t.ftol * cost;
        cost = cn; cur = nxt; ++accepted;
        double* sw = hc; hc = hn; hn = sw;
        sw = xc; xc = xn; xn = sw;
        lambda = fmax(lambda * 0.1, TRI_LAMBDA_MIN);
        if (conv) break;
      } else {
        if (!lost && cn - cost <= t.ftol * cost) { conv = true; break; }  // no change the tolerance can tell apart
        lambda *= 10.0;
      }
    }
    if (conv) status |= RBA_RES_CONVERGED;
    if (accepted > 0) {
      __syncthreads();
      if (tid == 0) res_round<S>(xc);
      __syncthreads();
      const double cr = res_eval(D, o, T, it, mem, mx, xc, 1, vb, cur, cur, s_mc, sacc, hn, lost);
      if (cr < c_start) {
        if (tid == 0)
          for (int k = 0; k < 10; ++k) s_cam[0][k] = xc[k];
        cost = cr;
        changed = true;
        status |= RBA_RES_REFINED;
      } else {
        cost = c_start;
      }
    }
  }
  if (changed) status |= RBA_RES_WRITTEN;
  __syncthreads();
  if (tid == 0) {
    if (changed) {  // the lead, then every other member M_j T_lead from the stored lead
      S* cl = D.cams + 10 * (size_t)it.lead;
      for (int k = 0; k < 10; ++k) cl[k] = (S)s_cam[0][k];
      for (int q = 0; q < it.nm; ++q) {
        const int cam = mem[it.m0 + q].cam;
        if (cam != it.lead) retie_pose(D.cams, cam, it.lead, mx + RES_MX * (size_t)(it.m0 + q));
      }
    }
    status_out[blockIdx.x] = (uint8_t)status;
    points_out[blockIdx.x] = pts;
    cost_out[blockIdx.x] = cost;
  }
}

}  // namespace rba
