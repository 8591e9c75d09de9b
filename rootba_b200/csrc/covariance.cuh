// Marginal covariances of the cameras and landmarks (rba_compute_covariance, DESIGN.md section 16).
//
// Everything here is float64, also for a float32 handle (the state, observations and prior arrays are widened).  The
// pipeline, on the solver stream:
//   1. k_cov_landmark     per landmark: weighted Jp, Jl; Hll = Jl^T Jl = V Lambda V^T; K_i = Lambda+^-1/2 V+^T Jl_i^T Jp_i
//   2. k_cov_assemble     lower triangle of the reduced camera matrix S = sum_l (delta_ij Jp_i^T Jp_i - K_i^T K_j), one
//                         warp per co-visible camera pair over a host-built term list (fixed order, no atomics)
//      k_cov_priors       + the absolute and pair priors' blocks, re-evaluated in double in the unscaled space
//      k_cov_diag/_equil  held rows and columns -> identity, equilibration D S D with D = diag(S)^-1/2, padding -> identity
//   3. dense SPD inverse in place: blocked potrf, trtri, lauum (LAPACK's potri) with the diagonal-tile kernels and one
//      FP64 tensor-core GEMM (mma.sync m8n8k4 .f64) for every O(N^3) update
//   4. cov_sinv           entry of D S^-1 D;  cov_lm_block  landmark pair W_l (delta_lm I + sum_ab K_a S^-1_ab K_b^T) W_m^T,
//                         W = V Lambda^-1/2
//   5. (DESIGN.md section 20) k_cov_cam_cross, k_cov_cam_lm, k_cov_lm_cross, k_cov_rel_pose: the blocks of chosen camera
//                         pairs, camera-landmark pairs, landmark pairs and relative poses.  The marginals cam_cov and lm_cov
//                         are the diagonal requests (k, k) of k_cov_cam_cross and k_cov_lm_cross
// The dense matrix is column-major with a leading dimension padded to a multiple of COV_TB; only its lower triangle is
// meaningful.
#pragma once

#include "kernels.cuh"

namespace rba {

constexpr int COV_TB = 64;               // diagonal tile of the blocked factorisation = GEMM block tile
constexpr int COV_BK = 16;               // k slice of the GEMM held in shared memory
constexpr int COV_LDS = COV_TB + 4;      // shared row stride: = 4 (mod 16) doubles, conflict-free fragment loads
constexpr double COV_EIG_DROP = 1e-10;   // eigenvalues of Hll <= this * lambda_max are dropped (pseudo-inverse)
constexpr double COV_PIVOT_TAU = 1e-10;  // a Cholesky pivot <= this of the equilibrated reduced matrix: singular (no gauge)

// ------------------------------------------------------------------------------------------------
// 1. per-landmark elimination
// ------------------------------------------------------------------------------------------------
// symmetric NxN eigendecomposition by cyclic Jacobi rotations, pairs (p, q) in row order: on return A holds the eigenvalues
// on its diagonal and the columns of V (row-major) the eigenvectors.  Fixed number of sweeps: the same operations on every
// run.  N = 3: the landmark blocks here; N = 4: the homogeneous triangulation (triangulate.cuh).
template <int N>
__device__ __forceinline__ void sym_eig(double (&A)[N * N], double (&V)[N * N]) {
#pragma unroll
  for (int k = 0; k < N * N; ++k) V[k] = (k % (N + 1) == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 8; ++sweep) {
#pragma unroll
    for (int p = 0; p < N - 1; ++p) {
#pragma unroll
      for (int q = p + 1; q < N; ++q) {
        const double apq = A[N * p + q];
        if (apq == 0.0) continue;
        const double th = (A[N * q + q] - A[N * p + p]) / (2.0 * apq);
        const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
        for (int k = 0; k < N; ++k) {  // columns p, q
          const double akp = A[N * k + p], akq = A[N * k + q];
          A[N * k + p] = c * akp - s * akq;
          A[N * k + q] = s * akp + c * akq;
        }
#pragma unroll
        for (int k = 0; k < N; ++k) {  // rows p, q
          const double apk = A[N * p + k], aqk = A[N * q + k];
          A[N * p + k] = c * apk - s * aqk;
          A[N * q + k] = s * apk + c * aqk;
        }
#pragma unroll
        for (int k = 0; k < N; ++k) {
          const double vkp = V[N * k + p], vkq = V[N * k + q];
          V[N * k + p] = c * vkp - s * vkq;
          V[N * k + q] = s * vkp + c * vkq;
        }
      }
    }
  }
}

// Landmark prior lp of this shard at the position pw, in double from the unweighted L (D.lmp_Lu): r = L (pw - x0), returns
// s = |r|^2.  lmp_loss gives err = rho(s)/2 and w = rho'(s) of its loss record (only while D.lmp_loss is set).
template <class S>
__device__ __forceinline__ double lmp_residual(const DevPtrs<S>& D, int lp, const double* pw, double (&r)[3]) {
  const S* Lp = D.lmp_Lu + 9 * (size_t)lp;
  const double e[3] = {pw[0] - (double)D.lmp_mean[3 * lp], pw[1] - (double)D.lmp_mean[3 * lp + 1], pw[2] - (double)D.lmp_mean[3 * lp + 2]};
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double v = (double)Lp[3 * i] * e[0] + (double)Lp[3 * i + 1] * e[1] + (double)Lp[3 * i + 2] * e[2];
    r[i] = v;
    s += v * v;
  }
  return s;
}
template <class S>
__device__ __forceinline__ void lmp_loss(const DevPtrs<S>& D, int lp, double s, double& err, double& w) {
  unsigned kind;
  S a;
  slot_loss(D.lmp_loss, D.lmp_n, (size_t)lp, kind, a);
  observation_loss<double>(kind, (double)a, s, err, w);
}

// Warp per landmark (problem order).  Re-linearises every observation in double with the weights and validity rule of
// rba_linearize (unscaled), then writes per slot jpw [18] = sqrt(w) Jp and kb [27] = K (3x9 row-major, rows of dropped
// eigenvalues zero), and per landmark wl [9] = V Lambda^-1/2 (row-major; columns of dropped eigenvalues zero) and its rank.
// LMP (landmark priors, DESIGN.md section 17): Hll += L^T L (unscaled, in double) for a landmark with prior slot
// lmp_of_lm[lm] >= 0, so a landmark with fewer than 2 valid observations can be full rank.
// OBSW (observation information, DESIGN.md section 19): the rows are whitened in double, sqrt(w) W [Jp | Jl], w from |W r|^2.
// OBSL (observation losses, DESIGN.md section 21): w from the slot's own loss, evaluated in double.
// LMPL (losses on the landmark priors, DESIGN.md section 22; implies LMP): Hll += w L^T L, with the unweighted L (D.lmp_Lu)
// and w of the prior's loss on |L (x - x0)|^2, evaluated in double at the current state.
template <class S, bool LMP = false, bool OBSW = false, bool OBSL = false, bool LMPL = false>
__global__ void __launch_bounds__(128) k_cov_landmark(DevPtrs<S> D, KOpts o, const int* __restrict__ lm_slot0,
                                                      const int* __restrict__ lm_n, int nl, double* __restrict__ jpw,
                                                      double* __restrict__ kb, double* __restrict__ wl, int* __restrict__ rank,
                                                      const int* __restrict__ lmp_of_lm = nullptr) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int lm = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); lm < nl; lm += warps) {
    const int s0 = lm_slot0[lm], n = lm_n[lm];
    const double pw[3] = {(double)D.lms[3 * lm], (double)D.lms[3 * lm + 1], (double)D.lms[3 * lm + 2]};
    double h[6] = {0, 0, 0, 0, 0, 0};  // Hll: 00 01 02 11 12 22
    for (int i = lane; i < n; i += 32) {
      const int s = s0 + i;
      const double obs[2] = {(double)D.slot_xy[2 * s], (double)D.slot_xy[2 * s + 1]};
      double cam[10];
      const S* cp = D.cams + 10 * (size_t)D.slot_cam[s];
#pragma unroll
      for (int k = 0; k < 10; ++k) cam[k] = (double)cp[k];
      double res[2], Jp[18], Jl[6];
      linearize_point<double, true>(obs, pw, cam, res, Jp, Jl);
      bool keep = true;
      if constexpr (OBSW) keep = !whiten_observation<double, true>(D.obs_W, s, res, Jp, Jl);
      if (keep && o.use_valid_projections_only) {  // the handle's own validity threshold (that of its Scalar)
        double R[9];
        quat_to_rot(cam, R);
        const double z = R[6] * pw[0] + R[7] * pw[1] + R[8] * pw[2] + cam[6];
        keep = z >= (double)ST<S>::eps_sqrt();
      }
      double sw = 0.0;
      if (keep) {
        double err, w;
        slot_error_weight<OBSL>(o, D.obs_loss, D.nslots, s, res[0] * res[0] + res[1] * res[1], err, w);
        sw = sqrt(w);
      }
#pragma unroll
      for (int k = 0; k < 18; ++k) jpw[18 * (size_t)s + k] = sw * Jp[k];
#pragma unroll
      for (int k = 0; k < 6; ++k) { Jl[k] *= sw; kb[27 * (size_t)s + k] = Jl[k]; }  // Jl parked in kb until K replaces it
      h[0] += Jl[0] * Jl[0] + Jl[3] * Jl[3];
      h[1] += Jl[0] * Jl[1] + Jl[3] * Jl[4];
      h[2] += Jl[0] * Jl[2] + Jl[3] * Jl[5];
      h[3] += Jl[1] * Jl[1] + Jl[4] * Jl[4];
      h[4] += Jl[1] * Jl[2] + Jl[4] * Jl[5];
      h[5] += Jl[2] * Jl[2] + Jl[5] * Jl[5];
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) h[k] = warp_sum(h[k]);  // butterfly: the same sum in every lane
    if constexpr (LMP) {
      const int lp = lmp_of_lm[lm];
      if (lp >= 0) {
        const S* Lp = (LMPL ? D.lmp_Lu : D.lmp_L) + 9 * (size_t)lp;
        double sw = 1.0;
        if constexpr (LMPL) {
          double rp[3], err, w;
          lmp_loss(D, lp, lmp_residual(D, lp, pw, rp), err, w);
          sw = sqrt(w);
        }
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          double a0 = (double)Lp[3 * r], a1 = (double)Lp[3 * r + 1], a2 = (double)Lp[3 * r + 2];
          if constexpr (LMPL) { a0 *= sw; a1 *= sw; a2 *= sw; }  // the row of sqrt(w) L
          h[0] += a0 * a0; h[1] += a0 * a1; h[2] += a0 * a2; h[3] += a1 * a1; h[4] += a1 * a2; h[5] += a2 * a2;
        }
      }
    }
    double A[9] = {h[0], h[1], h[2], h[1], h[3], h[4], h[2], h[4], h[5]}, V[9];
    sym_eig<3>(A, V);
    const double lmax = fmax(A[0], fmax(A[4], A[8]));
    double W[9];
    int r = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double ev = A[4 * k];
      const bool kept = lmax > 0.0 && ev > COV_EIG_DROP * lmax;
      r += kept ? 1 : 0;
      const double f = kept ? 1.0 / sqrt(ev) : 0.0;
#pragma unroll
      for (int row = 0; row < 3; ++row) W[3 * row + k] = V[3 * row + k] * f;
    }
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < 9; ++k) wl[9 * (size_t)lm + k] = W[k];
      rank[lm] = r;
    }
    for (int i = lane; i < n; i += 32) {
      const int s = s0 + i;
      double Jl[6], Jp[18];
#pragma unroll
      for (int k = 0; k < 6; ++k) Jl[k] = kb[27 * (size_t)s + k];
#pragma unroll
      for (int k = 0; k < 18; ++k) Jp[k] = jpw[18 * (size_t)s + k];
      // K = W^T (Jl^T Jp)
#pragma unroll
      for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int c = 0; c < 9; ++c) {
          double v = 0.0;
#pragma unroll
          for (int a = 0; a < 3; ++a) v += W[3 * a + k] * (Jl[a] * Jp[c] + Jl[3 + a] * Jp[9 + c]);
          kb[27 * (size_t)s + 9 * k + c] = v;
        }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// 2. assembly of the reduced camera matrix (unscaled), priors, held parameters, equilibration
// ------------------------------------------------------------------------------------------------
// Warp per co-visible camera pair (ca >= cb): block(ca, cb) = sum over its terms (sa, sb) of
// [sa == sb] Jp_sa^T Jp_sa - K_sa^T K_sb, in the term order of the list.  Writes the lower triangle only.
__global__ void __launch_bounds__(256) k_cov_assemble(const int2* __restrict__ blk_cam, const int* __restrict__ blk_ptr,
                                                      const int2* __restrict__ terms, int nblk, const double* __restrict__ jpw,
                                                      const double* __restrict__ kb, double* __restrict__ A, long long ld) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int bi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); bi < nblk; bi += warps) {
    const int2 cc = blk_cam[bi];
    const int t0 = blk_ptr[bi], t1 = blk_ptr[bi + 1];
#pragma unroll
    for (int u = 0; u < 3; ++u) {
      const int e = lane + 32 * u, p = e / 9, q = e % 9;
      if (e >= 81 || (cc.x == cc.y && p < q)) continue;
      double acc = 0.0;
      for (int t = t0; t < t1; ++t) {
        const int2 st = terms[t];
        const double* ka = kb + 27 * (size_t)st.x;
        const double* kq = kb + 27 * (size_t)st.y;
        double v = 0.0;
        if (st.x == st.y) {
          const double* j = jpw + 18 * (size_t)st.x;
          v = j[p] * j[q] + j[9 + p] * j[9 + q];
        }
        v -= ka[p] * kq[q] + ka[9 + p] * kq[9 + q] + ka[18 + p] * kq[18 + q];
        acc += v;
      }
      A[(9 * (long long)cc.x + p) + (9 * (long long)cc.y + q) * ld] = acc;
    }
  }
}

// Thread per camera c: adds to its block row (lower triangle) the absolute prior's A^T A and, over its incident pair sides
// in list order, the pair blocks A_s^T A_s (diagonal) and A_s^T A_o (to the column block of the other camera o < c).
// The rows are those of k_prior_linearize / k_pair_linearize (prior_jac_row, pair_jac_rows), unscaled, evaluated in double
// from the stored means and L.
// LOSS (losses on the priors, DESIGN.md section 22): the rows of a prior with a loss record (ploss over the nc cameras,
// qloss over the nq pairs; nullptr = every prior of that kind NONE) are those of sqrt(w) L, w of its loss on |L e|^2,
// evaluated in double at the current state from the unweighted L.
template <int NR, class S>
__device__ __forceinline__ double cov_prior_sqrt_weight(const S* __restrict__ loss, int n, int p, const S* __restrict__ Lp,
                                                        const double* e) {
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < NR; ++i) {
    double v = 0.0;
#pragma unroll
    for (int k = 0; k < NR; ++k) v += (double)Lp[NR * i + k] * e[k];
    s += v * v;
  }
  unsigned kind;
  S a;
  slot_loss(loss, n, (size_t)p, kind, a);
  double err, w;
  observation_loss<double>(kind, (double)a, s, err, w);
  return sqrt(w);
}
template <class S, bool LOSS = false>
__global__ void k_cov_priors(const S* __restrict__ cams, int nc, const S* __restrict__ pmean, const S* __restrict__ pL,
                             const int* __restrict__ pairs, const S* __restrict__ qmean, const S* __restrict__ qL,
                             const int* __restrict__ qptr, const int* __restrict__ qitem, const int* __restrict__ qnbr,
                             double* __restrict__ A, long long ld, const S* __restrict__ ploss = nullptr,
                             const S* __restrict__ qloss = nullptr, int nq = 0) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nc) return;
  double* Acc = A + 9 * (long long)c + 9 * (long long)c * ld;  // diagonal block (c, c)
  if (pmean) {
    double cam[10], mean[10], e[9], Jinv[9], R[9];
#pragma unroll
    for (int k = 0; k < 10; ++k) { cam[k] = (double)cams[10 * (size_t)c + k]; mean[k] = (double)pmean[10 * (size_t)c + k]; }
    prior_residual<double, true>(cam, mean, e, Jinv, R);
    double sw = 1.0;
    if constexpr (LOSS) {
      if (ploss) sw = cov_prior_sqrt_weight<9>(ploss, nc, c, pL + 81 * (size_t)c, e);
    }
    for (int i = 0; i < 9; ++i) {
      double l[9], row[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) l[k] = (double)pL[81 * (size_t)c + 9 * i + k];
      if constexpr (LOSS) {
#pragma unroll
        for (int k = 0; k < 9; ++k) l[k] *= sw;
      }
      prior_jac_row(l, R, Jinv, row);
      for (int a = 0; a < 9; ++a)
        for (int b = 0; b <= a; ++b) Acc[a + b * ld] += row[a] * row[b];
    }
  }
  if (qptr) {
    for (int q = qptr[c]; q < qptr[c + 1]; ++q) {
      const int it = qitem[q], p = it >> 1, side = it & 1, o = qnbr[q];
      double ci[10], cj[10], mean[7], e[6], M[9], tr[3], Jinv[9], JM[9];
#pragma unroll
      for (int k = 0; k < 10; ++k) {
        ci[k] = (double)cams[10 * (size_t)pairs[2 * p] + k];
        cj[k] = (double)cams[10 * (size_t)pairs[2 * p + 1] + k];
      }
#pragma unroll
      for (int k = 0; k < 7; ++k) mean[k] = (double)qmean[7 * (size_t)p + k];
      pair_residual<double, true>(ci, cj, mean, e, M, tr, Jinv, JM);
      double* Aco = A + 9 * (long long)c + 9 * (long long)o * ld;  // block (c, o), used when o < c
      double sw = 1.0;
      if constexpr (LOSS) {
        if (qloss) sw = cov_prior_sqrt_weight<6>(qloss, nq, p, qL + 36 * (size_t)p, e);
      }
      for (int i = 0; i < 6; ++i) {
        double l[6], ri[6], rj[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) l[k] = (double)qL[36 * (size_t)p + 6 * i + k];
        if constexpr (LOSS) {
#pragma unroll
          for (int k = 0; k < 6; ++k) l[k] *= sw;
        }
        pair_jac_rows(l, M, tr, Jinv, JM, ri, rj);
        const double* own = side ? rj : ri;
        const double* oth = side ? ri : rj;
        for (int a = 0; a < 6; ++a) {
          for (int b = 0; b <= a; ++b) Acc[a + b * ld] += own[a] * own[b];
          if (o < c)
            for (int b = 0; b < 6; ++b) Aco[a + b * ld] += own[a] * oth[b];
        }
      }
    }
  }
}

__device__ __forceinline__ bool cov_fixed(const uint8_t* __restrict__ cam_fixed, long long k) {
  return cam_fixed && ((fixed_entry_mask(cam_fixed[k / 9]) >> (k % 9)) & 1u);
}

// d [np] = diag(S)^-1/2 (1 for held entries, the padding and a non-positive diagonal).  Thread per entry.
__global__ void k_cov_diag(const double* __restrict__ A, long long ld, long long n, long long np,
                           const uint8_t* __restrict__ cam_fixed, double* __restrict__ d) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k >= np) return;
  double v = 1.0;
  if (k < n && !cov_fixed(cam_fixed, k)) {
    const double s = A[k + k * ld];
    if (s > 0.0) v = 1.0 / sqrt(s);
  }
  d[k] = v;
}

// S <- D S D on the lower triangle; rows and columns of held entries and of the padding -> identity; upper triangle -> 0.
// Thread per entry of a 32 x 8 patch, grid over the np x np matrix.
__global__ void k_cov_equil(double* __restrict__ A, long long ld, long long n, long long np, const uint8_t* __restrict__ cam_fixed,
                            const double* __restrict__ d) {
  const long long r = blockIdx.x * 32LL + threadIdx.x;
  const long long c = blockIdx.y * 8LL + threadIdx.y;
  if (r >= np || c >= np) return;
  double& a = A[r + c * ld];
  if (r < c) { a = 0.0; return; }
  if (r >= n || c >= n || cov_fixed(cam_fixed, r) || cov_fixed(cam_fixed, c)) { a = r == c ? 1.0 : 0.0; return; }
  a = a * d[r] * d[c];
}

// ------------------------------------------------------------------------------------------------
// 3. dense SPD inverse: diagonal-tile kernels (one CTA per COV_TB x COV_TB tile, in shared memory) and the DMMA GEMM
// ------------------------------------------------------------------------------------------------
// Cholesky of the lower triangle of tile (k0, k0), in place; upper part of the tile -> 0.  A pivot <= tau (or NaN) stores
// the smallest such global index in *fail.
__global__ void __launch_bounds__(256) k_cov_tile_potrf(double* __restrict__ A, long long ld, long long k0, double tau,
                                                        int* __restrict__ fail) {
  __shared__ double T[COV_TB][COV_TB + 1];
  const int tid = threadIdx.x;
  for (int e = tid; e < COV_TB * COV_TB; e += blockDim.x) T[e % COV_TB][e / COV_TB] = A[(k0 + e % COV_TB) + (k0 + e / COV_TB) * ld];
  __syncthreads();
  for (int j = 0; j < COV_TB; ++j) {
    const double piv = T[j][j];
    const double ljj = sqrt(piv);
    if (tid == 0 && !(piv > tau)) atomicMin(fail, (int)(k0 + j));
    __syncthreads();
    if (tid == 0) T[j][j] = ljj;
    for (int r = j + 1 + tid; r < COV_TB; r += blockDim.x) T[r][j] /= ljj;
    __syncthreads();
    const int m = COV_TB - 1 - j;
    for (int e = tid; e < m * m; e += blockDim.x) {
      const int r = j + 1 + e % m, c = j + 1 + e / m;
      if (c <= r) T[r][c] -= T[r][j] * T[c][j];
    }
    __syncthreads();
  }
  for (int e = tid; e < COV_TB * COV_TB; e += blockDim.x) {
    const int r = e % COV_TB, c = e / COV_TB;
    A[(k0 + r) + (k0 + c) * ld] = r >= c ? T[r][c] : 0.0;
  }
}

// Inverse of the lower-triangular tile (k0, k0) of A -> out (ldo), upper part 0.  Thread per column, forward substitution;
// a thread reads back only the column it writes.
__global__ void __launch_bounds__(COV_TB) k_cov_tile_trtri(const double* __restrict__ A, long long ld, long long k0,
                                                           double* __restrict__ out, long long ldo) {
  __shared__ double T[COV_TB][COV_TB + 1];
  const int j = threadIdx.x;
  for (int r = 0; r < COV_TB; ++r) T[r][j] = A[(k0 + r) + (k0 + j) * ld];
  __syncthreads();
  double* X = out + j * ldo;
  for (int i = 0; i < COV_TB; ++i) {
    double v = i == j ? 1.0 : 0.0;
    for (int k = j; k < i; ++k) v -= T[i][k] * X[k];
    X[i] = i >= j ? v / T[i][i] : 0.0;
  }
}

// Tile (k0, k0) <- L^T L of its lower triangle L (LAPACK lauu2), lower triangle written, upper part 0.
__global__ void __launch_bounds__(256) k_cov_tile_lauu2(double* __restrict__ A, long long ld, long long k0) {
  __shared__ double T[COV_TB][COV_TB + 1];
  const int tid = threadIdx.x;
  for (int e = tid; e < COV_TB * COV_TB; e += blockDim.x) {
    const int r = e % COV_TB, c = e / COV_TB;
    T[r][c] = r >= c ? A[(k0 + r) + (k0 + c) * ld] : 0.0;
  }
  __syncthreads();
  double out[COV_TB * COV_TB / 256];
#pragma unroll
  for (int u = 0; u < COV_TB * COV_TB / 256; ++u) {
    const int e = tid + 256 * u, r = e % COV_TB, c = e / COV_TB;
    double v = 0.0;
    if (r >= c)
      for (int k = r; k < COV_TB; ++k) v += T[k][r] * T[k][c];
    out[u] = v;
  }
#pragma unroll
  for (int u = 0; u < COV_TB * COV_TB / 256; ++u) {
    const int e = tid + 256 * u;
    A[(k0 + e % COV_TB) + (k0 + e / COV_TB) * ld] = out[u];
  }
}

__device__ __forceinline__ void dmma_8x8x4(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// C = alpha op(A) op(B) + beta C for column-major operands whose M, N, K are multiples of COV_TB; op(A)(i, k) = A(k, i) when
// TA, op(B)(k, j) = B(j, k) when TB.  beta == 0 does not read C.  lower: only the tiles with row tile >= column tile.
// ktri: op(A) is lower triangular by tiles (the k range of row tile i ends at (i + 1) COV_TB).
// 256 threads = 8 warps as 2 (rows) x 4 (columns), a warp computes 32 x 16 of the 64 x 64 tile with 4 x 2 DMMA 8x8x4
// fragments per k4 step; the next k slice is loaded into registers while the current one is multiplied.
template <bool TA, bool TB>
__global__ void __launch_bounds__(256) k_cov_dgemm(int M, int N, int K, double alpha, const double* __restrict__ A, long long lda,
                                                   const double* __restrict__ B, long long ldb, double beta, double* __restrict__ C,
                                                   long long ldc, int lower, int ktri) {
  const int ti = blockIdx.x, tj = blockIdx.y;
  if (lower && tj > ti) return;
  __shared__ double As[COV_BK][COV_LDS];
  __shared__ double Bs[COV_BK][COV_LDS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gid = lane >> 2, tig = lane & 3;
  const int wm = warp >> 2, wn = warp & 3;
  const long long i0 = (long long)ti * COV_TB, j0 = (long long)tj * COV_TB;
  const int kend = ktri ? min(K, (ti + 1) * COV_TB) : K;
  constexpr int LD = COV_TB * COV_BK / 256;  // elements of each operand a thread loads per k slice
  double ra[LD], rb[LD];
  auto load = [&](int kt) {
#pragma unroll
    for (int u = 0; u < LD; ++u) {
      const int e = tid + 256 * u;
      if (!TA) ra[u] = A[(i0 + e % COV_TB) + (long long)(kt + e / COV_TB) * lda];
      else ra[u] = A[(long long)(kt + e % COV_BK) + (i0 + e / COV_BK) * lda];
      if (!TB) rb[u] = B[(long long)(kt + e % COV_BK) + (j0 + e / COV_BK) * ldb];
      else rb[u] = B[(j0 + e % COV_TB) + (long long)(kt + e / COV_TB) * ldb];
    }
  };
  auto stash = [&]() {
#pragma unroll
    for (int u = 0; u < LD; ++u) {
      const int e = tid + 256 * u;
      if (!TA) As[e / COV_TB][e % COV_TB] = ra[u];
      else As[e % COV_BK][e / COV_BK] = ra[u];
      if (!TB) Bs[e % COV_BK][e / COV_BK] = rb[u];
      else Bs[e / COV_TB][e % COV_TB] = rb[u];
    }
  };
  double acc[4][2][2];
#pragma unroll
  for (int mi = 0; mi < 4; ++mi)
#pragma unroll
    for (int ni = 0; ni < 2; ++ni) acc[mi][ni][0] = acc[mi][ni][1] = 0.0;
  if (kend > 0) load(0);
  for (int kt = 0; kt < kend; kt += COV_BK) {
    __syncthreads();
    stash();
    __syncthreads();
    if (kt + COV_BK < kend) load(kt + COV_BK);
#pragma unroll
    for (int ks = 0; ks < COV_BK / 4; ++ks) {
      double a[4], b[2];
#pragma unroll
      for (int mi = 0; mi < 4; ++mi) a[mi] = As[4 * ks + tig][32 * wm + 8 * mi + gid];
#pragma unroll
      for (int ni = 0; ni < 2; ++ni) b[ni] = Bs[4 * ks + tig][16 * wn + 8 * ni + gid];
#pragma unroll
      for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 2; ++ni) dmma_8x8x4(acc[mi][ni][0], acc[mi][ni][1], a[mi], b[ni]);
    }
  }
#pragma unroll
  for (int mi = 0; mi < 4; ++mi)
#pragma unroll
    for (int ni = 0; ni < 2; ++ni)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long r = i0 + 32 * wm + 8 * mi + gid, c = j0 + 16 * wn + 8 * ni + 2 * tig + h;
        double& out = C[r + c * ldc];
        out = beta == 0.0 ? alpha * acc[mi][ni][h] : alpha * acc[mi][ni][h] + beta * out;
      }
}

// ------------------------------------------------------------------------------------------------
// 4. extraction
// ------------------------------------------------------------------------------------------------
// entry (r, c) of D S_eq^-1 D from the lower triangle; 0 in the rows and columns of held entries
__device__ __forceinline__ double cov_sinv(const double* __restrict__ A, long long ld, const double* __restrict__ d,
                                           const uint8_t* __restrict__ cam_fixed, long long r, long long c) {
  if (cov_fixed(cam_fixed, r) || cov_fixed(cam_fixed, c)) return 0.0;
  const double v = r >= c ? A[r + c * ld] : A[c + r * ld];
  return v * d[r] * d[c];
}

// One warp: the 3x3 block W_l (delta_lm I + sum_ab K_a Sigma_ab K_b^T) W_m^T of landmarks l and m (a over the slots of l,
// b over those of m), lanes over the n_l n_m slot pairs, fixed-order butterfly sum, written by lane 0 to out [9]; all NaN
// when the Hll of either has rank < 3.  With l == m it is the marginal W (I + sum_ab K_a Sigma_ab K_b^T) W^T over the n^2
// camera pairs of the landmark's track.
__device__ __forceinline__ void cov_lm_block(const double* __restrict__ A, long long ld, const double* __restrict__ d,
                                             const uint8_t* __restrict__ cam_fixed, const int* __restrict__ slot_cam,
                                             const int* __restrict__ lm_slot0, const int* __restrict__ lm_n,
                                             const double* __restrict__ kb, const double* __restrict__ wl,
                                             const int* __restrict__ rank, int l, int m, int lane, double* __restrict__ out) {
  if (rank[l] < 3 || rank[m] < 3) {
    if (lane < 9) out[lane] = __longlong_as_double(0x7ff8000000000000LL);
    return;
  }
  const int s0 = lm_slot0[l], n = lm_n[l], s1 = lm_slot0[m], nm = lm_n[m];
  double acc[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) acc[k] = 0.0;
  for (int t = lane; t < n * nm; t += 32) {
    const int a = t / nm, b = t % nm;
    const long long ra = 9LL * slot_cam[s0 + a], rb = 9LL * slot_cam[s1 + b];
    const double* ka = kb + 27 * (size_t)(s0 + a);
    const double* kq = kb + 27 * (size_t)(s1 + b);
    for (int p = 0; p < 9; ++p) {
      double u[3] = {0.0, 0.0, 0.0};  // (Sigma_ab K_b^T) row p
      for (int q = 0; q < 9; ++q) {
        const double sv = cov_sinv(A, ld, d, cam_fixed, ra + p, rb + q);
#pragma unroll
        for (int j = 0; j < 3; ++j) u[j] += sv * kq[9 * j + q];
      }
#pragma unroll
      for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int j = 0; j < 3; ++j) acc[3 * k + j] += ka[9 * k + p] * u[j];
    }
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) acc[k] = warp_sum(acc[k]);
  if (lane == 0) {
    const double* Wl = wl + 9 * (size_t)l;
    const double* Wm = wl + 9 * (size_t)m;
    const double diag = l == m ? 1.0 : 0.0;
    double X[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) X[k] = acc[k] + (k % 4 == 0 ? diag : 0.0);
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        double v = 0.0;
        for (int k = 0; k < 3; ++k)
          for (int j = 0; j < 3; ++j) v += Wl[3 * r + k] * X[3 * k + j] * Wm[3 * c + j];
        out[3 * r + c] = v;
      }
  }
}

// ------------------------------------------------------------------------------------------------
// 5. covariance blocks of chosen pairs (DESIGN.md section 20).  Grid-stride loops over the requests, fixed-order sums, no
//    atomics: the same output on every run, and request k depends on request k alone.
// ------------------------------------------------------------------------------------------------
// camera_cross [m][81] = Cov(d_a, d_b) of the requests (a, b), thread per entry.  req == nullptr: request k is (k, k), the
// marginals cam_cov.
__global__ void __launch_bounds__(256) k_cov_cam_cross(const double* __restrict__ A, long long ld, const double* __restrict__ d,
                                                       const uint8_t* __restrict__ cam_fixed, const int2* __restrict__ req, int m,
                                                       double* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < 81LL * m; e += stride) {
    const int2 ab = req ? req[e / 81] : make_int2((int)(e / 81), (int)(e / 81));
    const int p = (int)(e % 81) / 9, q = (int)(e % 9);
    out[e] = cov_sinv(A, ld, d, cam_fixed, 9LL * ab.x + p, 9LL * ab.y + q);
  }
}

// camera_landmark_cross [m][27] = Cov(d_c, d_l) = -(sum_i Sigma_{c,a_i} K_i^T) W_l^T of the requests (c, l), warp per request,
// lanes over the slots i of landmark l (camera a_i), fixed-order butterfly sum; all NaN when Hll has rank < 3.
__global__ void __launch_bounds__(128) k_cov_cam_lm(const double* __restrict__ A, long long ld, const double* __restrict__ d,
                                                    const uint8_t* __restrict__ cam_fixed, const int* __restrict__ slot_cam,
                                                    const int* __restrict__ lm_slot0, const int* __restrict__ lm_n,
                                                    const double* __restrict__ kb, const double* __restrict__ wl,
                                                    const int* __restrict__ rank, const int2* __restrict__ req, int m,
                                                    double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < m; k += warps) {
    const int2 cl = req[k];
    double* o = out + 27 * (size_t)k;
    if (rank[cl.y] < 3) {
      if (lane < 27) o[lane] = __longlong_as_double(0x7ff8000000000000LL);
      continue;
    }
    const int s0 = lm_slot0[cl.y], n = lm_n[cl.y];
    const long long rc = 9LL * cl.x;
    double u[27];  // (sum_i Sigma_{c,a_i} K_i^T) [9][3]
#pragma unroll
    for (int e = 0; e < 27; ++e) u[e] = 0.0;
    for (int i = lane; i < n; i += 32) {
      const long long ra = 9LL * slot_cam[s0 + i];
      const double* ki = kb + 27 * (size_t)(s0 + i);
#pragma unroll
      for (int p = 0; p < 9; ++p)
        for (int q = 0; q < 9; ++q) {
          const double sv = cov_sinv(A, ld, d, cam_fixed, rc + p, ra + q);
#pragma unroll
          for (int j = 0; j < 3; ++j) u[3 * p + j] += sv * ki[9 * j + q];
        }
    }
#pragma unroll
    for (int e = 0; e < 27; ++e) u[e] = warp_sum(u[e]);
    if (lane == 0) {
      const double* W = wl + 9 * (size_t)cl.y;
#pragma unroll
      for (int p = 0; p < 9; ++p)
#pragma unroll
        for (int r = 0; r < 3; ++r) o[3 * p + r] = -(u[3 * p] * W[3 * r] + u[3 * p + 1] * W[3 * r + 1] + u[3 * p + 2] * W[3 * r + 2]);
    }
  }
}

// landmark_cross [m][9] = Cov(d_l, d_m) of the requests (l, m), warp per request (cov_lm_block: (l, l) is l's marginal).
// MARGINALS: request k is (k, k) and req is not read, the marginals lm_cov.  That is an instantiation of its own because
// with l == m known the kernel needs 70 registers instead of 94, and the higher occupancy makes the marginals faster.
template <bool MARGINALS>
__global__ void __launch_bounds__(128) k_cov_lm_cross(const double* __restrict__ A, long long ld, const double* __restrict__ d,
                                                      const uint8_t* __restrict__ cam_fixed, const int* __restrict__ slot_cam,
                                                      const int* __restrict__ lm_slot0, const int* __restrict__ lm_n,
                                                      const double* __restrict__ kb, const double* __restrict__ wl,
                                                      const int* __restrict__ rank, const int2* __restrict__ req, int m,
                                                      double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < m; k += warps) {
    const int2 lm = MARGINALS ? make_int2(k, k) : req[k];
    cov_lm_block(A, ld, d, cam_fixed, slot_cam, lm_slot0, lm_n, kb, wl, rank, lm.x, lm.y, lane, out + 9 * (size_t)k);
  }
}

// relative_cov [m][36] of the requests (i, j), thread per request: the covariance A Sigma_P A^T of the pair-prior residual
// e = (e_t, e_r) at the mean equal to the current relative pose (e = 0, J_l^-1 = I), Sigma_P [12][12] the pose entries
// (v_i, w_i, v_j, w_j) of the joint block of cameras i and j, A = [A_i | A_j] the rows pair_jac_rows builds with L = I.
// Each thread keeps its A [6][12] in shared memory, entry-major (a warp's accesses are conflict-free): in registers it would
// need dynamic indexing, and holding Sigma_P instead spills.  The lower triangle is computed and mirrored, so the output is
// exactly symmetric.
constexpr int COV_REL_THREADS = 64;
template <class S>
__global__ void __launch_bounds__(COV_REL_THREADS) k_cov_rel_pose(const double* __restrict__ A, long long ld, const double* __restrict__ d,
                                                                  const uint8_t* __restrict__ cam_fixed, const S* __restrict__ cams,
                                                                  const int2* __restrict__ req, int m, double* __restrict__ out) {
  __shared__ double As[72][COV_REL_THREADS];
  const int tid = threadIdx.x;
  const int stride = gridDim.x * blockDim.x;
  for (int k = blockIdx.x * blockDim.x + tid; k < m; k += stride) {
    const int2 ij = req[k];
    double ci[10], cj[10];
#pragma unroll
    for (int e = 0; e < 10; ++e) { ci[e] = (double)cams[10 * (size_t)ij.x + e]; cj[e] = (double)cams[10 * (size_t)ij.y + e]; }
    const double ident[7] = {0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0};  // e is not used: only M and t_rel
    const double I3[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0};
    double e6[6], M[9], tr[3];
    pair_residual<double, false>(ci, cj, ident, e6, M, tr, nullptr, nullptr);
    for (int r = 0; r < 6; ++r) {  // row r of A: the rows of pair_jac_rows for the row e_r of L = I
      double l[6], ri[6], rj[6];
#pragma unroll
      for (int q = 0; q < 6; ++q) l[q] = q == r ? 1.0 : 0.0;
      pair_jac_rows(l, M, tr, I3, M, ri, rj);
#pragma unroll
      for (int q = 0; q < 6; ++q) { As[12 * r + q][tid] = ri[q]; As[12 * r + 6 + q][tid] = rj[q]; }
    }
    auto idx = [&](int q) { return q < 6 ? 9LL * ij.x + q : 9LL * ij.y + q - 6; };
    double* o = out + 36 * (size_t)k;
    for (int r = 0; r < 6; ++r) {
      double t[12];  // row r of A Sigma_P
#pragma unroll
      for (int q = 0; q < 12; ++q) t[q] = 0.0;
      for (int p = 0; p < 12; ++p) {
        const double arp = As[12 * r + p][tid];
        const long long rp = idx(p);
#pragma unroll
        for (int q = 0; q < 12; ++q) t[q] += arp * cov_sinv(A, ld, d, cam_fixed, rp, idx(q));
      }
      for (int c = 0; c <= r; ++c) {
        double v = 0.0;
#pragma unroll
        for (int q = 0; q < 12; ++q) v += t[q] * As[12 * c + q][tid];
        o[6 * r + c] = v;
        o[6 * c + r] = v;
      }
    }
  }
}

}  // namespace rba
