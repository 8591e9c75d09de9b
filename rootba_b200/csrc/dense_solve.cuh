// Exact solve of the reduced camera system by a dense Cholesky factorisation (linear_solver_type = DENSE_SCHUR, DESIGN.md
// section 27).
//
// The system is the one PCG iterates on, in the Jacobi-scaled space of the handle:
//   H = D (Jp^T Jp - Jp^T Jl (Jl^T Jl + lambda sl^-2)^-1 Jl^T Jp + priors) D + lambda I,   inc = -H_ff^-1 b_f
// (with intrinsics groups, rigs and sensors: the tied system, D the scaling of the merged columns).  Everything here is
// float64 for either Scalar, re-linearised at the current state like the covariances (covariance.cuh); the increment is
// rounded to Scalar once, at the end.  The pipeline, on the solver stream, with no host synchronisation:
//   1. k_dense_landmark   per landmark: sqrt(w) Jp per slot and K_i(lambda) = (Lambda + lambda)^-1/2 V^T Jls_i^T Jp_i
//   2. k_cov_assemble, k_cov_priors, the group and rig passes (covariance.cuh, groups.cuh, rigs.cuh) -> P^T S P
//      k_dense_scaling (+ k_dense_tied_scaling), k_cov_equil -> D S D, held entries and padding -> identity
//      k_dense_gather     + lambda on the free diagonal, b -> the padded float64 vector
//   3. the blocked potrf of the covariances (dense_potrf in solver.cu), the pivot flag left on the device
//   4. k_dense_trsv_fwd / k_dense_trsv_bwd per tile: L y = b, L^T x = y
//   5. k_dense_finish     inc = -x (0 held, NaN free entries on a failed pivot) and the PcgState of the solve
#pragma once

#include "covariance.cuh"
#include "rigs.cuh"

namespace rba {

constexpr int DENSE_TRSV_ROWS = 128;  // rows of the forward panel update per CTA (thread per row)
constexpr int DENSE_TRSV_COLS = 64;   // columns of the backward panel update per CTA (8 warps, 8 columns each)

// Warp per landmark (problem order).  The per-slot rows are those of k_cov_landmark: re-linearised in double with the
// weights, losses, observation information and validity rule of rba_linearize, unscaled; jpw [18] = sqrt(w) Jp per slot.
// Hll = sum Jl^T Jl (+ the landmark prior's (sqrt(w)) L^T L while lmp_of_lm is given) is scaled by the landmark's Jacobi
// scaling jls = 1 / (eps + |column|), whose column norms are the diagonal of Hll, and diag(jls) Hll diag(jls) = V Lambda V^T.
// kb [27] per slot = K = W^T Jl^T Jp with W = diag(jls) V (Lambda + lambda)^-1/2, so that K_a^T K_b is the camera term
// Jp_a^T Jl_a (Hll + lambda sl^-2)^-1 Jl_b^T Jp_b of the damped elimination.  The columns of W whose shifted eigenvalue is
// <= COV_EIG_DROP of the largest are zero (only reachable at lambda = 0: the null directions of a rank-deficient landmark).
template <class S>
__global__ void __launch_bounds__(128, 1) k_dense_landmark(DevPtrs<S> D, KOpts o, const int* __restrict__ lm_slot0,
                                                           const int* __restrict__ lm_n, int nl, double lambda,
                                                           double* __restrict__ jpw, double* __restrict__ kb,
                                                           const int* __restrict__ lmp_of_lm) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  const double eps = (double)(S)o.jacobi_eps;
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
      if (D.obs_W) keep = !whiten_observation<double, true>(D.obs_W, s, res, Jp, Jl);
      if (keep && o.use_valid_projections_only) {
        double R[9];
        quat_to_rot(cam, R);
        const double z = R[6] * pw[0] + R[7] * pw[1] + R[8] * pw[2] + cam[6];
        keep = z >= (double)ST<S>::eps_sqrt();
      }
      double sw = 0.0;
      if (keep) {
        const double sq = res[0] * res[0] + res[1] * res[1];
        double err, w;
        if (D.obs_loss) slot_error_weight<true>(o, D.obs_loss, D.nslots, s, sq, err, w);
        else slot_error_weight<false>(o, D.obs_loss, D.nslots, s, sq, err, w);
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
    const int lp = lmp_of_lm ? lmp_of_lm[lm] : -1;
    if (lp >= 0) {
      const S* Lp = (D.lmp_loss ? D.lmp_Lu : D.lmp_L) + 9 * (size_t)lp;
      double sw = 1.0;
      if (D.lmp_loss) {
        double rp[3], err, w;
        lmp_loss(D, lp, lmp_residual(D, lp, pw, rp), err, w);
        sw = sqrt(w);
      }
      for (int r = 0; r < 3; ++r) {
        const double a0 = sw * (double)Lp[3 * r], a1 = sw * (double)Lp[3 * r + 1], a2 = sw * (double)Lp[3 * r + 2];
        h[0] += a0 * a0; h[1] += a0 * a1; h[2] += a0 * a2; h[3] += a1 * a1; h[4] += a1 * a2; h[5] += a2 * a2;
      }
    }
    const double jls[3] = {1.0 / (eps + sqrt(h[0])), 1.0 / (eps + sqrt(h[3])), 1.0 / (eps + sqrt(h[5]))};
    double A[9] = {jls[0] * h[0] * jls[0], jls[0] * h[1] * jls[1], jls[0] * h[2] * jls[2],
                   jls[1] * h[1] * jls[0], jls[1] * h[3] * jls[1], jls[1] * h[4] * jls[2],
                   jls[2] * h[2] * jls[0], jls[2] * h[4] * jls[1], jls[2] * h[5] * jls[2]};
    double V[9];
    sym_eig<3>(A, V);
    const double mmax = fmax(A[0], fmax(A[4], A[8])) + lambda;
    double W[9];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double mu = A[4 * k] + lambda;
      const double f = mmax > 0.0 && mu > COV_EIG_DROP * mmax ? 1.0 / sqrt(mu) : 0.0;
#pragma unroll
      for (int row = 0; row < 3; ++row) W[3 * row + k] = jls[row] * V[3 * row + k] * f;
    }
    for (int i = lane; i < n; i += 32) {
      const int s = s0 + i;
      double Jl[6], Jp[18];
#pragma unroll
      for (int k = 0; k < 6; ++k) Jl[k] = kb[27 * (size_t)s + k];
#pragma unroll
      for (int k = 0; k < 18; ++k) Jp[k] = jpw[18 * (size_t)s + k];
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

// d [np] = the handle's Jacobi scaling, widened (1 on the padding).  Thread per entry.
template <class S>
__global__ void k_dense_scaling(const S* __restrict__ scaling, long long n, long long np, double* __restrict__ d) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k < np) d[k] = k < n ? (double)scaling[k] : 1.0;
}

// Rigs (DESIGN.md sections 23, 24): the pose entries of each rig's lead take D_u of the rig, those of each sensor's home
// D_s of the sensor (the scaling of the merged columns; intrinsics groups need nothing: every member carries the group's).
// Thread per rig, then per sensor.
template <class S>
__global__ void k_dense_tied_scaling(RigView<S> R, const S* __restrict__ ds, const int* __restrict__ sptr, const int* __restrict__ smem,
                                     int ns, double* __restrict__ d) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < R.nr) {
    const size_t lead = R.mem[R.ptr[t]];
#pragma unroll
    for (int k = 0; k < 6; ++k) d[9 * lead + k] = (double)R.du[6 * (size_t)t + k];
  } else if (t < R.nr + ns) {
    const int s = t - R.nr;
    const size_t home = smem[sptr[s]];
#pragma unroll
    for (int k = 0; k < 6; ++k) d[9 * home + k] = (double)ds[6 * (size_t)s + k];
  }
}

// + lambda on the free diagonal of the scaled matrix, and x [np] = b (0 on the padding; b is 0 on held entries already).
// A diagonal entry that is not finite is flagged like a failed pivot (k_cov_tile_potrf's test lets +inf through).
template <class S>
__global__ void k_dense_gather(double* __restrict__ A, long long ld, long long n, long long np, const uint8_t* __restrict__ held,
                               double lambda, const S* __restrict__ b, double* __restrict__ x, int* __restrict__ fail) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k >= np) return;
  x[k] = k < n ? (double)b[k] : 0.0;
  if (k < n && !cov_fixed(held, k)) {
    const double a = A[k + k * ld] + lambda;
    A[k + k * ld] = a;
    if (!isfinite(a)) atomicMin(fail, (int)k);
  }
}

// Loads the lower triangle of the diagonal tile (k0, k0) into T (T[r][c], r >= c; the rest is not read).
__device__ __forceinline__ void dense_load_tile(const double* __restrict__ A, long long ld, long long k0, double (*T)[COV_TB + 1]) {
  for (int e = threadIdx.x; e < COV_TB * COV_TB; e += blockDim.x) {
    const int r = e % COV_TB, c = e / COV_TB;
    if (r >= c) T[r][c] = A[(k0 + r) + (k0 + c) * ld];
  }
}

// Forward step of tile k0: every CTA solves L_kk y_k = x_k (warp 0, lane l owns rows l and l + 32, in the fixed order of
// the columns), CTA 0 stores y_k into y, and the CTAs then update the rows below, thread per row:
// x_r -= sum_c L(r, k0 + c) y_c.  Rows k0 .. k0 + 63 of x are only read here, so the launch has no race.
__global__ void __launch_bounds__(DENSE_TRSV_ROWS) k_dense_trsv_fwd(const double* __restrict__ A, long long ld, long long np,
                                                                    long long k0, double* __restrict__ x, double* __restrict__ y) {
  __shared__ double T[COV_TB][COV_TB + 1];
  __shared__ double ys[COV_TB];
  dense_load_tile(A, ld, k0, T);
  __syncthreads();
  if (threadIdx.x < 32) {
    const int l = threadIdx.x;
    double v0 = x[k0 + l], v1 = x[k0 + 32 + l];
    for (int j = 0; j < COV_TB; ++j) {
      if (j < 32 && l == j) v0 /= T[j][j];
      if (j >= 32 && l == j - 32) v1 /= T[j][j];
      const double yj = __shfl_sync(0xffffffffu, j < 32 ? v0 : v1, j & 31);
      if (l > j) v0 -= T[l][j] * yj;
      if (l + 32 > j) v1 -= T[l + 32][j] * yj;
    }
    ys[l] = v0;
    ys[l + 32] = v1;
  }
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x < COV_TB) y[k0 + threadIdx.x] = ys[threadIdx.x];
  const long long r = k0 + COV_TB + (long long)blockIdx.x * DENSE_TRSV_ROWS + threadIdx.x;
  if (r >= np) return;
  double acc = x[r];
  const double* col = A + r + k0 * ld;
  for (int c = 0; c < COV_TB; ++c) acc -= col[c * ld] * ys[c];
  x[r] = acc;
}

// Backward step of tile k0: every CTA solves L_kk^T z_k = y_k (warp 0, from the last row up), CTA 0 stores z_k into z, and
// the CTAs then update the entries above, warp per column c < k0: y_c -= sum_r L(k0 + r, c) z_r (the 64 entries of the
// column in the tile's rows are contiguous), fixed-order butterfly sum.
__global__ void __launch_bounds__(256) k_dense_trsv_bwd(const double* __restrict__ A, long long ld, long long k0, double* __restrict__ y,
                                                        double* __restrict__ z) {
  __shared__ double T[COV_TB][COV_TB + 1];
  __shared__ double zs[COV_TB];
  dense_load_tile(A, ld, k0, T);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp == 0) {
    double v0 = y[k0 + lane], v1 = y[k0 + 32 + lane];
    for (int i = COV_TB - 1; i >= 0; --i) {
      if (i < 32 && lane == i) v0 /= T[i][i];
      if (i >= 32 && lane == i - 32) v1 /= T[i][i];
      const double zi = __shfl_sync(0xffffffffu, i < 32 ? v0 : v1, i & 31);
      if (lane < i) v0 -= T[i][lane] * zi;
      if (lane + 32 < i) v1 -= T[i][lane + 32] * zi;
    }
    zs[lane] = v0;
    zs[lane + 32] = v1;
  }
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x < COV_TB) z[k0 + threadIdx.x] = zs[threadIdx.x];
  const double z0 = zs[lane], z1 = zs[lane + 32];
  for (int u = 0; u < DENSE_TRSV_COLS / 8; ++u) {
    const long long c = (long long)blockIdx.x * DENSE_TRSV_COLS + 8 * u + warp;
    if (c >= k0) break;
    const double* col = A + k0 + c * ld;
    const double v = warp_sum(col[lane] * z0 + col[lane + 32] * z1);
    if (lane == 0) y[c] -= v;
  }
}

// inc [9 nc] = -x on the free entries, 0 on the held ones; NaN on the free entries when a pivot failed (*fail < np).
// Thread 0 writes the PcgState of the solve: SUCCESS (reason 7) or FAILURE (reason 8), no iterations.
template <class S>
__global__ void k_dense_finish(const double* __restrict__ x, long long n, long long np, const uint8_t* __restrict__ held,
                               const int* __restrict__ fail, S* __restrict__ inc, PcgState* __restrict__ st) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const bool failed = *fail < np;
  if (k == 0) {
    st->iter = 0;
    st->done = 1;
    st->term = failed ? 2 : 1;
    st->reason = failed ? 8 : 7;
  }
  if (k >= n) return;
  inc[k] = cov_fixed(held, k) ? S(0) : failed ? S(__longlong_as_double(0x7ff8000000000000LL)) : (S)(-x[k]);
}

}  // namespace rba
