// preconditioner_type = CLUSTER_JACOBI (DESIGN.md section 28): the block diagonal of the Jacobi-scaled, damped reduced
// camera matrix S over clusters of co-visible cameras (rba_cluster_cameras, ClusterPlan in layout.hpp), factorised once
// per solve in float64, M = L L^T.
//   k_cluster_build  once per solve, one CTA per cluster: the cluster's (9k) x (9k) block of S in shared memory -- the
//                    SCHUR_JACOBI blocks k_precond_invert has just written (damping, camera and pair priors' diagonal
//                    blocks) on the diagonal, every cross block summed over its terms in list order, the pair priors'
//                    O_ab of the cluster's pairs, held rows and columns set to the identity -- written out for
//                    rba_get_cluster_preconditioner, then its Cholesky factorisation.  A pivot <= 0 or not finite makes
//                    the cluster fall back to its cameras' diagonal blocks alone (the SCHUR_JACOBI matrix), status 1.
//   k_cluster_fwd    y = L^-1 u, one CTA per cluster; u = the operator output + lambda w (+ the camera and pair priors'
//                    terms, in the order of k_pcg_vec's P1), or a plain vector (b).
//   k_cluster_back   y = L^-T v, one CTA per cluster, in place allowed.
// PCG then runs unchanged on L^-1 S L^-T with right-hand side L^-1 b and identity blocks (masked on held entries) as its
// preconditioner; in exact arithmetic its iterates x^ = L^T x and its scalars (rho = r^T M^-1 r, the Nash-Sofer
// quantity x^T (b + r), p^T S p) are those of PCG on S with M, and the increment is -L^-T x^.
#pragma once

#include "kernels.cuh"
#include "layout.hpp"

namespace rba {

constexpr int CLUSTER_THREADS = 160;  // >= 9 CLUSTER_MAX_CAMERAS: a thread per row in the substitutions
static_assert(CLUSTER_THREADS >= 9 * CLUSTER_MAX_CAMERAS, "a thread per row of the largest cluster");

struct ClusterView {
  int ncl;
  const int* ptr;              // [ncl + 1] into cams
  const int* cams;             // cluster by cluster, ascending
  const long long* blk_off;    // [ncl + 1] offsets of the (9k)^2 blocks
  const long long* fac_off;    // [ncl + 1] offsets of the packed lower factors
  const int* xb_ptr;           // [ncl + 1] into xb
  const ClusterBlock* xb;      // the cross blocks
  const int2* slots;           // [nt] (slot_a, slot_b)
  const AsmTerm* panel_terms;  // [nt] panel addresses; nullptr: the implicit form's -q1d_a^T q1d_b
  double* blocks;              // the unfactorised blocks (read back by rba_get_cluster_preconditioner)
  double* factor;              // the packed factors
  int* status;                 // [ncl] 0 factorised, 1 fell back to the diagonal blocks
};

// In-place Cholesky of the m x m matrix A (row-major, lower triangle used) in shared memory: right-looking, column by
// column, every entry updated in a fixed order.  Returns false (uniform over the CTA) on a pivot <= 0 or not finite.
__device__ __forceinline__ bool cluster_potrf(double* A, int m, int* bad) {
  for (int j = 0; j < m; ++j) {
    if (threadIdx.x == 0) {
      const double d = A[j * m + j];
      *bad = !(d > 0.0) || isinf(d);
      A[j * m + j] = sqrt(d);
    }
    __syncthreads();
    if (*bad) return false;
    const double djj = A[j * m + j];
    const double rd = __drcp_rn(djj);  // (a division here would be a subroutine call that spills)
    for (int i = j + 1 + threadIdx.x; i < m; i += blockDim.x) A[i * m + j] *= rd;
    __syncthreads();
    const int r = m - j - 1;  // trailing lower triangle, (r (r + 1) / 2 entries) dealt over the threads
    for (int t = threadIdx.x; t < r * (r + 1) / 2; t += blockDim.x) {
      int i = (int)((sqrtf(8.0f * t + 1.0f) - 1.0f) * 0.5f);  // corrected below
      while (i * (i + 1) / 2 > t) --i;
      while ((i + 1) * (i + 2) / 2 <= t) ++i;
      const int k = t - i * (i + 1) / 2;
      const int ii = j + 1 + i, kk = j + 1 + k;
      A[ii * m + kk] -= A[ii * m + j] * A[kk * m + j];
    }
    __syncthreads();
  }
  return true;
}

template <class S>
__global__ void __launch_bounds__(256) k_cluster_build(ClusterView cv, DevPtrs<S> D, S* __restrict__ eye) {
  extern __shared__ double A[];
  __shared__ int bad;
  const int cl = blockIdx.x;
  const int c0 = cv.ptr[cl], k = cv.ptr[cl + 1] - c0, m = 9 * k;
  const int* cams = cv.cams + c0;
  // the diagonal blocks (k_precond_invert's blocks_out) and zero cross blocks
  for (int t = threadIdx.x; t < m * m; t += blockDim.x) {
    const int i = t / m, j = t - i * m, u = i / 9, v = j / 9;
    A[t] = u == v ? (double)D.blocks[81 * (size_t)cams[u] + 9 * (i - 9 * u) + (j - 9 * v)] : 0.0;
  }
  __syncthreads();
  // the cross blocks: thread per entry (p, q) of a block S[a, b] (a > b), its terms added in list order; the transpose
  // goes to S[b, a]
  const int x0 = cv.xb_ptr[cl], nx = cv.xb_ptr[cl + 1] - x0;
  for (int t = threadIdx.x; t < 81 * nx; t += blockDim.x) {
    const ClusterBlock xb = cv.xb[x0 + t / 81];
    const int e = t % 81, p = e / 9, q = e % 9;
    double s = 0;
    for (int w = xb.t0; w < xb.t1; ++w) {
      double acc = 0;
      if (cv.panel_terms) {  // P_a^T P_b over all 2n panel rows, the damping rows of this solve included
        const AsmTerm at = cv.panel_terms[w];
        const int n = at.meta & 0x7fff, lg = (at.meta >> 15) & 7, KP = at.meta >> 18, G = 1 << lg;
        const int ca = 9 * (at.ij & 0xffff) + p, cb = 9 * (at.ij >> 16) + q;
        const int off_a = 2 * (((ca >> 1) >> lg) * 32 + ((ca >> 1) & (G - 1))) + (ca & 1);
        const int off_b = 2 * (((cb >> 1) >> lg) * 32 + ((cb >> 1) & (G - 1))) + (cb & 1);
        const S* lmp = D.panel + at.base;
        const size_t rstride = (size_t)KP * 64;
        for (int r = 0; r < 2 * n; ++r) acc = fma((double)lmp[r * rstride + off_a], (double)lmp[r * rstride + off_b], acc);
      } else {  // -q1d_a^T q1d_b (Jp_a^T Jp_b = 0 for two cameras)
        const int2 sl = cv.slots[w];
        const S* qa = D.q1d + 28 * (size_t)sl.x;
        const S* qb = D.q1d + 28 * (size_t)sl.y;
#pragma unroll
        for (int d = 0; d < 3; ++d) acc = fma((double)qa[9 * d + p], (double)qb[9 * d + q], acc);
        acc = -acc;
      }
      s += acc;
    }
    A[(9 * xb.la + p) * m + 9 * xb.lb + q] = s;
    A[(9 * xb.lb + q) * m + 9 * xb.la + p] = s;
  }
  __syncthreads();
  // the pair priors' O_ab (pose 6 x 6) of every pair of the cluster, edges in CSR order; thread per entry of a's row
  if (D.pair_ov) {
    for (int t = threadIdx.x; t < 36 * k; t += blockDim.x) {
      const int u = t / 36, e = t % 36, p = e / 6, q = e % 6, a = cams[u];
      for (int g = D.pair_ptr[a]; g < D.pair_ptr[a + 1]; ++g) {
        const int b = D.pair_nbr[g];
        if (b >= a) continue;
        int v = 0;
        while (v < k && cams[v] != b) ++v;
        if (v == k) continue;  // another cluster
        const double o = (double)D.pair_O[36 * (size_t)g + e];
        A[(9 * u + p) * m + 9 * v + q] += o;
        A[(9 * v + q) * m + 9 * u + p] += o;
      }
    }
    __syncthreads();
  }
  // held entries: identity rows and columns; the identity blocks of the vector step, zero on the held entries
  for (int t = threadIdx.x; t < m * m; t += blockDim.x) {
    const int i = t / m, j = t - i * m;
    const unsigned fi = D.cam_fixed ? fixed_entry_mask(D.cam_fixed[cams[i / 9]]) >> (i % 9) : 0u;
    const unsigned fj = D.cam_fixed ? fixed_entry_mask(D.cam_fixed[cams[j / 9]]) >> (j % 9) : 0u;
    if ((fi | fj) & 1u) A[t] = i == j ? 1.0 : 0.0;
    if (i / 9 == j / 9)
      eye[81 * (size_t)cams[i / 9] + 9 * (i % 9) + j % 9] = (i == j && !(fi & 1u)) ? S(1) : S(0);
  }
  __syncthreads();
  double* out = cv.blocks + cv.blk_off[cl];
  for (int t = threadIdx.x; t < m * m; t += blockDim.x) out[t] = A[t];
  __syncthreads();
  // the cluster block, then (a pivot <= 0 or not finite) the cameras' own blocks alone: the SCHUR_JACOBI matrix
  bool ok = true, ok2 = true;
  for (int attempt = 0; attempt < 2; ++attempt) {
    if (attempt) {
      for (int t = threadIdx.x; t < m * m; t += blockDim.x) {
        const int i = t / m, j = t - i * m;
        A[t] = i / 9 == j / 9 ? out[t] : 0.0;
      }
      __syncthreads();
    }
    const bool done = cluster_potrf(A, m, &bad);
    if (attempt) ok2 = done; else ok = done;
    if (done) break;
  }
  if (threadIdx.x == 0) cv.status[cl] = ok ? 0 : 1;
  // (a camera block that is not positive definite either leaves a NaN factor, as SCHUR_JACOBI's inverse would be)
  double* f = cv.factor + cv.fac_off[cl];
  for (int t = threadIdx.x; t < m * (m + 1) / 2; t += blockDim.x) {
    int i = (int)((sqrtf(8.0f * t + 1.0f) - 1.0f) * 0.5f);  // corrected below
    while (i * (i + 1) / 2 > t) --i;
    while ((i + 1) * (i + 2) / 2 <= t) ++i;
    f[t] = ok2 ? A[i * m + (t - i * (i + 1) / 2)] : __longlong_as_double(0x7ff8000000000000LL);
  }
}

// the cluster's packed factor into shared memory (dynamic, 9 k_max (9 k_max + 1) / 2 doubles) and its row count
__device__ __forceinline__ int cluster_load_factor(const ClusterView& cv, int cl, double* Lf) {
  const int m = 9 * (cv.ptr[cl + 1] - cv.ptr[cl]);
  const double* f = cv.factor + cv.fac_off[cl];
  for (int t = threadIdx.x; t < m * (m + 1) / 2; t += blockDim.x) Lf[t] = __ldg(f + t);
  return m;
}

// y = L^-1 u (u: WITH_OP the camera-reduced operator output of w -- D.y, or the per-segment partial sums when item_ptr is
// given -- plus lambda w and the priors' terms; else the vector y_in itself).  Returns at once when the solve has ended.
template <class S>
__global__ void __launch_bounds__(CLUSTER_THREADS) k_cluster_fwd(ClusterView cv, DevPtrs<S> D, const S* __restrict__ y_in,
                                                                  const int* __restrict__ item_ptr, const S* __restrict__ w,
                                                                  S lambda, S* __restrict__ y_out, const int* __restrict__ done) {
  extern __shared__ double Lf[];
  __shared__ double u[9 * CLUSTER_MAX_CAMERAS];
  if (done && *done) return;
  const int cl = blockIdx.x;
  const int m = cluster_load_factor(cv, cl, Lf);
  const int* cams = cv.cams + cv.ptr[cl];
  const int i = threadIdx.x;
  if (i < m) {
    const int cam = cams[i / 9], c = i % 9;
    const size_t e = 9 * (size_t)cam + c;
    S q;
    if (item_ptr) {  // the segment sums in their fixed order (k_pcg_vec)
      q = 0;
      for (int s = item_ptr[cam]; s < item_ptr[cam + 1]; ++s) q += __ldcg(D.partial + 9 * (size_t)s + c);
    } else {
      q = __ldcg(y_in + e);
    }
    if (w) {  // + lambda w (+ A^T A w) (+ sum_j O_ij w_j): the operator of k_pcg_vec's P1 and k_pcg_q
      q = q + lambda * w[e];
      if (D.prior_H) {
        const S* hr = D.prior_H + 81 * (size_t)cam + 9 * c;
        S h = 0;
#pragma unroll
        for (int kk = 0; kk < 9; ++kk) h += hr[kk] * w[9 * (size_t)cam + kk];
        q += h;
      }
      if (D.pair_ov) q += pair_ov_entry(D, w, 9 * cam + c);
    }
    u[i] = (double)q;
  }
  __syncthreads();
  // forward substitution, column by column: step j fixes u[j] and removes it from the rows below
  for (int j = 0; j < m; ++j) {
    const double yj = u[j] / Lf[j * (j + 1) / 2 + j];
    __syncthreads();
    if (i == j) u[j] = yj;
    else if (i > j && i < m) u[i] -= Lf[i * (i + 1) / 2 + j] * yj;
    __syncthreads();
  }
  if (i < m) y_out[9 * (size_t)cams[i / 9] + i % 9] = (S)u[i];
}

// y = L^-T v (y may be v).  Returns at once when the solve has ended (done given).
template <class S>
__global__ void __launch_bounds__(CLUSTER_THREADS) k_cluster_back(ClusterView cv, const S* v, S* y_out, const int* __restrict__ done) {
  extern __shared__ double Lf[];
  __shared__ double u[9 * CLUSTER_MAX_CAMERAS];
  if (done && *done) return;
  const int cl = blockIdx.x;
  const int m = cluster_load_factor(cv, cl, Lf);
  const int* cams = cv.cams + cv.ptr[cl];
  const int i = threadIdx.x;
  if (i < m) u[i] = (double)v[9 * (size_t)cams[i / 9] + i % 9];
  __syncthreads();
  // back substitution with L^T, row by row from the last: step j fixes u[j] and removes it from the rows above
  for (int j = m - 1; j >= 0; --j) {
    const double xj = u[j] / Lf[j * (j + 1) / 2 + j];
    __syncthreads();
    if (i == j) u[j] = xj;
    else if (i < j) u[i] -= Lf[j * (j + 1) / 2 + i] * xj;
    __syncthreads();
  }
  if (i < m) y_out[9 * (size_t)cams[i / 9] + i % 9] = (S)u[i];
}

}  // namespace rba
