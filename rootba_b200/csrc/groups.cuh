// Intrinsics shared across groups of cameras (rba_set_intrinsics_groups, DESIGN.md section 18).
// The tied problem has a pose per camera and one (f, k1, k2) per group; its vectors u are kept in the 9 nc layout with
// the group's intrinsics in the lead's entries 6..8 and the other members' entries 6..8 held at zero (x = P u, P copies
// the lead's entries into the members').  These kernels apply P (expand) and P^T (contract) around the unchanged operator
// kernels, and merge the scaling, the gradient and the preconditioner blocks over each group.  Only groups of >= 2
// cameras exist here: a group of one is an ungrouped camera.  Every sum over a group runs in a fixed order (members
// ascending per thread, then a fixed tree), so the results are deterministic.
#pragma once

#include "kernels.cuh"

namespace rba {

constexpr int GROUP_THREADS = 128;

struct GroupView {
  const int* lead;  // [nc] the lead (lowest-index member) of the camera's group, -1 = the camera keeps its own intrinsics
  const int* ptr;   // [ng + 1] members of group g: mem[ptr[g] .. ptr[g + 1]), ascending, so the lead first
  const int* mem;
  int ng;
};

// v[0..N) summed over the GROUP_THREADS threads of the block, in a fixed tree; every thread receives the totals
template <class S, int N>
__device__ __forceinline__ void group_block_sum(S (&v)[N]) {
  __shared__ S sh[GROUP_THREADS][N];
  const int t = threadIdx.x;
#pragma unroll
  for (int k = 0; k < N; ++k) sh[t][k] = v[k];
  __syncthreads();
  for (int s = GROUP_THREADS / 2; s > 0; s >>= 1) {
    if (t < s)
#pragma unroll
      for (int k = 0; k < N; ++k) sh[t][k] += sh[t + s][k];
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < N; ++k) v[k] = sh[0][k];
}

// linearize: every member's squared column norms of f, k1, k2 become the group's (the norms of the merged columns J P:
// the members' columns have disjoint rows), so every member gets the group's Jacobi scaling and P commutes with D.
// Block per group.
template <class S>
__global__ void __launch_bounds__(GROUP_THREADS) k_group_sum_diag2(S* __restrict__ diag2, GroupView G) {
  const int m0 = G.ptr[blockIdx.x], m1 = G.ptr[blockIdx.x + 1];
  S s[3] = {0, 0, 0};
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS)
#pragma unroll
    for (int k = 0; k < 3; ++k) s[k] += diag2[9 * (size_t)G.mem[q] + 6 + k];
  group_block_sum<S, 3>(s);
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS)
#pragma unroll
    for (int k = 0; k < 3; ++k) diag2[9 * (size_t)G.mem[q] + 6 + k] = s[k];
}

// solve, ahead of k_precond_invert: the preconditioner blocks in the block partition of the tied problem and the
// contracted gradient.  Blocks [0, ncb): thread per camera, blocks [ncb, ncb + ng): one per group.
//   ungrouped camera:  out = src (+ prior_H), b += prior_g
//   grouped camera:    pose 6x6 of out = that of src (+ prior_H), pose-intrinsics entries 0, b[0..5] += prior_g[0..5]
//   group:             the lead's intrinsics 3x3 of out = sum over the members of src (+ prior_H), its b[6..8] = sum over
//                      the members of b + prior_g; the other members' intrinsics entries of out and b are 0
// k_precond_invert then adds lambda once per parameter of the tied problem (a group's intrinsics once, on the lead) and
// masks the members' entries 6..8 as held, which gives blkdiag(pose^-1, G^-1) on the lead and the pose inverse on the
// other members.  The two roles touch disjoint entries, so out may be src (SCHUR_JACOBI).
template <class S>
__global__ void __launch_bounds__(GROUP_THREADS) k_group_precond(const S* src, const S* __restrict__ prior_H,
                                                                 const S* __restrict__ prior_g, S* __restrict__ b, S* out,
                                                                 GroupView G, int nc, int ncb) {
  if ((int)blockIdx.x < ncb) {
    const int cam = blockIdx.x * GROUP_THREADS + threadIdx.x;
    if (cam >= nc) return;
    const bool grouped = G.lead[cam] >= 0;
    const size_t o = 81 * (size_t)cam;
    for (int r = 0; r < 9; ++r)
      for (int c = 0; c < 9; ++c) {
        if (grouped && r >= 6 && c >= 6) continue;
        S a = src[o + 9 * r + c];
        if (prior_H) a += prior_H[o + 9 * r + c];
        out[o + 9 * r + c] = (grouped && (r >= 6) != (c >= 6)) ? S(0) : a;
      }
    if (prior_g)
      for (int d = 0; d < (grouped ? 6 : 9); ++d) b[9 * (size_t)cam + d] += prior_g[9 * (size_t)cam + d];
    return;
  }
  const int g = blockIdx.x - ncb;
  const int m0 = G.ptr[g], m1 = G.ptr[g + 1];
  S s[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) s[k] = 0;
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
    const size_t cam = G.mem[q];
#pragma unroll
    for (int k = 0; k < 3; ++k) s[k] += b[9 * cam + 6 + k] + (prior_g ? prior_g[9 * cam + 6 + k] : S(0));
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const size_t e = 81 * cam + 9 * (6 + r) + 6 + c;
        s[3 + 3 * r + c] += src[e] + (prior_H ? prior_H[e] : S(0));
      }
  }
  group_block_sum<S, 12>(s);  // every read above precedes its barriers, every write below follows them
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
    const size_t cam = G.mem[q];
    const bool lead = q == m0;
#pragma unroll
    for (int k = 0; k < 3; ++k) b[9 * cam + 6 + k] = lead ? s[k] : S(0);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) out[81 * cam + 9 * (6 + r) + 6 + c] = lead ? s[3 + 3 * r + c] : S(0);
  }
}

// out = P v: the members' entries 6..8 take the lead's.  out may be v (then only the members' entries are written).  In
// a solve (st set) it is launched dependent on its predecessor and returns once the solve has ended, like k_pair_ov.
template <class S>
__global__ void __launch_bounds__(256) k_group_expand(const S* v, S* out, const int* __restrict__ lead, int nc,
                                                      const PcgState* st) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (st && *reinterpret_cast<const volatile int*>(&st->done)) return;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < 9 * nc; e += gridDim.x * blockDim.x) {
    const int cam = e / 9, a = e - 9 * cam, ld = lead[cam];
    const int from = (a >= 6 && ld >= 0) ? 9 * ld + a : e;
    if (from != e || out != v) out[e] = v[from];
  }
}

// Row a of camera cam of the full operator at the expanded vector ve: the camera-reduced operator output y = D.y plus the
// camera priors' and pair priors' terms.  The pair priors act on poses only, so rows 6..8 carry no pair term.
template <class S>
__device__ __forceinline__ S operator_row(const DevPtrs<S>& D, const S* __restrict__ ve, size_t cam, int a) {
  S t = __ldcg(D.y + 9 * cam + a);
  if (D.prior_H) {
    const S* hr = D.prior_H + 81 * cam + 9 * a;
    S h = 0;
#pragma unroll
    for (int k = 0; k < 9; ++k) h += hr[k] * ve[9 * cam + k];
    t += h;
  }
  if (D.pair_ov && a < 6) t += pair_ov_entry(D, ve, (int)(9 * cam) + a);
  return t;
}

// out = P^T (y + A^T A ve + O ve): the rows of the full operator at the expanded vector ve = P v (operator_row),
// contracted into the leads.  The vector step that follows adds lambda v on the contracted v (lambda once per group) and
// runs without prior terms of its own.  Blocks [0, ncb): thread per camera (pose rows, and every row of an ungrouped
// camera), blocks [ncb, ncb + ng): one per group (the lead's rows 6..8 = the members' sum, the other members' 0).
template <class S>
__global__ void __launch_bounds__(GROUP_THREADS) k_group_contract(DevPtrs<S> D, const S* __restrict__ ve, S* __restrict__ out,
                                                                  GroupView G, int ncb, const PcgState* st) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (*reinterpret_cast<const volatile int*>(&st->done)) return;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  auto row = [&](size_t cam, int a) -> S { return operator_row(D, ve, cam, a); };
  if ((int)blockIdx.x < ncb) {
    const int cam = blockIdx.x * GROUP_THREADS + threadIdx.x;
    if (cam >= D.nc) return;
    const int na = G.lead[cam] >= 0 ? 6 : 9;
    for (int a = 0; a < na; ++a) out[9 * (size_t)cam + a] = row(cam, a);
    return;
  }
  const int g = blockIdx.x - ncb;
  const int m0 = G.ptr[g], m1 = G.ptr[g + 1];
  S s[3] = {0, 0, 0};
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS)
#pragma unroll
    for (int k = 0; k < 3; ++k) s[k] += row(G.mem[q], 6 + k);
  group_block_sum<S, 3>(s);
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS)
#pragma unroll
    for (int k = 0; k < 3; ++k) out[9 * (size_t)G.mem[q] + 6 + k] = q == m0 ? s[k] : S(0);
}

// ---- rba_compute_covariance (DESIGN.md sections 16 and 18) on the dense np x np column-major matrix A (ld) ----
// The upper triangle := the lower one, so that the row and column passes below see the full symmetric matrix.
__global__ void k_cov_group_symmetrize(double* __restrict__ A, long long ld, long long n) {
  const long long r = blockIdx.x * 32LL + threadIdx.x;
  const long long c = blockIdx.y * 8LL + threadIdx.y;
  if (r < n && c < n && r < c) A[r + c * ld] = A[c + r * ld];
}
// Row pass (thread per column c, which it alone touches) or column pass (thread per row r) over every group's intrinsics
// rows / columns: contract (expand = 0) adds the other members' row / column 6..8 to the lead's, in member order, which
// applied as rows then columns gives P^T A P; expand (expand = 1) copies the lead's into the other members', which applied
// to the inverse gives P A P^T.
__global__ void k_cov_group_pass(double* __restrict__ A, long long ld, long long n, GroupView G, int columns, int expand) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  // entry (j, i) of the row pass, (i, j) of the column pass
  auto at = [&](long long j) -> double& { return columns ? A[i + j * ld] : A[j + i * ld]; };
  for (int g = 0; g < G.ng; ++g) {
    const int m0 = G.ptr[g], m1 = G.ptr[g + 1];
    const long long lead = 9LL * G.mem[m0] + 6;
    for (int k = 0; k < 3; ++k) {
      if (expand) {
        const double v = at(lead + k);
        for (int q = m0 + 1; q < m1; ++q) at(9LL * G.mem[q] + 6 + k) = v;
      } else {
        double s = at(lead + k);
        for (int q = m0 + 1; q < m1; ++q) s += at(9LL * G.mem[q] + 6 + k);
        at(lead + k) = s;
      }
    }
  }
}
// the equilibration of the members' entries 6..8 := the lead's (after the expansion of the inverse).  One thread.
__global__ void k_cov_group_d(double* __restrict__ d, GroupView G) {
  for (int g = 0; g < G.ng; ++g)
    for (int q = G.ptr[g] + 1; q < G.ptr[g + 1]; ++q)
      for (int k = 0; k < 3; ++k) d[9LL * G.mem[q] + 6 + k] = d[9LL * G.mem[G.ptr[g]] + 6 + k];
}

}  // namespace rba
