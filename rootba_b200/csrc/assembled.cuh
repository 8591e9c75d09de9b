// The reduced camera matrix S = sum_l P_l^T P_l assembled from the Q2 panels P_l, and its block-row product (DESIGN.md
// section 4, "Assembled operator").  With one GPU and operator_form = DENSE the PCG operator is applied as (P^T P) x
// instead of P^T (P x): the same products of panel entries, associated differently, and S (9 x 9 blocks over the
// co-visible camera pairs) is several times smaller than the panels it is built from.
//   k_rcs_terms     once per linearisation: S_u = sum over panel rows 0..2n-4 (lambda-independent, the reference's rows
//   k_rcs_combine   3..2n-1 of the landmark block);  once per solve: S = S_u + sum over the three damping rows that
//                   k_stage2 has just written (rows 2n-3..2n-1).  The 9 x 9 block of every term (slot_a, slot_b) of every
//                   landmark is evaluated landmark by landmark into a staging buffer that holds all of them, then every
//                   co-visible camera pair (ca >= cb) adds its terms in the order of the host-built list
//                   (build_pair_list, layout.hpp): no atomics, fixed order.
//   k_rcs_spmv      y = S x over a camera-major block-row CSR of the full matrix (both triangles, diagonal included).
#pragma once

#include "kernels.cuh"

namespace rba {

// Landmark-major evaluation of the nt terms (landmarks in problem order): warp per three consecutive terms, lane 9 g + p
// (g = 0..2, p = 0..8; lanes 27..31 idle) computes row p of the 9 x 9 block of term 3 k + g over the panel rows
// [0, 2n - 3) (damping = 0: the lambda-independent rows) or [2n - 3, 2n) (damping = 1: the damping rows of the last
// k_stage2) into stage[81 w].  Neighbouring warps read the same landmark's panel, so it is read from HBM about once.
// Block entry (p, q) = sum_r P[r][9 ia + p] P[r][9 ib + q]; on the diagonal (sa == sb) it is symmetric bit for bit (fma
// commutes).
template <class S>
__global__ void __launch_bounds__(256) k_rcs_terms(const S* __restrict__ panel, const AsmTerm* __restrict__ terms, long long nt,
                                                   int damping, S* __restrict__ stage) {
  using V2 = typename ST<S>::V2;
  const int lane = threadIdx.x & 31;
  const int g = lane / 9, p = lane - 9 * g;
  if (lane >= 27) return;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long w = 3 * (blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5)) + g; w < nt; w += 3 * warps) {
    const AsmTerm at = terms[w];
    const int n = at.meta & 0x7fff, lg = (at.meta >> 15) & 7, KP = at.meta >> 18, G = 1 << lg;
    const int ia = at.ij & 0xffff, ib = at.ij >> 16;
    // column 9 ia + p of slot a: one scalar; columns 9 ib .. 9 ib + 8 of slot b: five two-scalar loads
    const int ca = 9 * ia + p, pa = ca >> 1;
    const int off_a = 2 * ((pa >> lg) * 32 + (pa & (G - 1))) + (ca & 1);
    const int cb0 = 9 * ib, pb0 = cb0 >> 1;
    const bool odd = cb0 & 1;
    int off_b[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) off_b[k] = ((pb0 + k) >> lg) * 32 + ((pb0 + k) & (G - 1));
    const size_t rstride = (size_t)KP * 64;
    const S* __restrict__ lmp = panel + at.base;
    const int r0 = damping ? 2 * n - 3 : 0, r1 = damping ? 2 * n : 2 * n - 3;
    S acc[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) acc[q] = 0;
#pragma unroll 3
    for (int r = r0; r < r1; ++r) {
      const S* row = lmp + (size_t)r * rstride;
      const V2* row2 = reinterpret_cast<const V2*>(row);
      const S va = __ldg(row + off_a);
      V2 b[5];
#pragma unroll
      for (int k = 0; k < 5; ++k) b[k] = __ldg(row2 + off_b[k]);
      const S el[10] = {b[0].x, b[0].y, b[1].x, b[1].y, b[2].x, b[2].y, b[3].x, b[3].y, b[4].x, b[4].y};
#pragma unroll
      for (int q = 0; q < 9; ++q) acc[q] = fma(va, odd ? el[q + 1] : el[q], acc[q]);
    }
    S* o = stage + 81 * (size_t)w + 9 * p;
#pragma unroll
    for (int q = 0; q < 9; ++q) o[q] = acc[q];
  }
}

// Thread per entry of a pair block (ca >= cb): `base` (the lambda-independent part S_u) or 0, plus the pair's staged terms
// in the pair's list order (landmark order); wpos[t] = landmark-major index of the pair-sorted term t.  The sum goes to
// out[81 pos.x] (pos == nullptr: out[81 bi], S_u), and off the diagonal its transpose to out[81 pos.y] (the full CSR).
template <class S>
__global__ void k_rcs_combine(const int* __restrict__ blk_ptr, const int* __restrict__ wpos, int nblk, const S* __restrict__ stage,
                              const S* __restrict__ base, const int2* __restrict__ pos, S* __restrict__ out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= 81LL * nblk) return;
  const int bi = (int)(i / 81), e = (int)(i - 81LL * bi);
  const S* st = stage + e;
  S s = base ? base[81 * (size_t)bi + e] : S(0);
  for (int t = blk_ptr[bi]; t < blk_ptr[bi + 1]; ++t) s += st[81 * (size_t)wpos[t]];
  const int2 ps = pos ? pos[bi] : make_int2(bi, -1);
  out[81 * (size_t)ps.x + e] = s;
  if (ps.y >= 0) out[81 * (size_t)ps.y + 9 * (e % 9) + e / 9] = s;
}

// y[9 row .. 9 row + 8] = sum over the blocks k of the row of S_k x[col_k]: CTA of 4 warps per block row, warp w takes the
// blocks k0 + w, k0 + w + 4, ... in that order, lane l entries l, l + 32, l + 64 of each 81-entry block (coalesced); the
// partial rows are added in shared memory in a fixed order (warp, then column).  A row without blocks (a camera without
// observations) gets y = 0.  In PCG it is launched dependent on the vector step and returns at once when the solve has
// ended (the `done` flag, as k_matvec_small_tma).
constexpr int SPMV_WARPS = 4;
constexpr int SPMV_UNROLL = 4;
template <class S>
__global__ void __launch_bounds__(SPMV_WARPS * 32) k_rcs_spmv(const int* __restrict__ row_ptr, const int* __restrict__ col,
                                                               const S* __restrict__ val, const S* __restrict__ x, S* __restrict__ y,
                                                               const int* done, int pdl) {
  __shared__ S part[SPMV_WARPS][81];
  if (done && *reinterpret_cast<const volatile int*>(done)) return;
  const int row = blockIdx.x, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = row_ptr[row], k1 = row_ptr[row + 1];
  int qe[3];
#pragma unroll
  for (int u = 0; u < 3; ++u) qe[u] = (lane + 32 * u) % 9;
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  if (done && *done) return;
  if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  S acc[3] = {0, 0, 0};
  for (int k = k0 + w; k < k1; k += SPMV_WARPS * SPMV_UNROLL) {
    S v[SPMV_UNROLL][3], xv[SPMV_UNROLL][3];
#pragma unroll
    for (int j = 0; j < SPMV_UNROLL; ++j) {
      const int kk = k + SPMV_WARPS * j;
      const bool in = kk < k1;
      const S* blk = val + 81 * (size_t)(in ? kk : k0);
      const S* xc = x + 9 * (size_t)(in ? __ldg(col + kk) : 0);
#pragma unroll
      for (int u = 0; u < 3; ++u) {
        const bool e_in = in && lane + 32 * u < 81;
        v[j][u] = e_in ? __ldg(blk + lane + 32 * u) : S(0);
        xv[j][u] = e_in ? __ldcg(xc + qe[u]) : S(0);
      }
    }
#pragma unroll
    for (int j = 0; j < SPMV_UNROLL; ++j)
#pragma unroll
      for (int u = 0; u < 3; ++u) acc[u] = fma(v[j][u], xv[j][u], acc[u]);
  }
#pragma unroll
  for (int u = 0; u < 3; ++u)
    if (lane + 32 * u < 81) part[w][lane + 32 * u] = acc[u];
  __syncthreads();
  if (threadIdx.x < 9) {
    const int p = threadIdx.x;
    S s = 0;
#pragma unroll
    for (int ww = 0; ww < SPMV_WARPS; ++ww)
#pragma unroll
      for (int q = 0; q < 9; ++q) s += part[ww][9 * p + q];
    y[9 * (size_t)row + p] = s;
  }
}

}  // namespace rba
