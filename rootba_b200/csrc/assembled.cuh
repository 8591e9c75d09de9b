// The reduced camera matrix S = sum_l P_l^T P_l assembled from the Q2 panels P_l, and its block-row product (DESIGN.md
// section 4, "Assembled operator").  With one GPU and operator_form = DENSE the PCG operator is applied as (P^T P) x
// instead of P^T (P x): the same products of panel entries, associated differently, and S (9 x 9 blocks over the
// co-visible camera pairs) is several times smaller than the panels it is built from.
//   k_rcs_terms     once per linearisation: S_u = sum over panel rows 0..2n-4 (lambda-independent, the reference's rows
//   k_rcs_combine   3..2n-1 of the landmark block).  The 9 x 9 block of every term (slot_a, slot_b) of every landmark is
//                   evaluated landmark by landmark into a staging buffer that holds all of them, then every co-visible
//                   camera pair (ca >= cb) adds its terms in the order of the host-built list (build_pair_list,
//                   layout.hpp): no atomics, fixed order.
//   k_rcs_damping   once per solve that reaches iteration asm_switch: S = S_u + sum over the three damping rows that
//   k_rcs_mirror    k_stage2 has just written, every term formed from the two slots' dmp records (no staging), added in
//                   the same list order; then the upper blocks as transposes of the lower ones.
//                   All four return at once when the solve has ended before.
//   k_rcs_spmv      y = S x over a camera-major block-row CSR of the full matrix (both triangles, diagonal included).
#pragma once

#include "kernels.cuh"

namespace rba {

// Landmark-major evaluation of the nt terms (landmarks in problem order): warp per three consecutive terms, lane 9 g + p
// (g = 0..2, p = 0..8; lanes 27..31 idle) computes row p of the 9 x 9 block of term 3 k + g over the panel rows
// [0, 2n - 3) (damping = 0: the lambda-independent rows, the only range that is launched) or [2n - 3, 2n) (damping = 1)
// into stage[81 w].  Neighbouring warps read the same landmark's panel, so it is read from HBM about once.  (The row range
// stays a run-time argument: with the bounds fixed at compile time ptxas allots 56 registers instead of 44 in float32 and
// the kernel is a sixth slower, DESIGN.md section 11 item 6.)
// Block entry (p, q) = sum_r P[r][9 ia + p] P[r][9 ib + q]; on the diagonal (sa == sb) it is symmetric bit for bit (fma
// commutes).  Enqueued by the host ahead of PCG iteration asm_switch, after the vector step of the iteration before, so it
// reads the solve's `done` flag in stream order and returns at once when the solve has already ended (as k_rcs_combine).
template <class S>
__global__ void __launch_bounds__(256) k_rcs_terms(const S* __restrict__ panel, const AsmTerm* __restrict__ terms, long long nt,
                                                   int damping, S* __restrict__ stage, const int* __restrict__ done) {
  using V2 = typename ST<S>::V2;
  if (*done) return;
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

// S_u: thread per entry of a pair block (ca >= cb), the pair's staged terms added in the pair's list order (landmark
// order); wpos[t] = landmark-major index of the pair-sorted term t.  Nothing is written when the solve has ended (`done`).
template <class S>
__global__ void k_rcs_combine(const int* __restrict__ blk_ptr, const int* __restrict__ wpos, int nblk, const S* __restrict__ stage,
                              S* __restrict__ out, const int* __restrict__ done) {
  if (*done) return;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= 81LL * nblk) return;
  const int bi = (int)(i / 81), e = (int)(i - 81LL * bi);
  const S* st = stage + e;
  S s = 0;
  for (int t = blk_ptr[bi]; t < blk_ptr[bi + 1]; ++t) s += st[81 * (size_t)wpos[t]];
  out[i] = s;
}

// S = S_u + the damping rows' part, lower blocks: warp per pair block (ca >= cb).  The damping rows of a slot are the 3 x 9
// record dmp[slot] (k_stage2 writes the same values into the panel rows 2n-3..2n-1), so a term (slot_a, slot_b) is formed
// from two records instead of being staged: entry (p, q) = fma over d = 0, 1, 2 of a[d][p] b[d][q] starting from 0, added
// to the entry in the pair's list order -- the arithmetic of k_rcs_terms(damping rows) + k_rcs_combine, bit for bit.  The
// records of DMP_BATCH terms are fetched together (16-byte loads, all in flight) into shared memory; lane l < 27 owns the
// entries (l / 3, 3 (l % 3) + 0..2).  Written to out[81 pos.x]; k_rcs_mirror fills the upper blocks.
constexpr int DMP_WARPS = 4;
constexpr int DMP_BATCH = 16;
template <class S>
__global__ void __launch_bounds__(DMP_WARPS * 32) k_rcs_damping(const int* __restrict__ blk_ptr, const int2* __restrict__ terms, int nblk,
                                                                 const S* __restrict__ dmp, const S* __restrict__ base,
                                                                 const int2* __restrict__ pos, S* __restrict__ out,
                                                                 const int* __restrict__ done) {
  constexpr int B = DMP_BATCH, NV = 28 * sizeof(S) / 16;  // 16-byte vectors per record
  constexpr int ROUNDS = (2 * B * NV + 31) / 32;
  __shared__ __align__(16) S rec[DMP_WARPS][B][2][28];
  if (*done) return;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int bi = blockIdx.x * DMP_WARPS + w;
  if (bi >= nblk) return;
  const bool own = lane < 27;
  const int p = lane / 3, q = 3 * (lane - 3 * p);
  S s[3] = {0, 0, 0};
  if (own) {
#pragma unroll
    for (int u = 0; u < 3; ++u) s[u] = base[81 * (size_t)bi + 3 * lane + u];
  }
  int4* rv = reinterpret_cast<int4*>(&rec[w][0][0][0]);
  const int t1 = blk_ptr[bi + 1];
  for (int t0 = blk_ptr[bi]; t0 < t1; t0 += B) {
    const int nb = min(B, t1 - t0);
    int4 v[ROUNDS];
#pragma unroll
    for (int c = 0; c < ROUNDS; ++c) {
      const int i = lane + 32 * c, r = i / NV, k = i - r * NV;  // record r = 2 term + (0: slot_a, 1: slot_b), vector k of it
      v[c] = make_int4(0, 0, 0, 0);
      if (i < 2 * nb * NV) {
        const int2 tt = __ldg(terms + t0 + (r >> 1));
        v[c] = __ldg(reinterpret_cast<const int4*>(dmp + 28 * (size_t)(r & 1 ? tt.y : tt.x)) + k);
      }
    }
#pragma unroll
    for (int c = 0; c < ROUNDS; ++c)
      if (lane + 32 * c < 2 * nb * NV) rv[lane + 32 * c] = v[c];
    __syncwarp();
    if (own) {
      for (int j = 0; j < nb; ++j) {
        const S* a = rec[w][j][0];
        const S* b = rec[w][j][1];
#pragma unroll
        for (int u = 0; u < 3; ++u) {
          S t = fma(a[p], b[q + u], S(0));
          t = fma(a[9 + p], b[9 + q + u], t);
          t = fma(a[18 + p], b[18 + q + u], t);
          s[u] += t;
        }
      }
    }
    __syncwarp();
  }
  if (own) {
    S* o = out + 81 * (size_t)pos[bi].x + 3 * lane;
#pragma unroll
    for (int u = 0; u < 3; ++u) o[u] = s[u];
  }
}

// The upper blocks of S: thread per entry of an off-diagonal pair, the transpose of its lower block (written by
// k_rcs_damping) into val[81 pos.y].
template <class S>
__global__ void k_rcs_mirror(const int2* __restrict__ pos, int nblk, S* val, const int* __restrict__ done) {
  if (*done) return;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= 81LL * nblk) return;
  const int bi = (int)(i / 81), e = (int)(i - 81LL * bi);
  const int2 ps = pos[bi];
  if (ps.y >= 0) val[81 * (size_t)ps.y + e] = val[81 * (size_t)ps.x + 9 * (e % 9) + e / 9];
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
