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
//   k_rcs_spmv      y = S x over a camera-major block-row CSR of the full matrix (both triangles, diagonal included), its
//                   rows dealt over one wave of persistent CTAs and S staged through shared memory by bulk copies.
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

// y = S x over the rows of the host's deal (deal_spmv, layout.hpp): a grid of co-resident CTAs of SPMV_CLASSES warps, each
// taking its chunks in order.  Thread 0 brings a chunk's blocks of S into one stage of an SPMV_NS-stage shared-memory ring
// with a cp.async.bulk copy (mbarrier complete_tx), under an L2 evict_last policy: S is read again by every later PCG
// iteration.  A bulk copy wants 16-byte addresses and sizes and a block is 81 scalars, so each copy starts at the 16-byte
// boundary at or below the chunk's first entry and its size is rounded up (the buffer of S ends in 16 bytes of padding);
// the stage is read from that offset.  x is gathered window by window: the col entries of a window of whole chunks (at
// most XWIN blocks, usually all of a CTA's chunks) into shared memory, then x[col] of all of them at once, so that the
// latency of the gathers is paid once per window and not once per chunk.  The first stages and the first window's col
// entries are requested before griddepcontrol.wait; only x and `done` are read after it.  That needs S and col written
// before the kernel right before this one: col and the deal are uploaded with the handle, and S is written by the
// assembly, after which the host launches the next k_rcs_spmv without PDL (Solver::s_fresh), so that stream order puts it
// after the assembly has completed.  Every later launch of the solve follows k_pcg_vec, with S unchanged since.  Warp c runs chain c (layout.hpp): blocks c, c + SPMV_CLASSES, ... of every chunk of the row in order, lane l
// entries l, l + 32, l + 64 of each block; at the row's last chunk the chains' partials are added in shared memory in the
// fixed order (chain, then column).  A row without blocks (a camera without observations) gets y = 0.  In PCG it is
// launched dependent on the vector step and returns at once when the solve has ended (the `done` flag, as
// k_matvec_small_tma).
constexpr int SPMV_NS = 3;
template <class S>
__global__ void __launch_bounds__(SPMV_CLASSES * 32) k_rcs_spmv(const SpmvChunk* __restrict__ chunks, const int* __restrict__ chunk_ptr,
                                                                 const int* __restrict__ col, const S* __restrict__ val,
                                                                 const S* __restrict__ x, S* __restrict__ y, const int* done, int pdl) {
  constexpr int CH = SPMV_STAGE_BYTES / (81 * (int)sizeof(S)), U = CH / SPMV_CLASSES;  // spmv_chunk_blocks
  constexpr int VB = CH * 81 * (int)sizeof(S) + 16;                                     // stage bytes, alignment slack included
  constexpr int XWIN = sizeof(S) == 4 ? 256 : 128;                                      // blocks per x window
  static_assert(CH % SPMV_CLASSES == 0 && VB % 16 == 0 && XWIN >= CH, "k_rcs_spmv stage layout");
  __shared__ __align__(128) unsigned char sval[SPMV_NS][VB];
  __shared__ S sx[XWIN * 9];
  __shared__ int scol[XWIN];
  __shared__ __align__(8) uint64_t bars[SPMV_NS];
  __shared__ S part[SPMV_CLASSES][81];
  __shared__ int quit;
  // `done` only ever goes 0 -> 1 inside one solve, and may do so while the vector step runs: thread 0 reads it once for
  // the whole CTA (a stale 0 is harmless, it is read again after griddepcontrol.wait)
  if (threadIdx.x == 0) {
    quit = done && *reinterpret_cast<const volatile int*>(done);
    if (!quit) {
      for (int s = 0; s < SPMV_NS; ++s) mbar_init(&bars[s], 1);
      mbar_fence_init();
    }
  }
  __syncthreads();
  if (quit) return;
  const int c0 = chunk_ptr[blockIdx.x], n = chunk_ptr[blockIdx.x + 1] - c0;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint64_t policy = l2_evict_last_policy();
  constexpr uintptr_t A16 = ~(uintptr_t)15;
  // (thread 0) chunk i into stage i % SPMV_NS.  An empty chunk copies nothing when its start is 16-byte aligned and the
  // 16 bytes at that boundary otherwise (inside the padding at the end of S when it is the last); nothing of it is read
  auto request = [&](int i) {
    const SpmvChunk ch = chunks[c0 + i];
    const int s = i % SPMV_NS;
    const uintptr_t v0 = (uintptr_t)(val + 81 * (size_t)ch.kb) & A16, v1 = ((uintptr_t)(val + 81 * (size_t)ch.ke) + 15) & A16;
    mbar_expect_tx(&bars[s], (uint32_t)(v1 - v0));
    if (v1 > v0) bulk_g2s(sval[s], (const void*)v0, (uint32_t)(v1 - v0), &bars[s], policy);
  };
  // the window from chunk i0: whole chunks while their blocks fit in XWIN; its col entries into scol (warp c takes chunks
  // c, c + SPMV_CLASSES, ... of it).  Returns its end and block count.
  auto window = [&](int i0, int& nblk) {
    int i = i0, off = 0;
    for (; i < n; ++i) {
      const SpmvChunk ch = chunks[c0 + i];
      const int nb = ch.ke - ch.kb;
      if (off + nb > XWIN) break;
      if ((i - i0) % SPMV_CLASSES == w)
        for (int t = lane; t < nb; t += 32) scol[off + t] = __ldg(col + ch.kb + t);
      off += nb;
    }
    nblk = off;
    return i;
  };
  // x[col] of the window's blocks into sx, all loads of a thread in flight together
  auto gather_x = [&](int nblk) {
    constexpr int B = 8;
    for (int t0 = threadIdx.x; t0 < 9 * nblk; t0 += B * SPMV_CLASSES * 32) {
      S v[B];
#pragma unroll
      for (int j = 0; j < B; ++j) {
        const int t = t0 + j * SPMV_CLASSES * 32;
        v[j] = t < 9 * nblk ? __ldcg(x + 9 * (size_t)scol[t / 9] + t % 9) : S(0);
      }
#pragma unroll
      for (int j = 0; j < B; ++j) {
        const int t = t0 + j * SPMV_CLASSES * 32;
        if (t < 9 * nblk) sx[t] = v[j];
      }
    }
  };
  const int primed = min(n, SPMV_NS);
  if (threadIdx.x == 0)
    for (int i = 0; i < primed; ++i) request(i);
  int nblk = 0;
  int wend = window(0, nblk);
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  if (done && *done) {
    // drain the bulk copies already in flight before the CTA may exit
    for (int i = 0; i < primed; ++i) mbar_wait(&bars[i], 0);
    return;
  }
  if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  __syncthreads();  // scol of the first window
  gather_x(nblk);
  __syncthreads();
  int qe[3];
#pragma unroll
  for (int u = 0; u < 3; ++u) qe[u] = (lane + 32 * u) % 9;
  S acc[3] = {0, 0, 0};
  for (int i = 0, jb = 0; i < n; ++i) {
    if (i == wend) {  // the next window (the last iteration ended in __syncthreads: scol and sx are free)
      wend = window(i, nblk);
      __syncthreads();
      gather_x(nblk);
      __syncthreads();
      jb = 0;
    }
    const SpmvChunk ch = chunks[c0 + i];
    const int s = i % SPMV_NS, nb = ch.ke - ch.kb;
    if (ch.flags & SPMV_FIRST) acc[0] = acc[1] = acc[2] = 0;
    mbar_wait(&bars[s], (i / SPMV_NS) & 1u);
    const S* vs = reinterpret_cast<const S*>(sval[s] + ((uintptr_t)(val + 81 * (size_t)ch.kb) & 15));
    const S* xs = sx + 9 * jb;
    S v[U][3], xv[U][3];
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const int b = w + SPMV_CLASSES * j;
#pragma unroll
      for (int u = 0; u < 3; ++u) {
        const bool e_in = b < nb && lane + 32 * u < 81;
        v[j][u] = e_in ? vs[81 * b + lane + 32 * u] : S(0);
        xv[j][u] = e_in ? xs[9 * b + qe[u]] : S(0);
      }
    }
#pragma unroll
    for (int j = 0; j < U; ++j)
      if (w + SPMV_CLASSES * j < nb) {
#pragma unroll
        for (int u = 0; u < 3; ++u) acc[u] = fma(v[j][u], xv[j][u], acc[u]);
      }
    jb += nb;
    if (ch.flags & SPMV_LAST) {
#pragma unroll
      for (int u = 0; u < 3; ++u)
        if (lane + 32 * u < 81) part[w][lane + 32 * u] = acc[u];
      __syncthreads();
      if (threadIdx.x < 9) {
        const int p = threadIdx.x;
        S t = 0;
#pragma unroll
        for (int c = 0; c < SPMV_CLASSES; ++c)
#pragma unroll
          for (int q = 0; q < 9; ++q) t += part[c][9 * p + q];
        y[9 * (size_t)ch.row + p] = t;
      }
    }
    __syncthreads();  // every warp is done with the stage (and with `part`) before the stage is requested again
    if (threadIdx.x == 0 && i + SPMV_NS < n) request(i + SPMV_NS);
  }
}

}  // namespace rba
