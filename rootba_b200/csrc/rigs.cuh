// Rigid camera rigs (rba_set_camera_rigs, DESIGN.md section 23).
// A rig is one placement of a rigid multi-camera body; its lead is its lowest-index camera and every member j is kept at
// T_j = M_j T_lead, M_j = E_j E_lead^-1 from the fixed extrinsics E (cam_from_rig).  A lead increment d moves member j by
// A_j d to first order, A_j = [[R_m, [t_m]x R_m], [0, R_m]] on (v, w).  The tied problem has one pose per rig and every
// camera's own intrinsics; its vectors u are kept in the 9 nc layout with the rig's pose in the lead's entries 0..5 and the
// other members' entries 0..5 held at zero.  In the x-space of the per-camera Jacobi scaling D the map is
// P~_j = D_j^-1 A_j D_u (P~_lead = D_lead^-1 D_u), D_u the Jacobi scaling of the merged pose columns, so that
// D_u P^T H P D_u = P~^T K P~ with K the existing x-space operator.  These kernels build D_u and P~ once per linearisation,
// apply P~ (expand) and P~^T (contract) around the unchanged operator kernels, merge the preconditioner blocks and re-tie
// the members' poses after every update.  Only rigs of >= 2 cameras exist here: a rig of one is a free camera.  Every sum
// over a rig runs in a fixed order (members ascending per thread, then the fixed tree of group_block_sum), so the results
// are deterministic.
#pragma once

#include "groups.cuh"

namespace rba {

template <class S>
struct RigView {
  const int* lead;   // [nc] the lead of the camera's rig, -1 = a free camera
  const int* ptr;    // [nr + 1] members of rig r: mem[ptr[r] .. ptr[r + 1]), ascending, so the lead first
  const int* mem;
  const S* adj;      // [nc][36] A_j row-major (the identity for a lead), rigged cameras only
  const double* M;   // [nc][7] M_j = (qx, qy, qz, qw, tx, ty, tz), rigged cameras only
  S* pt;             // [nc][36] P~_j row-major, rigged cameras only (k_rig_scaling)
  S* du;             // [nr][6] D_u
  int nr;
};

// linearize, after k_scaling and the priors' scaled blocks: D_u of every rig and P~ of its members.  Block per rig.
//   n_k^2 = sum_j (A_j e_k)^T G_j (A_j e_k) + sum over the directed pair edges (j, i) inside the rig of (A_j e_k)^T O_ji^u (A_i e_k)
// with G_j = D_j^-1 B_j D_j^-1 the member's unscaled pose Gram (B_j: `blocks`, the scaled observation Gram, + prior_H when
// given) and O^u = D_j^-1 O D_i^-1 the unscaled cross block of a pair prior (D.pair_O).  D_u,k = 1 / (eps + n_k) as k_scaling.
template <class S>
__global__ void __launch_bounds__(GROUP_THREADS) k_rig_scaling(const S* __restrict__ blocks, const S* __restrict__ prior_H,
                                                               DevPtrs<S> D, RigView<S> R, S eps) {
  const int m0 = R.ptr[blockIdx.x], m1 = R.ptr[blockIdx.x + 1];
  const int lead = R.mem[m0];
  // (A_j e_k) / D_j of camera cam, entry r
  auto w = [&](int cam, int r, int k) -> S { return R.adj[36 * (size_t)cam + 6 * r + k] / D.scaling[9 * (size_t)cam + r]; };
  S s[6] = {0, 0, 0, 0, 0, 0};
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
    const int cam = R.mem[q];
    const S* B = blocks + 81 * (size_t)cam;
    const S* H = prior_H ? prior_H + 81 * (size_t)cam : nullptr;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      S wk[6];
#pragma unroll
      for (int r = 0; r < 6; ++r) wk[r] = w(cam, r, k);
      S t = 0;
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int c = 0; c < 6; ++c) t += wk[r] * (B[9 * r + c] + (H ? H[9 * r + c] : S(0))) * wk[c];
      if (D.pair_ov)
        for (int e = D.pair_ptr[cam], e1 = D.pair_ptr[cam + 1]; e < e1; ++e) {
          const int nb = D.pair_nbr[e];
          if (R.lead[nb] != lead) continue;
          const S* O = D.pair_O + 36 * (size_t)e;
#pragma unroll
          for (int r = 0; r < 6; ++r)
#pragma unroll
            for (int c = 0; c < 6; ++c) t += wk[r] * O[6 * r + c] * w(nb, c, k);
        }
      s[k] += t;
    }
  }
  group_block_sum<S, 6>(s);
  S du[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) du[k] = S(1) / (eps + sqrt(s[k] > S(0) ? s[k] : S(0)));
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < 6; ++k) R.du[6 * (size_t)blockIdx.x + k] = du[k];
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
    const size_t cam = R.mem[q];
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
      for (int k = 0; k < 6; ++k) R.pt[36 * cam + 6 * r + k] = R.adj[36 * cam + 6 * r + k] * du[k] / D.scaling[9 * cam + r];
  }
}

// out = P~ v: every member's entries 0..5 (the lead's included) become P~_j times the lead's entries 0..5 of v; entries
// 6..8 and the free cameras are copied.  host = 1 (a host increment given to rba_apply): the lead keeps its entries x and
// the other members take D_j^-1 A_j D_lead x = P~_j (x / diag P~_lead).  out may be v: a rig's block reads the lead's
// entries before its barrier and writes after it.  Blocks [0, ncb): thread per camera (the copies), blocks
// [ncb, ncb + nr): one per rig.  In a solve (st set) it is launched dependent on its predecessor and returns once the
// solve has ended, like k_group_expand.
template <class S>
__global__ void __launch_bounds__(GROUP_THREADS) k_rig_expand(const S* v, S* out, RigView<S> R, int nc, int ncb, int host,
                                                              const PcgState* st) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (st && *reinterpret_cast<const volatile int*>(&st->done)) return;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if ((int)blockIdx.x < ncb) {
    const int cam = blockIdx.x * GROUP_THREADS + threadIdx.x;
    if (cam >= nc || out == v) return;
    for (int a = R.lead[cam] >= 0 ? 6 : 0; a < 9; ++a) out[9 * (size_t)cam + a] = v[9 * (size_t)cam + a];
    return;
  }
  const int r = blockIdx.x - ncb;
  const int m0 = R.ptr[r], m1 = R.ptr[r + 1];
  const size_t ld = R.mem[m0];
  S x[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) x[k] = v[9 * ld + k] / (host ? R.pt[36 * ld + 7 * k] : S(1));
  __syncthreads();
  for (int q = m0 + (host ? 1 : 0) + threadIdx.x; q < m1; q += GROUP_THREADS) {
    const size_t cam = R.mem[q];
    const S* P = R.pt + 36 * cam;
#pragma unroll
    for (int a = 0; a < 6; ++a) {
      S t = 0;
#pragma unroll
      for (int k = 0; k < 6; ++k) t += P[6 * a + k] * x[k];
      out[9 * cam + a] = t;
    }
  }
}

// out = P~^T (y + A^T A ve + O ve) as k_group_contract: the rows of the full operator at the expanded vector ve, the
// members' pose rows contracted into the lead's (lead: sum_j P~_j^T row_j, the other members 0).  in == nullptr: the rows
// come from D (operator_row); else `in` holds them already (after k_group_contract) and only the rigs' pose rows are
// contracted, in place when out == in.  Blocks [0, ncb): thread per camera (rows of the free cameras and the rigged cameras'
// rows 6..8; nothing when in is given), blocks [ncb, ncb + nr): one per rig.
template <class S>
__global__ void __launch_bounds__(GROUP_THREADS) k_rig_contract(DevPtrs<S> D, const S* __restrict__ ve, const S* in, S* out,
                                                                RigView<S> R, int ncb, const PcgState* st) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (*reinterpret_cast<const volatile int*>(&st->done)) return;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  auto row = [&](size_t cam, int a) -> S { return in ? in[9 * cam + a] : operator_row(D, ve, cam, a); };
  if ((int)blockIdx.x < ncb) {
    const int cam = blockIdx.x * GROUP_THREADS + threadIdx.x;
    if (cam >= D.nc || in) return;
    for (int a = R.lead[cam] >= 0 ? 6 : 0; a < 9; ++a) out[9 * (size_t)cam + a] = row(cam, a);
    return;
  }
  const int r = blockIdx.x - ncb;
  const int m0 = R.ptr[r], m1 = R.ptr[r + 1];
  S s[6] = {0, 0, 0, 0, 0, 0};
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
    const size_t cam = R.mem[q];
    S y[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) y[a] = row(cam, a);
    const S* P = R.pt + 36 * cam;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
      for (int k = 0; k < 6; ++k) s[k] += P[6 * a + k] * y[a];
  }
  group_block_sum<S, 6>(s);  // every read above precedes its barriers, every write below follows them
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS)
#pragma unroll
    for (int k = 0; k < 6; ++k) out[9 * (size_t)R.mem[q] + k] = q == m0 ? s[k] : S(0);
}

// solve, ahead of k_precond_invert: the preconditioner blocks in the block partition of the tied problem and the contracted
// gradient.  Blocks [0, ncb): thread per camera, blocks [ncb, ncb + nr): one per rig.
//   free camera:     out = src (+ prior_H), b += prior_g
//   rigged camera:   intrinsics 3x3 of out = that of src (+ prior_H), pose-intrinsics entries 0, b[6..8] += prior_g[6..8]
//   rig:             the lead's pose 6x6 = sum_j P~_j^T B_j P~_j with B_j the member's pose 6x6 of src (+ prior_H), its
//                    b[0..5] = sum_j P~_j^T (b_j + prior_g_j)[0..5]; the other members' pose entries of out and b are 0
// The cross terms between members of one rig are not in the per-camera blocks and stay out.  k_precond_invert then adds
// lambda once per parameter of the tied problem and masks the members' entries 0..5 as held.  The two roles touch disjoint
// entries, so out may be src (SCHUR_JACOBI, and after k_group_precond).
template <class S>
__global__ void __launch_bounds__(GROUP_THREADS) k_rig_precond(const S* src, const S* __restrict__ prior_H,
                                                               const S* __restrict__ prior_g, S* __restrict__ b, S* out,
                                                               RigView<S> R, int nc, int ncb) {
  if ((int)blockIdx.x < ncb) {
    const int cam = blockIdx.x * GROUP_THREADS + threadIdx.x;
    if (cam >= nc) return;
    const bool rigged = R.lead[cam] >= 0;
    const size_t o = 81 * (size_t)cam;
    for (int r = 0; r < 9; ++r)
      for (int c = 0; c < 9; ++c) {
        if (rigged && r < 6 && c < 6) continue;
        S a = src[o + 9 * r + c];
        if (prior_H) a += prior_H[o + 9 * r + c];
        out[o + 9 * r + c] = (rigged && (r < 6) != (c < 6)) ? S(0) : a;
      }
    if (prior_g)
      for (int d = rigged ? 6 : 0; d < 9; ++d) b[9 * (size_t)cam + d] += prior_g[9 * (size_t)cam + d];
    return;
  }
  const int rg = blockIdx.x - ncb;
  const int m0 = R.ptr[rg], m1 = R.ptr[rg + 1];
  S s[27];  // [0, 21): the upper triangle of the rig's pose block, row by row; [21, 27): its b
#pragma unroll
  for (int k = 0; k < 27; ++k) s[k] = 0;
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
    const size_t cam = R.mem[q];
    const S* P = R.pt + 36 * cam;
    auto B = [&](int r, int c) -> S { return src[81 * cam + 9 * r + c] + (prior_H ? prior_H[81 * cam + 9 * r + c] : S(0)); };
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      S bp[6];  // B_j P~_j e_k
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        S t = 0;
#pragma unroll
        for (int c = 0; c < 6; ++c) t += B(r, c) * P[6 * c + k];
        bp[r] = t;
      }
      // entry (i, k), i <= k, of P~^T B P~
#pragma unroll
      for (int i = 0; i <= k; ++i) {
        S t = 0;
#pragma unroll
        for (int r = 0; r < 6; ++r) t += P[6 * r + i] * bp[r];
        s[i * 6 - i * (i - 1) / 2 + (k - i)] += t;
      }
      S g = 0;
#pragma unroll
      for (int r = 0; r < 6; ++r) g += P[6 * r + k] * (b[9 * cam + r] + (prior_g ? prior_g[9 * cam + r] : S(0)));
      s[21 + k] += g;
    }
  }
  group_block_sum<S, 27>(s);  // every read above precedes its barriers, every write below follows them
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
    const size_t cam = R.mem[q];
    const bool lead = q == m0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        const int lo = i < k ? i : k, hi = i < k ? k : i;
        out[81 * cam + 9 * i + k] = lead ? s[lo * 6 - lo * (lo - 1) / 2 + (hi - lo)] : S(0);
      }
      b[9 * cam + i] = lead ? s[21 + i] : S(0);
    }
  }
}

// every member's pose := M_j T_lead (R = R_m R_lead, t = R_m t_lead + t_m), in double, the quaternion normalised, rounded to
// S.  Deterministic, so replicated cameras stay bit-identical across ranks.  Thread per camera.
template <class S>
__global__ void k_rig_retie(S* __restrict__ cams, RigView<S> R, int nc) {
  const int cam = blockIdx.x * blockDim.x + threadIdx.x;
  if (cam >= nc) return;
  const int ld = R.lead[cam];
  if (ld < 0 || ld == cam) return;
  const double* m = R.M + 7 * (size_t)cam;
  const S* cl = cams + 10 * (size_t)ld;
  const double a0 = m[0], a1 = m[1], a2 = m[2], a3 = m[3];
  const double b0 = cl[0], b1 = cl[1], b2 = cl[2], b3 = cl[3];
  double q[4];
  q[3] = a3 * b3 - a0 * b0 - a1 * b1 - a2 * b2;
  q[0] = a3 * b0 + a0 * b3 + a1 * b2 - a2 * b1;
  q[1] = a3 * b1 + a1 * b3 + a2 * b0 - a0 * b2;
  q[2] = a3 * b2 + a2 * b3 + a0 * b1 - a1 * b0;
  const double n = 1.0 / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  // R_m from the unit quaternion of M (normalised on the host)
  const double Rm[9] = {1 - 2 * (a1 * a1 + a2 * a2), 2 * (a0 * a1 - a2 * a3), 2 * (a0 * a2 + a1 * a3),
                        2 * (a0 * a1 + a2 * a3), 1 - 2 * (a0 * a0 + a2 * a2), 2 * (a1 * a2 - a0 * a3),
                        2 * (a0 * a2 - a1 * a3), 2 * (a1 * a2 + a0 * a3), 1 - 2 * (a0 * a0 + a1 * a1)};
  const double t0 = cl[4], t1 = cl[5], t2 = cl[6];
  S* cm = cams + 10 * (size_t)cam;
#pragma unroll
  for (int k = 0; k < 4; ++k) cm[k] = (S)(q[k] * n);
#pragma unroll
  for (int r = 0; r < 3; ++r) cm[4 + r] = (S)(Rm[3 * r] * t0 + Rm[3 * r + 1] * t1 + Rm[3 * r + 2] * t2 + m[4 + r]);
}

// ---- rba_compute_covariance (DESIGN.md sections 16 and 23) on the dense np x np column-major matrix A (ld) ----
// A_j of M_j in double, row-major 6x6
__device__ __forceinline__ void rig_adjoint(const double* __restrict__ m, double (&A)[36]) {
  const double x = m[0], y = m[1], z = m[2], w = m[3];
  const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                       2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                       2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
  const double tx[9] = {0, -m[6], m[5], m[6], 0, -m[4], -m[5], m[4], 0};
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 3; ++k) {
      double t = 0;
      for (int i = 0; i < 3; ++i) t += tx[3 * r + i] * R[3 * i + k];
      A[6 * r + k] = R[3 * r + k];
      A[6 * r + 3 + k] = t;
      A[6 * (3 + r) + k] = 0.0;
      A[6 * (3 + r) + 3 + k] = R[3 * r + k];
    }
}
// Row pass (thread per column i, which it alone touches) or column pass (thread per row i) over every rig's pose rows /
// columns, members in order: contract (expand = 0) adds A_j^T times the member's rows / columns 0..5 to the lead's, which
// applied as rows then columns gives P^T A P; expand (expand = 1) sets the member's to A_j times the lead's, which applied to
// the (un-equilibrated) inverse gives P A P^T.  The full symmetric matrix is read (k_cov_group_symmetrize first).
template <class S>
__global__ void k_cov_rig_pass(double* __restrict__ A, long long ld, long long n, RigView<S> R, int columns, int expand) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  auto at = [&](long long j) -> double& { return columns ? A[i + j * ld] : A[j + i * ld]; };
  for (int r = 0; r < R.nr; ++r) {
    const int m0 = R.ptr[r], m1 = R.ptr[r + 1];
    const long long lead = 9LL * R.mem[m0];
    double x[6];
    for (int k = 0; k < 6; ++k) x[k] = at(lead + k);
    for (int q = m0 + 1; q < m1; ++q) {
      const long long cam = R.mem[q];
      double Aj[36];
      rig_adjoint(R.M + 7 * cam, Aj);
      if (expand) {
        for (int a = 0; a < 6; ++a) {
          double t = 0;
          for (int b = 0; b < 6; ++b) t += Aj[6 * a + b] * x[b];
          at(9 * cam + a) = t;
        }
      } else {
        double y[6];
        for (int b = 0; b < 6; ++b) y[b] = at(9 * cam + b);
        for (int a = 0; a < 6; ++a) {
          double t = 0;
          for (int b = 0; b < 6; ++b) t += Aj[6 * b + a] * y[b];
          x[a] += t;
        }
      }
    }
    if (!expand)
      for (int k = 0; k < 6; ++k) at(lead + k) = x[k];
  }
}
// the inverse of the equilibrated matrix back to the inverse of the matrix itself on the leading n x n (full) part, so that the
// expansion through the unscaled A_j agrees with the equilibration: A <- D A D, then d <- 1 (k_cov_unit_d)
__global__ void k_cov_unequil(double* __restrict__ A, long long ld, long long n, const double* __restrict__ d) {
  const long long r = blockIdx.x * 32LL + threadIdx.x;
  const long long c = blockIdx.y * 8LL + threadIdx.y;
  if (r < n && c < n) A[r + c * ld] *= d[r] * d[c];
}
__global__ void k_cov_unit_d(double* __restrict__ d, long long n) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k < n) d[k] = 1.0;
}

}  // namespace rba
