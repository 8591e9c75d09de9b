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
// Estimated extrinsics (rba_set_rig_sensors, DESIGN.md section 24) run in the SENS instances of these kernels, which take a
// SensorView: the sensor's pose sits in its home's entries 0..5 of u, and every camera j of the sensor adds Q~_j u_s.
#pragma once

#include <type_traits>

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

// Estimated extrinsics (rba_set_rig_sensors, DESIGN.md section 24), passed to the sensor instances of the rig kernels (the
// others take NoSensors, so that their parameters are those of section 23).  The lead of a rig is then its lowest-index
// camera with held extrinsics, first in its member list.  Sensor s has the home smem[sptr[s]] (its lowest-index camera),
// whose entries 0..5 of u carry the sensor's pose; every camera j of s moves by A_j d_lead + d_s.
template <class S>
struct SensorView {
  const int* home;   // [nc] the home of the camera's sensor, -1 = held extrinsics
  const int* sptr;   // [ns + 1] cameras of sensor s: smem[sptr[s] .. sptr[s + 1]), ascending, so the home first
  const int* smem;
  const double* K;   // [nc][7] E_lead(home) E_lead(j)^-1 of every sensor camera j (the identity for a home)
  S* qt;             // [nc][6] Q~_j = D_j^-1 D_s, diagonal (k_rig_scaling)
  S* ds;             // [ns][6] D_s
  const S* b;        // [9 nc] the copy of b that k_rig_precond reads
  const uint8_t* fixed;  // [nc] the tied mask (the homes' pose entries free), read by the covariance expansion
  int ns;
};
struct NoSensors {};
template <class S, bool SENS>
using SensorArg = std::conditional_t<SENS, SensorView<S>, NoSensors>;

// ---- poses in double: (qx, qy, qz, qw, tx, ty, tz), T(x) = R x + t ----
__device__ __forceinline__ void pose_mul(const double* a, const double* b, double* out) {  // a b
  out[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  out[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  out[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  out[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  const double x = a[0], y = a[1], z = a[2], w = a[3];
  const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                       2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                       2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
  for (int r = 0; r < 3; ++r) out[4 + r] = R[3 * r] * b[4] + R[3 * r + 1] * b[5] + R[3 * r + 2] * b[6] + a[4 + r];
}
__device__ __forceinline__ void pose_inv(const double* a, double* out) {
  const double q[7] = {-a[0], -a[1], -a[2], a[3], 0, 0, 0};
  double r[7];
  pose_mul(q, a, r);  // rotation R^T, translation R^T t
  for (int k = 0; k < 4; ++k) out[k] = q[k];
  for (int k = 0; k < 3; ++k) out[4 + k] = -r[4 + k];
}
template <class S>
__device__ __forceinline__ void load_pose(const S* cams, size_t cam, double* p) {
  for (int k = 0; k < 7; ++k) p[k] = (double)cams[10 * cam + k];
}
// M_j = T_home T_lead(home)^-1 K_j of sensor camera j from the current state, the quaternion normalised: the extrinsics
// E_s = T_home T_lead(home)^-1 E_lead(home) that the state defines, relative to j's lead
template <class S>
__device__ __forceinline__ void sensor_map(const S* cams, const RigView<S>& R, const SensorView<S>& Z, size_t cam, double* m) {
  const int h = Z.home[cam];
  double th[7], tl[7], il[7], hl[7];
  load_pose(cams, h, th);
  load_pose(cams, R.lead[h], tl);
  pose_inv(tl, il);
  pose_mul(th, il, hl);
  pose_mul(hl, Z.K + 7 * cam, m);
  const double n = 1.0 / sqrt(m[0] * m[0] + m[1] * m[1] + m[2] * m[2] + m[3] * m[3]);
  for (int k = 0; k < 4; ++k) m[k] *= n;
}

// linearize, after k_scaling and the priors' scaled blocks: D_u of every rig and P~ of its members.  Block per rig.
//   n_k^2 = sum_j (A_j e_k)^T G_j (A_j e_k) + sum over the directed pair edges (j, i) inside the rig of (A_j e_k)^T O_ji^u (A_i e_k)
// with G_j = D_j^-1 B_j D_j^-1 the member's unscaled pose Gram (B_j: `blocks`, the scaled observation Gram, + prior_H when
// given) and O^u = D_j^-1 O D_i^-1 the unscaled cross block of a pair prior (D.pair_O).  D_u,k = 1 / (eps + n_k) as k_scaling.
// SENS: blocks [nr, nr + ns) build D_s and Q~ of every sensor likewise, the sensor's column k being e_k on each of its cameras:
//   n_k^2 = sum_j G_j,kk + sum over the directed pair edges (j, i) between two cameras of the sensor of O^u_ji,kk
template <class S, bool SENS = false>
__global__ void __launch_bounds__(GROUP_THREADS) k_rig_scaling(const S* __restrict__ blocks, const S* __restrict__ prior_H,
                                                               DevPtrs<S> D, RigView<S> R, S eps,
                                                               SensorArg<S, SENS> Z) {
  if constexpr (SENS)
    if ((int)blockIdx.x >= R.nr) {
      const int sn = blockIdx.x - R.nr, m0 = Z.sptr[sn], m1 = Z.sptr[sn + 1];
      S s[6] = {0, 0, 0, 0, 0, 0};
      for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
        const size_t cam = Z.smem[q];
        const S* B = blocks + 81 * cam;
#pragma unroll
        for (int k = 0; k < 6; ++k) {
          const S dk = D.scaling[9 * cam + k];
          S t = (B[10 * k] + (prior_H ? prior_H[81 * cam + 10 * k] : S(0))) / (dk * dk);
          if (D.pair_ov)
            for (int e = D.pair_ptr[cam], e1 = D.pair_ptr[cam + 1]; e < e1; ++e) {
              const int nb = D.pair_nbr[e];
              if (Z.home[nb] != Z.home[cam]) continue;
              t += D.pair_O[36 * (size_t)e + 7 * k] / (dk * D.scaling[9 * (size_t)nb + k]);
            }
          s[k] += t;
        }
      }
      group_block_sum<S, 6>(s);
      S ds[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) ds[k] = S(1) / (eps + sqrt(s[k] > S(0) ? s[k] : S(0)));
      if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < 6; ++k) Z.ds[6 * (size_t)sn + k] = ds[k];
      for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
        const size_t cam = Z.smem[q];
#pragma unroll
        for (int k = 0; k < 6; ++k) Z.qt[6 * cam + k] = ds[k] / D.scaling[9 * cam + k];
      }
      return;
    }
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
// SENS: every camera j of a sensor adds Q~_j u_s, u_s the home's entries 0..5 of v, so out must not be v (the homes' entries
// are read across rigs).  host = 1: the home keeps its entries and u_s = (x_home - P~_home u_lead(home)) / Q~_home, which
// reads only leads' and homes' entries, neither of which is written, so out may be v.
template <class S, bool SENS = false>
__global__ void __launch_bounds__(GROUP_THREADS) k_rig_expand(const S* v, S* out, RigView<S> R, int nc, int ncb, int host,
                                                              const PcgState* st, SensorArg<S, SENS> Z) {
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
    S us[6] = {0, 0, 0, 0, 0, 0};
    if constexpr (SENS) {
      const int h = Z.home[cam];
      if (h >= 0) {
        if (host && h == (int)cam) continue;
        if (host) {
          const size_t hl = R.lead[h];
          S ul[6];
#pragma unroll
          for (int k = 0; k < 6; ++k) ul[k] = v[9 * hl + k] / R.pt[36 * hl + 7 * k];
#pragma unroll
          for (int a = 0; a < 6; ++a) {
            S t = v[9 * (size_t)h + a];
#pragma unroll
            for (int k = 0; k < 6; ++k) t -= R.pt[36 * (size_t)h + 6 * a + k] * ul[k];
            us[a] = t / Z.qt[6 * (size_t)h + a];
          }
        } else {
#pragma unroll
          for (int a = 0; a < 6; ++a) us[a] = v[9 * (size_t)h + a];
        }
#pragma unroll
        for (int a = 0; a < 6; ++a) us[a] *= Z.qt[6 * cam + a];
      }
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) {
      S t = 0;
#pragma unroll
      for (int k = 0; k < 6; ++k) t += P[6 * a + k] * x[k];
      if constexpr (SENS) t += us[a];
      out[9 * cam + a] = t;
    }
  }
}

// out = P~^T (y + A^T A ve + O ve) as k_group_contract: the rows of the full operator at the expanded vector ve, the
// members' pose rows contracted into the lead's (lead: sum_j P~_j^T row_j, the other members 0).  in == nullptr: the rows
// come from D (operator_row); else `in` holds them already (after k_group_contract) and only the rigs' pose rows are
// contracted, in place when out == in.  Blocks [0, ncb): thread per camera (rows of the free cameras and the rigged cameras'
// rows 6..8; nothing when in is given), blocks [ncb, ncb + nr): one per rig.
// SENS: blocks [ncb + nr, ncb + nr + ns) give each home's rows 0..5 u_s = sum_j Q~_j^T row_j over the sensor's cameras and
// the other cameras' 0; the rig blocks leave the sensor cameras' rows to them.  A camera's rows feed a rig block and a sensor
// block, so out must not be in: every block then reads rows no block writes.  The thread-per-camera blocks copy the rows
// they own when in is given.
template <class S, bool SENS = false>
__global__ void __launch_bounds__(GROUP_THREADS) k_rig_contract(DevPtrs<S> D, const S* __restrict__ ve, const S* in, S* out,
                                                                RigView<S> R, int ncb, const PcgState* st, SensorArg<S, SENS> Z) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (*reinterpret_cast<const volatile int*>(&st->done)) return;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  auto row = [&](size_t cam, int a) -> S { return in ? in[9 * cam + a] : operator_row(D, ve, cam, a); };
  if ((int)blockIdx.x < ncb) {
    const int cam = blockIdx.x * GROUP_THREADS + threadIdx.x;
    if (cam >= D.nc || (SENS ? in == out : in != nullptr)) return;
    for (int a = R.lead[cam] >= 0 ? 6 : 0; a < 9; ++a) out[9 * (size_t)cam + a] = row(cam, a);
    return;
  }
  if constexpr (SENS)
    if ((int)blockIdx.x >= ncb + R.nr) {
      const int sn = blockIdx.x - ncb - R.nr, m0 = Z.sptr[sn], m1 = Z.sptr[sn + 1];
      S s[6] = {0, 0, 0, 0, 0, 0};
      for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
        const size_t cam = Z.smem[q];
#pragma unroll
        for (int a = 0; a < 6; ++a) s[a] += Z.qt[6 * cam + a] * row(cam, a);
      }
      group_block_sum<S, 6>(s);
      for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS)
#pragma unroll
        for (int k = 0; k < 6; ++k) out[9 * (size_t)Z.smem[q] + k] = q == m0 ? s[k] : S(0);
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
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
    if constexpr (SENS)
      if (Z.home[R.mem[q]] >= 0) continue;
#pragma unroll
    for (int k = 0; k < 6; ++k) out[9 * (size_t)R.mem[q] + k] = q == m0 ? s[k] : S(0);
  }
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
// SENS: blocks [ncb + nr, ncb + nr + ns) put sum_j Q~_j B_j Q~_j (Q~ diagonal) and sum_j Q~_j (b_j + prior_g_j)[0..5] of
// each sensor into its home's pose entries and 0 into its other cameras'; the rig blocks leave the sensor cameras' pose
// entries to them.  A camera's pose block feeds a rig block and a sensor block, so every block reads src and Z.b, copies
// that no block writes (out and b are other buffers).
template <class S, bool SENS = false>
__global__ void __launch_bounds__(GROUP_THREADS) k_rig_precond(const S* src, const S* __restrict__ prior_H,
                                                               const S* __restrict__ prior_g, S* __restrict__ b, S* out,
                                                               RigView<S> R, int nc, int ncb, SensorArg<S, SENS> Z) {
  auto b_in = [&](size_t e) -> S {
    if constexpr (SENS) return Z.b[e];
    else return b[e];
  };
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
    if constexpr (SENS) {
      for (int d = rigged ? 6 : 0; d < 9; ++d) b[9 * (size_t)cam + d] = Z.b[9 * (size_t)cam + d] + (prior_g ? prior_g[9 * (size_t)cam + d] : S(0));
    } else if (prior_g) {
      for (int d = rigged ? 6 : 0; d < 9; ++d) b[9 * (size_t)cam + d] += prior_g[9 * (size_t)cam + d];
    }
    return;
  }
  if constexpr (SENS)
    if ((int)blockIdx.x >= ncb + R.nr) {
      const int sn = blockIdx.x - ncb - R.nr, m0 = Z.sptr[sn], m1 = Z.sptr[sn + 1];
      S s[27];  // [0, 21): the upper triangle of the sensor's pose block, row by row; [21, 27): its b
#pragma unroll
      for (int k = 0; k < 27; ++k) s[k] = 0;
      for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
        const size_t cam = Z.smem[q];
        const S* Q = Z.qt + 6 * cam;
#pragma unroll
        for (int i = 0; i < 6; ++i) {
#pragma unroll
          for (int k = i; k < 6; ++k)
            s[i * 6 - i * (i - 1) / 2 + (k - i)] +=
                Q[i] * (src[81 * cam + 9 * i + k] + (prior_H ? prior_H[81 * cam + 9 * i + k] : S(0))) * Q[k];
          s[21 + i] += Q[i] * (b_in(9 * cam + i) + (prior_g ? prior_g[9 * cam + i] : S(0)));
        }
      }
      group_block_sum<S, 27>(s);
      for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
        const size_t cam = Z.smem[q];
        const bool home = q == m0;
#pragma unroll
        for (int i = 0; i < 6; ++i) {
#pragma unroll
          for (int k = 0; k < 6; ++k) {
            const int lo = i < k ? i : k, hi = i < k ? k : i;
            out[81 * cam + 9 * i + k] = home ? s[lo * 6 - lo * (lo - 1) / 2 + (hi - lo)] : S(0);
          }
          b[9 * cam + i] = home ? s[21 + i] : S(0);
        }
      }
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
      for (int r = 0; r < 6; ++r) g += P[6 * r + k] * (b_in(9 * cam + r) + (prior_g ? prior_g[9 * cam + r] : S(0)));
      s[21 + k] += g;
    }
  }
  group_block_sum<S, 27>(s);  // every read above precedes its barriers, every write below follows them
  for (int q = m0 + threadIdx.x; q < m1; q += GROUP_THREADS) {
    const size_t cam = R.mem[q];
    if constexpr (SENS)
      if (Z.home[cam] >= 0) continue;
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
__device__ __forceinline__ void retie_pose(S* __restrict__ cams, int cam, int ld, const double* m) {
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
template <class S>
__global__ void k_rig_retie(S* __restrict__ cams, RigView<S> R, int nc) {
  const int cam = blockIdx.x * blockDim.x + threadIdx.x;
  if (cam >= nc) return;
  const int ld = R.lead[cam];
  if (ld < 0 || ld == cam) return;
  retie_pose(cams, cam, ld, R.M + 7 * (size_t)cam);
}
// with sensors (section 24), after every camera update and at every rba_set_state: a member with held extrinsics as
// k_rig_retie, a sensor camera other than the home at M_j = T_home T_lead(home)^-1 K_j from the state (sensor_map); the
// home keeps its pose, which defines E_s.  Reads only leads and homes, which it does not write.  Thread per camera.
template <class S>
__global__ void k_sensor_retie(S* __restrict__ cams, RigView<S> R, SensorView<S> Z, int nc) {
  const int cam = blockIdx.x * blockDim.x + threadIdx.x;
  if (cam >= nc) return;
  const int ld = R.lead[cam], h = Z.home[cam];
  if (ld < 0 || ld == cam || h == cam) return;
  double m[7];
  if (h >= 0) sensor_map(cams, R, Z, cam, m);
  else
    for (int k = 0; k < 7; ++k) m[k] = R.M[7 * (size_t)cam + k];
  retie_pose(cams, cam, ld, m);
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
// M_j and A_j of every sensor camera from the current state (sensor_map), ahead of k_rig_scaling and of the covariance
// passes: M in double, A_j rounded to S.  Thread per camera.
template <class S>
__global__ void k_sensor_tie(const S* __restrict__ cams, RigView<S> R, SensorView<S> Z, double* __restrict__ M, S* __restrict__ adj,
                             int nc) {
  const int cam = blockIdx.x * blockDim.x + threadIdx.x;
  if (cam >= nc || Z.home[cam] < 0) return;
  double m[7], A[36];
  sensor_map(cams, R, Z, cam, m);
  for (int k = 0; k < 7; ++k) M[7 * (size_t)cam + k] = m[k];
  rig_adjoint(m, A);
  for (int k = 0; k < 36; ++k) adj[36 * (size_t)cam + k] = (S)A[k];
}
// Row pass (thread per column i, which it alone touches) or column pass (thread per row i) over every rig's pose rows /
// columns, members in order: contract (expand = 0) adds A_j^T times the member's rows / columns 0..5 to the lead's, which
// applied as rows then columns gives P^T A P; expand (expand = 1) sets the member's to A_j times the lead's, which applied to
// the (un-equilibrated) inverse gives P A P^T.  The full symmetric matrix is read (k_cov_group_symmetrize first).
// SENS (section 24, M_j of the sensor cameras from k_sensor_tie): contract then sums every sensor's rows / columns into its
// home's, after the rigs' pass, which writes only leads; expand adds the home's to every camera of the sensor, the homes
// last, so that each reads the home's contracted entries.  The inverse holds identity rows at held entries (k_cov_equil);
// a sensor camera of a held rig is not held, so expand reads a held lead's entries as 0.
template <class S, bool SENS = false>
__global__ void k_cov_rig_pass(double* __restrict__ A, long long ld, long long n, RigView<S> R, int columns, int expand,
                               SensorArg<S, SENS> Z) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  auto at = [&](long long j) -> double& { return columns ? A[i + j * ld] : A[j + i * ld]; };
  for (int r = 0; r < R.nr; ++r) {
    const int m0 = R.ptr[r], m1 = R.ptr[r + 1];
    const long long lead = 9LL * R.mem[m0];
    double x[6];
    for (int k = 0; k < 6; ++k) x[k] = at(lead + k);
    if constexpr (SENS)
      if (expand)
        for (int k = 0; k < 6; ++k)
          if ((fixed_entry_mask(Z.fixed[lead / 9]) >> k) & 1u) x[k] = 0.0;
    for (int q = m0 + 1; q < m1; ++q) {
      const long long cam = R.mem[q];
      if constexpr (SENS)
        if (expand && Z.home[cam] == cam) continue;
      double Aj[36];
      rig_adjoint(R.M + 7 * cam, Aj);
      if (expand) {
        for (int a = 0; a < 6; ++a) {
          double t = 0;
          for (int b = 0; b < 6; ++b) t += Aj[6 * a + b] * x[b];
          if constexpr (SENS)
            if (Z.home[cam] >= 0) t += at(9LL * Z.home[cam] + a);
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
  if constexpr (SENS)
    for (int sn = 0; sn < Z.ns; ++sn) {
      const int m0 = Z.sptr[sn], m1 = Z.sptr[sn + 1];
      const long long h = Z.smem[m0];
      double x[6];
      for (int k = 0; k < 6; ++k) x[k] = at(9 * h + k);
      if (expand) {  // the home: A_home times its lead's entries plus the sensor's
        const long long hl = 9LL * R.lead[h];
        const unsigned lf = fixed_entry_mask(Z.fixed[R.lead[h]]);
        double Aj[36];
        rig_adjoint(R.M + 7 * h, Aj);
        for (int a = 0; a < 6; ++a) {
          double t = x[a];
          for (int b = 0; b < 6; ++b)
            if (!((lf >> b) & 1u)) t += Aj[6 * a + b] * at(hl + b);
          at(9 * h + a) = t;
        }
      } else {
        for (int q = m0 + 1; q < m1; ++q)
          for (int k = 0; k < 6; ++k) x[k] += at(9LL * Z.smem[q] + k);
        for (int k = 0; k < 6; ++k) at(9 * h + k) = x[k];
      }
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
