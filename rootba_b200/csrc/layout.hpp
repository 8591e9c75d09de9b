// Host-side data model: landmark sharding, track-length classes, warp tiles, matvec work items,
// the camera-major CSR used by the deterministic scatter (two-phase reduction), the co-visible camera
// pairs and the structure of the assembled reduced camera matrix.
//
// Replaces (reference, relative to src/rootba/):
//   qr/landmark_block.cpp:51-80      LandmarkBlockFactory: static classes n=2..8 + dynamic
//   qr/linearization_qr.hpp:80-111   LinearizationQR ctor: allocate every block, prefix sums
// Pure C++ (no CUDA) so it is unit-testable on a CPU-only box.
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <limits>
#include <numeric>
#include <string>
#include <utility>
#include <vector>

namespace rba {

// One warp works on a tile of W = 32/G landmarks that all have the same track length n.  Each landmark
// is owned by a group of G lanes; lane j of the group owns the 2*KP panel columns
//     c(k, v) = 2*j + 2*G*k + v,   k = 0..KP-1, v = 0,1          (columns >= 9n are zero padding)
// so that for a fixed k a warp-wide 2-scalar vector load covers 64 consecutive scalars of the tile:
//     panel[tile] layout = [2n rows][KP steps][32 lanes][2]       (fully coalesced 256 B / 512 B requests)
struct TileInfo {
  long long panel_off;  // scalar offset of the tile's panel
  int slot_base;        // first observation slot of the tile; landmark g owns slots slot_base + g*n .. +n
  int lm_base;          // index into sorted_lm of landmark g = 0
  short n;              // track length of every landmark of the tile
  short G;              // lanes per landmark (power of two)
  short KP;             // column pairs per lane
  short nvalid;         // real landmarks in the tile (<= 32/G); the rest are padding
};

// rcs_matvec work item: a row range of one tile.  Rows are independent (y = sum_r P_r^T (P_r x)), so long
// tracks are split across warps; every chunk writes its own y slots (deterministic, no atomics).
struct MatvecItem {
  int tile;
  short row0, nrows;
  int yslot_base;  // landmark g writes y slots yslot_base + g*n .. +n (9 scalars each)
  int pad;
};

// segment of a camera's slot list, reduced by one warp
struct ReduceItem {
  int cam, begin, end;
};

struct CameraCSR {
  std::vector<int> cam_ptr;        // [nc + 1] into slots
  std::vector<int> slots;          // slot ids, ascending per camera
  std::vector<ReduceItem> items;   // segments of <= seg_len entries
  std::vector<int> cam_item_ptr;   // [nc + 1] into items
};

struct Layout {
  int nc = 0;
  int lm_begin = 0, lm_end = 0;    // shard in problem order
  int nl_local = 0;
  long long nobs_local = 0;
  long long sum_n2 = 0;
  int max_n = 0;
  int kp_max = 0;                  // largest KP with a register-resident matvec variant
  std::vector<int> sorted_lm;      // sorted index -> local landmark id (0..nl_local-1); -1 for padding
  std::vector<int> sorted_of_lm;   // local landmark id -> sorted index
  std::vector<TileInfo> tiles;
  std::vector<int> tile_of_sorted; // sorted index -> tile
  int nslots = 0;                  // observation slots incl. padding landmarks
  std::vector<int> slot_cam;       // [nslots] camera of the slot (0 for padding)
  std::vector<int> slot_lm;        // [nslots] local landmark id (-1 for padding)
  std::vector<long long> slot_obs; // [nslots] global observation index (-1 for padding)
  long long panel_scalars = 0;
  std::vector<MatvecItem> items;   // sorted by decreasing work; [0, n_items_large) have KP > kp_small_max
  int n_items_large = 0;
  int nyslots = 0;                 // y slots = nslots + slots of extra row chunks
  CameraCSR csr_obs;               // over observation slots (gradient, column norms, preconditioner)
  CameraCSR csr_y;                 // over y slots (matvec); equals csr_obs when no track is chunked
  bool csr_y_is_obs = true;
  std::vector<ReduceItem> pb_items;   // csr_obs slot list cut into segments of PB_SEG_LEN (preconditioner blocks)
  std::vector<int> pb_cam_item_ptr;   // [nc + 1]
  int k4_scratch_per_warp = 0;     // scalars of shared memory per warp for the matvec kernel
};

constexpr int KP_SMALL_MAX = 9;    // classes with G <= 32 and <= 18 columns per lane
constexpr int ROWS_PER_ITEM = 32;  // row chunk of long tracks
constexpr int SEG_LEN = 96;        // camera slot-list segment reduced by one warp
constexpr int PB_SEG_LEN = 16;     // observations per thread in the preconditioner-block kernel

// group size for a track length (see DESIGN.md "track-length classes")
inline int group_size_for(int n) {
  if (n <= 2) return 1;
  if (n <= 4) return 2;
  if (n <= 8) return 4;
  if (n <= 16) return 8;
  if (n <= 32) return 16;
  return 32;
}
inline int kp_for(int n, int G) {
  int kp = (9 * n + 2 * G - 1) / (2 * G);
  if (kp > 9) kp = (kp + 1) & ~1;  // register-resident large classes exist for even KP only (10, 12, 14, 16)
  return kp;
}

// contiguous shards equalising sum n^2 (work and bytes are ~ n^2 per landmark)
inline void partition_landmarks(int nl, const int64_t* lm_off, int nranks, int* bounds) {
  std::vector<double> pre(nl + 1, 0.0);
  for (int l = 0; l < nl; ++l) {
    const double n = (double)(lm_off[l + 1] - lm_off[l]);
    pre[l + 1] = pre[l] + n * n + 4.0 * n;  // panel ~ n^2, per-observation records ~ n
  }
  bounds[0] = 0;
  for (int r = 1; r < nranks; ++r) {
    const double target = pre[nl] * r / nranks;
    int b = (int)(std::lower_bound(pre.begin(), pre.end(), target) - pre.begin());
    b = std::max(b, bounds[r - 1]);
    b = std::min(b, nl);
    bounds[r] = b;
  }
  bounds[nranks] = nl;
}

inline void build_csr(int nc, int nslots_total, const std::vector<int>& cam_of_slot /* -1 = skip */,
                      CameraCSR& out) {
  out.cam_ptr.assign(nc + 1, 0);
  for (int s = 0; s < nslots_total; ++s)
    if (cam_of_slot[s] >= 0) out.cam_ptr[cam_of_slot[s] + 1]++;
  for (int c = 0; c < nc; ++c) out.cam_ptr[c + 1] += out.cam_ptr[c];
  out.slots.assign(out.cam_ptr[nc], 0);
  std::vector<int> cur(out.cam_ptr.begin(), out.cam_ptr.end() - 1);
  for (int s = 0; s < nslots_total; ++s)
    if (cam_of_slot[s] >= 0) out.slots[cur[cam_of_slot[s]]++] = s;
  out.items.clear();
  out.cam_item_ptr.assign(nc + 1, 0);
  for (int c = 0; c < nc; ++c) {
    out.cam_item_ptr[c] = (int)out.items.size();
    for (int b = out.cam_ptr[c]; b < out.cam_ptr[c + 1]; b += SEG_LEN)
      out.items.push_back({c, b, std::min(b + SEG_LEN, out.cam_ptr[c + 1])});
  }
  out.cam_item_ptr[nc] = (int)out.items.size();
}

// Longest-processing-time-first dealing of jobs with the given costs to nw persistent warps, where warp w takes the
// positions w, w + nw, w + 2 nw, ... of the returned order: position k * nw + w holds the k-th job of warp w, and -1 pads
// the lists that end early.  Jobs are dealt in order of decreasing cost (equal costs in index order), each to the warp
// with the least load so far (equal loads: the lowest warp).
inline std::vector<int> deal_lpt(const std::vector<long long>& cost, int nw) {
  std::vector<int> idx(cost.size());
  std::iota(idx.begin(), idx.end(), 0);
  std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return cost[a] > cost[b]; });
  std::vector<std::vector<int>> lists(nw);
  std::vector<std::pair<long long, int>> heap(nw);  // (load, warp), min-heap
  for (int w = 0; w < nw; ++w) heap[w] = {0, w};
  auto cmp = [](const std::pair<long long, int>& a, const std::pair<long long, int>& b) { return a > b; };
  std::make_heap(heap.begin(), heap.end(), cmp);
  for (int j : idx) {
    std::pop_heap(heap.begin(), heap.end(), cmp);
    heap.back().first += cost[j];
    lists[heap.back().second].push_back(j);
    std::push_heap(heap.begin(), heap.end(), cmp);
  }
  size_t maxlen = 0;
  for (auto& l : lists) maxlen = std::max(maxlen, l.size());
  std::vector<int> order(maxlen * nw, -1);
  for (int w = 0; w < nw; ++w)
    for (size_t k = 0; k < lists[w].size(); ++k) order[k * nw + w] = lists[w][k];
  return order;
}

// Returns "" on success or an error message.
inline std::string build_layout(int nc, int nl, const int64_t* lm_off, const int32_t* obs_cam, int rank,
                                int nranks, int kp_max, Layout& L) {
  L = Layout();
  L.nc = nc;
  L.kp_max = kp_max;
  std::vector<int> bounds(nranks + 1);
  partition_landmarks(nl, lm_off, nranks, bounds.data());
  L.lm_begin = bounds[rank];
  L.lm_end = bounds[rank + 1];
  L.nl_local = L.lm_end - L.lm_begin;
  // track lengths; reference requires n >= 2 (ipp:73-76, landmark_block.cpp:54)
  std::vector<int> nloc(L.nl_local);
  for (int l = 0; l < L.nl_local; ++l) {
    const int64_t n = lm_off[L.lm_begin + l + 1] - lm_off[L.lm_begin + l];
    if (n < 2) return "landmark " + std::to_string(L.lm_begin + l) + " has fewer than 2 observations";
    if (n > 20000) return "track length > 20000 unsupported";
    nloc[l] = (int)n;
    L.sum_n2 += n * n;
    L.nobs_local += n;
    L.max_n = std::max(L.max_n, (int)n);
    for (int64_t o = lm_off[L.lm_begin + l]; o + 1 < lm_off[L.lm_begin + l + 1]; ++o)
      if (obs_cam[o] >= obs_cam[o + 1]) return "observations of a landmark must be sorted by ascending camera index";
    for (int64_t o = lm_off[L.lm_begin + l]; o < lm_off[L.lm_begin + l + 1]; ++o)
      if (obs_cam[o] < 0 || obs_cam[o] >= nc) return "camera index out of range";
  }
  // stable sort by n (keeps the original neighbourhood => camera locality inside a tile)
  std::vector<int> order(L.nl_local);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return nloc[a] < nloc[b]; });
  L.sorted_of_lm.assign(L.nl_local, -1);
  // tiles
  int slot = 0;
  long long panel = 0;
  size_t pos = 0;
  while (pos < order.size()) {
    const int n = nloc[order[pos]];
    size_t end = pos;
    while (end < order.size() && nloc[order[end]] == n) ++end;
    const int G = group_size_for(n), W = 32 / G, KP = kp_for(n, G);
    for (size_t p = pos; p < end; p += W) {
      TileInfo T;
      T.panel_off = panel;
      T.slot_base = slot;
      T.lm_base = (int)L.sorted_lm.size();
      T.n = (short)n; T.G = (short)G; T.KP = (short)KP;
      T.nvalid = (short)std::min<size_t>(W, end - p);
      for (int g = 0; g < W; ++g) {
        const bool real = g < T.nvalid;
        const int lm = real ? order[p + g] : -1;
        if (real) L.sorted_of_lm[lm] = (int)L.sorted_lm.size();
        L.sorted_lm.push_back(lm);
        L.tile_of_sorted.push_back((int)L.tiles.size());
        for (int i = 0; i < n; ++i) {
          if (real) {
            const int64_t o = lm_off[L.lm_begin + lm] + i;
            L.slot_cam.push_back(obs_cam[o]);
            L.slot_lm.push_back(lm);
            L.slot_obs.push_back(o);
          } else {
            L.slot_cam.push_back(0);
            L.slot_lm.push_back(-1);
            L.slot_obs.push_back(-1);
          }
        }
      }
      slot += W * n;
      panel += (long long)2 * n * KP * 64;
      L.tiles.push_back(T);
    }
    pos = end;
  }
  L.nslots = slot;
  L.panel_scalars = panel;
  // matvec items
  int extra = L.nslots;
  std::vector<int> ycam(L.slot_cam.size());
  for (int s = 0; s < L.nslots; ++s) ycam[s] = L.slot_lm[s] >= 0 ? L.slot_cam[s] : -1;
  for (int t = 0; t < (int)L.tiles.size(); ++t) {
    const TileInfo& T = L.tiles[t];
    const int rows = 2 * T.n, W = 32 / T.G;
    int nchunks = 1;
    if (rows > ROWS_PER_ITEM + ROWS_PER_ITEM / 2) nchunks = (rows + ROWS_PER_ITEM - 1) / ROWS_PER_ITEM;
    int r0 = 0;
    for (int c = 0; c < nchunks; ++c) {
      const int r1 = (int)((long long)rows * (c + 1) / nchunks);
      MatvecItem it;
      it.tile = t; it.row0 = (short)r0; it.nrows = (short)(r1 - r0); it.pad = 0;
      if (c == 0) {
        it.yslot_base = T.slot_base;
      } else {
        it.yslot_base = extra;
        for (int g = 0; g < W; ++g)
          for (int i = 0; i < T.n; ++i) {
            const int s = T.slot_base + g * T.n + i;
            ycam.push_back(L.slot_lm[s] >= 0 ? L.slot_cam[s] : -1);
          }
        extra += W * T.n;
        L.csr_y_is_obs = false;
      }
      L.items.push_back(it);
      r0 = r1;
    }
  }
  L.nyslots = extra;
  // large-KP items first, then by decreasing bytes
  auto work = [&](const MatvecItem& it) {
    const TileInfo& T = L.tiles[it.tile];
    return (long long)it.nrows * T.KP;
  };
  std::stable_sort(L.items.begin(), L.items.end(), [&](const MatvecItem& a, const MatvecItem& b) {
    const bool la = L.tiles[a.tile].KP > KP_SMALL_MAX, lb = L.tiles[b.tile].KP > KP_SMALL_MAX;
    if (la != lb) return la;
    return work(a) > work(b);
  });
  L.n_items_large = 0;
  for (auto& it : L.items) if (L.tiles[it.tile].KP > KP_SMALL_MAX) ++L.n_items_large;
  // CSRs
  {
    std::vector<int> ocam(ycam.begin(), ycam.begin() + L.nslots);
    build_csr(nc, L.nslots, ocam, L.csr_obs);
    if (!L.csr_y_is_obs) build_csr(nc, L.nyslots, ycam, L.csr_y);
    L.pb_cam_item_ptr.assign(nc + 1, 0);
    for (int c = 0; c < nc; ++c) {
      L.pb_cam_item_ptr[c] = (int)L.pb_items.size();
      for (int b = L.csr_obs.cam_ptr[c]; b < L.csr_obs.cam_ptr[c + 1]; b += PB_SEG_LEN)
        L.pb_items.push_back({c, b, std::min(b + PB_SEG_LEN, L.csr_obs.cam_ptr[c + 1])});
    }
    L.pb_cam_item_ptr[nc] = (int)L.pb_items.size();
  }
  // shared-memory scratch sizes (scalars per warp)
  for (const TileInfo& T : L.tiles) {
    const int W = 32 / T.G;
    const int CS = (2 * T.G * T.KP) | 1;
    L.k4_scratch_per_warp = std::max(L.k4_scratch_per_warp, T.KP > kp_max ? 2 * 64 * (int)T.KP : W * CS);
  }
  return "";
}

// Two ints; uploaded as the device's int2 (solver.cu checks that the sizes match).
struct IntPair {
  int x, y;
};

// Co-visible camera pairs, shared by the assembled operator and rba_compute_covariance.  Per landmark its first slot and
// track length; per co-visible camera pair (ca >= cb), ascending (ca, cb), the terms (slot_a, slot_b) of every landmark
// that sees both, landmarks in problem order and within a landmark in observation order: the fixed summation order of
// k_rcs_combine and k_cov_assemble.  wpos[t] = position of term t in the landmark-major enumeration (landmarks in
// problem order, then a = 0..n-1, b = 0..a), the order of k_rcs_terms.
struct PairList {
  std::vector<int> slot0, nn;      // [nl_local]
  std::vector<IntPair> blk_cam;    // [nblk] (ca, cb)
  std::vector<int> blk_ptr;        // [nblk + 1] into terms
  std::vector<IntPair> terms;      // (slot_a, slot_b)
  std::vector<int> wpos;           // landmark-major position of each term
};

// Returns "" on success or an error message.
inline std::string build_pair_list(const Layout& L, PairList& P) {
  const int nl = L.nl_local, nc = L.nc;
  P = PairList();
  P.slot0.resize(nl); P.nn.resize(nl);
  long long nt = 0;
  for (int lm = 0; lm < nl; ++lm) {
    const int sidx = L.sorted_of_lm[lm];
    const TileInfo& T = L.tiles[L.tile_of_sorted[sidx]];
    P.slot0[lm] = T.slot_base + (sidx - T.lm_base) * T.n;
    P.nn[lm] = T.n;
    nt += (long long)T.n * (T.n + 1) / 2;
  }
  if (nt > std::numeric_limits<int>::max()) return "more than 2^31 camera-pair terms";
  // landmark-major list, then two stable counting sorts of its positions (by cb, then by ca): ascending (ca, cb),
  // landmark order kept
  std::vector<IntPair> raw;
  raw.reserve((size_t)nt);
  for (int lm = 0; lm < nl; ++lm)
    for (int a = 0; a < P.nn[lm]; ++a)
      for (int b = 0; b <= a; ++b) raw.push_back({P.slot0[lm] + a, P.slot0[lm] + b});  // camera(a) >= camera(b)
  std::vector<int> idx(raw.size()), tmp(raw.size());
  std::iota(idx.begin(), idx.end(), 0);
  std::vector<long long> cnt((size_t)nc + 1);
  auto pass = [&](const std::vector<int>& src, std::vector<int>& dst, bool by_a) {
    std::fill(cnt.begin(), cnt.end(), 0LL);
    for (int w : src) ++cnt[L.slot_cam[by_a ? raw[w].x : raw[w].y] + 1];
    for (int c = 0; c < nc; ++c) cnt[c + 1] += cnt[c];
    for (int w : src) dst[cnt[L.slot_cam[by_a ? raw[w].x : raw[w].y]]++] = w;
  };
  pass(idx, tmp, false);
  pass(tmp, idx, true);
  tmp.clear(); tmp.shrink_to_fit();
  P.terms.resize(raw.size());
  for (size_t t = 0; t < idx.size(); ++t) P.terms[t] = raw[idx[t]];
  P.wpos.swap(idx);
  for (size_t t = 0; t < P.terms.size(); ++t) {
    const IntPair cc{L.slot_cam[P.terms[t].x], L.slot_cam[P.terms[t].y]};
    if (t == 0 || cc.x != P.blk_cam.back().x || cc.y != P.blk_cam.back().y) {
      P.blk_cam.push_back(cc);
      P.blk_ptr.push_back((int)t);
    }
  }
  P.blk_ptr.push_back((int)P.terms.size());
  return "";
}

// One term (slot_a, slot_b) of a pair, resolved on the host to what k_rcs_terms needs to address the panel: base = the
// tile's panel offset + 2 G g (g = the landmark inside the tile); ij = ia | ib << 16 (observations of slot_a / slot_b inside
// the landmark); meta = n | log2(G) << 15 | KP << 18.  Column c of the landmark in row r is at base + r KP 64 +
// 2 ((c/2 >> lg) 32 + (c/2 & (G - 1))) + c % 2 (the tile layout above).  Every field fits for n <= 20000 (build_layout).
struct AsmTerm {
  long long base;
  int ij, meta;
};
inline AsmTerm pack_asm_term(long long base, int ia, int ib, int n, int G, int KP) {
  int lg = 0;
  while ((1 << lg) < G) ++lg;
  return {base, ia | ib << 16, n | lg << 15 | KP << 18};
}

// Staging bound of the assembled operator: every term's 9 x 9 block is staged at once.  Range by range, with the combine
// searching every pair's terms once per range, the assembly cost more than the panel product saves (DESIGN.md section 11).
constexpr long long ASM_STAGE_BYTES = (long long)2 << 30;

// PCG iteration at which a solve switches to S: building it costs about twice its staging traffic (stage 1 + stage 2,
// each written and read once) in units of operator time, and every iteration with S saves the panel bytes minus the bytes
// of S.
inline int asm_switch_iteration(long long nt, long long panel_scalars, long long s_bytes, int scalar_size) {
  const double staged = 4.0 * (double)nt * 81 * scalar_size, saved = (double)panel_scalars * scalar_size - (double)s_bytes;
  return 1 + (int)std::ceil(2.0 * staged / std::max(saved, 1.0));
}

// The assembled operator's host-side structure.  `fits`: S is at most a quarter of the panel bytes and all terms stage
// in one pass; only then are row_ptr, col, pos and terms built.  `device_bytes`: what its device buffers take.
struct AsmPlan {
  long long nt = 0, nblk = 0, nnzb = 0, s_bytes = 0, device_bytes = 0;
  bool fits = false;
  int switch_iteration = 0;
  std::vector<int> row_ptr;        // [nc + 1] camera-major block-row CSR of the full S (both triangles, diagonal included)
  std::vector<int> col;            // [nnzb] ascending in every row
  std::vector<IntPair> pos;        // [nblk] the pair's lower (ca, cb) and upper (cb, ca) block in the CSR; -1: diagonal
  std::vector<AsmTerm> terms;      // [nt] landmark-major
};

inline void plan_assembled(const Layout& L, const PairList& P, int scalar_size, AsmPlan& A) {
  A = AsmPlan();
  const int nc = L.nc;
  A.nblk = (long long)P.blk_cam.size();
  A.nt = (long long)P.terms.size();
  long long ndiag = 0;
  for (const IntPair& c : P.blk_cam) ndiag += c.x == c.y;
  A.nnzb = 2 * A.nblk - ndiag;
  A.s_bytes = A.nnzb * 81 * scalar_size;
  A.switch_iteration = asm_switch_iteration(A.nt, L.panel_scalars, A.s_bytes, scalar_size);
  A.fits = 4 * A.s_bytes <= L.panel_scalars * scalar_size && 81 * A.nt * scalar_size <= ASM_STAGE_BYTES;
  if (!A.fits) return;
  // S, S_u and the staging buffer; the terms and wpos; blk_ptr, row_ptr, col; pos
  A.device_bytes = A.s_bytes + (A.nblk + A.nt) * 81 * scalar_size + A.nt * (long long)(sizeof(AsmTerm) + sizeof(int)) +
                   (A.nblk + A.nnzb + nc + 2) * (long long)sizeof(int) + A.nblk * (long long)sizeof(IntPair);
  // row ca gets (ca, cb) and row cb the transpose; iterating the pairs in (ca, cb) order fills every row in ascending
  // column order (lower blocks, the diagonal, then upper blocks)
  A.row_ptr.assign((size_t)nc + 1, 0);
  A.col.resize((size_t)A.nnzb);
  for (const IntPair& c : P.blk_cam) { ++A.row_ptr[c.x + 1]; if (c.x != c.y) ++A.row_ptr[c.y + 1]; }
  for (int c = 0; c < nc; ++c) A.row_ptr[c + 1] += A.row_ptr[c];
  std::vector<int> fill(A.row_ptr.begin(), A.row_ptr.end() - 1);
  A.pos.resize((size_t)A.nblk);
  for (long long b = 0; b < A.nblk; ++b) {
    const IntPair c = P.blk_cam[b];
    const int lo = fill[c.x]++;
    A.col[lo] = c.y;
    int up = -1;
    if (c.x != c.y) { up = fill[c.y]++; A.col[up] = c.x; }
    A.pos[b] = {lo, up};
  }
  A.terms.reserve((size_t)A.nt);
  for (int lm = 0; lm < L.nl_local; ++lm) {
    const int sidx = L.sorted_of_lm[lm];
    const TileInfo& T = L.tiles[L.tile_of_sorted[sidx]];
    const int g = sidx - T.lm_base;
    for (int a = 0; a < T.n; ++a)
      for (int b = 0; b <= a; ++b) A.terms.push_back(pack_asm_term(T.panel_off + 2LL * g * T.G, a, b, T.n, T.G, T.KP));
  }
}

}  // namespace rba
