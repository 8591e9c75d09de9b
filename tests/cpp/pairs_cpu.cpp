// CPU test driver for the camera-pair structure of the assembled operator and rba_compute_covariance (rba::build_pair_list,
// rba::plan_assembled, rba::pack_asm_term in rootba_b200/csrc/layout.hpp).  tests/test_pairs_cpu.py checks the output.
//
// stdin, mode "full" or "summary":  nc nl rank nranks scalar_size, then lm_off[nl + 1], then obs_cam[lm_off[nl]].
//   Prints one line "name v0 v1 ..." per quantity: the summary (nt, nblk, nnzb, s_bytes, panel_scalars, fits, switch), and
//   with "full" also the layout's slot_obs, every landmark's tile (panel offset, index g in the tile, n, G, KP), the pair
//   list, the CSR and positions of S and the packed AsmTerms (raw base / ij / meta).
// stdin, mode "pack":  k, then k lines "base ia ib n G KP".  Prints the packed "base ij meta" of each.
// An error prints "error <message>" and exits with 1.
#include <cstdio>
#include <iostream>
#include <string>
#include <vector>

#include "../../rootba_b200/csrc/layout.hpp"

template <class T, class F>
static void put(const char* name, const std::vector<T>& v, F f) {
  std::printf("%s", name);
  for (const T& x : v) f(x);
  std::printf("\n");
}
static void put(const char* name, const std::vector<int>& v) { put(name, v, [](int x) { std::printf(" %d", x); }); }
static void put(const char* name, const std::vector<long long>& v) { put(name, v, [](long long x) { std::printf(" %lld", x); }); }
static void put(const char* name, const std::vector<rba::IntPair>& v) {
  put(name, v, [](const rba::IntPair& p) { std::printf(" %d %d", p.x, p.y); });
}

int main() {
  std::string mode;
  if (!(std::cin >> mode)) return 2;
  if (mode == "pack") {
    int k = 0;
    if (!(std::cin >> k)) return 2;
    for (int i = 0; i < k; ++i) {
      long long base = 0;
      int ia = 0, ib = 0, n = 0, G = 0, KP = 0;
      if (!(std::cin >> base >> ia >> ib >> n >> G >> KP)) return 2;
      const rba::AsmTerm t = rba::pack_asm_term(base, ia, ib, n, G, KP);
      std::printf("%lld %d %d\n", t.base, t.ij, t.meta);
    }
    return 0;
  }
  if (mode != "full" && mode != "summary") return 2;
  int nc = 0, nl = 0, rank = 0, nranks = 0, scalar_size = 0;
  if (!(std::cin >> nc >> nl >> rank >> nranks >> scalar_size)) return 2;
  std::vector<int64_t> lm_off((size_t)nl + 1);
  for (auto& o : lm_off)
    if (!(std::cin >> o)) return 2;
  std::vector<int32_t> obs_cam((size_t)lm_off[nl]);
  for (auto& c : obs_cam)
    if (!(std::cin >> c)) return 2;
  rba::Layout L;
  std::string msg = rba::build_layout(nc, nl, lm_off.data(), obs_cam.data(), rank, nranks, scalar_size == 4 ? 16 : 10, L);
  rba::PairList P;
  if (msg.empty()) msg = rba::build_pair_list(L, P);
  if (!msg.empty()) {
    std::printf("error %s\n", msg.c_str());
    return 1;
  }
  rba::AsmPlan A;
  rba::plan_assembled(L, P, scalar_size, A);
  std::printf("lm_range %d %d\nnt %lld\nnblk %lld\nnnzb %lld\ns_bytes %lld\npanel_scalars %lld\nfits %d\nswitch %d\n", L.lm_begin,
              L.lm_end, A.nt, A.nblk, A.nnzb, A.s_bytes, L.panel_scalars, (int)A.fits, A.switch_iteration);
  if (mode == "summary") return 0;
  put("slot_obs", L.slot_obs);
  std::vector<long long> panel_off;
  std::vector<int> g, n, G, KP;
  for (int lm = 0; lm < L.nl_local; ++lm) {
    const int sidx = L.sorted_of_lm[lm];
    const rba::TileInfo& T = L.tiles[L.tile_of_sorted[sidx]];
    panel_off.push_back(T.panel_off);
    g.push_back(sidx - T.lm_base);
    n.push_back(T.n); G.push_back(T.G); KP.push_back(T.KP);
  }
  put("lm_panel_off", panel_off); put("lm_g", g); put("lm_n", n); put("lm_G", G); put("lm_KP", KP);
  put("slot0", P.slot0); put("nn", P.nn);
  put("terms", P.terms); put("wpos", P.wpos); put("blk_cam", P.blk_cam); put("blk_ptr", P.blk_ptr);
  put("row_ptr", A.row_ptr); put("col", A.col); put("pos", A.pos);
  std::vector<long long> base;
  std::vector<int> ij, meta;
  for (const rba::AsmTerm& t : A.terms) { base.push_back(t.base); ij.push_back(t.ij); meta.push_back(t.meta); }
  put("asm_base", base); put("asm_ij", ij); put("asm_meta", meta);
  return 0;
}
