// Prints the intra-cluster term list of plan_clusters (rootba_b200/csrc/layout.hpp) for a problem read from stdin:
//   nc nl / lm_off[nl + 1] / obs_cam[nobs] / cluster_of[nc]
// Output: one line "k ca cb lm slot_cam_a slot_cam_b" per term, clusters and their cross blocks in list order.
#include <iostream>
#include <vector>

#include "../../rootba_b200/csrc/layout.hpp"

int main() {
  int nc = 0, nl = 0;
  std::cin >> nc >> nl;
  std::vector<int64_t> off(nl + 1);
  for (auto& v : off) std::cin >> v;
  std::vector<int32_t> cam(off[nl]);
  for (auto& v : cam) std::cin >> v;
  std::vector<int> cl(nc);
  for (auto& v : cl) std::cin >> v;
  rba::Layout L;
  std::string msg = rba::build_layout(nc, nl, off.data(), cam.data(), 0, 1, 16, L);
  if (!msg.empty()) { std::cerr << msg << "\n"; return 1; }
  rba::ClusterPlan C;
  msg = rba::plan_clusters(L, cl.data(), true, C);
  if (!msg.empty()) { std::cout << "error " << msg << "\n"; return 0; }
  for (int k = 0; k < C.ncl; ++k)
    for (int x = C.xb_ptr[k]; x < C.xb_ptr[k + 1]; ++x) {
      const rba::ClusterBlock& b = C.xb[x];
      const int ca = C.cams[C.ptr[k] + b.la], cb = C.cams[C.ptr[k] + b.lb];
      for (int t = b.t0; t < b.t1; ++t) {
        const rba::IntPair s = C.slots[t];
        std::cout << k << " " << ca << " " << cb << " " << L.slot_lm[s.x] << " " << L.slot_cam[s.x] << " " << L.slot_cam[s.y] << "\n";
      }
    }
  std::cout << "bytes " << C.device_bytes << " terms " << C.slots.size() << " panel " << C.panel_terms.size() << "\n";
  return 0;
}
