// CPU test driver for the longest-processing-time-first dealer of the persistent kernels (rba::deal_lpt,
// rootba_b200/csrc/layout.hpp).  Reads "nw n" and n costs from stdin and prints the dealt order (k * nw + w = the k-th job
// of warp w, -1 = padding) on one line.  tests/test_deal_cpu.py checks the order.
#include <cstdio>
#include <iostream>
#include <vector>

#include "../../rootba_b200/csrc/layout.hpp"

int main() {
  int nw = 0;
  size_t n = 0;
  if (!(std::cin >> nw >> n) || nw < 1) return 2;
  std::vector<long long> cost(n);
  for (auto& c : cost)
    if (!(std::cin >> c)) return 2;
  const std::vector<int> order = rba::deal_lpt(cost, nw);
  for (size_t i = 0; i < order.size(); ++i) std::printf(i ? " %d" : "%d", order[i]);
  std::printf("\n");
  return 0;
}
