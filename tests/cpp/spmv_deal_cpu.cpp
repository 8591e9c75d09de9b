// CPU test driver for the row deal of the assembled product k_rcs_spmv (rba::deal_spmv, rootba_b200/csrc/layout.hpp).
// Reads "ctas chunk_blocks nrows" and the nrows + 1 entries of row_ptr from stdin, and prints the deal: "ctas <n>", then
// "chunk_ptr ..." and one line "row kb ke flags" per chunk.  tests/test_spmv_deal_cpu.py checks it.
#include <cstdio>
#include <iostream>
#include <vector>

#include "../../rootba_b200/csrc/layout.hpp"

int main() {
  int ctas = 0, chunk = 0, nrows = 0;
  if (!(std::cin >> ctas >> chunk >> nrows) || ctas < 1 || chunk < 1 || nrows < 0) return 2;
  std::vector<int> row_ptr((size_t)nrows + 1);
  for (auto& r : row_ptr)
    if (!(std::cin >> r)) return 2;
  rba::SpmvDeal D;
  rba::deal_spmv(row_ptr, ctas, chunk, D);
  std::printf("ctas %d\nchunk_ptr", D.ctas);
  for (int p : D.chunk_ptr) std::printf(" %d", p);
  std::printf("\n");
  for (const rba::SpmvChunk& c : D.chunks) std::printf("%d %d %d %d\n", c.row, c.kb, c.ke, c.flags);
  return 0;
}
