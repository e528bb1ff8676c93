// Test tool for host/slab_layout.hpp (no GPU): every rank's SlabLayout of the ends tables on stdin.
//   slab_layout_tool < tables
// Each table is a line "u64|u32|f64 N world", then one line per rank:
//   first_key_bits last_key_bits last_run_start n_local no_dups
// Prints, for every table and rank, one line of name=value pairs (integers in decimal, the pivot as a C99 hex float).
#include <cstdio>
#include <iostream>
#include <string>
#include <vector>

#include "../../host/slab_layout.hpp"

using namespace rmihost;

template <class T> void print_layouts(const std::vector<rmi_shard_ends>& e, uint64_t N) {
  const int world = (int)e.size();
  for (int rank = 0; rank < world; ++rank) {
    const SlabLayout s = slab_layout<T>(e.data(), world, rank, N);
    std::printf("base=%llu n_global=%llu has_prev=%d is_last=%d is_first=%d has_next=%d prev_key_bits=%llu "
                "prev_F=%llu next_key_bits=%llu no_dups=%d first_key_bits=%llu last_key_bits=%llu last_F=%llu "
                "pivot_x=%a pivot_y=%a\n",
                (unsigned long long)s.base, (unsigned long long)s.n_global, s.has_prev, s.is_last, s.is_first,
                s.has_next, (unsigned long long)s.prev_key_bits, (unsigned long long)s.prev_F,
                (unsigned long long)s.next_key_bits, s.no_dups ? 1 : 0, (unsigned long long)s.first_key_bits, (unsigned long long)s.last_key_bits,
                (unsigned long long)s.last_F, s.pivot_x, s.pivot_y);
  }
}

int main() {
  std::string kt;
  uint64_t N = 0;
  int world = 0;
  while (std::cin >> kt >> N >> world) {
    std::vector<rmi_shard_ends> e(world);
    for (auto& r : e) std::cin >> r.first_key_bits >> r.last_key_bits >> r.last_run_start >> r.n_local >> r.no_dups;
    if (!std::cin || world < 1) return 2;
    if (kt == "u64") print_layouts<uint64_t>(e, N);
    else if (kt == "u32") print_layouts<uint32_t>(e, N);
    else if (kt == "f64") print_layouts<double>(e, N);
    else return 2;
  }
  return 0;
}
