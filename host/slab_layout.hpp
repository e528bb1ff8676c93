// slab_layout.hpp — where a rank's slab of range-partitioned keys sits among the others, derived from the
// table every rank gathers (one rmi_shard_ends per rank, include/rmi_b200.h).  The build
// (rmi_shard_build_create) and the evaluation (rmi_shard_eval_create) both take their layout from here, so every
// rank takes the same decisions about runs of equal keys that cross cuts, the global end keys and whether the key
// set is duplicate-free.  Host code only: g++ compiles it for the CPU test of the rule
// (tests/cxx/slab_layout_tool.cpp).
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

#include "../include/rmi_b200.h"

namespace rmihost {

// A key of type T from its raw bits (u32 zero-extended, the f64 bit pattern), and back.
template <class T> T key_from_bits(uint64_t bits) {
  T k;
  if (sizeof(T) == 4) { uint32_t v = (uint32_t)bits; memcpy(&k, &v, 4); }
  else memcpy(&k, &bits, 8);
  return k;
}
template <class T> uint64_t bits_from_key(T k) {
  uint64_t bits = 0;
  if (sizeof(T) == 4) { uint32_t v; memcpy(&v, &k, 4); bits = v; }
  else memcpy(&bits, &k, 8);
  return bits;
}

// The same on every rank for every field but the rank's own (base, has_prev / prev_*, is_first / is_last,
// has_next / next_key_bits).
struct SlabLayout {
  uint64_t base = 0, n_global = 0;
  int has_prev = 0, is_last = 0, is_first = 0, has_next = 0;
  uint64_t prev_key_bits = 0, prev_F = 0;   // last key before the slab, first global index of its run
  uint64_t next_key_bits = 0;               // first key of the next non-empty rank
  bool no_dups = false;                     // no two keys of the whole data set are equal
  uint64_t first_key_bits = 0, last_key_bits = 0;   // the data set's first and last key
  uint64_t last_F = 0;                      // first global index of the run of the last key
  double pivot_x = 0, pivot_y = 0;          // common pivot of the top model's sums (identical on every rank)
};

// Keys at the cuts are compared by value as T (-0.0 == 0.0; u32 keys as 32-bit values).  A slab that is one run of
// equal keys carries on the run start of the rank before it, which may lie several ranks back.  N: the leaves of the
// build (only the pivot depends on it).
template <class T> SlabLayout slab_layout(const rmi_shard_ends* e, int world, int rank, uint64_t N) {
  SlabLayout s;
  std::vector<uint64_t> base(world + 1, 0), last_F(world, 0);
  for (int g = 0; g < world; ++g) base[g + 1] = base[g] + e[g].n_local;
  s.base = base[rank];
  s.n_global = base[world];
  s.no_dups = true;
  int prev = -1, first = -1, last = -1;
  for (int g = 0; g < world; ++g) {
    if (!e[g].n_local) continue;
    const bool joins = prev >= 0 && key_from_bits<T>(e[prev].last_key_bits) == key_from_bits<T>(e[g].first_key_bits);
    last_F[g] = e[g].last_run_start == 0 && joins ? last_F[prev] : base[g] + e[g].last_run_start;
    if (joins || e[g].no_dups != 1) s.no_dups = false;
    if (g < rank) { s.has_prev = 1; s.prev_key_bits = e[g].last_key_bits; s.prev_F = last_F[g]; }
    if (g > rank && !s.has_next) { s.has_next = 1; s.next_key_bits = e[g].first_key_bits; }
    if (first < 0) first = g;
    last = g;
    prev = g;
  }
  s.is_first = rank == first;
  s.is_last = rank == last;
  if (last >= 0) {
    s.first_key_bits = e[first].first_key_bits;
    s.last_key_bits = e[last].last_key_bits;
    s.last_F = last_F[last];
  }
  const double x0 = 0.5 * (double)key_from_bits<T>(s.first_key_bits);
  const double x1 = 0.5 * (double)key_from_bits<T>(s.last_key_bits);
  s.pivot_x = x0 + x1;
  s.pivot_y = 0.5 * (double)N;
  return s;
}

}  // namespace rmihost
