// merge_path.cuh — the stable merge of two sorted key arrays by merge path (k_delta_merge, kernels_delta.cu).
//
// The merged order puts a[i] before b[j] unless b[j] < a[i]: on equal keys the first input wins, and keys compare by
// value, so -0.0 and 0.0 are equal and keep their inputs' order.  A NaN orders above every other key here, so the
// comparison is a total preorder even on float64 arrays that hold one, and every co-rank stays inside both arrays.
//
// Diagonal d of the merge (0 <= d <= na + nb) is the boundary after the first d merged keys; its co-rank is the
// number i of those keys that come from a (the other d - i come from b).  A block finds the co-ranks of its tile's two
// diagonals by a binary search over a and b, and its threads find theirs inside the block's slices the same way, then
// each merges its few keys sequentially.
//
// __host__ __device__ and free of CUDA intrinsics, so that g++ compiles it (tests/cxx/merge_path_tool.cpp checks the
// co-ranks and the tile merge against a stable merge).
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define RMI_MERGE_HD __host__ __device__ __forceinline__
#else
#define RMI_MERGE_HD inline
#endif

namespace rmi {

// k_delta_merge's block: MERGE_THREADS threads, each merging MERGE_ITEMS consecutive keys of a MERGE_TILE-key tile.
constexpr int MERGE_THREADS = 256;
constexpr int MERGE_ITEMS = 8;
constexpr uint64_t MERGE_TILE = (uint64_t)MERGE_THREADS * MERGE_ITEMS;

// Whether key y is merged before key x when y comes from b and x from a: y < x by value, with NaN above every key.
template <class T> RMI_MERGE_HD bool merge_b_first(const T& y, const T& x) { return y < x; }
template <> RMI_MERGE_HD bool merge_b_first<double>(const double& y, const double& x) {
  return y < x || (x != x && y == y);
}

// The co-rank of diagonal d: the number of a's keys among the first d merged keys.
template <class T>
RMI_MERGE_HD uint64_t merge_corank(const T* a, uint64_t na, const T* b, uint64_t nb, uint64_t d) {
  uint64_t lo = d > nb ? d - nb : 0, hi = d < na ? d : na;
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    // a[mid] is among the first d keys exactly when it is merged before b[d - 1 - mid]
    if (!merge_b_first(b[d - 1 - mid], a[mid])) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// The merged keys [d0, d1) into out[0, d1 - d0), from the co-ranks of both diagonals.  On sorted inputs the co-ranks
// are non-decreasing in d; the clamp keeps every read inside a and b even when they are not.
template <class T>
RMI_MERGE_HD void merge_tile(const T* a, uint64_t na, const T* b, uint64_t nb, uint64_t d0, uint64_t d1, T* out) {
  uint64_t i = merge_corank(a, na, b, nb, d0), j = d0 - i;
  uint64_t i1 = merge_corank(a, na, b, nb, d1);
  i1 = i1 < i ? i : (i1 > i + (d1 - d0) ? i + (d1 - d0) : i1);
  const uint64_t j1 = d1 - i1;
  for (uint64_t k = 0; k < d1 - d0; ++k) {
    const bool take_a = j >= j1 || (i < i1 && !merge_b_first(b[j], a[i]));
    out[k] = take_a ? a[i++] : b[j++];
  }
}

}  // namespace rmi
