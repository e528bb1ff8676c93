// multiset_diff.cuh — removed keys subtracted from a sorted key array (k_delta_subtract, kernels_delta.cu), and the
// check that a batch of removals holds no more copies of a value than the key set does (k_delta_check_remove).
//
// Both rest on one rule.  In a sorted array a, the key a[p] with value v is past the first c copies of v's run exactly
// when c == 0, or p >= c and a[p - c] == v: a[p - c] then lies in the same run, so at least c copies come before p.
//   - Subtract: removing v c times takes the first c copies of its run, so M[p] survives when it is past them, and
//     lands at p - #{removed <= v} (the removed keys below v, and the c copies of v, all come before p).
//   - Check: batch key j is the (r+1)-th copy of its run in the batch; the key set holds c(v) copies, so that copy is
//     missing exactly when r >= c(v), that is when batch[j] is past the first c(v) copies of its run in the batch.
//
// The counts #{removed < v} and #{removed <= v} use merge_path.cuh's order, in which a NaN is above every key: a NaN in
// a float64 base then counts every removed key below it (none equal), so every search and walk stays inside the
// removed array.  Keys compare by value (-0.0 == 0.0).
//
// __host__ __device__ and free of CUDA intrinsics, so that g++ compiles it (tests/cxx/multiset_diff_tool.cpp checks
// both rules and the kernel's decomposition against a std::map count of every value).
#pragma once
#include <cstdint>

#include "merge_path.cuh"

namespace rmi {

// Whether a[p] is past the first c copies of its value's run in the sorted array a.
template <class T> RMI_MERGE_HD bool past_first_copies(const T* a, uint64_t p, uint64_t c) {
  return c == 0 || (p >= c && a[p - c] == a[p]);
}

// Whether removed key x counts before v: x < v, or x <= v for LE, in merge_path.cuh's order (NaN above every key).
template <bool LE, class T> RMI_MERGE_HD bool diff_before(const T& x, const T& v) {
  return LE ? !merge_b_first(v, x) : merge_b_first(x, v);
}

// First index in [lo, hi) whose key does not count before v, or hi.
template <bool LE, class T> RMI_MERGE_HD uint64_t diff_search(const T* r, uint64_t lo, uint64_t hi, const T& v) {
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    if (diff_before<LE>(r[mid], v)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// The same answer, found by galloping forward from `from` (every key before `from` counts before v): O(1) probes
// when the answer is near `from`, O(log) when a long run lies between.
template <bool LE, class T> RMI_MERGE_HD uint64_t diff_gallop(const T* r, uint64_t from, uint64_t hi, const T& v) {
  if (from >= hi || !diff_before<LE>(r[from], v)) return from;
  uint64_t good = from, step = 1;   // r[good] counts before v
  for (;;) {
    const uint64_t probe = hi - good > step ? good + step : hi;
    if (probe == hi || !diff_before<LE>(r[probe], v)) return diff_search<LE>(r, good + 1, probe, v);
    good = probe;
    step <<= 1;
  }
}

// The keys M[p0, p0 + len), sorted (keys[k] == M[p0 + k]; m is M itself, for the probe of M[p - c]), minus the
// removed keys r: emit(k, dest) for every key that survives, with its position in the difference.  [lo, hi) is a
// window of r that holds every removed key equal to one of the keys (their tile's two searches).  The first key
// searches the window; every later one gallops on from the previous key's counts, so a thread's keys cost O(1)
// probes each unless a long run of removed copies lies between them.
template <class T, class Emit>
RMI_MERGE_HD void subtract_keys(const T* keys, uint64_t p0, uint64_t len, const T* m, const T* r, uint64_t lo,
                                uint64_t hi, Emit&& emit) {
  uint64_t i = lo, j = lo;   // #{r < v} and #{r <= v}, as indices into r
  for (uint64_t k = 0; k < len; ++k) {
    const T v = keys[k];
    if (k == 0) {
      i = diff_search<false>(r, lo, hi, v);
      j = diff_search<true>(r, i, hi, v);
    } else if (!(v == keys[k - 1])) {
      i = diff_gallop<false>(r, j, hi, v);
      j = diff_gallop<true>(r, i, hi, v);
    }
    if (past_first_copies(m, p0 + k, j - i)) emit(k, p0 + k - j);
  }
}

}  // namespace rmi
