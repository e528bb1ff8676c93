// lookup_search.cuh — the exact search of a lookup's error window, shared by the single-GPU lookup kernels
// (kernels_lookup.cu) and the search over a rank's slab of a range-partitioned data set (kernels_shard_lookup.cu).
//
// For a window [lo, hi] of candidate answers over keys[0, n): a branchless binary search over keys [lo, hi),
// confirmed by the keys just outside the window (lo == 0 and hi == n need no confirmation), and a galloping search
// outward from the window's edge when the window does not bracket the answer (counted in `misses`).
#pragma once
#include "models.cuh"

namespace rmi {
namespace {

// First index in [lo, hi) whose key is not < q, or hi.
template <class T> __device__ __forceinline__ u64 search_range(const T* __restrict__ keys, u64 lo, u64 hi, T q) {
  while (lo < hi) {
    u64 mid = lo + ((hi - lo) >> 1);
    if (keys[mid] < q) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// The window [lo, hi] missed: the answer is below lo (!left_ok: keys[lo-1] is not < q) or above hi
// (keys[hi] < q).  Gallop outward from that edge until the answer is bracketed, then search the bracket.
template <class T>
__device__ __noinline__ u64 lookup_fallback(const T* __restrict__ keys, u64 n, T q, u64 lo, u64 hi, bool left_ok) {
  if (!left_ok) {
    u64 R = lo - 1, step = 1, L = 0;   // answer <= R
    while (true) {
      if (R < step) { L = 0; break; }
      u64 c = R - step;
      if (keys[c] < q) { L = c + 1; break; }
      R = c;
      step <<= 1;
    }
    return search_range(keys, L, R, q);
  }
  u64 L = hi + 1, step = 1, R = n;     // answer >= L
  while (true) {
    if (n - L < step) { R = n; break; }
    u64 c = L + step - 1;
    if (!(keys[c] < q)) { R = c; break; }
    L = c + 1;
    step <<= 1;
  }
  return search_range(keys, L, R, q);
}

// Q queries in lockstep (keeps Q independent probes in flight per step).  Windows [lo[j], hi[j]] with
// lo[j] <= hi[j] <= n and n >= 1.  For every live query, emit(j, r) receives r = the exact lower bound of q[j] over
// keys[0, n).
template <class T, int Q, class Emit>
__device__ __forceinline__ void window_search(const T* __restrict__ keys, u64 n, const T (&q)[Q], const bool (&live)[Q],
                                              const u64 (&lo)[Q], const u64 (&hi)[Q], unsigned& misses, Emit&& emit) {
  u64 b[Q], len[Q];
  T edge_l[Q], edge_r[Q];
#pragma unroll
  for (int j = 0; j < Q; ++j) {
    b[j] = lo[j];
    len[j] = live[j] ? hi[j] - lo[j] : 0;
    // the confirmation probes do not depend on the search: issued with its first probe
    edge_l[j] = keys[lo[j] > 0 ? lo[j] - 1 : 0];
    edge_r[j] = keys[hi[j] < n ? hi[j] : n - 1];
  }
  while (true) {
    bool more = false;
#pragma unroll
    for (int j = 0; j < Q; ++j) {
      if (len[j] > 1) {
        u64 h = len[j] >> 1;
        b[j] = keys[b[j] + h] < q[j] ? b[j] + h : b[j];
        len[j] -= h;
        more |= len[j] > 1;
      }
    }
    if (!more) break;
  }
#pragma unroll
  for (int j = 0; j < Q; ++j) {
    u64 r = b[j];
    if (len[j] == 1) r += keys[r] < q[j] ? 1 : 0;
    bool left_ok = lo[j] == 0 || edge_l[j] < q[j];
    bool right_ok = hi[j] == n || !(edge_r[j] < q[j]);
    if (live[j]) {
      if (!(left_ok && (r < hi[j] || right_ok))) {
        ++misses;
        r = lookup_fallback(keys, n, q[j], lo[j], hi[j], left_ok);
      }
      emit(j, r);
    }
  }
}

}  // namespace
}  // namespace rmi
