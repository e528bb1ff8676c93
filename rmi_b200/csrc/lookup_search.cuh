// lookup_search.cuh — the exact search of a lookup's error window, shared by the single-GPU lookup kernels
// (kernels_lookup.cu) and the searches over a rank's slab of a range-partitioned data set (kernels_shard_lookup.cu,
// kernels_shard_bounded.cu), with the pieces of a bounded lookup both bounded kernels take: the knot-window search,
// the key-line step and the packed leaf record.
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

// The key-line step of a bounded lookup (kernels_lookup.cu k_lookup_bounded, kernels_shard_bounded.cu): r = the exact
// lower bound of q over keys[0, n) from the window [lo, hi] (lo <= hi <= n, hi - lo <= width).  Windows of up to
// BOUNDED_COUNT_MAX keys (width <= BOUNDED_COUNT_MAX) are searched by loading every key independently and counting
// those below q (no dependent probe chain); longer ones by the branchless binary search.  The keys just outside the
// window are read only when the search ends on that edge, so a present key touches its own line alone unless its
// lower bound is the line's first index.  A window that does not bracket the answer takes the galloping fallback and
// is counted in `misses`.
// A statement macro, not a function: the same code as an inlined function compiles to different SASS in
// k_lookup_bounded (the edge flags are materialised as bytes before the fallback call), and the move was to leave that
// kernel's SASS as it was.
constexpr u64 BOUNDED_COUNT_MAX = 16;

#define RMI_LINE_SEARCH(keys, n, q, lo, hi, width, misses, r)                  \
  do {                                                                         \
    r = lo;                                                                    \
    if ((width) <= BOUNDED_COUNT_MAX) {                                        \
      _Pragma("unroll") for (u64 j_ = 0; j_ < BOUNDED_COUNT_MAX; ++j_)         \
        if (lo + j_ < hi) r += keys[lo + j_] < q ? 1 : 0;                      \
    } else {                                                                   \
      u64 kb_ = lo, klen_ = hi - lo;                                           \
      while (klen_ > 1) {                                                      \
        const u64 h_ = klen_ >> 1;                                             \
        kb_ = keys[kb_ + h_] < q ? kb_ + h_ : kb_;                             \
        klen_ -= h_;                                                           \
      }                                                                        \
      r = klen_ == 1 && keys[kb_] < q ? kb_ + 1 : kb_;                         \
    }                                                                          \
    const bool left_ok_ = r > lo || lo == 0 || keys[lo - 1] < q;               \
    const bool right_ok_ = r < hi || hi == n || !(keys[hi] < q);               \
    if (!(left_ok_ && right_ok_)) {                                            \
      ++misses;                                                                \
      r = lookup_fallback(keys, n, q, lo, hi, left_ok_);                       \
    }                                                                          \
  } while (0)

// The packed leaf record (kernels_lookup.cu pack_leaf_records): parameters, then the error bound, in 16-byte vectors.
//   32 B: {f0, f1}, {f2, err}               linear family, loglinear, normal, lognormal (f2 = 0 for 2 params)
//   64 B: {f0, f1}, {f2, f3}, {err, 0}, pad  cubic
template <int LEAF> struct Rec {
  static constexpr int VECS = LEAF == M_CUBIC ? 4 : 2;   // stride in 16-byte vectors
  static constexpr int LOADS = LEAF == M_CUBIC ? 3 : 2;  // vectors a lookup reads
  __device__ __forceinline__ static void unpack(const ulonglong2 (&v)[LOADS], double* f, u64& err) {
    f[0] = __longlong_as_double((long long)v[0].x);
    f[1] = __longlong_as_double((long long)v[0].y);
    f[2] = __longlong_as_double((long long)v[1].x);
    if (LEAF == M_CUBIC) {
      f[3] = __longlong_as_double((long long)v[1].y);
      err = v[LOADS - 1].x;
    } else {
      f[3] = 0.0;
      err = v[1].y;
    }
  }
};

// First index in [lo, hi) whose knot key is not < q, or hi: the generated spline lookup's search of the knot window
// (codegen.rs:410-437), on {key, offset} knots.
__device__ __forceinline__ u64 knot_window_search(const ulonglong2* __restrict__ knots, u64 lo, u64 hi, u64 q) {
  u64 b = lo, len = hi - lo;
  while (len > 1) {
    const u64 h = len >> 1;
    b = knots[b + h].x < q ? b + h : b;
    len -= h;
  }
  return len == 1 && knots[b].x < q ? b + 1 : b;
}

}  // namespace
}  // namespace rmi
