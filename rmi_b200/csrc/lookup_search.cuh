// lookup_search.cuh — the exact search of a lookup's error window, shared by the single-GPU lookup kernels
// (kernels_lookup.cu, kernels_lookup_range.cu) and the searches over a rank's slab of a range-partitioned data set
// (kernels_shard_lookup.cu, kernels_shard_bounded.cu), with the steps every lookup kernel takes: the packed leaf
// record and the RMI step over it, the error window, the bounded index's spline step and key-line search, the
// fallback count and the grid.
//
// For a window [lo, hi] of candidate answers over keys[0, n): a branchless binary search over keys [lo, hi),
// confirmed by the keys just outside the window (lo == 0 and hi == n need no confirmation), and a galloping search
// outward from the window's edge when the window does not bracket the answer (counted in `misses`).
//
// Every search counts the keys k before q under one predicate: k < q (strict: the lower bound, what the predict /
// lower_bound kernels run) or k <= q (UPPER: the upper bound, kernels_lookup_range.cu).  Both compare by value, so
// -0.0 and 0.0 are equal, and a NaN q has no key before it under either.
#pragma once
#include <type_traits>

#include "kernels.h"
#include "models.cuh"
#include "spline.cuh"

namespace rmi {
namespace {

// Threads per block of the lookup kernels, each thread one query at a time (grid-stride).  Measured on an H100 SXM
// (DESIGN §11) on the headline index (linear,linear 2^20 over 200M uint64 keys, 2^27 random present keys):
// lower_bound took 27.4 / 34.2 / 36.6 / 37.0 ms at 1 / 2 / 4 / 8 queries per thread with 128 threads (28.4 / 33.9 /
// 35.2 / 37.2 ms with 256); predict was 2.65-2.72 ms at 1, 2 and 4 and 2.95 ms at 8.  One query per thread needs 32
// registers, so 64 warps fit on an SM, and those warps keep more probes in flight than fewer warps carrying several
// queries each: a lockstep search waits for the longest window of its queries, and the registers it needs cost warps.
constexpr int LOOKUP_THREADS = 128;
constexpr int LOOKUP_MAX_BLOCKS_PER_SM = 32;   // grid cap; beyond it the blocks stride over the queries

// The grid of a grid-stride kernel over n items: one block per `threads` items, at most per_sm blocks per SM.
inline unsigned capped_grid(const Launch& L, u64 n, int threads, int per_sm) {
  const u64 blocks = (n + threads - 1) / threads, cap = (u64)L.num_sms * per_sm;
  return (unsigned)(blocks < cap ? blocks : cap);
}

// Adds the warp's misses to *fallbacks (may be null): the epilogue of every lookup kernel.  Every lane of the warp
// calls it.
__device__ __forceinline__ void flush_fallbacks(unsigned misses, u64* fallbacks) {
  if (fallbacks) {
    misses = __reduce_add_sync(0xffffffffu, misses);
    if ((threadIdx.x & 31) == 0 && misses) atomicAdd((unsigned long long*)fallbacks, (unsigned long long)misses);
  }
}

// The window [pos-err, pos+err] ∩ [0, rows] for pos < rows, without wrapping.  The arguments are references: taken
// by value, the comparisons inline with their operands swapped, the same logic in different SASS.
struct Window { u64 lo, hi; };
__device__ __forceinline__ Window error_window(const u64& pos, const u64& err, const u64& rows) {
  return {pos >= err ? pos - err : 0, err >= rows - pos ? rows : pos + err};
}

// Whether key k counts before q: k < q, or k <= q for UPPER.  search_range and lookup_fallback spell the same
// conditional out: through this helper the float64 instances of the strict fallback compiled to different SASS.
template <bool UPPER, class T> __device__ __forceinline__ bool before(T k, T q) { return UPPER ? k <= q : k < q; }

// First index in [lo, hi) whose key does not count before q, or hi.
template <class T, bool UPPER = false>
__device__ __forceinline__ u64 search_range(const T* __restrict__ keys, u64 lo, u64 hi, T q) {
  while (lo < hi) {
    u64 mid = lo + ((hi - lo) >> 1);
    if (UPPER ? keys[mid] <= q : keys[mid] < q) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// The window [lo, hi] missed: the answer is below lo (!left_ok: keys[lo-1] does not count before q) or above hi
// (keys[hi] counts before q).  Gallop outward from that edge until the answer is bracketed, then search the bracket.
template <class T, bool UPPER = false>
__device__ __noinline__ u64 lookup_fallback(const T* __restrict__ keys, u64 n, T q, u64 lo, u64 hi, bool left_ok) {
  if (!left_ok) {
    u64 R = lo - 1, step = 1, L = 0;   // answer <= R
    while (true) {
      if (R < step) { L = 0; break; }
      u64 c = R - step;
      if (UPPER ? keys[c] <= q : keys[c] < q) { L = c + 1; break; }
      R = c;
      step <<= 1;
    }
    return search_range<T, UPPER>(keys, L, R, q);
  }
  u64 L = hi + 1, step = 1, R = n;     // answer >= L
  while (true) {
    if (n - L < step) { R = n; break; }
    u64 c = L + step - 1;
    if (!(UPPER ? keys[c] <= q : keys[c] < q)) { R = c; break; }
    L = c + 1;
    step <<= 1;
  }
  return search_range<T, UPPER>(keys, L, R, q);
}

// Q queries in lockstep (keeps Q independent probes in flight per step).  Windows [lo[j], hi[j]] with
// lo[j] <= hi[j] <= n and n >= 1.  For every live query, emit(j, r) receives r = the exact lower bound of q[j] over
// keys[0, n), or its upper bound where bit j of UPPER is set (lanes over the same window, as equal_range runs them,
// share the edge loads).
template <class T, int Q, unsigned UPPER = 0u, class Emit>
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
      const bool up = (UPPER >> j) & 1u;
      if (len[j] > 1) {
        u64 h = len[j] >> 1;
        const T k = keys[b[j] + h];
        b[j] = (up ? before<true>(k, q[j]) : before<false>(k, q[j])) ? b[j] + h : b[j];
        len[j] -= h;
        more |= len[j] > 1;
      }
    }
    if (!more) break;
  }
#pragma unroll
  for (int j = 0; j < Q; ++j) {
    const bool up = (UPPER >> j) & 1u;
    u64 r = b[j];
    if (len[j] == 1) r += (up ? before<true>(keys[r], q[j]) : before<false>(keys[r], q[j])) ? 1 : 0;
    bool left_ok = lo[j] == 0 || (up ? before<true>(edge_l[j], q[j]) : before<false>(edge_l[j], q[j]));
    bool right_ok = hi[j] == n || !(up ? before<true>(edge_r[j], q[j]) : before<false>(edge_r[j], q[j]));
    if (live[j]) {
      if (!(left_ok && (r < hi[j] || right_ok))) {
        ++misses;
        r = up ? lookup_fallback<T, true>(keys, n, q[j], lo[j], hi[j], left_ok)
               : lookup_fallback<T, false>(keys, n, q[j], lo[j], hi[j], left_ok);
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
// Statement macros, not functions: the same code as an inlined function compiles to different SASS in
// k_lookup_bounded (the edge flags are materialised as bytes before the fallback call), and the move was to leave that
// kernel's SASS as it was.
//   RMI_LINE_SEARCH_AS  the same with the predicate of UPPER (a constant): r = the upper bound for true
//   RMI_LINE_RANGE      both ends, r (lower) and ru (upper), over one window; the counting branch counts both from one
//                       set of loads; each end is confirmed on its own, and `misses` grows by one per end that missed
constexpr u64 BOUNDED_COUNT_MAX = 16;

#define RMI_LINE_BSEARCH_(keys, q, lo, hi, r, UPPER)                           \
  do {                                                                         \
    u64 kb_ = lo, klen_ = hi - lo;                                             \
    while (klen_ > 1) {                                                        \
      const u64 h_ = klen_ >> 1;                                               \
      kb_ = before<UPPER>(keys[kb_ + h_], q) ? kb_ + h_ : kb_;                 \
      klen_ -= h_;                                                             \
    }                                                                          \
    r = klen_ == 1 && before<UPPER>(keys[kb_], q) ? kb_ + 1 : kb_;             \
  } while (0)

#define RMI_LINE_CONFIRM_(keys, n, q, lo, hi, misses, r, UPPER)                          \
  do {                                                                                   \
    const bool left_ok_ = r > lo || lo == 0 || before<UPPER>(keys[lo - 1], q);           \
    const bool right_ok_ = r < hi || hi == n || !before<UPPER>(keys[hi], q);             \
    if (!(left_ok_ && right_ok_)) {                                                      \
      ++misses;                                                                          \
      r = lookup_fallback<std::remove_cv_t<std::remove_reference_t<decltype(keys[0])>>,  \
                          UPPER>(keys, n, q, lo, hi, left_ok_);                          \
    }                                                                                    \
  } while (0)

#define RMI_LINE_SEARCH_AS(keys, n, q, lo, hi, width, misses, r, UPPER)        \
  do {                                                                         \
    r = lo;                                                                    \
    if ((width) <= BOUNDED_COUNT_MAX) {                                        \
      _Pragma("unroll") for (u64 j_ = 0; j_ < BOUNDED_COUNT_MAX; ++j_)         \
        if (lo + j_ < hi) r += before<UPPER>(keys[lo + j_], q) ? 1 : 0;        \
    } else {                                                                   \
      RMI_LINE_BSEARCH_(keys, q, lo, hi, r, UPPER);                            \
    }                                                                          \
    RMI_LINE_CONFIRM_(keys, n, q, lo, hi, misses, r, UPPER);                   \
  } while (0)

#define RMI_LINE_SEARCH(keys, n, q, lo, hi, width, misses, r) \
  RMI_LINE_SEARCH_AS(keys, n, q, lo, hi, width, misses, r, false)

#define RMI_LINE_RANGE(keys, n, q, lo, hi, width, misses, r, ru)               \
  do {                                                                         \
    r = lo;                                                                    \
    ru = lo;                                                                   \
    if ((width) <= BOUNDED_COUNT_MAX) {                                        \
      _Pragma("unroll") for (u64 j_ = 0; j_ < BOUNDED_COUNT_MAX; ++j_) {       \
        if (lo + j_ < hi) {                                                    \
          const auto k_ = keys[lo + j_];                                       \
          r += before<false>(k_, q) ? 1 : 0;                                   \
          ru += before<true>(k_, q) ? 1 : 0;                                   \
        }                                                                      \
      }                                                                        \
    } else {                                                                   \
      RMI_LINE_BSEARCH_(keys, q, lo, hi, r, false);                            \
      RMI_LINE_BSEARCH_(keys, q, lo, hi, ru, true);                            \
    }                                                                          \
    RMI_LINE_CONFIRM_(keys, n, q, lo, hi, misses, r, false);                   \
    RMI_LINE_CONFIRM_(keys, n, q, lo, hi, misses, ru, true);                   \
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

// The RMI step of a lookup: leaf t = min(N-1, top(q)), then from its record the position min(rows-1, leaf_t(q)),
// returned, and the leaf's error bound err.  rows: the keys of a plain index, the knots of a bounded one.
template <int TOP, int LEAF, class T>
__device__ __forceinline__ u64 rmi_predict(const TopModel& top, const ulonglong2* __restrict__ recs, u64 N, u64 rows,
                                           T q, u64& err) {
  using R = Rec<LEAF>;
  u64 t = top_predict<TOP>(top, q);
  t = t < N - 1 ? t : N - 1;
  ulonglong2 v[R::LOADS];
#pragma unroll
  for (int k = 0; k < R::LOADS; ++k) v[k] = __ldg(recs + t * R::VECS + k);
  double f[4];
  R::unpack(v, f, err);
  u64 pos = leaf_predict64<LEAF>(f, Key<T>::as_float(q));
  pos = pos < rows - 1 ? pos : rows - 1;
  return pos;
}

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

// The spline step of a bounded lookup over K knots and n keys, from the knot window [lower, upper) of the RMI step:
// res = the window's first knot whose key is not < q; n - 1 past the last knot, 0 before the first, else the spline
// between knots res-1 and res rounded down to its line (codegen.rs:410-437).  knots holds the global knots from k_lo
// on (0 on one GPU), the window among them.
__device__ __forceinline__ u64 bounded_pos(const ulonglong2* __restrict__ knots, u64 k_lo, u64 lower, u64 upper, u64 K,
                                           u64 n, u64 line, u64 q) {
  const u64 res = knot_window_search(knots, lower - k_lo, upper - k_lo, q) + k_lo;
  if (res == K) return n - 1;
  if (res == 0) return 0;
  const ulonglong2 p0 = knots[res - k_lo - 1], p1 = knots[res - k_lo];
  return cache_fix_interp(q, p0.x, p0.y, p1.x, p1.y) / line * line;
}

}  // namespace
}  // namespace rmi
