// kernels_lookup_range.cu — upper bounds and equal ranges on a trained two-layer RMI (DESIGN §18), beside the
// predict / lower_bound kernels of kernels_lookup.cu.
//
// upper_bound:  the number of keys k with k <= q (std::upper_bound; 0 for a NaN query, compared by value so that
//               -0.0 <= 0.0).  The reference widens every leaf's error bound by the longest run of equal keys in
//               that leaf (two_layer.rs:250-251), so for a key of the data set the end of its run lies in the same
//               window [pos-err, pos+err] as its start.  The one run that bound does not record is the data set's
//               last one, whose upper bound is n: a query >= the last key gets n without a search.
// equal_range:  (lower_bound, upper_bound) from one top evaluation, one leaf record and one window: the two searches
//               run in lockstep over the window (lookup_search.cuh window_search, one lane per end), so the edge keys
//               are loaded once and the second search's probes hit the lines the first one brought in.  The lower end
//               is bit-equal to lower_bound's answer.
// Both are exact: a window that misses takes the galloping fallback and counts the query once (either end).
//
// Thread mapping: k_lookup's (one query per thread, LOOKUP_THREADS per block, grid-stride over the queries).
#include "kernels.h"
#include "lookup_search.cuh"

namespace rmi {

namespace {

template <class T, int TOP, int LEAF>
__global__ void __launch_bounds__(LOOKUP_THREADS)
k_lookup_range(const __grid_constant__ TopModel top, const ulonglong2* __restrict__ recs, const T* __restrict__ keys,
               u64 n, T last, u64 N, const T* __restrict__ qs, u64 nq, u64* __restrict__ out_first,
               u64* __restrict__ out_last, u64* fallbacks, int equal_range) {
  unsigned misses = 0;
  for (u64 i = (u64)blockIdx.x * LOOKUP_THREADS + threadIdx.x; i < nq; i += (u64)gridDim.x * LOOKUP_THREADS) {
    const T q = __ldcs(qs + i);
    u64 err;
    const u64 pos = rmi_predict<TOP, LEAF>(top, recs, N, n, q, err);
    const Window w = error_window(pos, err, n);
    const bool past = q >= last;   // every key is <= q
    if (past) __stcs(out_last + i, n);
    // lane 0: lower bound (equal_range only), lane 1: upper bound
    const T qq[2] = {q, q};
    const bool live[2] = {equal_range != 0, !past};
    const u64 los[2] = {w.lo, w.lo}, his[2] = {w.hi, w.hi};
    unsigned m = 0;
    if (live[0] || live[1])
      window_search<T, 2, 2u>(keys, n, qq, live, los, his, m,
                              [&](int j, u64 r) { __stcs((j ? out_last : out_first) + i, r); });
    misses += m ? 1 : 0;
  }
  flush_fallbacks(misses, fallbacks);
}

// The bounded index's spline step as in k_lookup_bounded, then the key line [pos, pos + line] for both ends: for
// distinct keys a present key's upper bound is its lower bound + 1 <= pos + line; a run that ends past its line takes
// the counted fallback.
template <int TOP, int LEAF>
__global__ void __launch_bounds__(LOOKUP_THREADS)
k_lookup_bounded_range(const __grid_constant__ TopModel top, const ulonglong2* __restrict__ recs, u64 N,
                       const ulonglong2* __restrict__ knots, u64 K, u64 line, const u64* __restrict__ keys, u64 n,
                       u64 last, const u64* __restrict__ qs, u64 nq, u64* __restrict__ out_first,
                       u64* __restrict__ out_last, u64* fallbacks, int equal_range) {
  unsigned misses = 0;
  for (u64 i = (u64)blockIdx.x * LOOKUP_THREADS + threadIdx.x; i < nq; i += (u64)gridDim.x * LOOKUP_THREADS) {
    const u64 q = __ldcs(qs + i);
    u64 e;
    const u64 start = rmi_predict<TOP, LEAF>(top, recs, N, K, q, e);
    const Window kw = error_window(start, e, K);
    const u64 pos = bounded_pos(knots, 0, kw.lo, kw.hi, K, n, line, q);
    const u64 lo = pos < n ? pos : n;
    const u64 hi = line >= n - lo ? n : lo + line;
    unsigned m = 0;
    u64 r, ru;
    if (q >= last) {   // every key is <= q
      __stcs(out_last + i, n);
      if (equal_range) {
        RMI_LINE_SEARCH_AS(keys, n, q, lo, hi, line, m, r, false);
        __stcs(out_first + i, r);
      }
    } else if (equal_range) {
      RMI_LINE_RANGE(keys, n, q, lo, hi, line, m, r, ru);
      __stcs(out_first + i, r);
      __stcs(out_last + i, ru);
    } else {
      RMI_LINE_SEARCH_AS(keys, n, q, lo, hi, line, m, ru, true);
      __stcs(out_last + i, ru);
    }
    misses += m ? 1 : 0;
  }
  flush_fallbacks(misses, fallbacks);
}

}  // namespace

template <class T>
void launch_range(const Launch& L, LookupMode mode, const TopModel& top, int leaf_kind, const void* recs, u64 N,
                  const T* keys, u64 n, T last, const T* q, u64 nq, u64* out, u64* out2, u64* fallbacks) {
  const bool eq = mode == LOOKUP_EQUAL_RANGE;
  with_groups(top.kind, leaf_kind, [&](auto tk, auto lk) {
    k_lookup_range<T, decltype(tk)::value, decltype(lk)::value>
        <<<capped_grid(L, nq, LOOKUP_THREADS, LOOKUP_MAX_BLOCKS_PER_SM), LOOKUP_THREADS, 0, L.stream>>>(
            top, (const ulonglong2*)recs, keys, n, last, N, q, nq, eq ? out : nullptr, eq ? out2 : out, fallbacks,
            eq ? 1 : 0);
  });
}

void launch_bounded_range(const Launch& L, LookupMode mode, const TopModel& top, int leaf_kind, const void* recs, u64 N,
                          const void* knots, u64 K, u64 line, const u64* keys, u64 n, u64 last, const u64* q, u64 nq,
                          u64* out, u64* out2, u64* fallbacks) {
  const bool eq = mode == LOOKUP_EQUAL_RANGE;
  with_groups(top.kind, leaf_kind, [&](auto tk, auto lk) {
    k_lookup_bounded_range<decltype(tk)::value, decltype(lk)::value>
        <<<capped_grid(L, nq, LOOKUP_THREADS, LOOKUP_MAX_BLOCKS_PER_SM), LOOKUP_THREADS, 0, L.stream>>>(
            top, (const ulonglong2*)recs, N, (const ulonglong2*)knots, K, line, keys, n, last, q, nq,
            eq ? out : nullptr, eq ? out2 : out, fallbacks, eq ? 1 : 0);
  });
}

#define RMI_LAUNCH_RANGE_INST(T)                                                                                    \
  template void launch_range<T>(const Launch&, LookupMode, const TopModel&, int, const void*, u64, const T*, u64, T, \
                                const T*, u64, u64*, u64*, u64*);
RMI_LAUNCH_RANGE_INST(u64)
RMI_LAUNCH_RANGE_INST(u32)
RMI_LAUNCH_RANGE_INST(double)
#undef RMI_LAUNCH_RANGE_INST

}  // namespace rmi
