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
#include <type_traits>

#include "kernels.h"
#include "lookup_search.cuh"
#include "spline.cuh"

namespace rmi {

namespace {

template <class T, int TOP, int LEAF>
__global__ void __launch_bounds__(LOOKUP_THREADS)
k_lookup_range(const __grid_constant__ TopModel top, const ulonglong2* __restrict__ recs, const T* __restrict__ keys,
               u64 n, T last, u64 N, const T* __restrict__ qs, u64 nq, u64* __restrict__ out_first,
               u64* __restrict__ out_last, u64* fallbacks, int equal_range) {
  using R = Rec<LEAF>;
  unsigned misses = 0;
  for (u64 i = (u64)blockIdx.x * LOOKUP_THREADS + threadIdx.x; i < nq; i += (u64)gridDim.x * LOOKUP_THREADS) {
    const T q = __ldcs(qs + i);
    u64 t = top_predict<TOP>(top, q);
    t = t < N - 1 ? t : N - 1;
    ulonglong2 v[R::LOADS];
#pragma unroll
    for (int k = 0; k < R::LOADS; ++k) v[k] = __ldg(recs + t * R::VECS + k);
    double f[4];
    u64 err;
    R::unpack(v, f, err);
    u64 pos = leaf_predict64<LEAF>(f, Key<T>::as_float(q));
    pos = pos < n - 1 ? pos : n - 1;
    const u64 lo = pos >= err ? pos - err : 0;
    const u64 hi = err >= n - pos ? n : pos + err;
    const bool past = q >= last;   // every key is <= q
    if (past) __stcs(out_last + i, n);
    // lane 0: lower bound (equal_range only), lane 1: upper bound
    const T qq[2] = {q, q};
    const bool live[2] = {equal_range != 0, !past};
    const u64 los[2] = {lo, lo}, his[2] = {hi, hi};
    unsigned m = 0;
    if (live[0] || live[1])
      window_search<T, 2, 2u>(keys, n, qq, live, los, his, m,
                              [&](int j, u64 r) { __stcs((j ? out_last : out_first) + i, r); });
    misses += m ? 1 : 0;
  }
  if (fallbacks) {
    misses = __reduce_add_sync(0xffffffffu, misses);
    if ((threadIdx.x & 31) == 0 && misses) atomicAdd((unsigned long long*)fallbacks, (unsigned long long)misses);
  }
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
  using R = Rec<LEAF>;
  unsigned misses = 0;
  for (u64 i = (u64)blockIdx.x * LOOKUP_THREADS + threadIdx.x; i < nq; i += (u64)gridDim.x * LOOKUP_THREADS) {
    const u64 q = __ldcs(qs + i);
    u64 t = top_predict<TOP>(top, q);
    t = t < N - 1 ? t : N - 1;
    ulonglong2 v[R::LOADS];
#pragma unroll
    for (int k = 0; k < R::LOADS; ++k) v[k] = __ldg(recs + t * R::VECS + k);
    double f[4];
    u64 e;
    R::unpack(v, f, e);
    u64 start = leaf_predict64<LEAF>(f, Key<u64>::as_float(q));
    start = start < K - 1 ? start : K - 1;
    const u64 lower = e > start ? 0 : start - e;
    const u64 upper = e >= K - start ? K : start + e;
    const u64 res = knot_window_search(knots, lower, upper, q);
    u64 pos;
    if (res == K) {
      pos = n - 1;
    } else if (res == 0) {
      pos = 0;
    } else {
      const ulonglong2 p0 = knots[res - 1], p1 = knots[res];
      pos = cache_fix_interp(q, p0.x, p0.y, p1.x, p1.y) / line * line;
    }
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
  if (fallbacks) {
    misses = __reduce_add_sync(0xffffffffu, misses);
    if ((threadIdx.x & 31) == 0 && misses) atomicAdd((unsigned long long*)fallbacks, (unsigned long long)misses);
  }
}

unsigned range_blocks(const Launch& L, u64 nq) {
  u64 blocks = (nq + LOOKUP_THREADS - 1) / LOOKUP_THREADS;
  const u64 cap = (u64)L.num_sms * LOOKUP_MAX_BLOCKS_PER_SM;
  return (unsigned)(blocks < cap ? blocks : cap);
}

template <int K> using Kind = std::integral_constant<int, K>;

// f(Kind<TOP>, Kind<LEAF>) for the kernel group of the given top and leaf model kinds (lookup_top_group,
// lookup_leaf_group), as lookup_batch dispatches.
template <class F> void with_groups(int top_kind, int leaf_kind, F&& f) {
  auto leaf = [&](auto top) {
    switch (lookup_leaf_group(leaf_kind)) {
      case M_LINEAR: f(top, Kind<M_LINEAR>{}); break;
      case M_CUBIC: f(top, Kind<M_CUBIC>{}); break;
      case M_LOGLINEAR: f(top, Kind<M_LOGLINEAR>{}); break;
      case M_NORMAL: f(top, Kind<M_NORMAL>{}); break;
      default: f(top, Kind<M_LOGNORMAL>{}); break;
    }
  };
  switch (lookup_top_group(top_kind)) {
    case M_LINEAR: leaf(Kind<M_LINEAR>{}); break;
    case M_CUBIC: leaf(Kind<M_CUBIC>{}); break;
    case M_LOGLINEAR: leaf(Kind<M_LOGLINEAR>{}); break;
    case M_NORMAL: leaf(Kind<M_NORMAL>{}); break;
    case M_LOGNORMAL: leaf(Kind<M_LOGNORMAL>{}); break;
    case M_RADIX: leaf(Kind<M_RADIX>{}); break;
    case M_RADIX_TABLE: leaf(Kind<M_RADIX_TABLE>{}); break;
    case M_BRADIX: leaf(Kind<M_BRADIX>{}); break;
    default: leaf(Kind<M_HISTOGRAM>{}); break;
  }
}

}  // namespace

template <class T>
void lookup_range_batch(const Launch& L, const TopModel& top, int leaf_kind, const void* recs, u64 N, const T* keys,
                        u64 n, T last, const T* q, u64 nq, u64* out_first, u64* out_last, u64* fallbacks) {
  if (nq == 0) return;
  with_groups(top.kind, leaf_kind, [&](auto tk, auto lk) {
    k_lookup_range<T, decltype(tk)::value, decltype(lk)::value><<<range_blocks(L, nq), LOOKUP_THREADS, 0, L.stream>>>(
        top, (const ulonglong2*)recs, keys, n, last, N, q, nq, out_first, out_last, fallbacks, out_first ? 1 : 0);
  });
  count_launch();
}

void lookup_bounded_range_batch(const Launch& L, const TopModel& top, int leaf_kind, const void* recs, u64 N,
                                const void* knots, u64 K, u64 line, const u64* keys, u64 n, u64 last, const u64* q,
                                u64 nq, u64* out_first, u64* out_last, u64* fallbacks) {
  if (nq == 0) return;
  with_groups(top.kind, leaf_kind, [&](auto tk, auto lk) {
    k_lookup_bounded_range<decltype(tk)::value, decltype(lk)::value><<<range_blocks(L, nq), LOOKUP_THREADS, 0,
                                                                       L.stream>>>(
        top, (const ulonglong2*)recs, N, (const ulonglong2*)knots, K, line, keys, n, last, q, nq, out_first, out_last,
        fallbacks, out_first ? 1 : 0);
  });
  count_launch();
}

#define RMI_LOOKUP_RANGE_INST(T)                                                                                   \
  template void lookup_range_batch<T>(const Launch&, const TopModel&, int, const void*, u64, const T*, u64, T,      \
                                      const T*, u64, u64*, u64*, u64*);
RMI_LOOKUP_RANGE_INST(u64)
RMI_LOOKUP_RANGE_INST(u32)
RMI_LOOKUP_RANGE_INST(double)
#undef RMI_LOOKUP_RANGE_INST

}  // namespace rmi
