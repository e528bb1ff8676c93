// kernels_lookup.cu — batched lookups on a trained two-layer RMI (DESIGN §11).
//
// predict:      t = min(N-1, top(q)),  pos = min(n-1, leaf[t](q)),  err = error bound of leaf t
//               — the generated code's lookup(key, &err) (codegen.rs:612-718), with NaN -> 0 where the
//               generated code's FCLAMP is undefined.
// lower_bound:  the number of keys k with k < q, found by a branchless binary search over the window
//               [pos-err, pos+err] (clamped to [0, n]) and confirmed by the keys just outside it.  A window
//               that does not bracket the answer falls back to a galloping search outward from its edge
//               and is counted.  For every key of the data set the window brackets the answer (the
//               reference's property, tests/simple_model_wiki/main.cpp:26-42), so the fallback only runs
//               for queries the index was not trained on.  The window search lives in lookup_search.cuh, shared
//               with the search over a rank's slab of a range-partitioned data set (kernels_shard_lookup.cu).
//
// Thread mapping: a block takes a tile of LOOKUP_THREADS consecutive queries, one per thread (grid-stride over tiles),
// so every query load and result store is coalesced.  DESIGN §11 gives the sweep over queries per thread that chose
// one.
#include <cstring>

#include "kernels.h"
#include "lookup_search.cuh"

namespace rmi {

namespace {

template <class T, int TOP, int LEAF>
__global__ void __launch_bounds__(LOOKUP_THREADS)
k_lookup(const __grid_constant__ TopModel top, const ulonglong2* __restrict__ recs, const T* __restrict__ keys, u64 n,
         u64 N, const T* __restrict__ qs, u64 nq, u64* __restrict__ out, u64* __restrict__ out_err, u64* fallbacks,
         int lower_bound) {
  unsigned misses = 0;
  // the loop runs over the blocks' tiles of queries, so a warp's lanes leave it together; a lane past nq computes on
  // a dummy query and stores nothing (on an H100, a per-lane loop condition made the headline lower_bound about 1%
  // slower)
  for (u64 base = (u64)blockIdx.x * LOOKUP_THREADS; base < nq; base += (u64)gridDim.x * LOOKUP_THREADS) {
    const u64 i = base + threadIdx.x;
    const bool live[1] = {i < nq};
    const T q[1] = {live[0] ? __ldcs(qs + i) : T(0)};
    u64 err;
    const u64 pos = rmi_predict<TOP, LEAF>(top, recs, N, n, q[0], err);
    if (!lower_bound) {
      if (!live[0]) continue;
      __stcs(out + i, pos);
      if (out_err) __stcs(out_err + i, err);
      continue;
    }
    const Window w = error_window(pos, err, n);
    const u64 lo[1] = {w.lo}, hi[1] = {w.hi};
    window_search<T, 1>(keys, n, q, live, lo, hi, misses, [&](int, u64 r) { __stcs(out + i, r); });
  }
  flush_fallbacks(misses, fallbacks);
}

// ---- bounded (`--bounded`, cache-fix) index ------------------------------------------------------------------
// The RMI runs over the K spline knots.  predict: (start, e) as above with K rows; res = the first knot in
// [start-e, start+e) ∩ [0, K) whose key is not < q; the spline between knots res-1 and res gives the key's
// position, rounded down to its line (codegen.rs:410-437).  lower_bound: the answer lies in [pos, pos + line]
// for every key of the data set (the spline's construction), so the kernel searches that window only.
//
// The spline step and the key-line step are lookup_search.cuh's (bounded_pos, RMI_LINE_SEARCH), shared with the
// search over a rank's slab of a range-partitioned data set (kernels_shard_bounded.cu).

template <int TOP, int LEAF>
__global__ void __launch_bounds__(LOOKUP_THREADS)
k_lookup_bounded(const __grid_constant__ TopModel top, const ulonglong2* __restrict__ recs, u64 N,
                 const ulonglong2* __restrict__ knots, u64 K, u64 line, const u64* __restrict__ keys, u64 n,
                 const u64* __restrict__ qs, u64 nq, u64* __restrict__ out, u64* __restrict__ out_err, u64* fallbacks,
                 int lower_bound) {
  unsigned misses = 0;
  for (u64 i = (u64)blockIdx.x * LOOKUP_THREADS + threadIdx.x; i < nq; i += (u64)gridDim.x * LOOKUP_THREADS) {
    const u64 q = __ldcs(qs + i);
    u64 e;
    const u64 start = rmi_predict<TOP, LEAF>(top, recs, N, K, q, e);
    // knot window [lower, upper); upper saturates where start + e would pass K
    const Window kw = error_window(start, e, K);
    const u64 pos = bounded_pos(knots, 0, kw.lo, kw.hi, K, n, line, q);
    if (!lower_bound) {
      __stcs(out + i, pos);
      if (out_err) __stcs(out_err + i, line);
      continue;
    }
    const u64 lo = pos < n ? pos : n;
    const u64 hi = line >= n - lo ? n : lo + line;
    u64 r;
    RMI_LINE_SEARCH(keys, n, q, lo, hi, line, misses, r);
    __stcs(out + i, r);
  }
  flush_fallbacks(misses, fallbacks);
}

}  // namespace

// The upper-bound and equal-range launches of the two entries below (kernels_lookup_range.cu, which compiles apart so
// that the two files' kernel instances build in parallel).
template <class T>
void launch_range(const Launch& L, LookupMode mode, const TopModel& top, int leaf_kind, const void* recs, u64 N,
                  const T* keys, u64 n, T last, const T* q, u64 nq, u64* out, u64* out2, u64* fallbacks);
void launch_bounded_range(const Launch& L, LookupMode mode, const TopModel& top, int leaf_kind, const void* recs, u64 N,
                          const void* knots, u64 K, u64 line, const u64* keys, u64 n, u64 last, const u64* q, u64 nq,
                          u64* out, u64* out2, u64* fallbacks);

void pack_leaf_records(int leaf_kind, const double* params, const u64* errors, u64 N, void* out) {
  const int ppm = leaf_params_per_model(leaf_kind);
  const u64 words = lookup_record_bytes(leaf_kind) / 8;
  u64* o = (u64*)out;
  for (u64 j = 0; j < N; ++j, o += words) {
    for (u64 w = 0; w < words; ++w) o[w] = 0;
    for (int p = 0; p < ppm; ++p) memcpy(&o[p], &params[j * ppm + p], 8);
    o[leaf_kind == M_CUBIC ? 4 : 3] = errors[j];
  }
}

template <class T>
void lookup_batch(const Launch& L, LookupMode mode, const TopModel& top, int leaf_kind, const void* recs, u64 N,
                  const T* keys, u64 n, T last, const T* q, u64 nq, u64* out, u64* out2, u64* fallbacks) {
  if (nq == 0) return;
  if (mode == LOOKUP_UPPER || mode == LOOKUP_EQUAL_RANGE)
    launch_range<T>(L, mode, top, leaf_kind, recs, N, keys, n, last, q, nq, out, out2, fallbacks);
  else
    with_groups(top.kind, leaf_kind, [&](auto tk, auto lk) {
      k_lookup<T, decltype(tk)::value, decltype(lk)::value>
          <<<capped_grid(L, nq, LOOKUP_THREADS, LOOKUP_MAX_BLOCKS_PER_SM), LOOKUP_THREADS, 0, L.stream>>>(
              top, (const ulonglong2*)recs, keys, n, N, q, nq, out, out2, fallbacks, mode == LOOKUP_LOWER ? 1 : 0);
    });
  count_launch();
}

void lookup_bounded_batch(const Launch& L, LookupMode mode, const TopModel& top, int leaf_kind, const void* recs,
                          u64 N, const void* knots, u64 K, u64 line, const u64* keys, u64 n, u64 last, const u64* q,
                          u64 nq, u64* out, u64* out2, u64* fallbacks) {
  if (nq == 0) return;
  if (mode == LOOKUP_UPPER || mode == LOOKUP_EQUAL_RANGE)
    launch_bounded_range(L, mode, top, leaf_kind, recs, N, knots, K, line, keys, n, last, q, nq, out, out2, fallbacks);
  else
    with_groups(top.kind, leaf_kind, [&](auto tk, auto lk) {
      k_lookup_bounded<decltype(tk)::value, decltype(lk)::value>
          <<<capped_grid(L, nq, LOOKUP_THREADS, LOOKUP_MAX_BLOCKS_PER_SM), LOOKUP_THREADS, 0, L.stream>>>(
              top, (const ulonglong2*)recs, N, (const ulonglong2*)knots, K, line, keys, n, q, nq, out, out2,
              fallbacks, mode == LOOKUP_LOWER ? 1 : 0);
    });
  count_launch();
}

#define RMI_LOOKUP_INST(T)                                                                                          \
  template void lookup_batch<T>(const Launch&, LookupMode, const TopModel&, int, const void*, u64, const T*, u64, T, \
                                const T*, u64, u64*, u64*, u64*);
RMI_LOOKUP_INST(u64)
RMI_LOOKUP_INST(u32)
RMI_LOOKUP_INST(double)
#undef RMI_LOOKUP_INST

}  // namespace rmi
