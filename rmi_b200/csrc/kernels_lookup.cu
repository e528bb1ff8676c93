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
// Thread mapping: a block takes a tile of LOOKUP_THREADS * LOOKUP_Q consecutive queries (grid-stride over
// tiles); thread x owns queries x, x + LOOKUP_THREADS, ... of the tile, so every query load and result store
// is coalesced.  The thread carries its LOOKUP_Q queries through the dependent chain — top model, leaf record,
// key probes — in lockstep, which keeps LOOKUP_Q independent loads in flight per step.
#include <cstring>

#include "kernels.h"
#include "lookup_search.cuh"
#include "spline.cuh"

namespace rmi {

namespace {

template <class T, int TOP, int LEAF>
__global__ void __launch_bounds__(LOOKUP_THREADS)
k_lookup(const __grid_constant__ TopModel top, const ulonglong2* __restrict__ recs, const T* __restrict__ keys, u64 n,
         u64 N, const T* __restrict__ qs, u64 nq, u64* __restrict__ out, u64* __restrict__ out_err, u64* fallbacks,
         int lower_bound) {
  using R = Rec<LEAF>;
  constexpr int Q = LOOKUP_Q;
  const u64 tile = (u64)LOOKUP_THREADS * Q;
  unsigned misses = 0;
  for (u64 base = (u64)blockIdx.x * tile; base < nq; base += (u64)gridDim.x * tile) {
    T q[Q];
    bool live[Q];
    u64 t[Q];
#pragma unroll
    for (int j = 0; j < Q; ++j) {
      u64 i = base + threadIdx.x + (u64)j * LOOKUP_THREADS;
      live[j] = i < nq;
      q[j] = live[j] ? __ldcs(qs + i) : T(0);
    }
#pragma unroll
    for (int j = 0; j < Q; ++j) {
      u64 p = top_predict<TOP>(top, q[j]);
      t[j] = p < N - 1 ? p : N - 1;
    }
    ulonglong2 v[Q][R::LOADS];
#pragma unroll
    for (int j = 0; j < Q; ++j)
#pragma unroll
      for (int k = 0; k < R::LOADS; ++k) v[j][k] = __ldg(recs + t[j] * R::VECS + k);
    u64 pos[Q], err[Q];
#pragma unroll
    for (int j = 0; j < Q; ++j) {
      double f[4];
      R::unpack(v[j], f, err[j]);
      u64 p = leaf_predict64<LEAF>(f, Key<T>::as_float(q[j]));
      pos[j] = p < n - 1 ? p : n - 1;
    }
    if (!lower_bound) {
#pragma unroll
      for (int j = 0; j < Q; ++j) {
        u64 i = base + threadIdx.x + (u64)j * LOOKUP_THREADS;
        if (!live[j]) continue;
        __stcs(out + i, pos[j]);
        if (out_err) __stcs(out_err + i, err[j]);
      }
      continue;
    }
    // window [lo, hi] of candidate answers; the search covers keys [lo, hi)
    u64 lo[Q], hi[Q];
#pragma unroll
    for (int j = 0; j < Q; ++j) {
      lo[j] = pos[j] >= err[j] ? pos[j] - err[j] : 0;
      hi[j] = err[j] >= n - pos[j] ? n : pos[j] + err[j];
    }
    window_search<T, Q>(keys, n, q, live, lo, hi, misses,
                        [&](int j, u64 r) { __stcs(out + base + threadIdx.x + (u64)j * LOOKUP_THREADS, r); });
  }
  if (fallbacks) {
    misses = __reduce_add_sync(0xffffffffu, misses);
    if ((threadIdx.x & 31) == 0 && misses) atomicAdd((unsigned long long*)fallbacks, (unsigned long long)misses);
  }
}

template <class T, int TOP, int LEAF>
void launch_lookup(const Launch& L, const TopModel& top, const void* recs, u64 N, const T* keys, u64 n, const T* q,
                   u64 nq, u64* out, u64* out_err, u64* fallbacks, bool lower_bound) {
  const u64 tile = (u64)LOOKUP_THREADS * LOOKUP_Q;
  u64 blocks = (nq + tile - 1) / tile;
  const u64 cap = (u64)L.num_sms * LOOKUP_MAX_BLOCKS_PER_SM;
  if (blocks > cap) blocks = cap;
  k_lookup<T, TOP, LEAF><<<(unsigned)blocks, LOOKUP_THREADS, 0, L.stream>>>(
      top, (const ulonglong2*)recs, keys, n, N, q, nq, out, out_err, fallbacks, lower_bound ? 1 : 0);
  count_launch();
}

template <class T, int TOP>
void lookup_leaf(const Launch& L, const TopModel& top, int leaf_kind, const void* recs, u64 N, const T* keys, u64 n,
                 const T* q, u64 nq, u64* out, u64* out_err, u64* fallbacks, bool lb) {
  switch (lookup_leaf_group(leaf_kind)) {
    case M_LINEAR: launch_lookup<T, TOP, M_LINEAR>(L, top, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
    case M_CUBIC: launch_lookup<T, TOP, M_CUBIC>(L, top, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
    case M_LOGLINEAR: launch_lookup<T, TOP, M_LOGLINEAR>(L, top, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
    case M_NORMAL: launch_lookup<T, TOP, M_NORMAL>(L, top, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
    default: launch_lookup<T, TOP, M_LOGNORMAL>(L, top, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
  }
}

// ---- bounded (`--bounded`, cache-fix) index ------------------------------------------------------------------
// The RMI runs over the K spline knots.  predict: (start, e) as above with K rows; res = the first knot in
// [start-e, start+e) ∩ [0, K) whose key is not < q; the spline between knots res-1 and res gives the key's
// position, rounded down to its line (codegen.rs:410-437).  lower_bound: the answer lies in [pos, pos + line]
// for every key of the data set (the spline's construction), so the kernel searches that window only.
//
// The knot-window search and the key-line step are lookup_search.cuh's (knot_window_search, RMI_LINE_SEARCH), shared
// with the search over a rank's slab of a range-partitioned data set (kernels_shard_bounded.cu).

template <int TOP, int LEAF>
__global__ void __launch_bounds__(LOOKUP_THREADS)
k_lookup_bounded(const __grid_constant__ TopModel top, const ulonglong2* __restrict__ recs, u64 N,
                 const ulonglong2* __restrict__ knots, u64 K, u64 line, const u64* __restrict__ keys, u64 n,
                 const u64* __restrict__ qs, u64 nq, u64* __restrict__ out, u64* __restrict__ out_err, u64* fallbacks,
                 int lower_bound) {
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
    // knot window [lower, upper); upper saturates where start + e would pass K
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
  if (fallbacks) {
    misses = __reduce_add_sync(0xffffffffu, misses);
    if ((threadIdx.x & 31) == 0 && misses) atomicAdd((unsigned long long*)fallbacks, (unsigned long long)misses);
  }
}

template <int TOP, int LEAF>
void launch_lookup_bounded(const Launch& L, const TopModel& top, const void* recs, u64 N, const void* knots, u64 K,
                           u64 line, const u64* keys, u64 n, const u64* q, u64 nq, u64* out, u64* out_err,
                           u64* fallbacks, bool lower_bound) {
  u64 blocks = (nq + LOOKUP_THREADS - 1) / LOOKUP_THREADS;
  const u64 cap = (u64)L.num_sms * LOOKUP_MAX_BLOCKS_PER_SM;
  if (blocks > cap) blocks = cap;
  k_lookup_bounded<TOP, LEAF><<<(unsigned)blocks, LOOKUP_THREADS, 0, L.stream>>>(
      top, (const ulonglong2*)recs, N, (const ulonglong2*)knots, K, line, keys, n, q, nq, out, out_err, fallbacks,
      lower_bound ? 1 : 0);
  count_launch();
}

#define RMI_BOUNDED_ARGS recs, N, knots, K, line, keys, n, q, nq, out, out_err, fallbacks, lb
template <int TOP>
void lookup_bounded_leaf(const Launch& L, const TopModel& top, int leaf_kind, const void* recs, u64 N,
                         const void* knots, u64 K, u64 line, const u64* keys, u64 n, const u64* q, u64 nq, u64* out,
                         u64* out_err, u64* fallbacks, bool lb) {
  switch (lookup_leaf_group(leaf_kind)) {
    case M_LINEAR: launch_lookup_bounded<TOP, M_LINEAR>(L, top, RMI_BOUNDED_ARGS); break;
    case M_CUBIC: launch_lookup_bounded<TOP, M_CUBIC>(L, top, RMI_BOUNDED_ARGS); break;
    case M_LOGLINEAR: launch_lookup_bounded<TOP, M_LOGLINEAR>(L, top, RMI_BOUNDED_ARGS); break;
    case M_NORMAL: launch_lookup_bounded<TOP, M_NORMAL>(L, top, RMI_BOUNDED_ARGS); break;
    default: launch_lookup_bounded<TOP, M_LOGNORMAL>(L, top, RMI_BOUNDED_ARGS); break;
  }
}

}  // namespace

void lookup_bounded_batch(const Launch& L, const TopModel& top, int leaf_kind, const void* recs, u64 N,
                          const void* knots, u64 K, u64 line, const u64* keys, u64 n, const u64* q, u64 nq, u64* out,
                          u64* out_err, u64* fallbacks, bool lb) {
  if (nq == 0) return;
  switch (lookup_top_group(top.kind)) {
    case M_LINEAR: lookup_bounded_leaf<M_LINEAR>(L, top, leaf_kind, RMI_BOUNDED_ARGS); break;
    case M_CUBIC: lookup_bounded_leaf<M_CUBIC>(L, top, leaf_kind, RMI_BOUNDED_ARGS); break;
    case M_LOGLINEAR: lookup_bounded_leaf<M_LOGLINEAR>(L, top, leaf_kind, RMI_BOUNDED_ARGS); break;
    case M_NORMAL: lookup_bounded_leaf<M_NORMAL>(L, top, leaf_kind, RMI_BOUNDED_ARGS); break;
    case M_LOGNORMAL: lookup_bounded_leaf<M_LOGNORMAL>(L, top, leaf_kind, RMI_BOUNDED_ARGS); break;
    case M_RADIX: lookup_bounded_leaf<M_RADIX>(L, top, leaf_kind, RMI_BOUNDED_ARGS); break;
    case M_RADIX_TABLE: lookup_bounded_leaf<M_RADIX_TABLE>(L, top, leaf_kind, RMI_BOUNDED_ARGS); break;
    case M_BRADIX: lookup_bounded_leaf<M_BRADIX>(L, top, leaf_kind, RMI_BOUNDED_ARGS); break;
    default: lookup_bounded_leaf<M_HISTOGRAM>(L, top, leaf_kind, RMI_BOUNDED_ARGS); break;
  }
}
#undef RMI_BOUNDED_ARGS

int lookup_top_group(int kind) {
  if (kind == M_LINEAR || kind == M_ROBUST_LINEAR || kind == M_LINEAR_SPLINE) return M_LINEAR;
  return kind >= M_LINEAR && kind <= M_HISTOGRAM ? kind : -1;
}
int lookup_leaf_group(int kind) {
  if (kind == M_LINEAR || kind == M_ROBUST_LINEAR || kind == M_LINEAR_SPLINE) return M_LINEAR;
  return kind >= M_CUBIC && kind <= M_LOGNORMAL ? kind : -1;
}

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
void lookup_batch(const Launch& L, const TopModel& top, int leaf_kind, const void* recs, u64 N, const T* keys, u64 n,
                  const T* q, u64 nq, u64* out, u64* out_err, u64* fallbacks, bool lb) {
  if (nq == 0) return;
  switch (lookup_top_group(top.kind)) {
    case M_LINEAR: lookup_leaf<T, M_LINEAR>(L, top, leaf_kind, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
    case M_CUBIC: lookup_leaf<T, M_CUBIC>(L, top, leaf_kind, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
    case M_LOGLINEAR: lookup_leaf<T, M_LOGLINEAR>(L, top, leaf_kind, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
    case M_NORMAL: lookup_leaf<T, M_NORMAL>(L, top, leaf_kind, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
    case M_LOGNORMAL: lookup_leaf<T, M_LOGNORMAL>(L, top, leaf_kind, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
    case M_RADIX: lookup_leaf<T, M_RADIX>(L, top, leaf_kind, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
    case M_RADIX_TABLE: lookup_leaf<T, M_RADIX_TABLE>(L, top, leaf_kind, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
    case M_BRADIX: lookup_leaf<T, M_BRADIX>(L, top, leaf_kind, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
    default: lookup_leaf<T, M_HISTOGRAM>(L, top, leaf_kind, recs, N, keys, n, q, nq, out, out_err, fallbacks, lb); break;
  }
}

#define RMI_LOOKUP_INST(T)                                                                                        \
  template void lookup_batch<T>(const Launch&, const TopModel&, int, const void*, u64, const T*, u64, const T*, u64, \
                                u64*, u64*, u64*, bool);
RMI_LOOKUP_INST(u64)
RMI_LOOKUP_INST(u32)
RMI_LOOKUP_INST(double)
#undef RMI_LOOKUP_INST

}  // namespace rmi
