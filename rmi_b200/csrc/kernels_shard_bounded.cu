// kernels_shard_bounded.cu — `--bounded` lookups over a range-partitioned data set (DESIGN §17).
//
// Rank r holds its key slab (global keys [base, base + n_local)) and its knot slab: the knots whose key routes to r by
// §14's rule, global knots [a0, a1), with a halo of knots on each side, global knots [k_lo, k_lo + k_len) in all.
//
// search   lower bounds of queries routed to r BY KEY.  The knot RMI gives (start, e) and the knot window
//          [lower, upper) as on one GPU.  When the closed window [lower, upper] meets [a0, a1], the answer knot lies in
//          the knot slab or is the first knot after it, and the window lies inside the halo: the single-GPU knot search
//          and spline step over the extended knots give the single-GPU pos, bit for bit.  The key line [pos, pos + line]
//          is shifted by -base and clamped to the slab, and searched with the single-GPU key-line step; the slab's edges
//          confirm themselves (§14).  A "far" query, whose window misses [a0, a1], may need knots past the halo: it
//          searches the whole slab instead, exactly, and is always counted as a fallback.  Any other query is counted
//          when its global line [pos, pos + line] does not hold its lower bound, as on one GPU.
// upper    (UPPER) upper bounds of queries routed to r by key with <= (DESIGN §18): the same steps with k <= q.  A query
//          equal to r's first key F may have its answer knot up to two knots before a0 (the knots with keys F - 1 and F
//          route to an earlier rank), but a non-far query's reads lie in [lower - 1, upper] wherever that knot is, and
//          the window meets [a0, a1], so they stay inside the halo of 2 e_max + 2.  A query >= the slab's last key gets
//          base + n_local without a search, uncounted.
// predict  pos of queries routed to r BY KNOT INDEX (the rank whose knot slab holds lower = start - e): the window and
//          the knot before it lie inside the halo, so every pos is the single-GPU one.
// The route by knot index reuses §14's route over the values lower + 1 (knot_route_keys), then moves the queries
// themselves to the positions the route gave (scatter_queries).
#include "kernels.h"
#include "lookup_search.cuh"

namespace rmi {

namespace {

constexpr int SB_THREADS = 128;
constexpr int SB_MAX_BLOCKS_PER_SM = 32;

template <int TOP, int LEAF, bool UPPER>
__global__ void __launch_bounds__(SB_THREADS)
k_shard_bounded(const __grid_constant__ TopModel top, const ulonglong2* __restrict__ recs, u64 N,
                const __grid_constant__ BoundedKnotSlab ks, const u64* __restrict__ keys, u64 n_local, u64 base,
                u64 n_global, const u64* __restrict__ qs, u64 m, u64* __restrict__ out, u64* fallbacks,
                int lower_bound, u64 last) {
  const ulonglong2* __restrict__ kext = (const ulonglong2*)ks.knots;
  const u64 K = ks.K, line = ks.line;
  unsigned misses = 0, local_misses = 0;
  for (u64 i = (u64)blockIdx.x * SB_THREADS + threadIdx.x; i < m; i += (u64)gridDim.x * SB_THREADS) {
    const u64 q = __ldcs(qs + i);
    if (UPPER && q >= last) {
      __stcs(out + i, base + n_local);
      continue;
    }
    u64 e;
    const u64 start = rmi_predict<TOP, LEAF>(top, recs, N, K, q, e);
    const Window kw = error_window(start, e, K);
    u64 r;
    if (lower_bound && (kw.hi < ks.a0 || kw.lo > ks.a1)) {
      // far: the whole slab, whose edges confirm themselves
      RMI_LINE_SEARCH_AS(keys, n_local, q, (u64)0, n_local, n_local, local_misses, r, UPPER);
      ++misses;
      __stcs(out + i, base + r);
      continue;
    }
    const u64 pos = bounded_pos(kext, ks.k_lo, kw.lo, kw.hi, K, n_global, line, q);
    if (!lower_bound) {
      __stcs(out + i, pos);
      continue;
    }
    // the global line, then its part inside this slab
    const u64 glo = pos < n_global ? pos : n_global;
    const u64 ghi = line >= n_global - glo ? n_global : glo + line;
    const u64 lo = glo <= base ? 0 : (glo - base < n_local ? glo - base : n_local);
    const u64 hi = ghi <= base ? 0 : (ghi - base < n_local ? ghi - base : n_local);
    RMI_LINE_SEARCH_AS(keys, n_local, q, lo, hi, line, local_misses, r, UPPER);
    if (base + r < glo || base + r > ghi) ++misses;
    __stcs(out + i, base + r);
  }
  flush_fallbacks(misses, fallbacks);
}

__global__ void __launch_bounds__(256)
k_knot_route_keys(const u64* pos, const u64* err, u64 n, u64* out) {   // out may be pos (in place)
  for (u64 i = (u64)blockIdx.x * 256 + threadIdx.x; i < n; i += (u64)gridDim.x * 256) {
    const u64 p = __ldcs(pos + i), e = __ldcs(err + i);
    __stcs(out + i, (p >= e ? p - e : 0) + 1);
  }
}

__global__ void __launch_bounds__(256)
k_scatter_queries(const u64* __restrict__ q, const u64* __restrict__ slot, u64 n, u64* __restrict__ send) {
  for (u64 i = (u64)blockIdx.x * 256 + threadIdx.x; i < n; i += (u64)gridDim.x * 256)
    send[__ldcs(slot + i)] = __ldcs(q + i);
}

__global__ void __launch_bounds__(256) k_fill(u64 v, u64 n, u64* __restrict__ out) {
  for (u64 i = (u64)blockIdx.x * 256 + threadIdx.x; i < n; i += (u64)gridDim.x * 256) __stcs(out + i, v);
}

}  // namespace

void shard_bounded_search(const Launch& L, const TopModel& top, int leaf_kind, const void* recs, u64 N,
                          const BoundedKnotSlab& ks, const u64* keys, u64 n_local, u64 base, u64 n_global, const u64* q,
                          u64 m, u64* out, u64* fallbacks, bool lb, bool upper, u64 last) {
  if (m == 0) return;
  const unsigned blocks = capped_grid(L, m, SB_THREADS, SB_MAX_BLOCKS_PER_SM);
  with_groups(top.kind, leaf_kind, [&](auto tk, auto lk) {
    constexpr int TOP = decltype(tk)::value, LEAF = decltype(lk)::value;
    if (upper)
      k_shard_bounded<TOP, LEAF, true><<<blocks, SB_THREADS, 0, L.stream>>>(
          top, (const ulonglong2*)recs, N, ks, keys, n_local, base, n_global, q, m, out, fallbacks, 1, last);
    else
      k_shard_bounded<TOP, LEAF, false><<<blocks, SB_THREADS, 0, L.stream>>>(
          top, (const ulonglong2*)recs, N, ks, keys, n_local, base, n_global, q, m, out, fallbacks, lb ? 1 : 0, last);
  });
  count_launch();
}

void shard_knot_route_keys(const Launch& L, const u64* d_pos, const u64* d_err, u64 n, u64* d_out) {
  if (n == 0) return;
  k_knot_route_keys<<<capped_grid(L, n, 256, 16), 256, 0, L.stream>>>(d_pos, d_err, n, d_out);
  count_launch();
}

void shard_scatter_queries(const Launch& L, const u64* d_q, const u64* d_slot, u64 n, u64* d_send) {
  if (n == 0) return;
  k_scatter_queries<<<capped_grid(L, n, 256, 16), 256, 0, L.stream>>>(d_q, d_slot, n, d_send);
  count_launch();
}

void shard_fill(const Launch& L, u64 value, u64 n, u64* d_out) {
  if (n == 0) return;
  k_fill<<<capped_grid(L, n, 256, 16), 256, 0, L.stream>>>(value, n, d_out);
  count_launch();
}

}  // namespace rmi
