// kernels_shard_lookup.cu — lookups over a range-partitioned data set (DESIGN §14).
//
// Rank r holds global keys [base_r, base_r + n_r).  A query q belongs to the last non-empty rank whose first key is
// < q (the first non-empty rank if none is, which includes a NaN query): every key before that rank's slab is < q and
// every key after it is not, so the global lower bound is base_r + the lower bound inside the slab.
//
// Upper bounds route by <= instead (DESIGN §18): the last non-empty rank whose first key is <= q, or the first non-empty
// rank.  Every key before that rank's slab is <= q and every key after it is > q, so the global upper bound is base_r +
// the upper bound inside the slab.  The two rules differ only for a query equal to some slab's first key.
//
// route    count / scan / scatter: each block takes a tile of ROUTE_THREADS * ROUTE_Q queries, finds every query's
//          rank by a binary search over the first keys (in shared memory) and counts queries per rank; one block scans
//          the (rank, block) counts rank-major; the scatter repeats the search and writes each query into its rank's
//          segment of the send buffer, and the position it got into slot[i].  Within a segment the order is that of
//          the warps' atomic reservations, not the callers' order; the answers come back by slot, so it does not
//          matter.
// search   over the queries a rank received: the predict kernel (kernels_lookup.cu, n = n_global) leaves pos / err in
//          scratch; the global window [pos - err, pos + err] is clamped to [0, n_global], shifted by -base and clamped
//          to [0, n_local], then searched with the single-GPU window search (lookup_search.cuh) over the slab.  The
//          slab's edges confirm themselves (lo == 0, hi == n_local) by the routing rule, so no key outside the slab is
//          read.
// gather   out[i] = returned[slot[i]].
#include "kernels.h"
#include "lookup_search.cuh"

namespace rmi {

namespace {

constexpr int ROUTE_THREADS = 256;
constexpr int ROUTE_Q = 16;   // queries per thread: a block's tile is 4096 queries, so the scan has n / 4096 x world entries
constexpr u64 ROUTE_TILE = (u64)ROUTE_THREADS * ROUTE_Q;
constexpr int SCAN_THREADS = 1024;
constexpr int SEARCH_THREADS = 128;
constexpr int SEARCH_MAX_BLOCKS_PER_SM = 32;

// Index into route.rank of the non-empty rank that owns q: the number of first keys < q (<= q for UPPER), less one
// (0 if none).  The first keys are in order, so the ones < q (<= q) are a prefix.
template <class T, bool UPPER = false> __device__ __forceinline__ int route_slot(const T* s_first, int count, T q) {
  int lo = 0, len = count;
  while (len > 0) {
    const int h = len >> 1;
    if (UPPER ? s_first[lo + h] <= q : s_first[lo + h] < q) { lo += h + 1; len -= h + 1; } else { len = h; }
  }
  return lo > 0 ? lo - 1 : 0;
}

template <class T>
__device__ __forceinline__ void route_load(const ShardRoute<T>& route, T* s_first, unsigned char* s_rank) {
  if ((int)threadIdx.x < route.count) {
    s_first[threadIdx.x] = route.first[threadIdx.x];
    s_rank[threadIdx.x] = route.rank[threadIdx.x];
  }
}

template <class T, bool UPPER>
__global__ void __launch_bounds__(ROUTE_THREADS)
k_route_count(const __grid_constant__ ShardRoute<T> route, const T* __restrict__ qs, u64 n, int world, u64 nblocks,
              u32* __restrict__ block_counts) {
  __shared__ T s_first[SHARD_ROUTE_MAX];
  __shared__ unsigned char s_rank[SHARD_ROUTE_MAX];
  __shared__ u32 s_count[SHARD_ROUTE_MAX];
  route_load(route, s_first, s_rank);
  if ((int)threadIdx.x < world) s_count[threadIdx.x] = 0;
  __syncthreads();
  const unsigned lane = threadIdx.x & 31;
  const u64 tile = (u64)blockIdx.x * ROUTE_TILE;
#pragma unroll 4
  for (int j = 0; j < ROUTE_Q; ++j) {
    const u64 i = tile + (u64)j * ROUTE_THREADS + threadIdx.x;
    const unsigned active = __ballot_sync(0xffffffffu, i < n);
    if (i < n) {
      const int d = s_rank[route_slot<T, UPPER>(s_first, route.count, __ldg(qs + i))];
      const unsigned peers = __match_any_sync(active, d);
      if (lane == (unsigned)(__ffs(peers) - 1)) atomicAdd(&s_count[d], (u32)__popc(peers));
    }
  }
  __syncthreads();
  if ((int)threadIdx.x < world) block_counts[(u64)threadIdx.x * nblocks + blockIdx.x] = s_count[threadIdx.x];
}

// One block: exclusive scan of the world x nblocks counts (rank-major), and every rank's total.
__global__ void __launch_bounds__(SCAN_THREADS)
k_route_scan(const u32* __restrict__ counts, u64 total, u64 nblocks, int world, u64* __restrict__ offsets,
             u64* __restrict__ send_counts) {
  __shared__ u64 s_warp[SCAN_THREADS / 32];
  const u64 chunk = (total + SCAN_THREADS - 1) / SCAN_THREADS;
  const u64 a = (u64)threadIdx.x * chunk, b = a + chunk < total ? a + chunk : total;
  u64 sum = 0;
  for (u64 k = a; k < b; ++k) sum += counts[k];
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  u64 incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const u64 v = __shfl_up_sync(0xffffffffu, incl, o);
    if ((int)lane >= o) incl += v;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    u64 w = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const u64 v = __shfl_up_sync(0xffffffffu, w, o);
      if ((int)lane >= o) w += v;
    }
    s_warp[lane] = w;   // inclusive over warps
  }
  __syncthreads();
  u64 run = incl - sum + (warp > 0 ? s_warp[warp - 1] : 0);
  for (u64 k = a; k < b; ++k) {
    offsets[k] = run;
    run += counts[k];
  }
  __syncthreads();
  if ((int)threadIdx.x < world) {
    const u64 grand = s_warp[SCAN_THREADS / 32 - 1];
    const u64 d = threadIdx.x;
    const u64 start = offsets[d * nblocks];
    const u64 end = d + 1 < (u64)world ? offsets[(d + 1) * nblocks] : grand;
    send_counts[d] = end - start;
  }
}

template <class T, bool UPPER>
__global__ void __launch_bounds__(ROUTE_THREADS)
k_route_scatter(const __grid_constant__ ShardRoute<T> route, const T* __restrict__ qs, u64 n, int world, u64 nblocks,
                const u64* __restrict__ offsets, T* __restrict__ send, u64* __restrict__ slot) {
  __shared__ T s_first[SHARD_ROUTE_MAX];
  __shared__ unsigned char s_rank[SHARD_ROUTE_MAX];
  __shared__ unsigned long long s_next[SHARD_ROUTE_MAX];
  route_load(route, s_first, s_rank);
  if ((int)threadIdx.x < world) s_next[threadIdx.x] = offsets[(u64)threadIdx.x * nblocks + blockIdx.x];
  __syncthreads();
  const unsigned lane = threadIdx.x & 31;
  const unsigned below = (1u << lane) - 1u;
  const u64 tile = (u64)blockIdx.x * ROUTE_TILE;
#pragma unroll 4
  for (int j = 0; j < ROUTE_Q; ++j) {
    const u64 i = tile + (u64)j * ROUTE_THREADS + threadIdx.x;
    const unsigned active = __ballot_sync(0xffffffffu, i < n);
    if (i < n) {
      const T q = __ldcs(qs + i);
      const int d = s_rank[route_slot<T, UPPER>(s_first, route.count, q)];
      const unsigned peers = __match_any_sync(active, d);
      const int leader = __ffs(peers) - 1;
      unsigned long long p = 0;
      if ((int)lane == leader) p = atomicAdd(&s_next[d], (unsigned long long)__popc(peers));
      p = __shfl_sync(peers, p, leader) + __popc(peers & below);
      send[p] = q;
      __stcs(slot + i, (u64)p);
    }
  }
}

// UPPER: upper bounds of queries routed by <=; last = keys[n_local - 1], and a query >= it gets base + n_local without
// a search (the slab's final run is the one a leaf bound may not record).
template <class T, bool UPPER>
__global__ void __launch_bounds__(SEARCH_THREADS)
k_shard_search(const T* __restrict__ keys, u64 n_local, u64 base, u64 n_global, const T* __restrict__ qs, u64 m,
               const u64* __restrict__ pos, const u64* __restrict__ err, u64* __restrict__ out, u64* fallbacks,
               T last) {
  unsigned misses = 0;
  for (u64 i = (u64)blockIdx.x * SEARCH_THREADS + threadIdx.x; i < m; i += (u64)gridDim.x * SEARCH_THREADS) {
    const T q[1] = {__ldcs(qs + i)};
    if (UPPER && q[0] >= last) {
      __stcs(out + i, base + n_local);
      continue;
    }
    const bool live[1] = {true};
    const u64 p = __ldcs(pos + i), e = __ldcs(err + i);
    // the global window, then its part inside this slab
    const Window g = error_window(p, e, n_global);
    const u64 glo = g.lo, ghi = g.hi;
    u64 lo[1], hi[1];
    lo[0] = glo <= base ? 0 : (glo - base < n_local ? glo - base : n_local);
    hi[0] = ghi <= base ? 0 : (ghi - base < n_local ? ghi - base : n_local);
    window_search<T, 1, UPPER ? 1u : 0u>(keys, n_local, q, live, lo, hi, misses,
                                         [&](int, u64 r) { __stcs(out + i, base + r); });
  }
  flush_fallbacks(misses, fallbacks);
}

__global__ void __launch_bounds__(256)
k_shard_gather(const u64* __restrict__ slot, const u64* __restrict__ returned, u64 n, u64* __restrict__ out) {
  for (u64 i = (u64)blockIdx.x * 256 + threadIdx.x; i < n; i += (u64)gridDim.x * 256)
    __stcs(out + i, __ldg(returned + __ldcs(slot + i)));
}

}  // namespace

u64 shard_route_blocks(u64 n) { return (n + ROUTE_TILE - 1) / ROUTE_TILE; }

template <class T>
void shard_route(const Launch& L, const ShardRoute<T>& route, int world, const T* q, u64 n, u32* d_block_counts,
                 u64* d_block_offsets, T* d_send, u64* d_slot, u64* d_send_counts, bool upper) {
  if (n == 0) {
    cudaMemsetAsync(d_send_counts, 0, sizeof(u64) * world, L.stream);
    return;
  }
  const u64 nb = shard_route_blocks(n);
  if (upper)
    k_route_count<T, true><<<(unsigned)nb, ROUTE_THREADS, 0, L.stream>>>(route, q, n, world, nb, d_block_counts);
  else
    k_route_count<T, false><<<(unsigned)nb, ROUTE_THREADS, 0, L.stream>>>(route, q, n, world, nb, d_block_counts);
  count_launch();
  k_route_scan<<<1, SCAN_THREADS, 0, L.stream>>>(d_block_counts, nb * world, nb, world, d_block_offsets, d_send_counts);
  count_launch();
  if (upper)
    k_route_scatter<T, true><<<(unsigned)nb, ROUTE_THREADS, 0, L.stream>>>(route, q, n, world, nb, d_block_offsets,
                                                                            d_send, d_slot);
  else
    k_route_scatter<T, false><<<(unsigned)nb, ROUTE_THREADS, 0, L.stream>>>(route, q, n, world, nb, d_block_offsets,
                                                                             d_send, d_slot);
  count_launch();
}

template <class T>
void shard_search(const Launch& L, const T* keys, u64 n_local, u64 base, u64 n_global, const T* q, u64 m,
                  const u64* d_pos, const u64* d_err, u64* d_out, u64* d_fallbacks, bool upper, T last) {
  if (m == 0) return;
  const unsigned blocks = capped_grid(L, m, SEARCH_THREADS, SEARCH_MAX_BLOCKS_PER_SM);
  if (upper)
    k_shard_search<T, true><<<blocks, SEARCH_THREADS, 0, L.stream>>>(keys, n_local, base, n_global, q, m, d_pos, d_err,
                                                                     d_out, d_fallbacks, last);
  else
    k_shard_search<T, false><<<blocks, SEARCH_THREADS, 0, L.stream>>>(keys, n_local, base, n_global, q, m, d_pos, d_err,
                                                                      d_out, d_fallbacks, last);
  count_launch();
}

void shard_gather(const Launch& L, const u64* d_slot, const u64* d_returned, u64 n, u64* d_out) {
  if (n == 0) return;
  k_shard_gather<<<capped_grid(L, n, 256, 16), 256, 0, L.stream>>>(d_slot, d_returned, n, d_out);
  count_launch();
}

#define RMI_SHARD_LOOKUP_INST(T)                                                                                    \
  template void shard_route<T>(const Launch&, const ShardRoute<T>&, int, const T*, u64, u32*, u64*, T*, u64*, u64*, \
                               bool);                                                                              \
  template void shard_search<T>(const Launch&, const T*, u64, u64, u64, const T*, u64, const u64*, const u64*, u64*,  \
                                u64*, bool, T);
RMI_SHARD_LOOKUP_INST(u64)
RMI_SHARD_LOOKUP_INST(u32)
RMI_SHARD_LOOKUP_INST(double)
#undef RMI_SHARD_LOOKUP_INST

}  // namespace rmi
