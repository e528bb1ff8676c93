// kernels_delta.cu — the sorted delta of an updatable index (rmi_delta, DESIGN §19): the stable merge that inserts a
// batch into the delta or folds the delta into the base keys, and the pass that adds the delta's share to a lookup's
// answers.
//
// k_delta_merge:  merge path (merge_path.cuh).  Block b writes merged keys [b * MERGE_TILE, (b + 1) * MERGE_TILE): two
//                 of its threads find the co-ranks of the tile's diagonals by binary search over both inputs, the
//                 block copies the two slices between them into shared memory with coalesced loads, every thread
//                 merges MERGE_ITEMS keys from its own diagonal there, and the block stores the tile coalesced.  Each
//                 input key is loaded by exactly one block, so the NaN check of the second input (an f64 batch) is
//                 one comparison per key on the way in.
// k_delta_count:  one query per thread with k_lookup's mapping (LOOKUP_THREADS per block, grid-stride): a
//                 branchless binary search over the m delta keys adds #{d < q} (lower), #{d <= q} (upper) or both, in
//                 lockstep, to the answers the base index's launch left in place.  The queries and answers stream
//                 (ld/st.global.cs); the probes read the delta, which at 2^20 u64 keys (8 MiB) stays in L2.
#include "kernels.h"
#include "lookup_search.cuh"
#include "merge_path.cuh"

namespace rmi {

namespace {

template <class T>
__global__ void __launch_bounds__(MERGE_THREADS)
k_delta_merge(const T* __restrict__ a, u64 na, const T* __restrict__ b, u64 nb, T* __restrict__ out,
              unsigned* status) {
  __shared__ T s_in[MERGE_TILE];    // a's slice, then b's
  __shared__ T s_out[MERGE_TILE];
  __shared__ u64 s_rank[2];
  const u64 total = na + nb;
  const u64 d0 = (u64)blockIdx.x * MERGE_TILE;
  const u64 d1 = total - d0 < MERGE_TILE ? total : d0 + MERGE_TILE;
  if (threadIdx.x < 2) s_rank[threadIdx.x] = merge_corank(a, na, b, nb, threadIdx.x ? d1 : d0);
  __syncthreads();
  const u64 i0 = s_rank[0];
  u64 i1 = s_rank[1];
  i1 = i1 < i0 ? i0 : (i1 > i0 + (d1 - d0) ? i0 + (d1 - d0) : i1);   // as merge_tile: reads stay in bounds
  const u64 j0 = d0 - i0;
  const u64 la = i1 - i0, len = d1 - d0;
  bool nan = false;
  for (u64 t = threadIdx.x; t < len; t += MERGE_THREADS) {
    const T v = t < la ? a[i0 + t] : b[j0 + (t - la)];
    s_in[t] = v;
    nan |= t >= la && v != v;
  }
  if (status && nan) atomicOr(status, DELTA_ST_NAN);
  __syncthreads();
  const u64 t0 = (u64)threadIdx.x * MERGE_ITEMS;
  if (t0 < len) merge_tile(s_in, la, s_in + la, len - la, t0, t0 + MERGE_ITEMS < len ? t0 + MERGE_ITEMS : len, s_out + t0);
  __syncthreads();
  for (u64 t = threadIdx.x; t < len; t += MERGE_THREADS) out[d0 + t] = s_out[t];
}

template <class T>
__global__ void __launch_bounds__(LOOKUP_THREADS)
k_delta_count(const T* __restrict__ delta, u64 m, const T* __restrict__ qs, u64 nq, u64* __restrict__ out_first,
              u64* __restrict__ out_last, int mode) {
  const bool lower = mode != DELTA_UPPER, upper = mode != DELTA_LOWER;
  for (u64 i = (u64)blockIdx.x * LOOKUP_THREADS + threadIdx.x; i < nq; i += (u64)gridDim.x * LOOKUP_THREADS) {
    const T q = __ldcs(qs + i);
    // lane 0 counts d < q, lane 1 d <= q; in DELTA_BOTH both walk the same halvings
    u64 b0 = 0, b1 = 0, len = m;
    while (len > 1) {
      const u64 h = len >> 1;
      if (lower) b0 = before<false>(__ldg(delta + b0 + h), q) ? b0 + h : b0;
      if (upper) b1 = before<true>(__ldg(delta + b1 + h), q) ? b1 + h : b1;
      len -= h;
    }
    if (lower) {
      const u64 r = b0 + (before<false>(__ldg(delta + b0), q) ? 1 : 0);
      __stcs(out_first + i, __ldcs(out_first + i) + r);
    }
    if (upper) {
      const u64 r = b1 + (before<true>(__ldg(delta + b1), q) ? 1 : 0);
      __stcs(out_last + i, __ldcs(out_last + i) + r);
    }
  }
}

}  // namespace

template <class T>
void delta_merge(const Launch& L, const T* a, u64 na, const T* b, u64 nb, T* out, unsigned* d_status) {
  const u64 tiles = (na + nb + MERGE_TILE - 1) / MERGE_TILE;
  if (tiles == 0) return;
  k_delta_merge<T><<<(unsigned)tiles, MERGE_THREADS, 0, L.stream>>>(a, na, b, nb, out, d_status);
  count_launch();
}

template <class T>
void delta_count(const Launch& L, DeltaCountMode mode, const T* delta, u64 m, const T* qs, u64 nq, u64* out_first,
                 u64* out_last) {
  if (m == 0 || nq == 0) return;
  k_delta_count<T><<<capped_grid(L, nq, LOOKUP_THREADS, LOOKUP_MAX_BLOCKS_PER_SM), LOOKUP_THREADS, 0, L.stream>>>(
      delta, m, qs, nq, out_first, out_last, (int)mode);
  count_launch();
}

#define RMI_DELTA_INST(T)                                                                             \
  template void delta_merge<T>(const Launch&, const T*, u64, const T*, u64, T*, unsigned*);           \
  template void delta_count<T>(const Launch&, DeltaCountMode, const T*, u64, const T*, u64, u64*, u64*);
RMI_DELTA_INST(u64)
RMI_DELTA_INST(u32)
RMI_DELTA_INST(double)
#undef RMI_DELTA_INST

}  // namespace rmi
