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
// k_delta_adjust: k_delta_count's mapping, for a delta with removed keys: per query, the branchless searches over the
//                 inserted keys (m may be 0) and over the removed keys run interleaved, so their dependent probes
//                 overlap, and the answer gains #{inserted before q} - #{removed before q} in place.
// k_delta_check_remove: one batch key per thread, grid-stride: given c(v), the copies of its value the logical key set
//                 holds (an equal range over the batch's own keys), flags a NaN or a copy the set does not hold
//                 (multiset_diff.cuh).
// k_delta_subtract: M minus the removed keys.  Block b owns M's keys [b * MERGE_TILE, (b + 1) * MERGE_TILE): two of
//                 its threads find the tile's window of removed keys, the block loads the tile into shared memory
//                 coalesced, every thread walks MERGE_ITEMS consecutive keys through the window (subtract_keys), the
//                 survivors are packed in shared memory at their offset from the tile's first destination, and the
//                 block stores them coalesced.
#include "kernels.h"
#include "lookup_search.cuh"
#include "merge_path.cuh"
#include "multiset_diff.cuh"

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

template <class T>
__global__ void __launch_bounds__(LOOKUP_THREADS)
k_delta_adjust(const T* __restrict__ ins, u64 m, const T* __restrict__ rem, u64 t, const T* __restrict__ qs, u64 nq,
               u64* __restrict__ out_first, u64* __restrict__ out_last, int mode) {
  const bool lower = mode != DELTA_UPPER, upper = mode != DELTA_LOWER;
  for (u64 i = (u64)blockIdx.x * LOOKUP_THREADS + threadIdx.x; i < nq; i += (u64)gridDim.x * LOOKUP_THREADS) {
    const T q = __ldcs(qs + i);
    // a0 / a1 search the inserted keys, r0 / r1 the removed ones; 0 counts k < q, 1 counts k <= q
    u64 a0 = 0, a1 = 0, la = m, r0 = 0, r1 = 0, lr = t;
    while (la > 1 || lr > 1) {   // both lengths are uniform over the grid: no divergence
      if (la > 1) {
        const u64 h = la >> 1;
        if (lower) a0 = before<false>(__ldg(ins + a0 + h), q) ? a0 + h : a0;
        if (upper) a1 = before<true>(__ldg(ins + a1 + h), q) ? a1 + h : a1;
        la -= h;
      }
      if (lr > 1) {
        const u64 h = lr >> 1;
        if (lower) r0 = before<false>(__ldg(rem + r0 + h), q) ? r0 + h : r0;
        if (upper) r1 = before<true>(__ldg(rem + r1 + h), q) ? r1 + h : r1;
        lr -= h;
      }
    }
    // removed ⊆ base ⊎ inserted as a multiset, so the difference never drops below 0 (DESIGN §19.5)
    if (lower) {
      u64 r = __ldcs(out_first + i) - (r0 + (before<false>(__ldg(rem + r0), q) ? 1 : 0));
      if (m) r += a0 + (before<false>(__ldg(ins + a0), q) ? 1 : 0);
      __stcs(out_first + i, r);
    }
    if (upper) {
      u64 r = __ldcs(out_last + i) - (r1 + (before<true>(__ldg(rem + r1), q) ? 1 : 0));
      if (m) r += a1 + (before<true>(__ldg(ins + a1), q) ? 1 : 0);
      __stcs(out_last + i, r);
    }
  }
}

template <class T>
__global__ void __launch_bounds__(LOOKUP_THREADS)
k_delta_check_remove(const T* __restrict__ batch, u64 n, const u64* __restrict__ first, const u64* __restrict__ last,
                     unsigned* status) {
  unsigned st = 0;
  for (u64 j = (u64)blockIdx.x * LOOKUP_THREADS + threadIdx.x; j < n; j += (u64)gridDim.x * LOOKUP_THREADS) {
    const T v = batch[j];
    if (v != v) st |= DELTA_ST_NAN;
    if (past_first_copies(batch, j, __ldcs(last + j) - __ldcs(first + j))) st |= DELTA_ST_MISSING;
  }
  if (st) atomicOr(status, st);
}

template <class T>
__global__ void __launch_bounds__(MERGE_THREADS)
k_delta_subtract(const T* __restrict__ M, u64 nm, const T* __restrict__ rem, u64 t, T* __restrict__ out, u64 nout) {
  __shared__ T s_in[MERGE_TILE];
  __shared__ T s_out[MERGE_TILE];
  __shared__ u64 s_win[2];
  __shared__ unsigned long long s_dest0;   // the tile's first destination
  __shared__ unsigned s_kept;
  const u64 p0 = (u64)blockIdx.x * MERGE_TILE;
  const u64 len = nm - p0 < MERGE_TILE ? nm - p0 : MERGE_TILE;
  if (threadIdx.x == 0) {
    s_win[0] = diff_search<false>(rem, 0, t, M[p0]);
    s_dest0 = ~0ull;
    s_kept = 0;
  }
  if (threadIdx.x == 1) s_win[1] = diff_search<true>(rem, 0, t, M[p0 + len - 1]);
  for (u64 k = threadIdx.x; k < len; k += MERGE_THREADS) s_in[k] = M[p0 + k];
  __syncthreads();
  const u64 lo = s_win[0], hi = s_win[1] < lo ? lo : s_win[1];   // on sorted keys lo <= hi already
  const u64 k0 = (u64)threadIdx.x * MERGE_ITEMS;
  const u64 kn = k0 < len ? (len - k0 < MERGE_ITEMS ? len - k0 : MERGE_ITEMS) : 0;
  // survivors' destinations are consecutive, so a thread needs only its first one and the mask of its survivors
  unsigned mask = 0;
  u64 first_dest = ~0ull;
  subtract_keys(s_in + k0, p0 + k0, kn, M, rem, lo, hi, [&](u64 k, u64 dest) {
    mask |= 1u << k;
    if (first_dest == ~0ull) first_dest = dest;
  });
  if (mask) {
    atomicMin(&s_dest0, (unsigned long long)first_dest);
    atomicAdd(&s_kept, (unsigned)__popc(mask));
  }
  __syncthreads();
  const u64 dest0 = s_dest0;
  u64 o = first_dest - dest0;
  for (int k = 0; k < MERGE_ITEMS; ++k)
    if (mask >> k & 1) {
      if (o < MERGE_TILE) s_out[o] = s_in[k0 + k];   // always, unless NaN keys sit out of order in a float64 base
      ++o;
    }
  __syncthreads();
  const u64 kept = s_kept;
  for (u64 k = threadIdx.x; k < kept; k += MERGE_THREADS)
    if (dest0 + k < nout) out[dest0 + k] = s_out[k];
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

template <class T>
void delta_adjust(const Launch& L, DeltaCountMode mode, const T* ins, u64 m, const T* rem, u64 t, const T* qs, u64 nq,
                  u64* out_first, u64* out_last) {
  if (t == 0 || nq == 0) return;
  k_delta_adjust<T><<<capped_grid(L, nq, LOOKUP_THREADS, LOOKUP_MAX_BLOCKS_PER_SM), LOOKUP_THREADS, 0, L.stream>>>(
      ins, m, rem, t, qs, nq, out_first, out_last, (int)mode);
  count_launch();
}

template <class T>
void delta_check_remove(const Launch& L, const T* batch, u64 n, const u64* first, const u64* last, unsigned* d_status) {
  if (n == 0) return;
  k_delta_check_remove<T><<<capped_grid(L, n, LOOKUP_THREADS, LOOKUP_MAX_BLOCKS_PER_SM), LOOKUP_THREADS, 0, L.stream>>>(
      batch, n, first, last, d_status);
  count_launch();
}

template <class T>
void delta_subtract(const Launch& L, const T* M, u64 nm, const T* rem, u64 t, T* out) {
  const u64 tiles = (nm + MERGE_TILE - 1) / MERGE_TILE;
  if (tiles == 0) return;
  k_delta_subtract<T><<<(unsigned)tiles, MERGE_THREADS, 0, L.stream>>>(M, nm, rem, t, out, nm - t);
  count_launch();
}

#define RMI_DELTA_INST(T)                                                                                        \
  template void delta_merge<T>(const Launch&, const T*, u64, const T*, u64, T*, unsigned*);                      \
  template void delta_count<T>(const Launch&, DeltaCountMode, const T*, u64, const T*, u64, u64*, u64*);         \
  template void delta_adjust<T>(const Launch&, DeltaCountMode, const T*, u64, const T*, u64, const T*, u64, u64*, \
                                u64*);                                                                           \
  template void delta_check_remove<T>(const Launch&, const T*, u64, const u64*, const u64*, unsigned*);          \
  template void delta_subtract<T>(const Launch&, const T*, u64, const T*, u64, T*);
RMI_DELTA_INST(u64)
RMI_DELTA_INST(u32)
RMI_DELTA_INST(double)
#undef RMI_DELTA_INST

}  // namespace rmi
