// device_util.cuh — small device helpers shared by the kernels: duplicate-run lookup,
// offset scaling, deterministic block reductions.
#pragma once
#include "rust_math.cuh"

namespace rmi {

// First index of the run of equal keys that contains index i (keys sorted ascending).
// This is the offset FixDupsIter reports for item i (reference models/mod.rs:154-185).
// One load when keys[i-1] != keys[i]; otherwise gallop + binary search, O(log run).
template <class T> __device__ __forceinline__ u64 run_start(const T* __restrict__ keys, u64 i) {
  if (i == 0) return 0;
  T v = keys[i];
  if (keys[i - 1] != v) return i;
  u64 hi = i - 1, step = 1, lo;
  for (;;) {
    if (hi < step) { lo = 0; break; }
    u64 c = hi - step;
    if (keys[c] == v) { hi = c; step <<= 1; } else { lo = c + 1; break; }
  }
  while (lo < hi) {
    u64 mid = lo + ((hi - lo) >> 1);
    if (keys[mid] == v) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// Duplicate-fixed GLOBAL offset of local item i on a rank's slab: the run may start on an
// earlier rank, whose last key and offset travel in (has_prev, prev_key, prev_F).
template <class T>
__device__ __forceinline__ u64 global_run_start(const T* __restrict__ keys, u64 i, u64 base, int has_prev, T prev_key,
                                                u64 prev_F) {
  u64 ls = run_start(keys, i);
  if (ls == 0 && has_prev && keys[0] == prev_key) return prev_F;
  return base + ls;
}

// Four consecutive keys starting at `base` (base % 4 == 0): two 128-bit loads for 8-byte
// keys, one for 4-byte keys, when the array is 16-byte aligned and all four are in range;
// scalar loads otherwise (entries past the end repeat the last key).  Returns how many are valid.
template <class T>
__device__ __forceinline__ int load_keys4(const T* __restrict__ keys, u64 base, u64 n, bool aligned16, T (&k)[4]) {
  int cnt = (n - base) < 4ull ? (int)(n - base) : 4;
  if (cnt == 4 && aligned16) {
    if (sizeof(T) == 8) {
      const ulonglong2* p = reinterpret_cast<const ulonglong2*>(keys + base);
      ulonglong2 a = __ldg(p), b = __ldg(p + 1);
      u64 raw[4] = {a.x, a.y, b.x, b.y};
#pragma unroll
      for (int e = 0; e < 4; ++e) k[e] = *reinterpret_cast<T*>(&raw[e]);
    } else {
      uint4 a = __ldg(reinterpret_cast<const uint4*>(keys + base));
      u32 raw[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) k[e] = *reinterpret_cast<T*>(&raw[e]);
    }
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) k[e] = keys[base + (u64)(e < cnt ? e : cnt - 1)];
  }
  return cnt;
}
__device__ __forceinline__ bool is_aligned16(const void* p) { return (reinterpret_cast<unsigned long long>(p) & 15ull) == 0; }

// createpolicy for an L2 eviction priority: 0 evict_normal, 1 evict_first, 2 evict_last.
__device__ __forceinline__ u64 l2_policy_of(int kind) {
  u64 p;
  if (kind == 1) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  else if (kind == 2) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  else asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// load_keys4 with an L2 eviction policy (l2_policy_of) on the 128-bit loads.
template <class T>
__device__ __forceinline__ int load_keys4_hint(const T* __restrict__ keys, u64 base, u64 n, bool aligned16, T (&k)[4],
                                               u64 policy) {
  int cnt = (n - base) < 4ull ? (int)(n - base) : 4;
  if (cnt == 4 && aligned16) {
    u64 raw8[4];
    u32 raw4[4];
    if (sizeof(T) == 8) {
      const T* p = keys + base;
      asm("ld.global.nc.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;" : "=l"(raw8[0]), "=l"(raw8[1]) : "l"(p), "l"(policy));
      asm("ld.global.nc.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;" : "=l"(raw8[2]), "=l"(raw8[3]) : "l"(p + 2), "l"(policy));
#pragma unroll
      for (int e = 0; e < 4; ++e) memcpy(&k[e], &raw8[e], sizeof(T));
    } else {
      asm("ld.global.nc.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
          : "=r"(raw4[0]), "=r"(raw4[1]), "=r"(raw4[2]), "=r"(raw4[3]) : "l"(keys + base), "l"(policy));
#pragma unroll
      for (int e = 0; e < 4; ++e) memcpy(&k[e], &raw4[e], sizeof(T));
    }
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) k[e] = keys[base + (u64)(e < cnt ? e : cnt - 1)];
  }
  return cnt;
}

// One key stored with an L2 eviction policy (l2_policy_of).
template <class T> __device__ __forceinline__ void store_key_hint(T* p, T v, u64 policy) {
  if (sizeof(T) == 8) {
    u64 b;
    memcpy(&b, &v, 8);
    asm volatile("st.global.L2::cache_hint.b64 [%0], %1, %2;" ::"l"(p), "l"(b), "l"(policy) : "memory");
  } else {
    u32 b;
    memcpy(&b, &v, 4);
    asm volatile("st.global.L2::cache_hint.b32 [%0], %1, %2;" ::"l"(p), "r"(b), "l"(policy) : "memory");
  }
}

// map_scale! (reference models/mod.rs:238-250): (offset as f64 * sf) as usize when the
// scale differs from 1.0 by more than f64::EPSILON.
__device__ __forceinline__ u64 scale_offset(u64 off, double sf, int use_sf) {
  return use_sf ? f64_to_u64_sat(__dmul_rn(__ull2double_rn(off), sf)) : off;
}

// The x a normal / lognormal model sees for a key (normal.rs:30-33, :56-63: ln(x), non-finite -> 0).
template <class T, int LOGN> __device__ __forceinline__ double normal_x(T k) {
  double x = Key<T>::as_float(k);
  if (LOGN) { double l = log(x); x = isfinite(l) ? l : 0.0; }
  return x;
}

// utils.rs:13-21
__device__ __forceinline__ int num_bits_of(u64 largest) {
  int nbits = 0;
  while (nbits + 1 < 64 && ((1ull << (nbits + 1)) - 1ull) <= largest) nbits += 1;
  return nbits;
}
// utils.rs:23-36 on a sorted key array: the leading bits on which ALL keys agree are the
// leading bits on which the smallest and the largest key agree.
__device__ __forceinline__ int common_prefix_sorted(u64 first_as_int, u64 last_as_int) {
  u64 diff = first_as_int ^ last_as_int;
  return diff == 0 ? 64 : __clzll((long long)diff);
}

// Deterministic block-wide sum (fixed shuffle tree, then warp 0 over the per-warp partials).
// Result valid in thread 0.  `sm` needs 32 doubles.
__device__ __forceinline__ double block_sum(double v, double* sm) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) sm[w] = v;
  __syncthreads();
  if (w == 0) {
    v = lane < nw ? sm[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
  }
  return v;
}
__device__ __forceinline__ u64 block_sum_u64(u64 v, u64* sm) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) sm[w] = v;
  __syncthreads();
  if (w == 0) {
    v = lane < nw ? sm[lane] : 0ull;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  }
  return v;
}

}  // namespace rmi
