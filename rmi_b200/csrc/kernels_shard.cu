// kernels_shard.cu — the pieces of a range-partitioned (multi-GPU) build that differ from the
// single-GPU path.  Every rank holds a contiguous slab of the globally sorted key array
// (Shard<T>, kernels.h); the top model and the leaf boundaries S are made global by small
// collectives issued by the host between these phases (rmi_b200/sharded.py):
//
//   phase TOP_LOCAL   k_shard_slr_partial / k_shard_slr_reduce   -> 5 partial sums per rank
//        [all-reduce SUM of 5 doubles]                             (linear, robust_linear, loglinear)
//                     bradix: the scalars, then shard_bradix_count (kernels_top.cu): per-bin key counts of all
//                     four candidates in one pass
//        [all-reduce SUM of 4 x N u32]                             (bradix)
//                     k_shard_cubic_local: this rank's candidates for the two interior points
//        [all-reduce MIN of 4 order-encoded u64]                   (cubic)
//                     k_shard_normal_partial<pass 0>: sum(x - pivot)
//        [all-reduce SUM]                                          (normal, lognormal)
//   phase TOP_MID     (two-round tops only) cubic: closed form from the gathered points, then
//                     the local part of the two L1 sums; normal: mean, then sum((x - mean)^2)
//        [all-reduce SUM]
//   phase TOP_FINISH  k_shard_slr_solve, k_shard_top_from_ends (linear_spline, radix: O(1)
//                     functions of the global first / last key), k_shard_cubic_pick,
//                     k_shard_normal_solve, shard_bradix_decide (kernels_top.cu)
//   phase BOUNDS      k_shard_bounds_search (monotone-by-construction tops) or the streaming
//                     k_shard_bounds_stream (cubic, loglinear, normal: also verifies monotonicity)
//                     -> S_local (global indices, n_global where none)
//        [all-reduce MIN of (N+1) u64]
//   phase SPLIT       k_split_from_S
//        [halo: each rank receives the keys of its last leaf that live on the next rank(s)]
//   phase LEAF        k_leaf (kernels_leaf.cu) on the leaves whose first key is local
//        [all-reduce SUM of the zero-initialised parameter / error / count arrays]
//   phase STATS       leaf_statistics
//
// The fits themselves are the same code as on one GPU; only offsets become global
// (base + local) and the item before local index 0 comes from the previous rank.
#include "device_util.cuh"
#include "kernels.h"
#include "spline.cuh"

namespace rmi {

namespace {

constexpr int SH_THREADS = 256;
constexpr int SH_MAX_BLOCKS = 132 * 8;   // 8 blocks per SM of an H100 (sh_grid: min(num_sms * 8, this))

__device__ __forceinline__ void set_status(BuildAux* aux, unsigned bit) { atomicOr(&aux->status, bit); }

// Partial sums of the top-level simple linear regression over the global item range
// [g0, g1) restricted to this rank's slab, about the common pivot (px, py).  MODE 0: y;  MODE 1: ln(y), items whose
// ln(y) is not finite dropped (loglinear, as k_slr_partial<T, 1>; the pivot is then (px, 0)).
template <class T, int MODE>
__global__ void __launch_bounds__(SH_THREADS)
k_shard_slr_partial(const T* __restrict__ keys, const Shard<T> sh, u64 g0, u64 g1, double sf, int use_sf, double px,
                    double py, double* __restrict__ partials) {
  __shared__ double sm[32];
  // local range
  u64 lo = g0 > sh.base ? g0 - sh.base : 0;
  u64 hi = g1 > sh.base ? g1 - sh.base : 0;
  if (hi > sh.n_local) hi = sh.n_local;
  double sx = 0, sy = 0, sxx = 0, sxy = 0;
  unsigned icnt = 0;
  const bool aligned = is_aligned16(keys);
  u64 stride = (u64)gridDim.x * blockDim.x * 4;
  for (u64 b = (lo & ~3ull) + ((u64)blockIdx.x * blockDim.x + threadIdx.x) * 4; b < hi; b += stride) {
    T k[4];
    int c = load_keys4(keys, b, sh.n_local, aligned, k);
    if (MODE == 0 && c == 4 && b >= lo && b + 4 <= hi) {
      const T before = b > 0 ? keys[b - 1] : sh.prev_key;
      const bool dup = ((b > 0 || sh.has_prev) && before == k[0]) || k[1] == k[0] || k[2] == k[1] || k[3] == k[2];
      if (!dup) {
        // every key starts its own run: offset = global index, floor(offset * sf) by the 2^52 trick
        const double bd = __ull2double_rn(sh.base + b);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          double x = Key<T>::as_float(k[e]);
          double y = bd + (double)e;
          if (use_sf) y = __dadd_rn(__dadd_rd(__dmul_rn(y, sf), 4503599627370496.0), -4503599627370496.0);
          double dx = x - px, dy = y - py;
          sx += dx; sy += dy; sxx = fma(dx, dx, sxx); sxy = fma(dx, dy, sxy);
        }
        icnt += 4;
        continue;
      }
    }
    u64 F = global_run_start(keys, b, sh.base, sh.has_prev, sh.prev_key, sh.prev_F);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (e >= c) break;
      u64 i = b + e;
      if (e > 0 && k[e] != k[e - 1]) F = sh.base + i;
      if (i < lo || i >= hi) continue;
      double x = Key<T>::as_float(k[e]);
      double y = __ull2double_rn(scale_offset(F, sf, use_sf));
      if (MODE == 1) { y = log(y); if (!isfinite(y)) continue; }
      double dx = x - px, dy = y - py;
      sx += dx; sy += dy; sxx = fma(dx, dx, sxx); sxy = fma(dx, dy, sxy);
      icnt += 1;
    }
  }
  double r0 = block_sum(sx, sm), r1 = block_sum(sy, sm), r2 = block_sum(sxx, sm), r3 = block_sum(sxy, sm),
         r4 = block_sum((double)icnt, sm);
  if (threadIdx.x == 0) {
    double* p = partials + (size_t)blockIdx.x * 5;
    p[0] = r0; p[1] = r1; p[2] = r2; p[3] = r3; p[4] = r4;
  }
}

// Block partials -> sums[0..5); the rank holding the global last key adds the drained
// iterator's repeated final item (models/mod.rs:180) when the fit drains the iterator (MODE 1: only if its ln(y) is
// finite, as k_slr_finish<T, 1>).
template <class T, int MODE>
__global__ void __launch_bounds__(SH_THREADS)
k_shard_slr_reduce(const T* __restrict__ keys, const Shard<T> sh, int repeat, double sf, int use_sf, double px, double py,
                   const double* __restrict__ partials, int nblocks, double* __restrict__ sums) {
  __shared__ double sm[32];
  double s[5] = {0, 0, 0, 0, 0};
  for (int b = threadIdx.x; b < nblocks; b += blockDim.x)
    for (int q = 0; q < 5; ++q) s[q] += partials[(size_t)b * 5 + q];
  double r[5];
  for (int q = 0; q < 5; ++q) r[q] = block_sum(s[q], sm);
  if (threadIdx.x != 0) return;
  if (repeat && sh.is_last && sh.n_local > 0) {
    u64 i = sh.n_local - 1;
    double x = Key<T>::as_float(keys[i]);
    u64 F = global_run_start(keys, i, sh.base, sh.has_prev, sh.prev_key, sh.prev_F);
    double y = __ull2double_rn(scale_offset(F, sf, use_sf));
    if (MODE == 1) y = log(y);
    if (MODE == 0 || isfinite(y)) {
      double dx = x - px, dy = y - py;
      r[0] += dx; r[1] += dy; r[2] += dx * dx; r[3] += dx * dy; r[4] += 1.0;
    }
  }
  for (int q = 0; q < 5; ++q) sums[q] = r[q];
}

// slr()'s closing formulas (linear.rs:36-58) on the globally reduced sums (loglinear: the same on the ln(y) sums,
// k_slr_finish<T, 1>).
__global__ void k_shard_slr_solve(const double* __restrict__ sums, double px, double py, TopModel* top, BuildAux* aux) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double sx = sums[0], sy = sums[1], sxx = sums[2], sxy = sums[3], cnt = sums[4];
  double alpha, beta;
  if (cnt == 0.0) { alpha = 0.0; beta = 0.0; }
  else {
    double mx = sx / cnt, my = sy / cnt;
    double mean_x = px + mx, mean_y = py + my;
    if (cnt == 1.0) { alpha = mean_y; beta = 0.0; }
    else {
      double m2 = sxx - sx * mx, c = sxy - sx * my;
      double cov = c / (cnt - 1.0), var = m2 / (cnt - 1.0);
      if (!(var >= 0.0)) {
        if (var > -1e-9 * fabs(sxx / cnt)) var = 0.0;
        else set_status(aux, ST_NEG_VARIANCE);
      }
      if (var == 0.0) { alpha = mean_y; beta = 0.0; }
      else { beta = cov / var; alpha = mean_y - beta * mean_x; }
    }
  }
  top->f[0] = alpha;
  top->f[1] = beta;
}

// Top models that are O(1) functions of the global first / last item:
// linear_spline (linear_spline.rs:13-35) and radix (radix.rs:18-40, utils.rs:13-36); bradix's prefix, bits and
// max_output (balanced_radix.rs:20-27).
template <class T>
__global__ void k_shard_top_from_ends(int kind, T first_key, T last_key, u64 last_F, u64 n, double sf, int use_sf,
                                      TopModel* top, BuildAux* aux) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (kind == M_LINEAR_SPLINE) {
    double alpha, beta;
    double y0 = __ull2double_rn(scale_offset(0, sf, use_sf));
    if (n == 0) { alpha = 0.0; beta = 0.0; }
    else if (n == 1 || first_key == last_key) { alpha = y0; beta = 0.0; }
    else {
      double y1 = __ull2double_rn(scale_offset(n - 1, sf, use_sf));
      double x0 = Key<T>::as_float(first_key), x1 = Key<T>::as_float(last_key);
      double slope = __ddiv_rn(__dadd_rn(y0, -y1), __dadd_rn(x0, -x1));
      alpha = __dadd_rn(y0, -__dmul_rn(slope, x0));
      beta = slope;
    }
    top->f[0] = alpha; top->f[1] = beta;
  } else if (kind == M_RADIX || kind == M_BRADIX) {   // bradix: the scalars its candidates start from (k_radix_scalars)
    int prefix = common_prefix_sorted(Key<T>::as_int(first_key), Key<T>::as_int(last_key));
    u64 largest = scale_offset(last_F, sf, use_sf);
    aux->max_scaled_y = largest;
    int bits = num_bits_of(largest);
    if (bits < 1) set_status(aux, ST_NUM_BITS);
    top->ip[0] = (u64)prefix; top->ip[1] = (u64)bits;
  } else if (kind == M_RADIX_TABLE) {   // radix.rs:90-100: the prefix; the table's width is fixed by the model name
    int prefix = common_prefix_sorted(Key<T>::as_int(first_key), Key<T>::as_int(last_key));
    aux->max_scaled_y = scale_offset(last_F, sf, use_sf);
    top->ip[0] = (u64)prefix;
  }
}

// ------------------------------------------------------------------------------------------
// Table tops over a range-partitioned array (radix8..28: radix.rs:90-134; histogram: histogram.rs:20-61).
// Both are "one writer per entry": a hint-table entry is written at the one key where the radix steps past
// it, a pivot is the key at one global index.  Every rank fills the entries its slab decides into a
// zero-initialised table (hint entries as value + 1), ONE all-reduce MAX merges the ranks' tables, and a
// decode pass restores the reference's values for the entries nobody wrote.
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void __launch_bounds__(SH_THREADS)
k_shard_table_fill(const T* __restrict__ keys, const Shard<T> sh, T first_key, T last_key, int bits, double sf, int use_sf,
                   u32* __restrict__ table, BuildAux* aux) {
  const unsigned prefix = (unsigned)common_prefix_sorted(Key<T>::as_int(first_key), Key<T>::as_int(last_key));
  const unsigned nb = (prefix + (unsigned)bits > 64u) ? 0u : 64u - (prefix + (unsigned)bits);
  const u64 len = 1ull << bits;
  auto radix_of = [&](T k) { return shr64(shr64(shl64(Key<T>::as_int(k), prefix), prefix), nb); };
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < sh.n_local; i += stride) {
    const u64 r = radix_of(keys[i]);
    const u64 rp = i > 0 ? radix_of(keys[i - 1]) : (sh.has_prev ? radix_of(sh.prev_key) : 0ull);
    if (r > rp) {
      if (r >= len) { atomicOr(&aux->status, (unsigned)ST_RADIX_TABLE_OOB); continue; }
      const u32 y = (u32)scale_offset(sh.base + i, sf, use_sf);   // a radix change implies a key change: F_i = i
      for (u64 q = rp + 1; q <= r; ++q) table[q] = y + 1u;
    }
  }
}
__global__ void __launch_bounds__(SH_THREADS)
k_shard_table_decode(u32* __restrict__ table, u64 len) {
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < len; q += stride) {
    const u32 v = table[q];
    table[q] = v ? v - 1u : (q == 0 ? 0u : (u32)len);   // hint[0] = 0; entries past the last key's radix = 2^bits
  }
}
template <class T>
__global__ void __launch_bounds__(SH_THREADS)
k_shard_hist_pivots(const T* __restrict__ keys, const Shard<T> sh, u64 num_bins, u64 items_per_bin, u64* __restrict__ pivots) {
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x; b < num_bins; b += stride) {
    const u64 g = b * items_per_bin;
    if (g >= sh.base && g < sh.base + sh.n_local) pivots[b] = Key<T>::as_int(keys[g - sh.base]);
  }
}


// ------------------------------------------------------------------------------------------
// cubic top (cubic_spline.rs:18-136) over a range-partitioned array.
// The closed form needs four points: the global first / last item (known everywhere from the
// gathered slab ends) and two interior ones — the first item whose scaled x is > 0 and the
// last raw item whose scaled x is < 1.  Each rank binary-searches its slab for its own
// candidates; ONE all-reduce MIN over four order-encoded u64 picks the winners:
//   slot 0: global index of the first candidate        slot 1: its key (order-preserving code)
//   slot 2: ~(global index + 1) of the last candidate  slot 3: ~(its key's code)
// Keys are sorted, so the smallest candidate index carries the smallest candidate key and
// index and key can be reduced independently.  The host reduces signed 64-bit integers, so
// every slot is stored with its top bit flipped (unsigned order == signed order).
// ------------------------------------------------------------------------------------------
constexpr u64 ORD_SIGN = 0x8000000000000000ull;
template <class T> __device__ __forceinline__ u64 key_code(T k) { return (u64)k; }
template <> __device__ __forceinline__ u64 key_code<double>(double k) {
  u64 b = (u64)__double_as_longlong(k);
  return (b & ORD_SIGN) ? ~b : (b | ORD_SIGN);
}
template <class T> __device__ __forceinline__ T key_decode(u64 c) { return (T)c; }
template <> __device__ __forceinline__ double key_decode<double>(u64 c) {
  u64 b = (c & ORD_SIGN) ? (c & ~ORD_SIGN) : ~c;
  return __longlong_as_double((long long)b);
}

template <class T>
__global__ void k_shard_cubic_local(const T* __restrict__ keys, const Shard<T> sh, T first_key, T last_key,
                                    u64* __restrict__ slots) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  u64 v0 = ~0ull, v1 = ~0ull, v2 = ~0ull, v3 = ~0ull;
  if (sh.n_global >= 2 && !(first_key == last_key) && sh.n_local > 0) {
    double xmin = Key<T>::as_float(first_key), xmax = Key<T>::as_float(last_key);
    u64 lo = 0, hi = sh.n_local;          // :46-54 first local item with scaled x > 0
    while (lo < hi) {
      u64 mid = lo + ((hi - lo) >> 1);
      if (scale3(Key<T>::as_float(keys[mid]), xmin, xmax) > 0.0) hi = mid; else lo = mid + 1;
    }
    if (lo < sh.n_local) { v0 = sh.base + lo; v1 = key_code<T>(keys[lo]); }
    u64 lo2 = 0, hi2 = sh.n_local;        // :56-65 first local index with !(scaled x < 1)
    while (lo2 < hi2) {
      u64 mid = lo2 + ((hi2 - lo2) >> 1);
      if (scale3(Key<T>::as_float(keys[mid]), xmin, xmax) < 1.0) lo2 = mid + 1; else hi2 = mid;
    }
    if (lo2 > 0) { v2 = ~(sh.base + lo2); v3 = ~key_code<T>(keys[lo2 - 1]); }
  }
  slots[0] = v0 ^ ORD_SIGN; slots[1] = v1 ^ ORD_SIGN; slots[2] = v2 ^ ORD_SIGN; slots[3] = v3 ^ ORD_SIGN;
}

// cand[0..4) = cubic (a,b,c,d), cand[4..6) = linear spline (alpha, beta)  — as k_spline_prepare
template <class T>
__global__ void k_shard_cubic_closed_form(const Shard<T> sh, T first_key, T last_key, double sf, int use_sf,
                                          const u64* __restrict__ slots, double* __restrict__ cand, BuildAux* aux) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const u64 n = sh.n_global;
  double y_first = __ull2double_rn(scale_offset(0, sf, use_sf));
  double la, lb, a, b, c, d;
  if (n == 1 || first_key == last_key) { la = y_first; lb = 0.0; a = b = c = 0.0; d = y_first; }   // :23-36
  else {
    double xmin = Key<T>::as_float(first_key), xmax = Key<T>::as_float(last_key);
    double ymin = y_first, ymax = __ull2double_rn(scale_offset(n - 1, sf, use_sf));
    double slope = __ddiv_rn(__dadd_rn(ymin, -ymax), __dadd_rn(xmin, -xmax));     // linear_spline.rs:28-33
    la = __dadd_rn(ymin, -__dmul_rn(slope, xmin));
    lb = slope;
    u64 v0 = slots[0] ^ ORD_SIGN, v1 = slots[1] ^ ORD_SIGN, v2 = slots[2] ^ ORD_SIGN, v3 = slots[3] ^ ORD_SIGN;
    if (v0 == ~0ull || v2 == ~0ull) {
      atomicOr(&aux->status, ST_CUBIC_UNWRAP);
      a = b = c = d = 0.0;
    } else {
      // the first item with scaled x > 0 starts a run of equal keys, so its duplicate-fixed
      // offset is its own index; the last item with scaled x < 1 is taken raw (:56-65)
      u64 lo = v0, ip = ~v2 - 1ull;
      cubic_from_points(xmin, ymin, xmax, ymax, Key<T>::as_float(key_decode<T>(v1)),
                        __ull2double_rn(scale_offset(lo, sf, use_sf)), Key<T>::as_float(key_decode<T>(~v3)),
                        __ull2double_rn(scale_offset(ip, sf, use_sf)), a, b, c, d);
    }
  }
  cand[0] = a; cand[1] = b; cand[2] = c; cand[3] = d; cand[4] = la; cand[5] = lb;
}

// cubic_spline.rs:117-126 over the local slab: partials[2b] = sum |cubic(x) - y|,
// partials[2b+1] = sum |linear_spline(x) - y|, y = scaled duplicate-fixed GLOBAL offset.
template <class T>
__global__ void __launch_bounds__(SH_THREADS)
k_shard_cubic_l1_partial(const T* __restrict__ keys, const Shard<T> sh, double sf, int use_sf,
                         const double* __restrict__ cand, double* __restrict__ partials) {
  __shared__ double sm[32];
  double cf[4] = {cand[0], cand[1], cand[2], cand[3]};
  double lf[2] = {cand[4], cand[5]};
  double ec = 0, el = 0;
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < sh.n_local; i += stride) {
    double x = Key<T>::as_float(keys[i]);
    u64 F = global_run_start(keys, i, sh.base, sh.has_prev, sh.prev_key, sh.prev_F);
    double y = __ull2double_rn(scale_offset(F, sf, use_sf));
    ec += fabs(predict_float<M_CUBIC>(cf, x) - y);
    el += fabs(predict_float<M_LINEAR>(lf, x) - y);
  }
  double r0 = block_sum(ec, sm), r1 = block_sum(el, sm);
  if (threadIdx.x == 0) { partials[2 * blockIdx.x] = r0; partials[2 * blockIdx.x + 1] = r1; }
}
template <class T>
__global__ void __launch_bounds__(SH_THREADS)
k_shard_cubic_l1_reduce(const T* __restrict__ keys, const Shard<T> sh, double sf, int use_sf,
                        const double* __restrict__ cand, const double* __restrict__ partials, int nblocks,
                        double* __restrict__ sums) {
  __shared__ double sm[32];
  double ec = 0, el = 0;
  for (int b = threadIdx.x; b < nblocks; b += blockDim.x) { ec += partials[2 * b]; el += partials[2 * b + 1]; }
  double r0 = block_sum(ec, sm), r1 = block_sum(el, sm);
  if (threadIdx.x != 0) return;
  if (sh.is_last && sh.n_local > 0) {   // the drained iterator's repeated final item
    u64 i = sh.n_local - 1;
    double x = Key<T>::as_float(keys[i]);
    u64 F = global_run_start(keys, i, sh.base, sh.has_prev, sh.prev_key, sh.prev_F);
    double y = __ull2double_rn(scale_offset(F, sf, use_sf));
    double lf[2] = {cand[4], cand[5]};
    r0 += fabs(predict_float<M_CUBIC>(cand, x) - y);
    r1 += fabs(predict_float<M_LINEAR>(lf, x) - y);
  }
  sums[0] = r0; sums[1] = r1;
  for (int q = 2; q < 8; ++q) sums[q] = 0.0;
}
// cubic_spline.rs:128-135: keep the linear spline (0, 0, beta, alpha) if it is strictly better.
__global__ void k_shard_cubic_pick(const double* __restrict__ sums, const double* __restrict__ cand, TopModel* top) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (sums[1] < sums[0]) { top->f[0] = 0.0; top->f[1] = 0.0; top->f[2] = cand[5]; top->f[3] = cand[4]; }
  else { top->f[0] = cand[0]; top->f[1] = cand[1]; top->f[2] = cand[2]; top->f[3] = cand[3]; }
}

// ------------------------------------------------------------------------------------------
// normal / lognormal top (normal.rs:28-76): mean over the drained stream (n+1 items, divisor
// n), then sum((x - mean)^2) — two rounds of one all-reduce SUM each.
// PASS 0: sums[0] = local sum(x - px), px a pivot every rank derives from the global end keys.
// PASS 1: state[0] = mean (from the reduced sums[0]); sums[0] = local sum((x - mean)^2).
// ------------------------------------------------------------------------------------------
template <class T, int LOGN> __device__ __forceinline__ double normal_pivot(T first_key, T last_key) {
  return 0.5 * normal_x<T, LOGN>(first_key) + 0.5 * normal_x<T, LOGN>(last_key);
}
template <class T, int LOGN, int PASS>
__global__ void __launch_bounds__(SH_THREADS)
k_shard_normal_partial(const T* __restrict__ keys, const Shard<T> sh, T first_key, T last_key,
                       const double* __restrict__ sums, double* __restrict__ partials) {
  __shared__ double sm[32];
  const double pivot = normal_pivot<T, LOGN>(first_key, last_key);
  double px = pivot;
  if (PASS == 1) px = (sums[0] + __ull2double_rn(sh.n_global + 1) * pivot) / __ull2double_rn(sh.n_global);   // mean
  double s = 0;
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < sh.n_local; i += stride) {
    double d = normal_x<T, LOGN>(keys[i]) - px;
    s += PASS == 0 ? d : d * d;
  }
  double r = block_sum(s, sm);
  if (threadIdx.x == 0) partials[blockIdx.x] = r;
}
template <class T, int LOGN, int PASS>
__global__ void __launch_bounds__(SH_THREADS)
k_shard_normal_reduce(const T* __restrict__ keys, const Shard<T> sh, T first_key, T last_key,
                      const double* __restrict__ partials, int nblocks, double* __restrict__ sums,
                      double* __restrict__ state) {
  __shared__ double sm[32];
  double s = 0;
  for (int b = threadIdx.x; b < nblocks; b += blockDim.x) s += partials[b];
  double r = block_sum(s, sm);
  if (threadIdx.x != 0) return;
  const double pivot = normal_pivot<T, LOGN>(first_key, last_key);
  double px = pivot;
  if (PASS == 1) {
    px = (sums[0] + __ull2double_rn(sh.n_global + 1) * pivot) / __ull2double_rn(sh.n_global);
    state[0] = px;
  }
  if (sh.is_last && sh.n_local > 0) {   // repeated final item
    double d = normal_x<T, LOGN>(keys[sh.n_local - 1]) - px;
    r += PASS == 0 ? d : d * d;
  }
  sums[0] = r;
  for (int q = 1; q < 8; ++q) sums[q] = 0.0;
}
__global__ void k_shard_normal_solve(const double* __restrict__ sums, const double* __restrict__ state, u64 n,
                                     u64 last_F, double sf, int use_sf, TopModel* top) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double stdev = sqrt(sums[0] / __ull2double_rn(n));
  double scale = __ull2double_rn(scale_offset(last_F, sf, use_sf));   // max y = y of the last run (n > 0)
  top->f[0] = state[0]; top->f[1] = stdev; top->f[2] = scale;
}

// ------------------------------------------------------------------------------------------
// Streaming leaf boundaries for tops whose prediction is not monotone by construction
// (cubic, normal, lognormal): as k_bounds (kernels_leaf.cu) on the local slab, writing global
// indices; the key before local index 0 is the previous rank's last key, so the
// non-decreasing-target assertion (two_layer.rs:50) is checked across cuts too.  S must be
// pre-filled with n_global; the all-reduce MIN then yields the global S.
// ------------------------------------------------------------------------------------------
__global__ void k_shard_fill(u64* __restrict__ p, u64 len, u64 v) {
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += stride) p[i] = v;
}
template <class T, int TOP>
__global__ void __launch_bounds__(SH_THREADS)
k_shard_bounds_stream(const T* __restrict__ keys, const Shard<T> sh, const TopModel* __restrict__ top_ptr, u64 N,
                      u64* __restrict__ S, BuildAux* aux) {
  TopModel m = *top_ptr;
  const bool aligned = is_aligned16(keys);
  constexpr bool nbc = !(TOP == M_CUBIC || TOP == M_RADIX || TOP == M_RADIX_TABLE || TOP == M_BRADIX || TOP == M_HISTOGRAM);
  u64 stride = (u64)gridDim.x * blockDim.x * 4;
  unsigned bad = 0;
  for (u64 b = ((u64)blockIdx.x * blockDim.x + threadIdx.x) * 4; b < sh.n_local; b += stride) {
    T k[4];
    int cnt = load_keys4(keys, b, sh.n_local, aligned, k);
    T kp = b > 0 ? keys[b - 1] : (sh.has_prev ? sh.prev_key : k[0]);
    u64 pp = top_predict<TOP>(m, kp);
    u64 tp = pp < N - 1 ? pp : N - 1;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (e >= cnt) break;
      u64 i = b + e;
      u64 p = top_predict<TOP>(m, k[e]);
      if (!nbc && p >= N) bad |= ST_TOP_OUT_OF_BOUNDS;
      u64 t = p < N - 1 ? p : N - 1;
      if (i == 0 && !sh.has_prev) {
        for (u64 q = 0; q <= t; ++q) S[q] = 0;
      } else {
        if (k[e] < kp) bad |= ST_NOT_SORTED;
        if (t < tp) bad |= ST_NON_MONOTONE;
        for (u64 q = tp + 1; q <= t; ++q) S[q] = sh.base + i;
      }
      kp = k[e]; tp = t;
    }
  }
  if (bad) set_status(aux, bad);
}

// S_local[j] = global index of the first LOCAL key whose prediction reaches j, n_global if
// none (the all-reduce MIN over ranks then yields the global S).
template <class T, int TOP>
__global__ void __launch_bounds__(SH_THREADS)
k_shard_bounds_search(const T* __restrict__ keys, const Shard<T> sh, const TopModel* __restrict__ top_ptr, u64 N,
                      u64* __restrict__ S) {
  TopModel m = *top_ptr;
  u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (j > N) return;
  u64 v;
  if (j == N) v = sh.n_global;
  else if (j == 0) v = 0;
  else if (sh.n_local == 0) v = sh.n_global;
  else {
    // Predictions are non-decreasing over the sorted keys (these tops are monotone by construction), so only the
    // leaves between the slab's first and last prediction can begin inside it: the others get what the search would
    // return without running it — on W ranks each rank searches about N / W boundaries instead of N.
    const u64 p_first = top_predict<TOP>(m, keys[0]), p_last = top_predict<TOP>(m, keys[sh.n_local - 1]);
    if (j <= p_first) v = sh.base;
    else if (j > p_last) v = sh.n_global;
    else {
      u64 lo = 1, hi = sh.n_local - 1;   // keys[0] predicts < j, keys[n_local - 1] predicts >= j
      while (lo < hi) {
        u64 mid = lo + ((hi - lo) >> 1);
        if (top_predict<TOP>(m, keys[mid]) >= j) hi = mid; else lo = mid + 1;
      }
      v = sh.base + lo;
    }
  }
  S[j] = v;
}

// two_layer.rs:131-159 from the global S alone: split = S[N/2]; the split key's leaf is the
// last j with S[j] == split (leaves N/2 .. that one - 1 are empty).
template <class T, int TOP>
__global__ void k_split_from_S(const T* __restrict__ keys, const Shard<T> sh, const TopModel* __restrict__ top_ptr,
                               u64 N, const u64* __restrict__ S, BuildAux* aux) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  TopModel m = *top_ptr;
  u64 n = sh.n_global;
  if (TOP == M_LINEAR && !(m.f[1] >= 0.0)) set_status(aux, ST_NON_MONOTONE);
  if (sh.is_last && sh.n_local > 0) {
    bool nbc = !(TOP == M_CUBIC || TOP == M_RADIX || TOP == M_RADIX_TABLE || TOP == M_BRADIX || TOP == M_HISTOGRAM);
    if (!nbc && top_predict<TOP>(m, keys[sh.n_local - 1]) >= N) set_status(aux, ST_TOP_OUT_OF_BOUNDS);
  }
  u64 split = S[N / 2];
  aux->split_idx = split;
  if (split >= n) { aux->has_split = 0; aux->split_target = 0; return; }
  aux->has_split = 1;
  if (split == 0) set_status(aux, ST_SPLIT_AT_ZERO);
  if (split + 1 >= n) set_status(aux, ST_SPLIT_AT_END);
  u64 lo = N / 2, hi = N;   // last j in [N/2, N) with S[j] == split  (S is non-decreasing)
  while (lo + 1 < hi) {
    u64 mid = lo + ((hi - lo) >> 1);
    if (S[mid] <= split) lo = mid; else hi = mid;
  }
  aux->split_target = lo;
}

__global__ void k_copy_status(const BuildAux* __restrict__ aux, unsigned* __restrict__ out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) out[0] = aux->status;
}

__global__ void k_copy_flags(const BuildAux* __restrict__ aux, unsigned* __restrict__ out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) { out[0] = aux->status; out[1] = aux->could_not_replace ? 1u : 0u; }
}

int sh_grid(u64 n, int num_sms) {
  u64 blocks = (n + SH_THREADS - 1) / SH_THREADS;
  u64 cap = (u64)num_sms * 8;
  if (cap > (u64)SH_MAX_BLOCKS) cap = SH_MAX_BLOCKS;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

}  // namespace

// block partials (5 doubles per block) followed by 8 doubles of per-build state:
// cand[0..6) (cubic / linear-spline candidates) and state[0] (normal: the mean)
// (bradix's TOP_FINISH takes the block partials' room for its chi2 partials and best candidate)
size_t shard_scratch_bytes() {
  return std::max(((size_t)SH_MAX_BLOCKS * 5 + 8) * sizeof(double), shard_bradix_scratch_bytes());
}
static inline double* shard_cand(void* scratch) { return (double*)scratch + (size_t)SH_MAX_BLOCKS * 5; }

template <class T>
unsigned shard_top_local(const Launch& L, const T* keys, const Shard<T>& sh, int kind, u64 N, double px, double py,
                         T first_key, T last_key, u64 last_F, void* scratch, double* d_sums, TopModel* d_top,
                         BuildAux* d_aux, u32* d_bradix_counts) {
  double sf = (double)N / (double)sh.n_global;
  int use_sf = std::fabs(sf - 1.0) > DBL_EPSILON ? 1 : 0;
  double* partials = (double*)scratch;
  if (kind == M_LINEAR || kind == M_ROBUST_LINEAR) {
    u64 g0 = 0, g1 = sh.n_global;
    int repeat = 1;
    if (kind == M_ROBUST_LINEAR) {
      u64 n = sh.n_global;
      if (n == 0) { g0 = g1 = 0; repeat = 0; }
      else {
        u64 bnd = (u64)((double)n * 0.0001);
        if (bnd < 1) bnd = 1;
        if (!(bnd * 2 + 1 < n)) return ST_ROBUST_TOO_SMALL;
        g0 = bnd; g1 = n - bnd; repeat = 0;
      }
    }
    int g = sh_grid((sh.n_local + 3) / 4 + 1, L.num_sms);
    k_shard_slr_partial<T, 0><<<g, SH_THREADS, 0, L.stream>>>(keys, sh, g0, g1, sf, use_sf, px, py, partials);
    count_launch();
    k_shard_slr_reduce<T, 0><<<1, SH_THREADS, 0, L.stream>>>(keys, sh, repeat, sf, use_sf, px, py, partials, g, d_sums);
    count_launch();
  } else if (kind == M_LOGLINEAR) {   // linear.rs:61-72: the whole stream, ln(y) about the pivot (px, 0)
    int g = sh_grid((sh.n_local + 3) / 4 + 1, L.num_sms);
    k_shard_slr_partial<T, 1><<<g, SH_THREADS, 0, L.stream>>>(keys, sh, 0, sh.n_global, sf, use_sf, px, 0.0, partials);
    count_launch();
    k_shard_slr_reduce<T, 1><<<1, SH_THREADS, 0, L.stream>>>(keys, sh, 1, sf, use_sf, px, 0.0, partials, g, d_sums);
    count_launch();
  } else if (kind == M_BRADIX) {      // the scalars from the global ends, then this rank's per-bin counts
    cudaMemsetAsync(d_sums, 0, 8 * sizeof(double), L.stream);
    k_shard_top_from_ends<T><<<1, 32, 0, L.stream>>>(kind, first_key, last_key, last_F, sh.n_global, sf, use_sf, d_top, d_aux);
    count_launch();
    shard_bradix_count<T>(L, keys, sh, N, d_top, d_aux, d_bradix_counts);
  } else if (kind == M_CUBIC) {
    cudaMemsetAsync(d_sums, 0, 8 * sizeof(double), L.stream);
    k_shard_cubic_local<T><<<1, 32, 0, L.stream>>>(keys, sh, first_key, last_key, (u64*)d_sums + 8);
    count_launch();
  } else if (kind == M_NORMAL || kind == M_LOGNORMAL) {
    int g = sh_grid(sh.n_local, L.num_sms);
    if (kind == M_NORMAL) {
      k_shard_normal_partial<T, 0, 0><<<g, SH_THREADS, 0, L.stream>>>(keys, sh, first_key, last_key, d_sums, partials);
      k_shard_normal_reduce<T, 0, 0><<<1, SH_THREADS, 0, L.stream>>>(keys, sh, first_key, last_key, partials, g, d_sums, shard_cand(scratch) + 6);
    } else {
      k_shard_normal_partial<T, 1, 0><<<g, SH_THREADS, 0, L.stream>>>(keys, sh, first_key, last_key, d_sums, partials);
      k_shard_normal_reduce<T, 1, 0><<<1, SH_THREADS, 0, L.stream>>>(keys, sh, first_key, last_key, partials, g, d_sums, shard_cand(scratch) + 6);
    }
    count_launch(); count_launch();
  } else {
    cudaMemsetAsync(d_sums, 0, 8 * sizeof(double), L.stream);
  }
  return 0;
}

// Second round of the two-round tops (between the two collectives).
template <class T>
void shard_top_mid(const Launch& L, const T* keys, const Shard<T>& sh, int kind, u64 N, T first_key, T last_key,
                   void* scratch, double* d_sums, BuildAux* d_aux) {
  double sf = (double)N / (double)sh.n_global;
  int use_sf = std::fabs(sf - 1.0) > DBL_EPSILON ? 1 : 0;
  double* partials = (double*)scratch;
  double* cand = shard_cand(scratch);
  if (kind == M_CUBIC) {
    k_shard_cubic_closed_form<T><<<1, 32, 0, L.stream>>>(sh, first_key, last_key, sf, use_sf, (const u64*)d_sums + 8, cand, d_aux);
    int g = sh_grid(sh.n_local, L.num_sms);
    k_shard_cubic_l1_partial<T><<<g, SH_THREADS, 0, L.stream>>>(keys, sh, sf, use_sf, cand, partials);
    k_shard_cubic_l1_reduce<T><<<1, SH_THREADS, 0, L.stream>>>(keys, sh, sf, use_sf, cand, partials, g, d_sums);
    count_launch(); count_launch(); count_launch();
  } else if (kind == M_NORMAL || kind == M_LOGNORMAL) {
    int g = sh_grid(sh.n_local, L.num_sms);
    if (kind == M_NORMAL) {
      k_shard_normal_partial<T, 0, 1><<<g, SH_THREADS, 0, L.stream>>>(keys, sh, first_key, last_key, d_sums, partials);
      k_shard_normal_reduce<T, 0, 1><<<1, SH_THREADS, 0, L.stream>>>(keys, sh, first_key, last_key, partials, g, d_sums, cand + 6);
    } else {
      k_shard_normal_partial<T, 1, 1><<<g, SH_THREADS, 0, L.stream>>>(keys, sh, first_key, last_key, d_sums, partials);
      k_shard_normal_reduce<T, 1, 1><<<1, SH_THREADS, 0, L.stream>>>(keys, sh, first_key, last_key, partials, g, d_sums, cand + 6);
    }
    count_launch(); count_launch();
  }
}

template <class T>
void shard_top_finish(const Launch& L, const Shard<T>& sh, int kind, u64 N, double px, double py, const double* d_sums,
                      T first_key, T last_key, u64 last_F, const void* scratch, const u32* d_bradix_counts,
                      TopModel* d_top, BuildAux* d_aux) {
  double sf = (double)N / (double)sh.n_global;
  int use_sf = std::fabs(sf - 1.0) > DBL_EPSILON ? 1 : 0;
  if (kind == M_LINEAR || kind == M_ROBUST_LINEAR) {
    k_shard_slr_solve<<<1, 32, 0, L.stream>>>(d_sums, px, py, d_top, d_aux);
  } else if (kind == M_LOGLINEAR) {
    k_shard_slr_solve<<<1, 32, 0, L.stream>>>(d_sums, px, 0.0, d_top, d_aux);
  } else if (kind == M_BRADIX) {   // chi2 over the merged counts, the strict minimum in candidate order, commit
    shard_bradix_decide(L, sh.n_global, N, d_bradix_counts, const_cast<void*>(scratch), d_top, d_aux);
    return;
  } else if (kind == M_CUBIC) {
    k_shard_cubic_pick<<<1, 32, 0, L.stream>>>(d_sums, shard_cand(const_cast<void*>(scratch)), d_top);
  } else if (kind == M_NORMAL || kind == M_LOGNORMAL) {
    k_shard_normal_solve<<<1, 32, 0, L.stream>>>(d_sums, shard_cand(const_cast<void*>(scratch)) + 6, sh.n_global, last_F, sf,
                                                 use_sf, d_top);
  } else {
    k_shard_top_from_ends<T><<<1, 32, 0, L.stream>>>(kind, first_key, last_key, last_F, sh.n_global, sf, use_sf, d_top, d_aux);
  }
  count_launch();
}

template <class T, int TOP>
static void shard_bounds_stream(const Launch& L, const T* keys, const Shard<T>& sh, const TopModel* d_top, u64 N, u64* d_S,
                                BuildAux* d_aux) {
  k_shard_fill<<<sh_grid(N + 1, L.num_sms), SH_THREADS, 0, L.stream>>>(d_S, N + 1, sh.n_global);
  count_launch();
  k_shard_bounds_stream<T, TOP><<<sh_grid((sh.n_local + 3) / 4, L.num_sms), SH_THREADS, 0, L.stream>>>(keys, sh, d_top, N, d_S, d_aux);
  count_launch();
}

template <class T>
void shard_bounds(const Launch& L, const T* keys, const Shard<T>& sh, int kind, const TopModel* d_top, u64 N, u64* d_S,
                  BuildAux* d_aux) {
  unsigned blocks = (unsigned)((N + 1 + SH_THREADS - 1) / SH_THREADS);
  switch (kind) {
    case M_RADIX: k_shard_bounds_search<T, M_RADIX><<<blocks, SH_THREADS, 0, L.stream>>>(keys, sh, d_top, N, d_S); count_launch(); break;
    case M_RADIX_TABLE: k_shard_bounds_search<T, M_RADIX_TABLE><<<blocks, SH_THREADS, 0, L.stream>>>(keys, sh, d_top, N, d_S); count_launch(); break;
    case M_HISTOGRAM: k_shard_bounds_search<T, M_HISTOGRAM><<<blocks, SH_THREADS, 0, L.stream>>>(keys, sh, d_top, N, d_S); count_launch(); break;
    case M_BRADIX: k_shard_bounds_search<T, M_BRADIX><<<blocks, SH_THREADS, 0, L.stream>>>(keys, sh, d_top, N, d_S); count_launch(); break;
    case M_CUBIC: shard_bounds_stream<T, M_CUBIC>(L, keys, sh, d_top, N, d_S, d_aux); break;
    case M_LOGLINEAR: shard_bounds_stream<T, M_LOGLINEAR>(L, keys, sh, d_top, N, d_S, d_aux); break;
    case M_NORMAL: shard_bounds_stream<T, M_NORMAL>(L, keys, sh, d_top, N, d_S, d_aux); break;
    case M_LOGNORMAL: shard_bounds_stream<T, M_LOGNORMAL>(L, keys, sh, d_top, N, d_S, d_aux); break;
    default: k_shard_bounds_search<T, M_LINEAR><<<blocks, SH_THREADS, 0, L.stream>>>(keys, sh, d_top, N, d_S); count_launch(); break;
  }
}

// A GIVEN top model (rmi_shard_eval) is not known to be monotone on the keys, so every top group takes the streaming
// pass, which also checks the order of the targets across the cuts.
template <class T>
void shard_bounds_given(const Launch& L, const T* keys, const Shard<T>& sh, int kind, const TopModel* d_top, u64 N,
                        u64* d_S, BuildAux* d_aux) {
  switch (kind) {
    case M_LINEAR: case M_ROBUST_LINEAR: case M_LINEAR_SPLINE: shard_bounds_stream<T, M_LINEAR>(L, keys, sh, d_top, N, d_S, d_aux); break;
    case M_CUBIC: shard_bounds_stream<T, M_CUBIC>(L, keys, sh, d_top, N, d_S, d_aux); break;
    case M_LOGLINEAR: shard_bounds_stream<T, M_LOGLINEAR>(L, keys, sh, d_top, N, d_S, d_aux); break;
    case M_NORMAL: shard_bounds_stream<T, M_NORMAL>(L, keys, sh, d_top, N, d_S, d_aux); break;
    case M_LOGNORMAL: shard_bounds_stream<T, M_LOGNORMAL>(L, keys, sh, d_top, N, d_S, d_aux); break;
    case M_RADIX: shard_bounds_stream<T, M_RADIX>(L, keys, sh, d_top, N, d_S, d_aux); break;
    case M_RADIX_TABLE: shard_bounds_stream<T, M_RADIX_TABLE>(L, keys, sh, d_top, N, d_S, d_aux); break;
    case M_BRADIX: shard_bounds_stream<T, M_BRADIX>(L, keys, sh, d_top, N, d_S, d_aux); break;
    default: shard_bounds_stream<T, M_HISTOGRAM>(L, keys, sh, d_top, N, d_S, d_aux); break;
  }
}

template <class T>
void shard_split(const Launch& L, const T* keys, const Shard<T>& sh, int kind, const TopModel* d_top, u64 N,
                 const u64* d_S, BuildAux* d_aux) {
  switch (kind) {
    case M_RADIX: k_split_from_S<T, M_RADIX><<<1, 32, 0, L.stream>>>(keys, sh, d_top, N, d_S, d_aux); break;
    case M_RADIX_TABLE: k_split_from_S<T, M_RADIX_TABLE><<<1, 32, 0, L.stream>>>(keys, sh, d_top, N, d_S, d_aux); break;
    case M_HISTOGRAM: k_split_from_S<T, M_HISTOGRAM><<<1, 32, 0, L.stream>>>(keys, sh, d_top, N, d_S, d_aux); break;
    case M_BRADIX: k_split_from_S<T, M_BRADIX><<<1, 32, 0, L.stream>>>(keys, sh, d_top, N, d_S, d_aux); break;
    case M_LOGLINEAR: k_split_from_S<T, M_LOGLINEAR><<<1, 32, 0, L.stream>>>(keys, sh, d_top, N, d_S, d_aux); break;
    case M_CUBIC: k_split_from_S<T, M_CUBIC><<<1, 32, 0, L.stream>>>(keys, sh, d_top, N, d_S, d_aux); break;
    case M_NORMAL: k_split_from_S<T, M_NORMAL><<<1, 32, 0, L.stream>>>(keys, sh, d_top, N, d_S, d_aux); break;
    case M_LOGNORMAL: k_split_from_S<T, M_LOGNORMAL><<<1, 32, 0, L.stream>>>(keys, sh, d_top, N, d_S, d_aux); break;
    default: k_split_from_S<T, M_LINEAR><<<1, 32, 0, L.stream>>>(keys, sh, d_top, N, d_S, d_aux); break;
  }
  count_launch();
}

void shard_copy_status(const Launch& L, const BuildAux* d_aux, unsigned* d_out) {
  k_copy_status<<<1, 32, 0, L.stream>>>(d_aux, d_out);
  count_launch();
}

template <class T>
void shard_table_local(const Launch& L, const T* keys, const Shard<T>& sh, int kind, int table_bits, u64 N, T first_key,
                       T last_key, BuildAux* d_aux, u32* d_table32, u64* d_pivots, u64 num_bins, u64 items_per_bin) {
  double sf = (double)N / (double)sh.n_global;
  int use_sf = std::fabs(sf - 1.0) > DBL_EPSILON ? 1 : 0;
  if (kind == M_RADIX_TABLE) {
    cudaMemsetAsync(d_table32, 0, sizeof(u32) << table_bits, L.stream);
    if (sh.n_local) {
      k_shard_table_fill<T><<<sh_grid(sh.n_local, L.num_sms), SH_THREADS, 0, L.stream>>>(keys, sh, first_key, last_key, table_bits, sf,
                                                                                        use_sf, d_table32, d_aux);
      count_launch();
    }
  } else if (kind == M_HISTOGRAM) {
    cudaMemsetAsync(d_pivots, 0, sizeof(u64) * (num_bins + 1), L.stream);
    if (sh.n_local && num_bins) {
      k_shard_hist_pivots<T><<<sh_grid(num_bins, L.num_sms), SH_THREADS, 0, L.stream>>>(keys, sh, num_bins, items_per_bin, d_pivots);
      count_launch();
    }
  }
}
void shard_table_decode(const Launch& L, int table_bits, u32* d_table32) {
  k_shard_table_decode<<<sh_grid(1ull << table_bits, L.num_sms), SH_THREADS, 0, L.stream>>>(d_table32, 1ull << table_bits);
  count_launch();
}

void shard_copy_flags(const Launch& L, const BuildAux* d_aux, unsigned* d_out2) {
  k_copy_flags<<<1, 32, 0, L.stream>>>(d_aux, d_out2);
  count_launch();
}

#define INST(T)                                                                                                     \
  template unsigned shard_top_local<T>(const Launch&, const T*, const Shard<T>&, int, u64, double, double, T, T, u64, \
                                       void*, double*, TopModel*, BuildAux*, u32*);                                 \
  template void shard_top_mid<T>(const Launch&, const T*, const Shard<T>&, int, u64, T, T, void*, double*, BuildAux*); \
  template void shard_top_finish<T>(const Launch&, const Shard<T>&, int, u64, double, double, const double*, T, T, u64,   \
                                    const void*, const u32*, TopModel*, BuildAux*);                                 \
  template void shard_bounds<T>(const Launch&, const T*, const Shard<T>&, int, const TopModel*, u64, u64*, BuildAux*); \
  template void shard_bounds_given<T>(const Launch&, const T*, const Shard<T>&, int, const TopModel*, u64, u64*, BuildAux*); \
  template void shard_split<T>(const Launch&, const T*, const Shard<T>&, int, const TopModel*, u64, const u64*, BuildAux*); \
  template void shard_table_local<T>(const Launch&, const T*, const Shard<T>&, int, int, u64, T, T, BuildAux*, u32*, u64*, u64, u64);
INST(u64)
INST(u32)
INST(double)
#undef INST

}  // namespace rmi
