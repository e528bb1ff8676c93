// kernels_shard_eval.cu — rmi_evaluate over a range-partitioned key array (DESIGN.md section 15).
//
// The single-GPU error pass (kernels_eval.cu) needs, per leaf, a maximum of per-key errors, a maximum run length and
// two widening terms.  Each is a MAX of contributions, and each contribution can be computed by the rank that holds
// the key it reads.  So every rank streams only its own slab, with global indices, into zero-initialised partials
// part_err | part_run (2N u64), the host all-reduces them with MAX, and every rank finishes the same leaves from the
// same arrays:
//
//   k_shard_eval_keys     k_eval_keys's tile walk over the local keys: leaf from the global S, offset from
//                         global_run_start, a run ends at the slab's last key when the next non-empty rank's first
//                         key differs (by value)                                      -> part_err, part_run
//   k_shard_eval_widen    per leaf, on the rank holding the key it reads: upper_error from key S[j+1] (max_value on
//                         the last non-empty rank when S[j+1] == n), lower_error from key S[j]-1 (zero_value on the
//                         first non-empty rank when S[j] == 0)                       -> part_err
//        [all-reduce MAX of part_err (| part_run when the key set holds equal keys)]
//   k_shard_eval_finish   errors = part_err + run_max, counts from S (k_eval_leaves without its key reads)
#include "device_util.cuh"
#include "kernels.h"

namespace rmi {

namespace {

constexpr int SE_THREADS = 256;
constexpr int SE_E = 4;                     // consecutive keys per lane per tile
constexpr u64 SE_TILE = 32 * SE_E;          // keys per warp tile

// Largest j in [j, N) with S[j] <= i, given S[j] <= i: a gallop forward, then a bisection (kernels_eval.cu leaf_at).
__device__ __forceinline__ u64 shard_leaf_at(const u64* __restrict__ S, u64 N, u64 j, u64 i) {
  u64 step = 1;
  while (j + step < N && __ldg(S + j + step) <= i) { j += step; step <<= 1; }
  u64 hi = j + step < N ? j + step : N;
  while (hi - j > 1) {
    const u64 mid = j + ((hi - j) >> 1);
    if (__ldg(S + mid) <= i) j = mid; else hi = mid;
  }
  return j;
}

// part_err[j] = max over this rank's keys in leaf j of error_between(pred_j(key), F, n_global); with DUPS
// part_run[j] = the longest run of equal keys that ENDS on this rank inside leaf j, unless it is the data set's last.
// A run that began on an earlier rank has its global start F from prev_F; one that continues on the next non-empty
// rank (has_next, next_key) does not end here.
template <class T, int LEAF, bool DUPS>
__global__ void __launch_bounds__(SE_THREADS, 4)
k_shard_eval_keys(const T* __restrict__ keys, const Shard<T> sh, int has_next, T next_key, const u64* __restrict__ S,
                  u64 N, const double* __restrict__ params, u64 chunk, u64* __restrict__ part_err,
                  u64* __restrict__ part_run) {
  constexpr int PPM = leaf_params_per_model(LEAF);
  const u64 nl = sh.n_local, n = sh.n_global, gb = sh.base;
  const int lane = threadIdx.x & 31;
  const u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const u64 c0 = warp * chunk;
  if (c0 >= nl) return;
  const u64 c1 = c0 + chunk < nl ? c0 + chunk : nl;
  const bool aligned = is_aligned16(keys);
  u64 jw = shard_leaf_at(S, N, 0, gb + c0);
  for (u64 t0 = c0; t0 < c1; t0 += SE_TILE) {
    const u64 b = t0 + (u64)lane * SE_E;   // local index of the lane's first key
    T k[SE_E];
    const int cnt = b < c1 ? load_keys4(keys, b, c1, aligned, k) : 0;
    u64 j = jw, seg_err = 0, seg_run = 0;
    if (cnt > 0) {
      j = shard_leaf_at(S, N, jw, gb + b);
      u64 next_start = __ldg(S + j + 1);
      double f[PPM];
#pragma unroll
      for (int q = 0; q < PPM; ++q) f[q] = __ldg(params + j * PPM + q);
      u64 F = DUPS ? global_run_start(keys, b, gb, sh.has_prev, sh.prev_key, sh.prev_F) : gb + b;
      const u64 after = b + (u64)cnt;
      bool after_exists = false;
      T k_after = T();
      if (DUPS) {
        if (after < nl) { k_after = keys[after]; after_exists = true; }
        else if (has_next) { k_after = next_key; after_exists = true; }
      }
#pragma unroll
      for (int e = 0; e < SE_E; ++e) {
        if (e >= cnt) break;
        const u64 i = gb + b + (u64)e;
        if (i >= next_start) {
          if (seg_err) atomicMax(&part_err[j], seg_err);
          if (DUPS && seg_run) atomicMax(&part_run[j], seg_run);
          seg_err = 0; seg_run = 0;
          j = shard_leaf_at(S, N, j, i);
          next_start = __ldg(S + j + 1);
#pragma unroll
          for (int q = 0; q < PPM; ++q) f[q] = __ldg(params + j * PPM + q);
        }
        if (DUPS) {
          if (e > 0 && k[e] != k[e - 1]) F = i;
        } else {
          F = i;
        }
        const u64 err = error_between(leaf_predict64<LEAF>(f, Key<T>::as_float(k[e])), F, n);
        seg_err = err > seg_err ? err : seg_err;
        if (DUPS && i + 1 < n) {
          const bool run_ends = e + 1 < cnt ? k[e + 1] != k[e] : (after_exists && k_after != k[e]);
          if (run_ends && i - F + 1 > seg_run) seg_run = i - F + 1;
        }
      }
    }
    const u64 jkey = cnt > 0 ? j : ~0ull;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const u64 oj = __shfl_up_sync(0xffffffffu, jkey, o);
      const u64 oe = __shfl_up_sync(0xffffffffu, seg_err, o);
      const u64 orun = __shfl_up_sync(0xffffffffu, seg_run, o);
      if (lane >= o && oj == jkey) {
        seg_err = oe > seg_err ? oe : seg_err;
        seg_run = orun > seg_run ? orun : seg_run;
      }
    }
    const u64 nj = __shfl_down_sync(0xffffffffu, jkey, 1);
    if (cnt > 0 && (lane == 31 || nj != jkey)) {
      if (seg_err) atomicMax(&part_err[j], seg_err);
      if (DUPS && seg_run) atomicMax(&part_run[j], seg_run);
    }
    const unsigned valid = __ballot_sync(0xffffffffu, cnt > 0);
    jw = __shfl_sync(0xffffffffu, j, 31 - __clz((int)valid));
  }
}

// The widening of leaf j (two_layer.rs:226-259, as k_eval_leaves), each term on the one rank that holds the key it
// reads: upper_error on the rank holding global index S[j+1] (or, when S[j+1] == n, the last non-empty rank with
// max_value); lower_error on the rank holding S[j]-1 (or, when S[j] == 0, the first non-empty rank with zero_value).
// Runs after k_shard_eval_keys on the same stream, one thread per leaf: a plain read-modify-write of part_err[j].
template <class T, int LEAF>
__global__ void __launch_bounds__(SE_THREADS)
k_shard_eval_widen(const T* __restrict__ keys, const Shard<T> sh, int is_first, const u64* __restrict__ S, u64 N,
                   const double* __restrict__ params, u64* __restrict__ part_err) {
  constexpr int PPM = leaf_params_per_model(LEAF);
  const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  const u64 n = sh.n_global, lo = sh.base, hi = sh.base + sh.n_local;
  const u64 g_lo = S[j], g_hi = S[j + 1];
  const bool up_here = g_hi < n ? (g_hi >= lo && g_hi < hi) : (sh.is_last != 0);
  const bool low_here = g_lo > 0 ? (g_lo - 1 >= lo && g_lo - 1 < hi) : (is_first != 0);
  if (!up_here && !low_here) return;
  double f[PPM];
#pragma unroll
  for (int q = 0; q < PPM; ++q) f[q] = params[j * PPM + q];
  u64 e = part_err[j];
  if (up_here) {
    const T next_key = g_hi < n ? keys[g_hi - lo] : Key<T>::max_value();
    const u64 up = leaf_predict64<LEAF>(f, Key<T>::as_float(Key<T>::minus_epsilon(next_key)));
    const u64 upper_error = error_between(up, g_hi + 1, n);
    if (upper_error > e) e = upper_error;
  }
  if (low_here) {
    const T prev_key = g_lo > 0 ? keys[g_lo - 1 - lo] : Key<T>::zero_value();
    const u64 first_idx = j == 0 ? S[1] : g_lo;
    const u64 lp = leaf_predict64<LEAF>(f, Key<T>::as_float(Key<T>::plus_epsilon(prev_key)));
    const u64 lower_error = error_between(lp, first_idx, n);
    if (lower_error > e) e = lower_error;
  }
  part_err[j] = e;
}

// errors[j] = part_err[j] + run_max[j], counts[j] from S (k_eval_leaves, with the maxima already combined over ranks).
__global__ void __launch_bounds__(SE_THREADS)
k_shard_eval_finish(u64 n, const u64* __restrict__ S, u64 N, int no_dups, const u64* __restrict__ part_err,
                    const u64* __restrict__ part_run, u64* __restrict__ errors, u64* __restrict__ counts) {
  const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  const u64 g_lo = S[j], g_hi = S[j + 1];
  u64 run_max;
  if (no_dups) {   // every run has length 1, and the data set's final run is never recorded
    const u64 recorded = g_hi < n ? (g_hi - g_lo) : (g_hi > g_lo ? g_hi - g_lo - 1 : 0);
    run_max = recorded > 0 ? 1 : 0;
  } else {
    run_max = part_run[j];
  }
  u64 cnt = g_hi - g_lo;
  if (g_hi == n && g_lo < g_hi) cnt += 1;
  errors[j] = part_err[j] + run_max;
  counts[j] = cnt;
}

template <class T, int LEAF, bool DUPS>
void launch_shard_eval(const Launch& L, const T* keys, const Shard<T>& sh, int is_first, int has_next, T next_key, u64 N,
                       const u64* d_S, const double* d_params, u64* d_part) {
  const u64 nl = sh.n_local;
  if (nl) {   // one warp per chunk of whole tiles, as launch_eval
    const u64 tiles = (nl + SE_TILE - 1) / SE_TILE;
    const u64 max_warps = (u64)L.num_sms * 32;
    const u64 warps = tiles < max_warps ? tiles : max_warps;
    const u64 chunk = (tiles + warps - 1) / warps * SE_TILE;
    const u64 used = (nl + chunk - 1) / chunk;
    const unsigned blocks = (unsigned)((used * 32 + SE_THREADS - 1) / SE_THREADS);
    k_shard_eval_keys<T, LEAF, DUPS><<<blocks, SE_THREADS, 0, L.stream>>>(keys, sh, has_next, next_key, d_S, N, d_params,
                                                                           chunk, d_part, d_part + N);
    count_launch();
  }
  k_shard_eval_widen<T, LEAF><<<(unsigned)((N + SE_THREADS - 1) / SE_THREADS), SE_THREADS, 0, L.stream>>>(
      keys, sh, is_first, d_S, N, d_params, d_part);
  count_launch();
}

template <class T, int LEAF>
void launch_shard_eval_dups(const Launch& L, const T* keys, const Shard<T>& sh, int is_first, int has_next, T next_key,
                            u64 N, const u64* d_S, const double* d_params, u64* d_part) {
  if (sh.no_dups) launch_shard_eval<T, LEAF, false>(L, keys, sh, is_first, has_next, next_key, N, d_S, d_params, d_part);
  else launch_shard_eval<T, LEAF, true>(L, keys, sh, is_first, has_next, next_key, N, d_S, d_params, d_part);
}

}  // namespace

template <class T>
void shard_evaluate_partials(const Launch& L, const T* keys, const Shard<T>& sh, int is_first, int has_next, T next_key,
                             int leaf_kind, u64 N, const u64* d_S, const double* d_params, u64* d_part) {
  cudaMemsetAsync(d_part, 0, sizeof(u64) * 2 * N, L.stream);
  switch (leaf_kind) {
    case M_LINEAR: case M_ROBUST_LINEAR: case M_LINEAR_SPLINE:   // one forward function (models.cuh)
      launch_shard_eval_dups<T, M_LINEAR>(L, keys, sh, is_first, has_next, next_key, N, d_S, d_params, d_part); break;
    case M_CUBIC: launch_shard_eval_dups<T, M_CUBIC>(L, keys, sh, is_first, has_next, next_key, N, d_S, d_params, d_part); break;
    case M_LOGLINEAR: launch_shard_eval_dups<T, M_LOGLINEAR>(L, keys, sh, is_first, has_next, next_key, N, d_S, d_params, d_part); break;
    case M_NORMAL: launch_shard_eval_dups<T, M_NORMAL>(L, keys, sh, is_first, has_next, next_key, N, d_S, d_params, d_part); break;
    default: launch_shard_eval_dups<T, M_LOGNORMAL>(L, keys, sh, is_first, has_next, next_key, N, d_S, d_params, d_part); break;
  }
}

void shard_evaluate_finish(const Launch& L, u64 n, u64 N, bool no_dups, const u64* d_S, const u64* d_part, u64* d_errors,
                           u64* d_counts) {
  k_shard_eval_finish<<<(unsigned)((N + SE_THREADS - 1) / SE_THREADS), SE_THREADS, 0, L.stream>>>(
      n, d_S, N, no_dups ? 1 : 0, d_part, d_part + N, d_errors, d_counts);
  count_launch();
}

#define INST(T)                                                                                                        \
  template void shard_evaluate_partials<T>(const Launch&, const T*, const Shard<T>&, int, int, T, int, u64, const u64*, \
                                           const double*, u64*);
INST(u64)
INST(u32)
INST(double)
#undef INST

}  // namespace rmi
