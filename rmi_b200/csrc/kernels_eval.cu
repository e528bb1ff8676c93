// kernels_eval.cu — the error pass of a build over GIVEN leaf tables (rmi_evaluate): two_layer.rs:205-259 without
// the fit and without the empty-leaf constants.
//
// Nothing in the pass depends on the order in which keys are visited: per leaf it needs the largest
// |pred - offset| of its keys, the longest run of equal keys that is not the data set's last, and its key count,
// which is S[j+1] - S[j].  So it runs key-parallel: every warp streams a contiguous chunk of the key array in
// 128-key tiles (four consecutive keys per lane, one 32-byte load), finds each key's leaf from the boundaries S
// (a gallop from the leaf of the warp's previous tile), evaluates the leaf's model with its parameters from L2,
// and reduces the per-leaf maxima with a segmented warp scan and one atomicMax per leaf segment.  A second,
// per-leaf kernel adds the widening by the neighbour keys (k_leaf's, kernels_leaf.cu) and the counts.
#include "device_util.cuh"
#include "kernels.h"

namespace rmi {

namespace {

constexpr int EVAL_THREADS = 256;
constexpr int EVAL_E = 4;                      // consecutive keys per lane per tile
constexpr u64 EVAL_TILE = 32 * EVAL_E;         // keys per warp tile

// Largest j in [j, N) with S[j] <= i, given S[j] <= i: a gallop forward, then a bisection.
__device__ __forceinline__ u64 leaf_at(const u64* __restrict__ S, u64 N, u64 j, u64 i) {
  u64 step = 1;
  while (j + step < N && __ldg(S + j + step) <= i) { j += step; step <<= 1; }
  u64 hi = j + step < N ? j + step : N;
  while (hi - j > 1) {
    const u64 mid = j + ((hi - j) >> 1);
    if (__ldg(S + mid) <= i) j = mid; else hi = mid;
  }
  return j;
}

// max_err[j] = max over leaf j's keys of error_between(pred_j(key), offset, n); with DUPS max_run[j] = the longest
// run of equal keys in leaf j that ends before n - 1 (lower_bound_correction.rs:101-119 records a run when the next
// one starts).  Both arrays start at 0.  Each warp owns `chunk` keys (a multiple of EVAL_TILE).
template <class T, int LEAF, bool DUPS>
__global__ void __launch_bounds__(EVAL_THREADS, 4)
k_eval_keys(const T* __restrict__ keys, u64 n, const u64* __restrict__ S, u64 N, const double* __restrict__ params,
            u64 chunk, u64* __restrict__ max_err, u64* __restrict__ max_run) {
  constexpr int PPM = leaf_params_per_model(LEAF);
  const int lane = threadIdx.x & 31;
  const u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const u64 c0 = warp * chunk;
  if (c0 >= n) return;
  const u64 c1 = c0 + chunk < n ? c0 + chunk : n;
  const bool aligned = is_aligned16(keys);
  u64 jw = leaf_at(S, N, 0, c0);   // leaf of the warp's next key
  for (u64 t0 = c0; t0 < c1; t0 += EVAL_TILE) {
    const u64 base = t0 + (u64)lane * EVAL_E;
    T k[EVAL_E];
    const int cnt = base < c1 ? load_keys4(keys, base, c1, aligned, k) : 0;
    u64 j = jw, seg_err = 0, seg_run = 0;
    if (cnt > 0) {
      j = leaf_at(S, N, jw, base);
      u64 next_start = __ldg(S + j + 1);
      double f[PPM];
#pragma unroll
      for (int q = 0; q < PPM; ++q) f[q] = __ldg(params + j * PPM + q);
      u64 F = DUPS ? run_start(keys, base) : base;
      // the key after the lane's last one: decides whether the lane's last run ends there
      const u64 after = base + (u64)cnt;
      const T k_after = DUPS && after < n ? keys[after] : T();
#pragma unroll
      for (int e = 0; e < EVAL_E; ++e) {
        if (e >= cnt) break;
        const u64 i = base + (u64)e;
        if (i >= next_start) {   // a new leaf: flush the previous one's maxima
          if (seg_err) atomicMax(&max_err[j], seg_err);
          if (DUPS && seg_run) atomicMax(&max_run[j], seg_run);
          seg_err = 0; seg_run = 0;
          j = leaf_at(S, N, j, i);
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
          const bool run_ends = e + 1 < cnt ? k[e + 1] != k[e] : k_after != k[e];
          if (run_ends && i - F + 1 > seg_run) seg_run = i - F + 1;
        }
      }
    }
    // segmented max over the lanes' last segments: lanes of one leaf are contiguous (keys sorted, lanes in order)
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
      if (seg_err) atomicMax(&max_err[j], seg_err);
      if (DUPS && seg_run) atomicMax(&max_run[j], seg_run);
    }
    // the next tile starts at or after the last valid lane's leaf
    const unsigned valid = __ballot_sync(0xffffffffu, cnt > 0);
    jw = __shfl_sync(0xffffffffu, j, 31 - __clz((int)valid));
  }
}

// Per leaf: count (two_layer.rs:207-217, with the drained iterator's repeated final item in the last key's leaf) and
// the widened bound (two_layer.rs:226-259), exactly as k_leaf finishes a leaf.
template <class T, int LEAF>
__global__ void __launch_bounds__(EVAL_THREADS)
k_eval_leaves(const T* __restrict__ keys, u64 n, const u64* __restrict__ S, u64 N, const double* __restrict__ params,
              int no_dups, const u64* __restrict__ max_err, const u64* __restrict__ max_run, u64* __restrict__ errors,
              u64* __restrict__ counts) {
  constexpr int PPM = leaf_params_per_model(LEAF);
  const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  const u64 g_lo = S[j], g_hi = S[j + 1];
  double f[PPM];
#pragma unroll
  for (int q = 0; q < PPM; ++q) f[q] = params[j * PPM + q];
  u64 run_max;
  if (no_dups) {   // every run has length 1, and the data set's final run is never recorded
    const u64 recorded = g_hi < n ? (g_hi - g_lo) : (g_hi > g_lo ? g_hi - g_lo - 1 : 0);
    run_max = recorded > 0 ? 1 : 0;
  } else {
    run_max = max_run[j];
  }
  u64 cnt = g_hi - g_lo;
  if (g_hi == n && g_lo < g_hi) cnt += 1;
  const T next_key = g_hi < n ? keys[g_hi] : Key<T>::max_value();
  const T prev_key = g_lo > 0 ? keys[g_lo - 1] : Key<T>::zero_value();
  const u64 first_idx = j == 0 ? S[1] : g_lo;   // lb.next_index(max(j-1, 0))
  const u64 up = leaf_predict64<LEAF>(f, Key<T>::as_float(Key<T>::minus_epsilon(next_key)));
  const u64 upper_error = error_between(up, g_hi + 1, n);
  const u64 lp = leaf_predict64<LEAF>(f, Key<T>::as_float(Key<T>::plus_epsilon(prev_key)));
  const u64 lower_error = error_between(lp, first_idx, n);
  u64 e = max_err[j];
  if (upper_error > e) e = upper_error;
  if (lower_error > e) e = lower_error;
  errors[j] = e + run_max;
  counts[j] = cnt;
}

template <class T, int LEAF, bool DUPS>
void launch_eval(const Launch& L, const T* keys, u64 n, u64 N, const u64* d_S, const double* d_params, u64* d_max_err,
                 u64* d_max_run, u64* d_errors, u64* d_counts) {
  // one warp per chunk of whole tiles; enough warps for every SM, no more than there are tiles
  const u64 tiles = (n + EVAL_TILE - 1) / EVAL_TILE;
  const u64 max_warps = (u64)L.num_sms * 32;   // 4 blocks of 8 warps per SM
  const u64 warps = tiles < max_warps ? tiles : max_warps;
  const u64 chunk = (tiles + warps - 1) / warps * EVAL_TILE;
  const u64 used = (n + chunk - 1) / chunk;
  const unsigned blocks = (unsigned)((used * 32 + EVAL_THREADS - 1) / EVAL_THREADS);
  k_eval_keys<T, LEAF, DUPS><<<blocks, EVAL_THREADS, 0, L.stream>>>(keys, n, d_S, N, d_params, chunk, d_max_err, d_max_run);
  count_launch();
  k_eval_leaves<T, LEAF><<<(unsigned)((N + EVAL_THREADS - 1) / EVAL_THREADS), EVAL_THREADS, 0, L.stream>>>(
      keys, n, d_S, N, d_params, DUPS ? 0 : 1, d_max_err, d_max_run, d_errors, d_counts);
  count_launch();
}

template <class T, int LEAF>
void launch_eval_dups(const Launch& L, const T* keys, u64 n, bool no_dups, u64 N, const u64* d_S, const double* d_params,
                      u64* d_scratch, u64* d_errors, u64* d_counts) {
  if (no_dups) launch_eval<T, LEAF, false>(L, keys, n, N, d_S, d_params, d_scratch, d_scratch + N, d_errors, d_counts);
  else launch_eval<T, LEAF, true>(L, keys, n, N, d_S, d_params, d_scratch, d_scratch + N, d_errors, d_counts);
}

}  // namespace

template <class T>
void evaluate_leaves(const Launch& L, const T* keys, u64 n, bool no_dups, int leaf_kind, u64 N, const u64* d_S,
                     const double* d_params, u64* d_scratch, u64* d_errors, u64* d_counts) {
  cudaMemsetAsync(d_scratch, 0, sizeof(u64) * 2 * N, L.stream);
  switch (leaf_kind) {
    case M_LINEAR: case M_ROBUST_LINEAR: case M_LINEAR_SPLINE:   // one forward function (models.cuh)
      launch_eval_dups<T, M_LINEAR>(L, keys, n, no_dups, N, d_S, d_params, d_scratch, d_errors, d_counts); break;
    case M_CUBIC: launch_eval_dups<T, M_CUBIC>(L, keys, n, no_dups, N, d_S, d_params, d_scratch, d_errors, d_counts); break;
    case M_LOGLINEAR: launch_eval_dups<T, M_LOGLINEAR>(L, keys, n, no_dups, N, d_S, d_params, d_scratch, d_errors, d_counts); break;
    case M_NORMAL: launch_eval_dups<T, M_NORMAL>(L, keys, n, no_dups, N, d_S, d_params, d_scratch, d_errors, d_counts); break;
    default: launch_eval_dups<T, M_LOGNORMAL>(L, keys, n, no_dups, N, d_S, d_params, d_scratch, d_errors, d_counts); break;
  }
}

template void evaluate_leaves<u64>(const Launch&, const u64*, u64, bool, int, u64, const u64*, const double*, u64*, u64*, u64*);
template void evaluate_leaves<u32>(const Launch&, const u32*, u64, bool, int, u64, const u64*, const double*, u64*, u64*, u64*);
template void evaluate_leaves<double>(const Launch&, const double*, u64, bool, int, u64, const u64*, const double*, u64*, u64*,
                                      u64*);

}  // namespace rmi
