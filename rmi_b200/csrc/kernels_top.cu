// kernels_top.cu — layer-0 (top) model fits on the full key array.
//
// Reference: train_two_layer step 1 (rmi_lib/src/train/two_layer.rs:109-110) calls
// train_model(layer1, data) with targets scaled by N/n; the per-model constructors are
// models/linear.rs:79-83,169-173,239-260, linear_spline.rs:13-35, cubic_spline.rs:18-136,
// normal.rs:28-76, radix.rs:18-40,90-120, balanced_radix.rs:20-98, histogram.rs:20-54.
//
// The item stream every constructor sees is RMITrainingData::iter(): for index i the pair
// (key_i, scale(F_i)) with F_i the first index of i's run of equal keys, followed — when the
// iterator is drained — by ONE repeat of the final item (FixDupsIter, models/mod.rs:154-185,
// the `None => self.last_item.take()` arm).  "repeat" below always means that extra item.
//
// HBM traffic: one coalesced read of the key array per full pass; the sums / comparison
// passes are grid-stride with a fixed grid so reductions are deterministic run to run.
#include "device_util.cuh"
#include "kernels.h"
#include "spline.cuh"

namespace rmi {

namespace {

constexpr int TOP_THREADS = 256;
constexpr int MAX_PARTIAL_BLOCKS = 132 * 8;   // 8 blocks per SM of an H100 (grid_for: min(num_sms * 8, this))

__device__ __forceinline__ void set_status(BuildAux* aux, unsigned bit) { atomicOr(&aux->status, bit); }

// (x, y) of stream item i.
template <class T>
__device__ __forceinline__ void stream_item(const T* __restrict__ keys, u64 i, double sf, int use_sf, double& x,
                                            u64& y) {
  x = Key<T>::as_float(keys[i]);
  y = scale_offset(run_start(keys, i), sf, use_sf);
}

// ------------------------------------------------------------------------------------------
// linear / robust_linear, parallel ("fast") fit: pivot-shifted sums, finished into
// slr()'s closing formulas (linear.rs:36-58).  MODE 0: y;  MODE 1: ln(y), non-finite dropped
// (loglinear_slr, linear.rs:61-72).
// partial layout per block: {Sx, Sy, Sxx, Sxy, count}
// sample (MODE 0, may be null): receives keys[s * BOUNDS_SAMPLE_R] for every s < bounds_sample_len(n), stored
// evict_last so that the sample is still in L2 when the boundary search reads it; the keys themselves are loaded
// evict_first, so that this 1.6 GB stream does not push the sample out.
// ------------------------------------------------------------------------------------------
template <class T, int MODE>
__global__ void __launch_bounds__(TOP_THREADS)
k_slr_partial(const T* __restrict__ keys, u64 n, u64 i0, u64 i1, double sf, int use_sf,
              double* __restrict__ partials, T* __restrict__ sample) {
  __shared__ double sm[32];
  u64 mid = i0 + ((i1 - i0) >> 1);
  double px = Key<T>::as_float(keys[mid]);
  double py = MODE == 0 ? __ull2double_rn(scale_offset(mid, sf, use_sf)) : 0.0;
  double sx = 0, sy = 0, sxx = 0, sxy = 0, cnt = 0;
  const bool aligned = is_aligned16(keys);
  const u64 ld_policy = l2_policy_of(1), st_policy = l2_policy_of(2);
  // each thread owns 4 consecutive keys per trip (128-bit loads); [i0, i1) is covered from the
  // 4-aligned index at or below i0
  const u64 tid = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  u64 stride = (u64)gridDim.x * blockDim.x * 4;
  unsigned icnt = 0;
  if (MODE == 0 && sample) {
    // sample points the loop below does not visit: robust_linear sums [i0, i1) only, the sample covers [0, n)
    const u64 lo_pts = ((i0 & ~3ull) + BOUNDS_SAMPLE_R - 1) / BOUNDS_SAMPLE_R;   // s * R < (i0 & ~3)
    const u64 hi_first = (i1 + BOUNDS_SAMPLE_R - 1) / BOUNDS_SAMPLE_R;           // s * R >= i1
    const u64 extra = lo_pts + (bounds_sample_len(n) - hi_first);
    for (u64 q = tid; q < extra; q += stride / 4) {
      const u64 s = q < lo_pts ? q : hi_first + (q - lo_pts);
      store_key_hint(sample + s, keys[s * BOUNDS_SAMPLE_R], st_policy);
    }
  }
  // One trip: the 4 keys at `base` (c of them valid), kprev = keys[base - 1].
  auto trip = [&](u64 base, const T (&k)[4], int c, T kprev) {
    if (MODE == 0 && sample && base % BOUNDS_SAMPLE_R == 0) store_key_hint(sample + base / BOUNDS_SAMPLE_R, k[0], st_policy);
    bool interior = MODE == 0 && c == 4 && base >= i0 && base + 4 <= i1;
    if (interior) {
      bool dup = (base > 0 && kprev == k[0]) || k[1] == k[0] || k[2] == k[1] || k[3] == k[2];
      if (!dup) {
        // fast path: every key starts its own run, so the offset of key e is base + e and the
        // scaled target floor(offset * sf) is taken with the 2^52 trick (0 <= value < 2^51)
        double bd = __ull2double_rn(base);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          double x = Key<T>::as_float(k[e]);
          double y = bd + (double)e;
          if (use_sf) y = __dadd_rn(__dadd_rd(__dmul_rn(y, sf), 4503599627370496.0), -4503599627370496.0);
          double dx = x - px, dy = y - py;
          sx += dx; sy += dy; sxx = fma(dx, dx, sxx); sxy = fma(dx, dy, sxy);
        }
        icnt += 4;
        return;
      }
    }
    // general path: duplicates, range edges, log targets
    u64 F = run_start(keys, base);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (e >= c) break;
      u64 i = base + e;
      if (e > 0 && k[e] != k[e - 1]) F = i;
      if (i < i0 || i >= i1) continue;
      double x = Key<T>::as_float(k[e]);
      double y = __ull2double_rn(scale_offset(F, sf, use_sf));
      if (MODE == 1) { y = log(y); if (!isfinite(y)) continue; }
      double dx = x - px, dy = y - py;
      sx += dx; sy += dy; sxx = fma(dx, dx, sxx); sxy = fma(dx, dy, sxy);
      icnt += 1;
    }
  };
  // Two trips per iteration, both loaded before either is summed, in the order a one-trip loop takes them (the sums do
  // not change).  The loop runs while the warp's first lane has keys, so every lane takes part in the shuffles: lane l
  // gets keys[base - 1] (lane l - 1's last key) from below, only lane 0 loads it.
  const unsigned FULL = 0xffffffffu;
  const unsigned lane = threadIdx.x & 31u;
  for (u64 wb = (i0 & ~3ull) + (tid - lane) * 4; wb < i1; wb += 2 * stride) {
    const u64 b0 = wb + lane * 4, b1 = b0 + stride;
    T k0[4] = {}, k1[4] = {};
    const int c0 = b0 < i1 ? load_keys4_hint(keys, b0, n, aligned, k0, ld_policy) : 0;
    const int c1 = b1 < i1 ? load_keys4_hint(keys, b1, n, aligned, k1, ld_policy) : 0;
    T p0 = __shfl_up_sync(FULL, k0[3], 1), p1 = __shfl_up_sync(FULL, k1[3], 1);
    if (lane == 0) {
      if (c0 && b0 > 0) p0 = keys[b0 - 1];
      if (c1) p1 = keys[b1 - 1];
    }
    if (c0) trip(b0, k0, c0, p0);
    if (c1) trip(b1, k1, c1, p1);
  }
  cnt = (double)icnt;
  double r0 = block_sum(sx, sm), r1 = block_sum(sy, sm), r2 = block_sum(sxx, sm), r3 = block_sum(sxy, sm),
         r4 = block_sum(cnt, sm);
  if (threadIdx.x == 0) {
    double* p = partials + (size_t)blockIdx.x * 5;
    p[0] = r0; p[1] = r1; p[2] = r2; p[3] = r3; p[4] = r4;
  }
}

template <class T, int MODE>
__global__ void __launch_bounds__(TOP_THREADS)
k_slr_finish(const T* __restrict__ keys, u64 i0, u64 i1, int repeat, double sf, int use_sf,
             const double* __restrict__ partials, int nblocks, TopModel* top, BuildAux* aux) {
  __shared__ double sm[32];
  double s[5] = {0, 0, 0, 0, 0};
  for (int b = threadIdx.x; b < nblocks; b += blockDim.x)
    for (int q = 0; q < 5; ++q) s[q] += partials[(size_t)b * 5 + q];
  double r[5];
  for (int q = 0; q < 5; ++q) r[q] = block_sum(s[q], sm);
  if (threadIdx.x != 0) return;
  u64 mid = i0 + ((i1 - i0) >> 1);
  double px = (i1 > i0) ? Key<T>::as_float(keys[mid]) : 0.0;
  double py = (MODE == 0 && i1 > i0) ? __ull2double_rn(scale_offset(mid, sf, use_sf)) : 0.0;
  double sx = r[0], sy = r[1], sxx = r[2], sxy = r[3], cnt = r[4];
  if (repeat && i1 > i0) {
    double x; u64 yi;
    stream_item(keys, i1 - 1, sf, use_sf, x, yi);
    double y = __ull2double_rn(yi);
    bool keep = true;
    if (MODE == 1) { y = log(y); keep = isfinite(y); }
    if (keep) {
      double dx = x - px, dy = y - py;
      sx += dx; sy += dy; sxx += dx * dx; sxy += dx * dy; cnt += 1.0;
    }
  }
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
        if (var > -1e-9 * fabs(sxx / cnt)) var = 0.0;   // rounding of a zero variance
        else set_status(aux, ST_NEG_VARIANCE);
      }
      if (var == 0.0) { alpha = mean_y; beta = 0.0; }
      else { beta = cov / var; alpha = mean_y - beta * mean_x; }
    }
  }
  top->f[0] = alpha;
  top->f[1] = beta;
}

// ------------------------------------------------------------------------------------------
// linear / robust_linear, exact fit: the reference's sequential Welford recurrence
// (linear.rs:17-34) in stream order on ONE warp.  Lanes load 32 keys coalesced and derive the
// duplicate-fixed targets with a warp max-scan; every lane then replays the 32 steps from
// shuffles (redundantly, so no divergence).  Latency-bound by design: ~5 dependent FP64 ops
// per item.  Bit-identical to the reference.
// ------------------------------------------------------------------------------------------
struct Welford {
  double mean_x, mean_y, c, m2;
  u64 n;
  __device__ __forceinline__ void init() { mean_x = mean_y = c = m2 = 0.0; n = 0; }
  __device__ __forceinline__ void push(double x, double y) {
    n += 1;
    double nf = __ull2double_rn(n);
    double dx = __dadd_rn(x, -mean_x);
    mean_x = __dadd_rn(mean_x, __ddiv_rn(dx, nf));
    mean_y = __dadd_rn(mean_y, __ddiv_rn(__dadd_rn(y, -mean_y), nf));
    c = __dadd_rn(c, __dmul_rn(dx, __dadd_rn(y, -mean_y)));
    double dx2 = __dadd_rn(x, -mean_x);
    m2 = __dadd_rn(m2, __dmul_rn(dx, dx2));
  }
  // linear.rs:36-58; returns false where the reference asserts (var >= 0)
  __device__ __forceinline__ bool finish(double& alpha, double& beta) const {
    if (n == 0) { alpha = 0.0; beta = 0.0; return true; }
    if (n == 1) { alpha = mean_y; beta = 0.0; return true; }
    double nm1 = __ull2double_rn(n - 1);
    double cov = __ddiv_rn(c, nm1), var = __ddiv_rn(m2, nm1);
    if (!(var >= 0.0)) { alpha = 0.0; beta = 0.0; return false; }
    if (var == 0.0) { alpha = mean_y; beta = 0.0; return true; }
    beta = __ddiv_rn(cov, var);
    alpha = __dadd_rn(mean_y, -__dmul_rn(beta, mean_x));
    return true;
  }
};

template <class T, int MODE>
__global__ void __launch_bounds__(32)
k_slr_exact(const T* __restrict__ keys, u64 i0, u64 i1, int repeat, double sf, int use_sf, TopModel* top,
            BuildAux* aux) {
  const unsigned FULL = 0xffffffffu;
  int lane = threadIdx.x;
  Welford w;
  w.init();
  u64 carryF = (i1 > i0) ? run_start(keys, i0) : 0;
  T carryK = (i1 > i0) ? keys[i0] : T();
  for (u64 base = i0; base < i1; base += 32) {
    u64 i = base + lane;
    bool valid = i < i1;
    T k = valid ? keys[i] : carryK;
    T kp = __shfl_up_sync(FULL, k, 1);
    if (lane == 0) kp = carryK;
    // a new run starts here iff the key differs from its predecessor (index i0 continues carryF)
    u64 f = (valid && i != i0 && k != kp) ? i : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      u64 t = __shfl_up_sync(FULL, f, o);
      if (lane >= o && t > f) f = t;
    }
    if (carryF > f) f = carryF;
    double x = Key<T>::as_float(k);
    double y = __ull2double_rn(scale_offset(f, sf, use_sf));
    if (MODE == 1) y = log(y);
    int cnt = (i1 - base) < 32 ? (int)(i1 - base) : 32;
    for (int j = 0; j < cnt; ++j) {
      double xj = __shfl_sync(FULL, x, j), yj = __shfl_sync(FULL, y, j);
      if (MODE == 1 && !isfinite(yj)) continue;
      w.push(xj, yj);
    }
    carryF = __shfl_sync(FULL, f, cnt - 1);
    carryK = __shfl_sync(FULL, k, cnt - 1);
  }
  if (repeat && i1 > i0) {
    // the repeated item is the stream's final item; in MODE 1 it is dropped if ln(y) is not finite
    double x; u64 yi;
    stream_item(keys, i1 - 1, sf, use_sf, x, yi);
    double y = __ull2double_rn(yi);
    if (MODE == 1) y = log(y);
    if (MODE == 0 || isfinite(y)) w.push(x, y);
  }
  if (lane == 0) {
    double a, b;
    if (!w.finish(a, b)) set_status(aux, ST_NEG_VARIANCE);
    top->f[0] = a;
    top->f[1] = b;
  }
}

// ------------------------------------------------------------------------------------------
// linear_spline (linear_spline.rs:13-35) and the closed-form part of cubic
// (cubic_spline.rs:18-101): O(1) gathers + two binary searches, one thread.
// cand[0..4) = cubic (a,b,c,d), cand[4..6) = linear spline (alpha, beta).
// ------------------------------------------------------------------------------------------
template <class T>
__device__ void linear_spline_params(const T* __restrict__ keys, u64 n, double sf, int use_sf, double& alpha,
                                     double& beta) {
  if (n == 0) { alpha = 0.0; beta = 0.0; return; }
  double y0 = __ull2double_rn(scale_offset(0, sf, use_sf));
  if (n == 1) { alpha = y0; beta = 0.0; return; }
  T k0 = keys[0], k1 = keys[n - 1];
  if (k0 == k1) { alpha = y0; beta = 0.0; return; }
  double y1 = __ull2double_rn(scale_offset(n - 1, sf, use_sf));
  double x0 = Key<T>::as_float(k0), x1 = Key<T>::as_float(k1);
  double slope = __ddiv_rn(__dadd_rn(y0, -y1), __dadd_rn(x0, -x1));
  alpha = __dadd_rn(y0, -__dmul_rn(slope, x0));
  beta = slope;
}

template <class T>
__global__ void k_spline_prepare(const T* __restrict__ keys, u64 n, double sf, int use_sf, int want_cubic,
                                 double* cand, TopModel* top, BuildAux* aux) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double la, lb;
  linear_spline_params(keys, n, sf, use_sf, la, lb);
  if (!want_cubic) { top->f[0] = la; top->f[1] = lb; return; }
  cand[4] = la; cand[5] = lb;
  double a, b, c, d;
  double y_first = __ull2double_rn(scale_offset(0, sf, use_sf));
  if (n == 0) { a = 0.0; b = 0.0; c = 1.0; d = 0.0; }
  else if (n == 1 || keys[0] == keys[n - 1]) { a = b = c = 0.0; d = y_first; }   // :23-36 (sorted: all equal)
  else {
    double xmin = Key<T>::as_float(keys[0]), ymin = y_first;
    double xmax = Key<T>::as_float(keys[n - 1]);
    double ymax = __ull2double_rn(scale_offset(n - 1, sf, use_sf));
    // :46-54 first stream item with scaled x > 0 (monotone in the index)
    u64 lo = 0, hi = n;
    while (lo < hi) {
      u64 mid = lo + ((hi - lo) >> 1);
      if (scale3(Key<T>::as_float(keys[mid]), xmin, xmax) > 0.0) hi = mid; else lo = mid + 1;
    }
    // :56-65 last raw item with scaled x < 1
    u64 lo2 = 0, hi2 = n;   // first index with !(sx < 1)
    while (lo2 < hi2) {
      u64 mid = lo2 + ((hi2 - lo2) >> 1);
      if (scale3(Key<T>::as_float(keys[mid]), xmin, xmax) < 1.0) lo2 = mid + 1; else hi2 = mid;
    }
    if (lo >= n || lo2 == 0) {
      set_status(aux, ST_CUBIC_UNWRAP);
      a = b = c = d = 0.0;
    } else {
      u64 ip = lo2 - 1;
      cubic_from_points(xmin, ymin, xmax, ymax, Key<T>::as_float(keys[lo]),
                        __ull2double_rn(scale_offset(run_start(keys, lo), sf, use_sf)), Key<T>::as_float(keys[ip]),
                        __ull2double_rn(scale_offset(ip, sf, use_sf)), a, b, c, d);
    }
  }
  cand[0] = a; cand[1] = b; cand[2] = c; cand[3] = d;
}

// cubic_spline.rs:117-126: sum |cubic(x) - y| and |linear_spline(x) - y| over the stream.
template <class T>
__global__ void __launch_bounds__(TOP_THREADS)
k_cubic_l1_partial(const T* __restrict__ keys, u64 n, double sf, int use_sf, const double* __restrict__ cand,
                   double* __restrict__ partials) {
  __shared__ double sm[32];
  double cf[4] = {cand[0], cand[1], cand[2], cand[3]};
  double lf[2] = {cand[4], cand[5]};
  double ec = 0, el = 0;
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double x; u64 yi;
    stream_item(keys, i, sf, use_sf, x, yi);
    double y = __ull2double_rn(yi);
    ec += fabs(predict_float<M_CUBIC>(cf, x) - y);
    el += fabs(predict_float<M_LINEAR>(lf, x) - y);
  }
  double r0 = block_sum(ec, sm), r1 = block_sum(el, sm);
  if (threadIdx.x == 0) { partials[2 * blockIdx.x] = r0; partials[2 * blockIdx.x + 1] = r1; }
}

template <class T>
__global__ void __launch_bounds__(TOP_THREADS)
k_cubic_finish(const T* __restrict__ keys, u64 n, double sf, int use_sf, const double* __restrict__ cand,
               const double* __restrict__ partials, int nblocks, TopModel* top) {
  __shared__ double sm[32];
  double ec = 0, el = 0;
  for (int b = threadIdx.x; b < nblocks; b += blockDim.x) { ec += partials[2 * b]; el += partials[2 * b + 1]; }
  double r0 = block_sum(ec, sm), r1 = block_sum(el, sm);
  if (threadIdx.x != 0) return;
  if (n > 0) {  // the repeated final item
    double x; u64 yi;
    stream_item(keys, n - 1, sf, use_sf, x, yi);
    double y = __ull2double_rn(yi);
    double lf[2] = {cand[4], cand[5]};
    r0 += fabs(predict_float<M_CUBIC>(cand, x) - y);
    r1 += fabs(predict_float<M_LINEAR>(lf, x) - y);
  }
  if (r1 < r0) { top->f[0] = 0.0; top->f[1] = 0.0; top->f[2] = cand[5]; top->f[3] = cand[4]; }
  else { top->f[0] = cand[0]; top->f[1] = cand[1]; top->f[2] = cand[2]; top->f[3] = cand[3]; }
}

// ------------------------------------------------------------------------------------------
// normal / lognormal (normal.rs:28-76).  Parallel: mean = sum(x)/n over the drained stream
// (n+1 items, divisor n), scale = max y, stdev = sqrt(sum((x-mean)^2)/n).
// ------------------------------------------------------------------------------------------
template <class T, int LOGN, int PASS>
__global__ void __launch_bounds__(TOP_THREADS)
k_normal_partial(const T* __restrict__ keys, u64 n, const double* __restrict__ state, double* __restrict__ partials) {
  __shared__ double sm[32];
  double px = PASS == 0 ? normal_x<T, LOGN>(keys[n >> 1]) : state[0];  // pass 0: pivot; pass 1: mean
  double s = 0;
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double d = normal_x<T, LOGN>(keys[i]) - px;
    s += PASS == 0 ? d : d * d;
  }
  double r = block_sum(s, sm);
  if (threadIdx.x == 0) partials[blockIdx.x] = r;
}
template <class T, int LOGN, int PASS>
__global__ void __launch_bounds__(TOP_THREADS)
k_normal_finish(const T* __restrict__ keys, u64 n, double sf, int use_sf, const double* __restrict__ partials,
                int nblocks, double* state, TopModel* top) {
  __shared__ double sm[32];
  double s = 0;
  for (int b = threadIdx.x; b < nblocks; b += blockDim.x) s += partials[b];
  double r = block_sum(s, sm);
  if (threadIdx.x != 0) return;
  double nf = __ull2double_rn(n);
  if (PASS == 0) {
    double mean = 0.0;
    if (n > 0) {
      double px = normal_x<T, LOGN>(keys[n >> 1]);
      r += normal_x<T, LOGN>(keys[n - 1]) - px;                      // repeated final item
      mean = (r + __ull2double_rn(n + 1) * px) / nf;
    }
    state[0] = mean;
  } else {
    double mean = state[0];
    if (n > 0) { double d = normal_x<T, LOGN>(keys[n - 1]) - mean; r += d * d; }
    double stdev = sqrt(r / nf);                                      // n == 0: 0/0 = NaN, as the reference
    double scale = -INFINITY;
    if (n > 0) scale = fmax(scale, __ull2double_rn(scale_offset(run_start(keys, n - 1), sf, use_sf)));
    top->f[0] = mean; top->f[1] = stdev; top->f[2] = scale;
  }
}
// Exact (serial) variant for `normal` (no libm on the path): normal.rs:36-48 verbatim.
template <class T>
__global__ void __launch_bounds__(32)
k_normal_exact(const T* __restrict__ keys, u64 n, double sf, int use_sf, TopModel* top) {
  const unsigned FULL = 0xffffffffu;
  int lane = threadIdx.x;
  double nf = __ull2double_rn(n);
  double mean = 0.0, stdev = 0.0;
  for (u64 base = 0; base < n; base += 32) {
    u64 i = base + lane;
    double x = i < n ? Key<T>::as_float(keys[i]) : 0.0;
    int cnt = (n - base) < 32 ? (int)(n - base) : 32;
    for (int j = 0; j < cnt; ++j) mean = __dadd_rn(mean, __ddiv_rn(__shfl_sync(FULL, x, j), nf));
  }
  if (n > 0) mean = __dadd_rn(mean, __ddiv_rn(Key<T>::as_float(keys[n - 1]), nf));
  for (u64 base = 0; base < n; base += 32) {
    u64 i = base + lane;
    double x = i < n ? Key<T>::as_float(keys[i]) : 0.0;
    int cnt = (n - base) < 32 ? (int)(n - base) : 32;
    for (int j = 0; j < cnt; ++j) {
      double d = __dadd_rn(__shfl_sync(FULL, x, j), -mean);
      stdev = __dadd_rn(stdev, __dmul_rn(d, d));
    }
  }
  if (n > 0) { double d = __dadd_rn(Key<T>::as_float(keys[n - 1]), -mean); stdev = __dadd_rn(stdev, __dmul_rn(d, d)); }
  if (lane == 0) {
    stdev = __dsqrt_rn(__ddiv_rn(stdev, nf));
    double scale = -INFINITY;
    if (n > 0) scale = fmax(scale, __ull2double_rn(scale_offset(run_start(keys, n - 1), sf, use_sf)));
    top->f[0] = mean; top->f[1] = stdev; top->f[2] = scale;
  }
}

// ------------------------------------------------------------------------------------------
// radix family.  k_radix_scalars: prefix, bits, max scaled y (radix.rs:18-40; bradix and the
// radix tables share the prefix).  One thread.
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void k_radix_scalars(const T* __restrict__ keys, u64 n, double sf, int use_sf, int kind, TopModel* top,
                                BuildAux* aux) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (n == 0) {
    top->ip[0] = 0; top->ip[1] = 0; top->ip[2] = 0; top->high = 1;
    aux->max_scaled_y = 0;
    return;
  }
  int prefix = common_prefix_sorted(Key<T>::as_int(keys[0]), Key<T>::as_int(keys[n - 1]));
  u64 largest = scale_offset(run_start(keys, n - 1), sf, use_sf);
  aux->max_scaled_y = largest;
  top->ip[0] = (u64)prefix;
  if (kind == M_RADIX || kind == M_BRADIX) {
    int bits = num_bits_of(largest);
    if (bits < 1) set_status(aux, ST_NUM_BITS);
    top->ip[1] = (u64)bits;
  }
}

// RadixTable::new (radix.rs:90-120): hint[r] = scaled offset of the first key whose radix
// is >= r, for 1 <= r <= radix(last key); hint[0] = 0; later entries = 2^bits.
__global__ void k_table_init(u32* __restrict__ table, u64 len) {
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += stride) table[i] = i == 0 ? 0u : (u32)len;
}
template <class T> __device__ __forceinline__ u64 table_radix(T key, unsigned prefix, unsigned nb) {
  return shr64(shr64(shl64(Key<T>::as_int(key), prefix), prefix), nb);
}
template <class T>
__global__ void __launch_bounds__(TOP_THREADS)
k_table_fill(const T* __restrict__ keys, u64 n, double sf, int use_sf, const TopModel* __restrict__ top, int bits,
             u32* __restrict__ table, BuildAux* aux) {
  unsigned prefix = (unsigned)top->ip[0];
  unsigned nb = (prefix + (unsigned)bits > 64u) ? 0u : 64u - (prefix + (unsigned)bits);
  u64 len = 1ull << bits;
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    u64 r = table_radix(keys[i], prefix, nb);
    u64 rp = i == 0 ? 0ull : table_radix(keys[i - 1], prefix, nb);
    if (r > rp) {
      if (r >= len) { set_status(aux, ST_RADIX_TABLE_OOB); continue; }
      u32 y = (u32)scale_offset(i, sf, use_sf);   // a radix change implies a key change: F_i = i
      for (u64 q = rp + 1; q <= r; ++q) table[q] = y;
    }
  }
}

// bradix (balanced_radix.rs:20-98).  The candidate's predictions are monotone in the key, so
// the per-bin counts of chi2() come from bin boundaries: B[b] = first index whose prediction
// is >= b.  k_bradix_bounds writes B (pre-filled with n); k_bradix_chi2 sums
// (count_b - expected)^2 / expected over the bins (the drained stream adds one to the bin of
// the last key); k_bradix_pick keeps the strict minimum in candidate order.
struct BradixCand { u64 prefix, bits, clamp; int high; };
template <class T> __device__ __forceinline__ u64 bradix_pred(const BradixCand& m, T key) {
  u64 res = shr64(shl64(Key<T>::as_int(key), (unsigned)m.prefix), (unsigned)((64u - (unsigned)m.bits) & 0xffu));
  if (m.high) return res < m.clamp ? res : m.clamp;
  return res < m.clamp ? 0ull : res - m.clamp;
}
__device__ __forceinline__ BradixCand bradix_candidate(const TopModel* top, const BuildAux* aux, int which) {
  BradixCand c;
  u64 max_output = aux->max_scaled_y;
  u64 bits = top->ip[1];
  u64 test_bits = bits + (u64)(which >> 1);
  c.prefix = top->ip[0];
  c.bits = test_bits;
  c.high = (which & 1) == 0;
  u64 bits_max = shl64(1ull, (unsigned)(test_bits + 1)) - 1ull;
  c.clamp = c.high ? max_output - 1ull : max_output - bits_max;   // wraps, as in release Rust
  return c;
}
__global__ void k_fill_u64(u64* __restrict__ p, u64 len, u64 v) {
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += stride) p[i] = v;
}
template <class T>
__global__ void __launch_bounds__(TOP_THREADS)
k_bradix_bounds(const T* __restrict__ keys, u64 n, const TopModel* __restrict__ top, BuildAux* aux, int which,
                u64* __restrict__ B) {
  BradixCand c = bradix_candidate(top, aux, which);
  u64 max_output = aux->max_scaled_y;
  if (c.bits >= 64) return;   // `for test_bits in bits..min(bits+2, 64)`
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    u64 p = bradix_pred(c, keys[i]);
    if (p >= max_output) { set_status(aux, ST_BRADIX_OOB); continue; }
    if (i == 0) { for (u64 q = 0; q <= p; ++q) B[q] = 0; }
    else {
      u64 pp = bradix_pred(c, keys[i - 1]);
      if (pp < max_output) for (u64 q = pp + 1; q <= p; ++q) B[q] = i;
    }
  }
}
// The count of bin b (< max_output) of one candidate, as chi2() sees it (the drained stream's extra item included):
// from the boundaries B of the whole array (single GPU) ...
struct BradixBoundsCounts {
  const u64* B;
  u64 n;
  __device__ __forceinline__ u64 operator()(u64 b, u64 max_output) const {
    u64 lo = B[b], hi = (b + 1 < max_output) ? B[b + 1] : n;
    u64 cnt = hi - lo;
    if (hi == n && lo < n) cnt += 1;                  // repeated final item
    return cnt;
  }
};
// ... or from the merged per-bin counts of a range-partitioned build (the sum over ranks mod 2^32)
struct BradixTableCounts {
  const u32* c;
  __device__ __forceinline__ u64 operator()(u64 b, u64) const { return c[b]; }
};
// The grid of the chi2 reduction: a function of N alone, so that every rank of a range-partitioned build sums the
// same terms in the same tree whatever its GPU, and takes the decision rmi_train takes.
int bradix_chi2_grid(u64 N) {
  u64 blocks = (N + TOP_THREADS - 1) / TOP_THREADS;
  if (blocks > (u64)MAX_PARTIAL_BLOCKS) blocks = MAX_PARTIAL_BLOCKS;
  return blocks < 1 ? 1 : (int)blocks;
}
template <class Counts>
__global__ void __launch_bounds__(TOP_THREADS)
k_bradix_chi2(u64 n, const BuildAux* __restrict__ aux, Counts count_of, double* __restrict__ partials) {
  __shared__ double sm[32];
  u64 max_output = aux->max_scaled_y;
  double expected = __ddiv_rn(__ull2double_rn(n), __ull2double_rn(max_output));
  double s = 0;
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x; b < max_output; b += stride) {
    u64 cnt = count_of(b, max_output);
    double cf = (double)(int)(unsigned)cnt;           // counts are i32 in the reference
    double dl = __dadd_rn(cf, -expected);
    s += __ddiv_rn(__dmul_rn(dl, dl), expected);
  }
  double r = block_sum(s, sm);
  if (threadIdx.x == 0) partials[blockIdx.x] = r;
}
__global__ void __launch_bounds__(TOP_THREADS)
k_bradix_pick(const double* __restrict__ partials, int nblocks, int which, TopModel* top, BuildAux* aux,
              BradixCand* best) {
  __shared__ double sm[32];
  double s = 0;
  for (int b = threadIdx.x; b < nblocks; b += blockDim.x) s += partials[b];
  double score = block_sum(s, sm);
  if (threadIdx.x != 0) return;
  BradixCand c = bradix_candidate(top, aux, which);
  if (c.bits >= 64) return;
  if (which == 0) { aux->best_score = INFINITY; aux->best_valid = 0; }
  if (score < aux->best_score) { aux->best_score = score; aux->best_valid = 1; *best = c; }
}
__global__ void k_bradix_commit(TopModel* top, BuildAux* aux, const BradixCand* best) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (!aux->best_valid) { set_status(aux, ST_NUM_BITS); return; }
  top->ip[0] = best->prefix; top->ip[1] = best->bits; top->ip[2] = best->clamp; top->high = best->high;
}

// bradix over a range-partitioned array: this rank's keys counted per bin, for all four candidates in ONE pass over
// the slab, into counts[which * N + bin] (zero-initialised u32, N > max_output).  Predictions are monotone in the key,
// so a bin's keys form one run; the lane that sees a run start subtracts its local index, the lane that sees it end
// adds the index one past it, and the wrapping u32 sum is the run's length — two atomics per run and candidate,
// whichever thread sees which end.  The rank holding the global last key counts the drained stream's extra item in
// that key's bin.  Summed over the ranks (mod 2^32) these are the counts k_bradix_chi2 takes from B on one GPU.
template <class T>
__global__ void __launch_bounds__(TOP_THREADS)
k_bradix_count(const T* __restrict__ keys, const Shard<T> sh, u64 N, const TopModel* __restrict__ top, BuildAux* aux,
               u32* __restrict__ counts) {
  const u64 max_output = aux->max_scaled_y;
  BradixCand c[4];
#pragma unroll
  for (int w = 0; w < 4; ++w) c[w] = bradix_candidate(top, aux, w);
  const bool aligned = is_aligned16(keys);
  const u64 n = sh.n_local;
  unsigned bad = 0;
  u64 stride = (u64)gridDim.x * blockDim.x * 4;
  for (u64 b = ((u64)blockIdx.x * blockDim.x + threadIdx.x) * 4; b < n; b += stride) {
    T k[4];
    const int cnt = load_keys4(keys, b, n, aligned, k);
    const T kp = b > 0 ? keys[b - 1] : k[0];
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      if (c[w].bits >= 64) continue;               // `for test_bits in bits..min(bits+2, 64)`
      u32* cw = counts + (u64)w * N;
      u64 pp = bradix_pred(c[w], kp);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (e >= cnt) break;
        const u64 i = b + e;
        const u64 p = bradix_pred(c[w], k[e]);
        if (p >= max_output) bad = ST_BRADIX_OOB;
        if (i == 0 || p != pp) {
          if (i > 0 && pp < max_output) atomicAdd(cw + pp, (u32)i);
          if (p < max_output) atomicAdd(cw + p, 0u - (u32)i);
        }
        if (i + 1 == n && p < max_output) atomicAdd(cw + p, (u32)n + (sh.is_last ? 1u : 0u));
        pp = p;
      }
    }
  }
  if (bad) set_status(aux, bad);
}

// histogram (histogram.rs:20-54, utils.rs:55-102): equi-depth pivots + 20-bit radix index.
template <class T>
__global__ void __launch_bounds__(TOP_THREADS)
k_hist_pivots(const T* __restrict__ keys, u64 num_bins, u64 items_per_bin, u64* __restrict__ pivots) {
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x; b < num_bins; b += stride)
    pivots[b] = Key<T>::as_int(keys[b * items_per_bin]);
}
__global__ void __launch_bounds__(TOP_THREADS)
k_hist_radix_index(const u64* __restrict__ pivots, u64 num_bins, u64* __restrict__ ri) {
  const u64 len = 1ull << 20;
  u64 last_radix = num_bins ? (pivots[num_bins - 1] >> 44) : 0;
  u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r <= len; r += stride) {
    u64 v;
    if (r == 0) v = 0;
    else if (r == len || r > last_radix) v = num_bins;
    else {  // first pivot whose radix is >= r
      u64 lo = 0, hi = num_bins;
      while (lo < hi) { u64 mid = lo + ((hi - lo) >> 1); if ((pivots[mid] >> 44) >= r) hi = mid; else lo = mid + 1; }
      v = lo;
    }
    ri[r] = v;
  }
}

int grid_for(u64 n, int num_sms) {
  u64 blocks = (n + TOP_THREADS - 1) / TOP_THREADS;
  u64 cap = (u64)num_sms * 8;
  if (cap > (u64)MAX_PARTIAL_BLOCKS) cap = MAX_PARTIAL_BLOCKS;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

}  // namespace

void hist_radix_index(const Launch& L, const u64* d_pivots, u64 num_bins, u64* d_radix_index) {
  k_hist_radix_index<<<grid_for((1ull << 20) + 1, L.num_sms), TOP_THREADS, 0, L.stream>>>(d_pivots, num_bins, d_radix_index);
  count_launch();
}

template <class T>
void shard_bradix_count(const Launch& L, const T* keys, const Shard<T>& sh, u64 N, const TopModel* d_top, BuildAux* d_aux,
                        u32* d_counts) {
  cudaMemsetAsync(d_counts, 0, sizeof(u32) * 4 * N, L.stream);
  if (sh.n_local == 0) return;
  k_bradix_count<T><<<grid_for((sh.n_local + 3) / 4, L.num_sms), TOP_THREADS, 0, L.stream>>>(keys, sh, N, d_top, d_aux, d_counts);
  count_launch();
}

void shard_bradix_decide(const Launch& L, u64 n, u64 N, const u32* d_counts, void* scratch, TopModel* d_top,
                         BuildAux* d_aux) {
  double* partials = (double*)scratch;
  BradixCand* best = (BradixCand*)(partials + MAX_PARTIAL_BLOCKS);
  const int gb = bradix_chi2_grid(N);
  for (int which = 0; which < 4; ++which) {
    k_bradix_chi2<<<gb, TOP_THREADS, 0, L.stream>>>(n, d_aux, BradixTableCounts{d_counts + (u64)which * N}, partials);
    count_launch();
    k_bradix_pick<<<1, TOP_THREADS, 0, L.stream>>>(partials, gb, which, d_top, d_aux, best);
    count_launch();
  }
  k_bradix_commit<<<1, 32, 0, L.stream>>>(d_top, d_aux, best);
  count_launch();
}
size_t shard_bradix_scratch_bytes() { return (size_t)MAX_PARTIAL_BLOCKS * sizeof(double) + sizeof(BradixCand); }

size_t top_scratch_bytes(u64 num_leaves) {
  // partials (5 doubles per block) + candidates + state + bradix boundaries (N+2 u64) + best cand
  return (size_t)MAX_PARTIAL_BLOCKS * 5 * sizeof(double) + 64 * sizeof(double) + (size_t)(num_leaves + 2) * sizeof(u64) + 256;
}

void histogram_bins(u64 n, u64 num_leaves, u64* num_bins, u64* items_per_bin) {
  // histogram.rs:23-27 with the scale of two_layer.rs:109; pure host scalars
  double sf = (double)num_leaves / (double)n;
  bool use_sf = std::fabs(sf - 1.0) > DBL_EPSILON;
  u64 last_off = n ? n - 1 : 0;
  *num_bins = use_sf ? (u64)((double)last_off * sf) : last_off;
  *items_per_bin = *num_bins ? n / *num_bins : 0;
}

template <class T>
unsigned fit_top_model(const Launch& L, const T* keys, u64 n, int kind, int table_bits, u64 num_leaves, bool exact,
                       TopModel* d_top, BuildAux* d_aux, void* scratch, u32* d_table32, u64* d_pivots,
                       u64* d_radix_index, T* d_sample) {
  cudaStream_t st = L.stream;
  // two_layer.rs:109: scale = N / n, applied per models/mod.rs:238-250
  double sf = (double)num_leaves / (double)n;
  int use_sf = std::fabs(sf - 1.0) > DBL_EPSILON ? 1 : 0;
  double* partials = (double*)scratch;
  double* cand = partials + (size_t)MAX_PARTIAL_BLOCKS * 5;
  double* state = cand + 32;
  u64* B = (u64*)(state + 32);
  BradixCand* best = (BradixCand*)(B + num_leaves + 2);
  int g = grid_for(n, L.num_sms);

  switch (kind) {
    case M_LINEAR:
    case M_ROBUST_LINEAR:
    case M_LOGLINEAR: {
      u64 i0 = 0, i1 = n;
      int repeat = 1;
      if (kind == M_ROBUST_LINEAR) {   // linear.rs:239-256
        if (n == 0) { i0 = i1 = 0; repeat = 0; }
        else {
          u64 bnd = (u64)((double)n * 0.0001);
          if (bnd < 1) bnd = 1;
          if (!(bnd * 2 + 1 < n)) return ST_ROBUST_TOO_SMALL;
          i0 = bnd; i1 = n - bnd; repeat = 0;
        }
      }
      if (kind == M_LOGLINEAR) {
        if (exact) { k_slr_exact<T, 1><<<1, 32, 0, st>>>(keys, i0, i1, repeat, sf, use_sf, d_top, d_aux); count_launch(); }
        else {
          int gg = i1 > i0 ? grid_for((i1 - i0 + 3) / 4 + 1, L.num_sms) : 1;
          if (i1 > i0) { k_slr_partial<T, 1><<<gg, TOP_THREADS, 0, st>>>(keys, n, i0, i1, sf, use_sf, partials, nullptr); count_launch(); }
          k_slr_finish<T, 1><<<1, TOP_THREADS, 0, st>>>(keys, i0, i1, repeat, sf, use_sf, partials, i1 > i0 ? gg : 0, d_top, d_aux);
          count_launch();
        }
      } else if (exact) {
        k_slr_exact<T, 0><<<1, 32, 0, st>>>(keys, i0, i1, repeat, sf, use_sf, d_top, d_aux);
        count_launch();
      } else {
        int gg = i1 > i0 ? grid_for((i1 - i0 + 3) / 4 + 1, L.num_sms) : 1;
        if (i1 > i0) {
          k_slr_partial<T, 0><<<gg, TOP_THREADS, 0, st>>>(keys, n, i0, i1, sf, use_sf, partials, d_sample);
          count_launch();
        }
        k_slr_finish<T, 0><<<1, TOP_THREADS, 0, st>>>(keys, i0, i1, repeat, sf, use_sf, partials, i1 > i0 ? gg : 0, d_top, d_aux);
        count_launch();
      }
      break;
    }
    case M_LINEAR_SPLINE:
      k_spline_prepare<T><<<1, 32, 0, st>>>(keys, n, sf, use_sf, 0, cand, d_top, d_aux);
      count_launch();
      break;
    case M_CUBIC:
      k_spline_prepare<T><<<1, 32, 0, st>>>(keys, n, sf, use_sf, 1, cand, d_top, d_aux);
      count_launch();
      if (n > 0) { k_cubic_l1_partial<T><<<g, TOP_THREADS, 0, st>>>(keys, n, sf, use_sf, cand, partials); count_launch(); }
      k_cubic_finish<T><<<1, TOP_THREADS, 0, st>>>(keys, n, sf, use_sf, cand, partials, n > 0 ? g : 0, d_top);
      count_launch();
      break;
    case M_NORMAL:
    case M_LOGNORMAL:
      if (kind == M_NORMAL && exact) {
        k_normal_exact<T><<<1, 32, 0, st>>>(keys, n, sf, use_sf, d_top);
        count_launch();
      } else if (kind == M_NORMAL) {
        if (n > 0) { k_normal_partial<T, 0, 0><<<g, TOP_THREADS, 0, st>>>(keys, n, state, partials); count_launch(); }
        k_normal_finish<T, 0, 0><<<1, TOP_THREADS, 0, st>>>(keys, n, sf, use_sf, partials, n > 0 ? g : 0, state, d_top); count_launch();
        if (n > 0) { k_normal_partial<T, 0, 1><<<g, TOP_THREADS, 0, st>>>(keys, n, state, partials); count_launch(); }
        k_normal_finish<T, 0, 1><<<1, TOP_THREADS, 0, st>>>(keys, n, sf, use_sf, partials, n > 0 ? g : 0, state, d_top); count_launch();
      } else {
        if (n > 0) { k_normal_partial<T, 1, 0><<<g, TOP_THREADS, 0, st>>>(keys, n, state, partials); count_launch(); }
        k_normal_finish<T, 1, 0><<<1, TOP_THREADS, 0, st>>>(keys, n, sf, use_sf, partials, n > 0 ? g : 0, state, d_top); count_launch();
        if (n > 0) { k_normal_partial<T, 1, 1><<<g, TOP_THREADS, 0, st>>>(keys, n, state, partials); count_launch(); }
        k_normal_finish<T, 1, 1><<<1, TOP_THREADS, 0, st>>>(keys, n, sf, use_sf, partials, n > 0 ? g : 0, state, d_top); count_launch();
      }
      break;
    case M_RADIX:
      k_radix_scalars<T><<<1, 32, 0, st>>>(keys, n, sf, use_sf, kind, d_top, d_aux);
      count_launch();
      break;
    case M_RADIX_TABLE: {
      k_radix_scalars<T><<<1, 32, 0, st>>>(keys, n, sf, use_sf, kind, d_top, d_aux);
      count_launch();
      u64 len = 1ull << table_bits;
      k_table_init<<<grid_for(len, L.num_sms), TOP_THREADS, 0, st>>>(d_table32, len);
      count_launch();
      if (n > 0) { k_table_fill<T><<<g, TOP_THREADS, 0, st>>>(keys, n, sf, use_sf, d_top, table_bits, d_table32, d_aux); count_launch(); }
      break;
    }
    case M_BRADIX: {
      k_radix_scalars<T><<<1, 32, 0, st>>>(keys, n, sf, use_sf, kind, d_top, d_aux);
      count_launch();
      if (n == 0) break;
      for (int which = 0; which < 4; ++which) {
        k_fill_u64<<<grid_for(num_leaves + 2, L.num_sms), TOP_THREADS, 0, st>>>(B, num_leaves + 2, n); count_launch();
        k_bradix_bounds<T><<<g, TOP_THREADS, 0, st>>>(keys, n, d_top, d_aux, which, B); count_launch();
        int gb = bradix_chi2_grid(num_leaves);
        k_bradix_chi2<<<gb, TOP_THREADS, 0, st>>>(n, d_aux, BradixBoundsCounts{B, n}, partials); count_launch();
        k_bradix_pick<<<1, TOP_THREADS, 0, st>>>(partials, gb, which, d_top, d_aux, best); count_launch();
      }
      k_bradix_commit<<<1, 32, 0, st>>>(d_top, d_aux, best);
      count_launch();
      break;
    }
    case M_HISTOGRAM: {
      if (n == 0) break;
      u64 num_bins, items_per_bin;
      histogram_bins(n, num_leaves, &num_bins, &items_per_bin);
      if (num_bins == 0 || items_per_bin < 1) return ST_HIST_BINS;
      k_hist_pivots<T><<<grid_for(num_bins, L.num_sms), TOP_THREADS, 0, st>>>(keys, num_bins, items_per_bin, d_pivots);
      count_launch();
      k_hist_radix_index<<<grid_for((1ull << 20) + 1, L.num_sms), TOP_THREADS, 0, st>>>(d_pivots, num_bins, d_radix_index);
      count_launch();
      break;
    }
    default:
      break;
  }
  return 0;
}

template void shard_bradix_count<u64>(const Launch&, const u64*, const Shard<u64>&, u64, const TopModel*, BuildAux*, u32*);
template void shard_bradix_count<u32>(const Launch&, const u32*, const Shard<u32>&, u64, const TopModel*, BuildAux*, u32*);
template void shard_bradix_count<double>(const Launch&, const double*, const Shard<double>&, u64, const TopModel*, BuildAux*, u32*);
template unsigned fit_top_model<u64>(const Launch&, const u64*, u64, int, int, u64, bool, TopModel*, BuildAux*, void*, u32*, u64*, u64*, u64*);
template unsigned fit_top_model<u32>(const Launch&, const u32*, u64, int, int, u64, bool, TopModel*, BuildAux*, void*, u32*, u64*, u64*, u32*);
template unsigned fit_top_model<double>(const Launch&, const double*, u64, int, int, u64, bool, TopModel*, BuildAux*, void*, u32*, u64*, u64*, double*);

}  // namespace rmi
