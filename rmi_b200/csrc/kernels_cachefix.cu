// kernels_cachefix.cu — the `--bounded` cache-fix spline (reference cache_fix.rs:106-150, restated on the host in
// host/cache_fix.hpp) fitted on the device, knot for knot equal to the host scan.  DESIGN.md section 12.
//
// The point stream p_0 .. p_{m-1} (DedupIter + minus_epsilon, cache_fix.hpp:83-91) is never materialised: point
// (key index i, sub) has id pid = 2i + sub, sub 0 = (keys[i] - 1, i), present iff i starts a run of equal keys and
// keys[i] - 1 != (i ? keys[i-1] : 0); sub 1 = (keys[i], i), present iff i starts a run.  pids increase along the
// stream, and so do the points' x values, so a knot is identified by its pid.
//
// add_point (cache_fix.rs:62-88) makes the next knot a pure function of the current one: after a knot s the spline
// is s -> p_{s+1}; each later p_k proposes s -> p_k, checked against p_{s+1} .. p_{k-1}; the first failing proposal
// makes p_{k-1} the next knot (next_knot below).  The first segment also holds p_0 itself, which always passes
// (t = 0 gives y0 exactly).  So the knots are p_0, next(p_0), next(next(p_0)), ... and finish()'s p_{m-1}, and two
// chains that share a knot are identical from there on.  The scan exploits that:
//   1. speculate  one thread per chunk of CACHEFIX_CHUNK key indices runs the chain from the chunk's first point as
//                 if it were a knot: its knot count inside the chunk, its first CACHEFIX_TARGETS knots (targets) and
//                 its exit (first knot at or past the chunk's end).  A segment still open CACHEFIX_CHUNK key indices
//                 past the chunk's end stops it (the chunk is "open").
//   2. stitch     one thread per chunk walks the true chain from the previous chunk's exit until it lands on one of
//                 the chunk's targets (from there the speculative chain is the true one) or leaves the chunk.
//   3. resolve    one block checks, in parallel, which stitches started from a true knot; from the first chunk whose
//                 did not, it walks the true chain itself (every thread of the block checks a share of each
//                 proposal's points) until the walk lands on a later chunk's speculative chain again; then it
//                 scans the per-chunk knot counts into output offsets.
//   4. emit       one thread per chunk re-walks the chain from the chunk's first true knot and writes its knots.
// All arithmetic goes through cache_fix_interp (spline.cuh), the host's expression with explicitly rounded
// intrinsics; the library is compiled with -fmad=false.
#include "kernels.h"
#include "spline.cuh"

namespace rmi {

namespace {

constexpr u64 PID_END = ~0ull;         // no further knot: the last segment stays open to the end of the data
constexpr u64 PID_OPEN = ~0ull - 1;    // a speculative walk gave up inside an open segment
constexpr int CF_THREADS = 128;
constexpr int CF_RESOLVE_THREADS = 1024;

struct Pt { u64 pid, x, y; };

__device__ __forceinline__ Pt pt_of(const u64* keys, u64 pid) {
  const u64 i = pid >> 1, k = keys[i];
  return Pt{pid, (pid & 1) ? k : k - 1, i};
}

// First index > i whose key differs from keys[i] (n if none): galloping, so a long run of equal keys costs log steps.
__device__ __forceinline__ u64 run_end(const u64* keys, u64 n, u64 i) {
  const u64 v = keys[i];
  if (i + 1 >= n || keys[i + 1] != v) return i + 1;
  u64 lo = i + 1, step = 1;
  while (lo + step < n && keys[lo + step] == v) { lo += step; step <<= 1; }
  u64 hi = lo + step < n ? lo + step : n;   // keys[lo] == v; hi == n or keys[hi] != v
  while (hi - lo > 1) {
    const u64 m = lo + (hi - lo) / 2;
    if (keys[m] == v) lo = m; else hi = m;
  }
  return hi;
}

// First index of the run of equal keys that holds index i.
__device__ __forceinline__ u64 run_start(const u64* keys, u64 i) {
  const u64 v = keys[i];
  if (i == 0 || keys[i - 1] != v) return i;
  u64 hi = i, step = 1;   // keys[hi] == v
  while (step <= hi && keys[hi - step] == v) { hi -= step; step <<= 1; }
  if (step > hi && keys[0] == v) return 0;
  u64 lo = step > hi ? 0 : hi - step;   // keys[lo] != v
  while (hi - lo > 1) {
    const u64 m = lo + (hi - lo) / 2;
    if (keys[m] == v) hi = m; else lo = m;
  }
  return hi;
}

// The first point of run start i (prev: the key before it, 0 for i == 0).
__device__ __forceinline__ Pt run_first_point(u64 i, u64 k, u64 prev) {
  return k - 1 != prev ? Pt{2 * i, k - 1, i} : Pt{2 * i + 1, k, i};
}

// The first point whose key index lies in [i, i_end); false if there is none.
__device__ __forceinline__ bool first_point_at(const u64* keys, u64 n, u64 i, u64 i_end, Pt& p) {
  if (i > 0 && keys[i] == keys[i - 1]) i = run_end(keys, n, i);
  if (i >= i_end) return false;
  p = run_first_point(i, keys[i], i ? keys[i - 1] : 0);
  return true;
}

// The point after p in the stream; false at the end of the data.
__device__ __forceinline__ bool next_point(const u64* keys, u64 n, const Pt& p, Pt& q) {
  const u64 i = p.pid >> 1;
  if (!(p.pid & 1)) { q = Pt{p.pid + 1, p.x + 1, i}; return true; }
  const u64 j = run_end(keys, n, i);
  if (j >= n) return false;
  q = run_first_point(j, keys[j], p.x);   // keys[j - 1] == keys[i] == p.x
  return true;
}

// Does the proposal s -> k put point p outside its line?  (SplineFit::check, cache_fix.rs:96-103)
__device__ __forceinline__ bool misses_line(const Pt& s, const Pt& k, u64 px, u64 py, u64 line) {
  return cache_fix_interp(px, s.x, s.y, k.x, k.y) / line != py / line;
}

// The knot after knot s.  Returns PID_END when the segment stays open to the last point, PID_OPEN when a proposal
// reaches pid `limit` first (speculation and stitching only; the true walks pass PID_END).  One thread.
__device__ Pt next_knot(const u64* keys, u64 n, u64 line, const Pt& s, u64 limit, u64& evals) {
  Pt a, prev, k;
  if (!next_point(keys, n, s, a)) return Pt{PID_END, 0, 0};
  prev = a;
  for (;;) {
    if (!next_point(keys, n, prev, k)) return Pt{PID_END, 0, 0};
    if (k.pid >= limit) return Pt{PID_OPEN, 0, 0};
    Pt j = a;
    for (;;) {
      ++evals;
      if (misses_line(s, k, j.x, j.y, line)) return prev;
      if (j.pid == prev.pid) break;
      next_point(keys, n, j, j);
    }
    prev = k;
  }
}

struct ChunkRange { u64 i0, i1, end_pid, limit; };
__device__ __forceinline__ ChunkRange chunk_range(u64 c, u64 chunk, u64 n) {
  ChunkRange r;
  r.i0 = c * chunk;
  r.i1 = r.i0 + chunk < n ? r.i0 + chunk : n;
  r.end_pid = 2 * r.i1;
  r.limit = r.i1 + chunk < n ? 2 * (r.i1 + chunk) : PID_END;
  return r;
}

// Adds every thread's v to *stat (all threads of the warp must call it).
__device__ __forceinline__ void add_stat(u64* stat, u64 v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0 && v) atomicAdd((unsigned long long*)stat, (unsigned long long)v);
}

// Number of points in the stream (statistics only).
__global__ void __launch_bounds__(CF_THREADS) k_cf_points(const u64* __restrict__ keys, u64 n, u64* stats) {
  u64 pts = 0;
  for (u64 i = (u64)blockIdx.x * CF_THREADS + threadIdx.x; i < n; i += (u64)gridDim.x * CF_THREADS) {
    const u64 k = keys[i], prev = i ? keys[i - 1] : 0;
    if (i == 0 || k != prev) pts += (k - 1 != prev) ? 2 : 1;
  }
  add_stat(stats + CF_STAT_POINTS, pts);
}

__global__ void __launch_bounds__(CF_THREADS)
k_cf_speculate(const u64* __restrict__ keys, u64 n, u64 line, u64 chunk, u64 nch, CacheFixScratch s) {
  const u64 c = (u64)blockIdx.x * CF_THREADS + threadIdx.x;
  u64 evals = 0;
  if (c < nch) {
    const ChunkRange r = chunk_range(c, chunk, n);
    u64* T = s.targets + c * CACHEFIX_TARGETS;
    Pt p;
    u64 cnt = 0, exit_pid = PID_OPEN;   // an empty chunk (inside a run of equal keys) has no chain to join
    if (first_point_at(keys, n, r.i0, r.i1, p)) {
      T[0] = p.pid;
      cnt = 1;
      for (;;) {
        p = next_knot(keys, n, line, p, r.limit, evals);
        if (p.pid >= r.end_pid) { exit_pid = p.pid; break; }   // PID_OPEN and PID_END included
        if (cnt < CACHEFIX_TARGETS) T[cnt] = p.pid;
        ++cnt;
      }
    }
    s.spec_count[c] = cnt;
    s.spec_exit[c] = exit_pid;
  }
  add_stat(s.stats + CF_STAT_EVALS, evals);
}

__global__ void __launch_bounds__(CF_THREADS)
k_cf_stitch(const u64* __restrict__ keys, u64 n, u64 line, u64 chunk, u64 nch, CacheFixScratch s) {
  const u64 c = (u64)blockIdx.x * CF_THREADS + threadIdx.x;
  u64 evals = 0, segs = 0;
  if (c < nch) {
    const ChunkRange r = chunk_range(c, chunk, n);
    u64 E;
    if (c == 0) { Pt p0; first_point_at(keys, n, 0, n, p0); E = p0.pid; }
    else E = s.spec_exit[c - 1];
    u32 ok = 0;
    u64 cnt = 0, exit_pid = PID_OPEN;
    if (E != PID_OPEN && E >= r.end_pid) {       // the segment open at the chunk's start spans the whole chunk
      ok = 1; exit_pid = E;
    } else if (E != PID_OPEN) {
      const u64 scnt = s.spec_count[c], sexit = s.spec_exit[c];
      const u64 nt = scnt < CACHEFIX_TARGETS ? scnt : CACHEFIX_TARGETS;
      const u64* T = s.targets + c * CACHEFIX_TARGETS;
      Pt p = pt_of(keys, E);
      for (;;) {
        if (sexit != PID_OPEN) {
          u64 t = 0;
          while (t < nt && T[t] < p.pid) ++t;
          if (t < nt && T[t] == p.pid) { ok = 1; cnt += scnt - t; exit_pid = sexit; break; }
          if (t == nt && scnt > nt) break;      // past the last target: the chains can no longer be seen to meet
        }
        ++cnt;
        ++segs;
        p = next_knot(keys, n, line, p, r.limit, evals);
        if (p.pid == PID_OPEN) break;
        if (p.pid >= r.end_pid) { ok = 1; exit_pid = p.pid; break; }
      }
    }
    s.entry[c] = E;
    s.count[c] = ok ? cnt : 0;
    s.stitch_exit[c] = exit_pid;
    s.stitch_ok[c] = ok;
  }
  add_stat(s.stats + CF_STAT_EVALS, evals);
  add_stat(s.stats + CF_STAT_STITCH_SEGMENTS, segs);
}

// The knot after knot s, found by the whole block: each proposal's points are split over the threads, which vote.
// Every thread follows the same cursor (the loads are broadcasts).  Returns PID_END at the end of the data.
__device__ u64 block_next_knot(const u64* keys, u64 n, u64 line, u64 s_pid, u64& evals, u64& walked) {
  const Pt s = pt_of(keys, s_pid);
  Pt a, prev, k;
  if (!next_point(keys, n, s, a)) return PID_END;
  prev = a;
  for (;;) {
    if (!next_point(keys, n, prev, k)) return PID_END;
    ++walked;
    bool miss = false;
    for (u64 i = a.y + threadIdx.x; i <= prev.y; i += CF_RESOLVE_THREADS) {
      const u64 key = keys[i], pk = i ? keys[i - 1] : 0;
      if (i > 0 && key == pk) continue;
      if (key - 1 != pk && 2 * i >= a.pid && 2 * i <= prev.pid) { ++evals; miss |= misses_line(s, k, key - 1, i, line); }
      if (2 * i + 1 >= a.pid && 2 * i + 1 <= prev.pid) { ++evals; miss |= misses_line(s, k, key, i, line); }
    }
    if (__syncthreads_or(miss)) return prev.pid;
    prev = k;
  }
}

__global__ void __launch_bounds__(CF_RESOLVE_THREADS)
k_cf_resolve(const u64* __restrict__ keys, u64 n, u64 line, u64 chunk, u64 nch, CacheFixScratch s) {
  __shared__ u64 s_first;
  __shared__ u64 s_part[CF_RESOLVE_THREADS];
  const unsigned tid = threadIdx.x;
  u64 evals = 0, walked = 0;
  u64 pos = 0;
  while (pos < nch) {
    // the first chunk whose stitched result cannot be trusted: its stitch failed, or it started from an exit the
    // previous chunk's stitch did not confirm
    if (tid == 0) s_first = nch;
    __syncthreads();
    for (u64 base = pos; base < nch; base += CF_RESOLVE_THREADS) {
      const u64 c = base + tid;
      const bool bad = c < nch && !(s.stitch_ok[c] && (c == 0 || s.stitch_exit[c - 1] == s.spec_exit[c - 1]));
      if (bad) atomicMin((unsigned long long*)&s_first, (unsigned long long)c);
      if (__syncthreads_or(bad)) break;
    }
    const u64 f = s_first;
    __syncthreads();
    if (f >= nch) break;
    // the sequential fallback: walk the true chain from the last true knot until it joins a later chunk's chain
    u64 E = f == 0 ? s.entry[0] : s.stitch_exit[f - 1];
    u64 c = f;
    for (;;) {
      const ChunkRange r = chunk_range(c, chunk, n);
      const u64 scnt = s.spec_count[c], sexit = s.spec_exit[c];
      const u64 nt = scnt < CACHEFIX_TARGETS ? scnt : CACHEFIX_TARGETS;
      const u64* T = s.targets + c * CACHEFIX_TARGETS;
      const u64 entry = E;
      u64 cnt = 0;
      while (E < r.end_pid) {
        if (sexit != PID_OPEN) {
          u64 t = 0;
          while (t < nt && T[t] < E) ++t;
          if (t < nt && T[t] == E) { cnt += scnt - t; E = sexit; break; }
        }
        ++cnt;
        E = block_next_knot(keys, n, line, E, evals, walked);
      }
      if (tid == 0) { s.entry[c] = entry; s.count[c] = cnt; }
      ++c;
      if (c >= nch) { pos = nch; break; }
      if (E == s.spec_exit[c - 1] && s.stitch_ok[c]) { pos = c + 1; break; }   // chunk c's stitch started from E
    }
    __syncthreads();
  }
  // exclusive scan of the knot counts -> output offsets; total = offsets[nch]
  __syncthreads();
  const u64 per = (nch + CF_RESOLVE_THREADS - 1) / CF_RESOLVE_THREADS;
  const u64 b = tid * per < nch ? tid * per : nch, e = b + per < nch ? b + per : nch;
  u64 sum = 0;
  for (u64 c = b; c < e; ++c) sum += s.count[c];
  s_part[tid] = sum;
  __syncthreads();
  for (unsigned o = 1; o < CF_RESOLVE_THREADS; o <<= 1) {
    const u64 v = tid >= o ? s_part[tid - o] : 0;
    __syncthreads();
    s_part[tid] += v;
    __syncthreads();
  }
  u64 off = s_part[tid] - sum;
  for (u64 c = b; c < e; ++c) { s.offsets[c] = off; off += s.count[c]; }
  if (tid == CF_RESOLVE_THREADS - 1) s.offsets[nch] = s_part[tid];
  if (tid == 0) {
    s.stats[CF_STAT_FALLBACK_POINTS] += walked;
    const u64 last = run_start(keys, n - 1);
    s.last_knot[0] = keys[n - 1];
    s.last_knot[1] = last;
  }
  add_stat(s.stats + CF_STAT_EVALS, evals);
}

__global__ void __launch_bounds__(CF_THREADS)
k_cf_emit(const u64* __restrict__ keys, u64 n, u64 line, u64 chunk, u64 nch, CacheFixScratch s, ulonglong2* out) {
  const u64 c = (u64)blockIdx.x * CF_THREADS + threadIdx.x;
  u64 evals = 0;
  if (c < nch) {
    const u64 cnt = s.count[c];
    if (cnt) {
      ulonglong2* o = out + s.offsets[c];
      Pt p = pt_of(keys, s.entry[c]);
      o[0] = make_ulonglong2(p.x, p.y);
      for (u64 j = 1; j < cnt; ++j) {
        p = next_knot(keys, n, line, p, PID_END, evals);
        o[j] = make_ulonglong2(p.x, p.y);
      }
    }
    if (c == 0) out[s.offsets[nch]] = make_ulonglong2(s.last_knot[0], s.last_knot[1]);   // finish() (cache_fix.rs:91-93)
  }
  add_stat(s.stats + CF_STAT_EVALS, evals);
}

unsigned blocks_for(u64 items) { return (unsigned)((items + CF_THREADS - 1) / CF_THREADS); }

}  // namespace

void cache_fix_scan(const Launch& L, const u64* keys, u64 n, u64 line, u64 chunk, const CacheFixScratch& s) {
  const u64 nch = (n + chunk - 1) / chunk;
  u64 pb = (n + CF_THREADS - 1) / CF_THREADS;
  if (pb > (u64)L.num_sms * 16) pb = (u64)L.num_sms * 16;
  k_cf_points<<<(unsigned)pb, CF_THREADS, 0, L.stream>>>(keys, n, s.stats);
  count_launch();
  k_cf_speculate<<<blocks_for(nch), CF_THREADS, 0, L.stream>>>(keys, n, line, chunk, nch, s);
  count_launch();
  k_cf_stitch<<<blocks_for(nch), CF_THREADS, 0, L.stream>>>(keys, n, line, chunk, nch, s);
  count_launch();
  k_cf_resolve<<<1, CF_RESOLVE_THREADS, 0, L.stream>>>(keys, n, line, chunk, nch, s);
  count_launch();
}

void cache_fix_emit(const Launch& L, const u64* keys, u64 n, u64 line, u64 chunk, const CacheFixScratch& s,
                    void* d_out) {
  const u64 nch = (n + chunk - 1) / chunk;
  k_cf_emit<<<blocks_for(nch), CF_THREADS, 0, L.stream>>>(keys, n, line, chunk, nch, s, (ulonglong2*)d_out);
  count_launch();
}

}  // namespace rmi
