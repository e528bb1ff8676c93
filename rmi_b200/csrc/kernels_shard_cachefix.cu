// kernels_shard_cachefix.cu — the cache-fix scan of kernels_cachefix.cu (DESIGN.md section 12) over one rank's slab of
// range-partitioned keys (DESIGN.md section 16).  The stream and its points are section 12's with GLOBAL indices: point
// (global key index g, sub) has pid 2g + sub.  A rank reads its own keys [0, n_local) and behind them the halo, the
// keys of the following ranks up to n_avail; the key before its local index 0 is the last key of the previous
// non-empty rank (0 before the first key), so a run of equal keys that began on an earlier rank has no point here.
//
// The passes are section 12's speculate / stitch / resolve / emit over the slab's chunks, with one change: chunk 0's
// stitch starts from a given entry pid E instead of the data's first point.  Speculation and the other chunks'
// stitches do not depend on E, so a scan with a new entry re-runs only chunk 0's stitch and the resolve, which starts
// from the stitched values saved by the first scan.  The resolve reports the rank's exit: the first knot of the chain
// from E at or past the slab's end (PID_END when the last segment stays open to the end of the data).
//
// A walk that needs a key past the halo, where the halo does not end the data, is PID_HALO: speculation and the
// stitch give up there (as at PID_OPEN); the resolve, which walks the true chain, stops and reports "halo too small"
// with the global index of the first key it could not read.  Exact or refused, never a wrong knot.
#include "kernels.h"
#include "spline.cuh"

namespace rmi {

namespace {

constexpr u64 PID_END = ~0ull;         // no further knot: the last segment stays open to the end of the data
constexpr u64 PID_OPEN = ~0ull - 1;    // a speculative walk gave up inside an open segment
constexpr u64 PID_HALO = ~0ull - 2;    // a walk needs a key past the halo
constexpr int SCF_THREADS = 128;
constexpr int SCF_RESOLVE_THREADS = 512;
// Under __launch_bounds__ ptxas holds these kernels to 64 registers and spills around the division's slow path; 96
// registers hold every walk without spills (DESIGN.md section 16), and 96 x 512 fits the resolve's one block.
constexpr int SCF_MAX_REGS = 96;

enum NextPoint { NP_OK = 0, NP_END = 1, NP_HALO = 2 };

struct Pt { u64 pid, x, y; };

__device__ __forceinline__ u64 key_before(const CacheFixSlab& S, u64 i) { return i ? S.keys[i - 1] : S.prev_key; }

// Does local index i start a run of equal keys?  (Global index 0 always does.)
__device__ __forceinline__ bool starts_run(const CacheFixSlab& S, u64 i) {
  return i ? S.keys[i] != S.keys[i - 1] : (!S.has_prev || S.keys[0] != S.prev_key);
}

__device__ __forceinline__ Pt pt_of(const CacheFixSlab& S, u64 pid) {
  const u64 g = pid >> 1, k = S.keys[g - S.base];
  return Pt{pid, (pid & 1) ? k : k - 1, g};
}

// First local index > i whose key differs from keys[i], n_avail if none is readable: galloping, so a long run of
// equal keys costs log steps.
__device__ __forceinline__ u64 run_end(const CacheFixSlab& S, u64 i) {
  const u64* keys = S.keys;
  const u64 n = S.n_avail, v = keys[i];
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

// The first point of the run that starts at local index i (prev: the key before it).
__device__ __forceinline__ Pt run_first_point(const CacheFixSlab& S, u64 i, u64 k, u64 prev) {
  const u64 g = S.base + i;
  return k - 1 != prev ? Pt{2 * g, k - 1, g} : Pt{2 * g + 1, k, g};
}

// The first point whose local key index lies in [i, i_end); false if there is none (i_end <= n_local).
__device__ __forceinline__ bool first_point_at(const CacheFixSlab& S, u64 i, u64 i_end, Pt& p) {
  if (!starts_run(S, i)) i = run_end(S, i);
  if (i >= i_end) return false;
  p = run_first_point(S, i, S.keys[i], key_before(S, i));
  return true;
}

// The point after p in the stream.
__device__ __forceinline__ int next_point(const CacheFixSlab& S, const Pt& p, Pt& q) {
  const u64 g = p.pid >> 1;
  if (!(p.pid & 1)) { q = Pt{p.pid + 1, p.x + 1, g}; return NP_OK; }
  const u64 j = run_end(S, g - S.base);
  if (j >= S.n_avail) return S.at_end ? NP_END : NP_HALO;
  q = run_first_point(S, j, S.keys[j], p.x);   // keys[j - 1] == p.x
  return NP_OK;
}

__device__ __forceinline__ u64 stop_pid(int r) { return r == NP_END ? PID_END : PID_HALO; }

// Does the proposal s -> k put point p outside its line?  (SplineFit::check, cache_fix.rs:96-103)
__device__ __forceinline__ bool misses_line(const Pt& s, const Pt& k, u64 px, u64 py, u64 line) {
  return cache_fix_interp(px, s.x, s.y, k.x, k.y) / line != py / line;
}

// The knot after knot s (kernels_cachefix.cu's next_knot): PID_END at the end of the data, PID_OPEN when a proposal
// reaches pid `limit` first, PID_HALO when a point past the halo is needed.  One thread.
__device__ __forceinline__ Pt next_knot(const CacheFixSlab& S, u64 line, const Pt& s, u64 limit) {
  Pt a, prev, k;
  int r = next_point(S, s, a);
  if (r != NP_OK) return Pt{stop_pid(r), 0, 0};
  prev = a;
  for (;;) {
    r = next_point(S, prev, k);
    if (r != NP_OK) return Pt{stop_pid(r), 0, 0};
    if (k.pid >= limit) return Pt{PID_OPEN, 0, 0};
    Pt j = a;
    for (;;) {
      if (misses_line(s, k, j.x, j.y, line)) return prev;
      if (j.pid == prev.pid) break;
      Pt q;
      next_point(S, j, q);   // j < prev: already read
      j = q;
    }
    prev = k;
  }
}

struct ChunkRange { u64 i0, i1, end_pid, limit; };
__device__ __forceinline__ ChunkRange chunk_range(const CacheFixSlab& S, u64 c, u64 chunk) {
  const u64 n = S.n_local;
  ChunkRange r;
  r.i0 = c * chunk;
  r.i1 = r.i0 + chunk < n ? r.i0 + chunk : n;
  r.end_pid = 2 * (S.base + r.i1);
  r.limit = r.i1 + chunk < n ? 2 * (S.base + r.i1 + chunk) : PID_END;
  return r;
}

__global__ void __maxnreg__(SCF_MAX_REGS)
k_scf_speculate(const CacheFixSlab S, u64 line, u64 chunk, u64 nch, ShardCacheFixScratch s) {
  const u64 c = (u64)blockIdx.x * SCF_THREADS + threadIdx.x;
  if (c >= nch) return;
  const ChunkRange r = chunk_range(S, c, chunk);
  u64* T = s.targets + c * CACHEFIX_TARGETS;
  Pt p;
  u64 cnt = 0, exit_pid = PID_OPEN;   // an empty chunk (inside a run of equal keys) has no chain to join
  if (first_point_at(S, r.i0, r.i1, p)) {
    T[0] = p.pid;
    cnt = 1;
    for (;;) {
      p = next_knot(S, line, p, r.limit);
      if (p.pid == PID_HALO) break;                          // speculation past the halo: open
      if (p.pid >= r.end_pid) { exit_pid = p.pid; break; }   // PID_OPEN and PID_END included
      if (cnt < CACHEFIX_TARGETS) T[cnt] = p.pid;
      ++cnt;
    }
  }
  s.spec_count[c] = cnt;
  s.spec_exit[c] = exit_pid;
}

// Chunks [0, c_end): chunk 0 from the entry (the first point at or after pid `entry`), chunk c > 0 from chunk c - 1's
// speculative exit.  Writes the stitched entries and counts to s.st_entry.
__global__ void __maxnreg__(SCF_MAX_REGS)
k_scf_stitch(const CacheFixSlab S, u64 line, u64 chunk, u64 c_end, u64 entry, ShardCacheFixScratch s) {
  const u64 c = (u64)blockIdx.x * SCF_THREADS + threadIdx.x;
  if (c >= c_end) return;
  const u64 nch = (S.n_local + chunk - 1) / chunk;
  const ChunkRange r = chunk_range(S, c, chunk);
  u64 E;
  if (c == 0) {
    Pt p0;
    if (!first_point_at(S, (entry >> 1) - S.base, S.n_local, p0)) E = 2 * (S.base + S.n_local);   // no point left
    else E = p0.pid < entry ? entry : p0.pid;   // an odd entry on a run's first index: the run's second point
  } else {
    E = s.spec_exit[c - 1];
  }
  u32 ok = 0;
  u64 cnt = 0, exit_pid = PID_OPEN;
  if (E != PID_OPEN && E >= r.end_pid) {       // the segment open at the chunk's start spans the whole chunk
    ok = 1; exit_pid = E;
  } else if (E != PID_OPEN) {
    const u64 scnt = s.spec_count[c], sexit = s.spec_exit[c];
    const u64 nt = scnt < CACHEFIX_TARGETS ? scnt : CACHEFIX_TARGETS;
    const u64* T = s.targets + c * CACHEFIX_TARGETS;
    Pt p = pt_of(S, E);
    for (;;) {
      if (sexit != PID_OPEN) {
        u64 t = 0;
        while (t < nt && T[t] < p.pid) ++t;
        if (t < nt && T[t] == p.pid) { ok = 1; cnt += scnt - t; exit_pid = sexit; break; }
        if (t == nt && scnt > nt) break;      // past the last target: the chains can no longer be seen to meet
      }
      ++cnt;
      p = next_knot(S, line, p, r.limit);
      if (p.pid == PID_OPEN || p.pid == PID_HALO) break;
      if (p.pid >= r.end_pid) { ok = 1; exit_pid = p.pid; break; }
    }
  }
  s.st_entry[c] = E;
  s.st_entry[nch + c] = ok ? cnt : 0;
  s.stitch_exit[c] = exit_pid;
  s.stitch_ok[c] = ok;
}

// The knot after knot s, found by the whole block (kernels_cachefix.cu's block_next_knot): PID_END at the end of the
// data, PID_HALO when a point past the halo is needed.
__device__ __forceinline__ u64 block_next_knot(const CacheFixSlab& S, u64 line, u64 s_pid) {
  const Pt s = pt_of(S, s_pid);
  Pt a, prev, k;
  int r = next_point(S, s, a);
  if (r != NP_OK) return stop_pid(r);
  prev = a;
  for (;;) {
    r = next_point(S, prev, k);
    if (r != NP_OK) return stop_pid(r);
    bool miss = false;
    for (u64 g = a.y + threadIdx.x; g <= prev.y; g += SCF_RESOLVE_THREADS) {
      const u64 i = g - S.base;
      const u64 key = S.keys[i], pk = key_before(S, i);
      if ((i > 0 || S.has_prev) && key == pk) continue;
      if (key - 1 != pk && 2 * g >= a.pid && 2 * g <= prev.pid) miss |= misses_line(s, k, key - 1, g, line);
      if (2 * g + 1 >= a.pid && 2 * g + 1 <= prev.pid) miss |= misses_line(s, k, key, g, line);
    }
    if (__syncthreads_or(miss)) return prev.pid;
    prev = k;
  }
}

// kernels_cachefix.cu's resolve over s.entry / s.count (copied from the stitched values before the launch), then the
// offsets and the scan's result: res = {exit pid, knots in the slab, status, reach}.
__global__ void __maxnreg__(SCF_MAX_REGS)
k_scf_resolve(const CacheFixSlab S, u64 line, u64 chunk, u64 nch, ShardCacheFixScratch s) {
  __shared__ u64 s_first;
  __shared__ u64 s_part[SCF_RESOLVE_THREADS];
  u64* entry = s.entry;
  u64* count = s.entry + nch;
  const unsigned tid = threadIdx.x;
  u64 exit_pid = s.stitch_exit[nch - 1];   // when the last chunk's stitch is confirmed
  bool halo = false;
  u64 pos = 0;
  while (pos < nch) {
    if (tid == 0) s_first = nch;
    __syncthreads();
    for (u64 base = pos; base < nch; base += SCF_RESOLVE_THREADS) {
      const u64 c = base + tid;
      const bool bad = c < nch && !(s.stitch_ok[c] && (c == 0 || s.stitch_exit[c - 1] == s.spec_exit[c - 1]));
      if (bad) atomicMin((unsigned long long*)&s_first, (unsigned long long)c);
      if (__syncthreads_or(bad)) break;
    }
    const u64 f = s_first;
    __syncthreads();
    if (f >= nch) break;
    u64 E = f == 0 ? entry[0] : s.stitch_exit[f - 1];
    u64 c = f;
    for (;;) {
      const ChunkRange r = chunk_range(S, c, chunk);
      const u64 scnt = s.spec_count[c], sexit = s.spec_exit[c];
      const u64 nt = scnt < CACHEFIX_TARGETS ? scnt : CACHEFIX_TARGETS;
      const u64* T = s.targets + c * CACHEFIX_TARGETS;
      const u64 first = E;
      u64 cnt = 0;
      while (E < r.end_pid) {
        if (sexit != PID_OPEN) {
          u64 t = 0;
          while (t < nt && T[t] < E) ++t;
          if (t < nt && T[t] == E) { cnt += scnt - t; E = sexit; break; }
        }
        ++cnt;
        E = block_next_knot(S, line, E);
      }
      if (E == PID_HALO) { halo = true; pos = nch; break; }
      if (tid == 0) { entry[c] = first; count[c] = cnt; }
      ++c;
      if (c >= nch) { exit_pid = E; pos = nch; break; }
      if (E == s.spec_exit[c - 1] && s.stitch_ok[c]) { pos = c + 1; break; }   // chunk c's stitch started from E
    }
    __syncthreads();
  }
  // exclusive scan of the knot counts -> output offsets; total = offsets[nch]
  __syncthreads();
  const u64 per = (nch + SCF_RESOLVE_THREADS - 1) / SCF_RESOLVE_THREADS;
  const u64 b = tid * per < nch ? tid * per : nch, e = b + per < nch ? b + per : nch;
  u64 sum = 0;
  for (u64 c = b; c < e; ++c) sum += count[c];
  s_part[tid] = sum;
  __syncthreads();
  for (unsigned o = 1; o < SCF_RESOLVE_THREADS; o <<= 1) {
    const u64 v = tid >= o ? s_part[tid - o] : 0;
    __syncthreads();
    s_part[tid] += v;
    __syncthreads();
  }
  u64 off = s_part[tid] - sum;
  for (u64 c = b; c < e; ++c) { s.offsets[c] = off; off += count[c]; }
  if (tid == SCF_RESOLVE_THREADS - 1) {
    s.offsets[nch] = s_part[tid];
    s.res[0] = halo ? PID_HALO : exit_pid;
    s.res[1] = s_part[tid];
    s.res[2] = halo ? 1 : 0;
    s.res[3] = halo ? S.base + S.n_avail : 0;
  }
}

__global__ void __maxnreg__(SCF_MAX_REGS)
k_scf_emit(const CacheFixSlab S, u64 line, u64 chunk, u64 nch, ShardCacheFixScratch s, ulonglong2* out) {
  const u64 c = (u64)blockIdx.x * SCF_THREADS + threadIdx.x;
  if (c >= nch) return;
  const u64 cnt = s.entry[nch + c];
  if (!cnt) return;
  const u64 off = s.offsets[c];
  Pt p = pt_of(S, s.entry[c]);
  for (u64 j = 0;;) {
    out[off + j] = make_ulonglong2(p.x, p.y);
    if (++j == cnt) break;
    p = next_knot(S, line, p, PID_END);
  }
}

unsigned blocks_for(u64 items) { return (unsigned)((items + SCF_THREADS - 1) / SCF_THREADS); }

}  // namespace

void shard_cache_fix_speculate(const Launch& L, const CacheFixSlab& S, u64 line, u64 chunk, const ShardCacheFixScratch& s) {
  const u64 nch = (S.n_local + chunk - 1) / chunk;
  k_scf_speculate<<<blocks_for(nch), SCF_THREADS, 0, L.stream>>>(S, line, chunk, nch, s);
  count_launch();
}

void shard_cache_fix_join(const Launch& L, const CacheFixSlab& S, u64 line, u64 chunk, u64 entry_pid, bool chunk0_only,
                          const ShardCacheFixScratch& s) {
  const u64 nch = (S.n_local + chunk - 1) / chunk;
  const u64 c_end = chunk0_only ? 1 : nch;
  k_scf_stitch<<<blocks_for(c_end), SCF_THREADS, 0, L.stream>>>(S, line, chunk, c_end, entry_pid, s);
  count_launch();
  cudaMemcpyAsync(s.entry, s.st_entry, sizeof(u64) * 2 * nch, cudaMemcpyDeviceToDevice, L.stream);
  k_scf_resolve<<<1, SCF_RESOLVE_THREADS, 0, L.stream>>>(S, line, chunk, nch, s);
  count_launch();
}

void shard_cache_fix_emit(const Launch& L, const CacheFixSlab& S, u64 line, u64 chunk, const ShardCacheFixScratch& s,
                          void* d_out) {
  const u64 nch = (S.n_local + chunk - 1) / chunk;
  k_scf_emit<<<blocks_for(nch), SCF_THREADS, 0, L.stream>>>(S, line, chunk, nch, s, (ulonglong2*)d_out);
  count_launch();
}

}  // namespace rmi
