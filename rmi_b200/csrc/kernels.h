// kernels.h — host-callable launchers of the CUDA kernels (kernels_top.cu, kernels_leaf.cu)
// used by the C-ABI layer (api.cu).  Internal; the public surface is include/rmi_b200.h.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include <type_traits>

#include "models.cuh"

namespace rmi {

// Conditions under which the reference panics (or this build gives up); set by kernels in a
// device status word, decoded by api.cu into rmi_last_error() text.
enum StatusBit : unsigned {
  ST_NOT_SORTED = 1u << 0,        // keys[i] < keys[i-1]
  ST_NON_MONOTONE = 1u << 1,      // two_layer.rs:50  assert!(target >= last_target)
  ST_SPLIT_AT_ZERO = 1u << 2,     // two_layer.rs:27  build_models_from(0, 0, ..): end_idx > start_idx
  ST_SPLIT_AT_END = 1u << 3,      // two_layer.rs:27  build_models_from(n, n, ..)
  ST_TOP_OUT_OF_BOUNDS = 1u << 4, // two_layer.rs:45  top model index out of bounds
  ST_NUM_BITS = 1u << 5,          // utils.rs:18      assert!(nbits >= 1)
  ST_CUBIC_UNWRAP = 1u << 6,      // cubic_spline.rs:50,61  find(..).unwrap() on None
  ST_ROBUST_TOO_SMALL = 1u << 7,  // linear.rs:248    assert!(bnd*2+1 < data.len())
  ST_HIST_BINS = 1u << 8,         // histogram.rs:25-27 division by zero / items_per_bin >= 1
  ST_NEG_VARIANCE = 1u << 9,      // linear.rs:48     assert!(var >= 0.0)
  ST_BRADIX_OOB = 1u << 10,       // balanced_radix.rs:28 counts[] index out of bounds
  ST_RADIX_TABLE_OOB = 1u << 11,  // radix.rs:103     assert!(current_radix < hint_table.len())
  ST_HALO_TOO_SMALL = 1u << 12    // sharded build: a leaf reaches past the keys copied from the next rank
};

// Small device-resident scalars shared between kernels of one build.
struct BuildAux {
  unsigned status;        // OR of StatusBit
  int has_split;          // two_layer.rs:147-175: 0 = single range, 1 = two halves
  u64 split_idx;          // first index whose clamped top prediction >= N/2
  u64 split_target;       // clamped prediction of keys[split_idx]
  u64 max_scaled_y;       // largest scaled offset (radix / bradix)
  // summary statistics (two_layer.rs:267-284)
  u64 max_error, max_error_idx, sum_n_err;
  double sum_l2, sum_log2;
  // bradix search state
  double best_score;
  int best_valid, _pad;
  u64 could_not_replace;
};

// Position of a rank's slab inside the global sorted key array (single-GPU: base 0, the whole
// array, no neighbours).  Kernels index the LOCAL slab; every offset that enters a fit or an
// error bound is global (base + local).
template <class T> struct Shard {
  u64 base;       // global index of local key 0
  u64 n_global;   // keys in the whole data set
  u64 n_local;    // keys this rank owns
  u64 n_avail;    // n_local + halo keys (copied from the following ranks) readable after them
  int has_prev;   // some earlier rank holds keys; prev_key / prev_F describe the last of them
  int is_last;    // this rank holds the data set's last key
  T prev_key;
  u64 prev_F;     // duplicate-fixed global offset of prev_key
  int no_dups;    // the whole data set is known to contain no two equal keys
};
template <class T> inline Shard<T> whole_array(u64 n) {
  Shard<T> s;
  s.base = 0; s.n_global = n; s.n_local = n; s.n_avail = n; s.has_prev = 0; s.is_last = 1; s.prev_key = T(); s.prev_F = 0; s.no_dups = 0;
  return s;
}

// Optional: hand the leaf results to the host slice by slice while later slices still compute
// (N x (8*ppm + 8) bytes cross PCIe in about the time the leaf kernel itself takes, so copied
// after the kernel they would be fully exposed).  The bulk leaf kernel is launched as
// LEAF_SLICES consecutive block ranges on separate streams (so a slice's tail overlaps the next
// slice's start); each slice's parameter / error (/ count) ranges are copied to pinned host
// memory on the slice's stream as soon as the slice is done.  streams[c] must have a higher
// priority than streams[c + 1], so that the slices are scheduled, and finish, in order.
constexpr int LEAF_SLICES = 5;
struct LeafCopyOut {
  double* h_params = nullptr;   // N x ppm (pinned)
  u64* h_errors = nullptr;      // N
  u64* h_counts = nullptr;      // N or null
  cudaStream_t streams[LEAF_SLICES] = {};
  cudaEvent_t ev_ready = nullptr;             // main stream: leaf boundaries are final
  cudaEvent_t ev_kernel[LEAF_SLICES] = {};    // slice kernel finished
  cudaEvent_t ev_copied[LEAF_SLICES] = {};    // slice results are on the host
  mutable int used = 0;                       // slices actually launched (set by fit_leaves)
};

struct Launch {
  cudaStream_t stream;
  int num_sms;
  const LeafCopyOut* copy = nullptr;   // optional sliced launch + overlapped result copies (fit_leaves)
  // optional leaf window [leaf_lo, leaf_hi) (leaf_hi == 0: all leaves): fit_leaves launches blocks only for the leaf
  // groups that intersect it and copies only its records — a rank of a range-partitioned build that already knows
  // which leaves it owns (the other lanes of the boundary groups are not its leaves and stay idle)
  u64 leaf_lo = 0, leaf_hi = 0;
  // optional fork/join resources for the long-leaf kernel (kernels_leaf.cu); all null = disabled
  cudaStream_t side = nullptr;       // high-priority stream
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  u32* d_long = nullptr;             // [0] = number of long leaves found, [1 + i] = their indices
};
constexpr u32 LONG_LEAF_CAP = 16;    // more long leaves than this: no separate kernel (skewed data; they stay in the bulk kernel)

void count_launch();   // bumps the process-wide kernel launch counter (api.cu)

// ---- key sample for the leaf-boundary search --------------------------------------------------
// The parallel linear / robust_linear top fit streams every key anyway; on the way it leaves
// sample[s] = keys[s * BOUNDS_SAMPLE_R] for s < bounds_sample_len(n) (25 MB at 200M u64 keys) with an L2 evict_last
// policy, and compute_leaf_bounds() then finds each leaf boundary in the sample (from L2) before it touches the keys
// (DESIGN.md section 4 gives the sweep of R).
constexpr u64 BOUNDS_SAMPLE_R = 64;
__host__ __device__ inline u64 bounds_sample_len(u64 n) { return (n + BOUNDS_SAMPLE_R - 1) / BOUNDS_SAMPLE_R; }
// The sample occupies whole 128-byte L2 lines of its own (compute_leaf_bounds discards them once the search is done):
// allocate bounds_sample_bytes() and place the sample at bounds_sample_at() of that allocation.
inline size_t bounds_sample_bytes(u64 n, size_t key_bytes) { return (bounds_sample_len(n) * key_bytes + 127) / 128 * 128 + 128; }
template <class T> inline T* bounds_sample_at(void* raw) { return (T*)(((uintptr_t)raw + 127) & ~(uintptr_t)127); }
// The top fits that stream the keys on the device and leave the sample behind.
inline bool top_fit_writes_sample(int kind, bool exact) { return (kind == M_LINEAR || kind == M_ROBUST_LINEAR) && !exact; }

// ---- top-model fits (kernels_top.cu) -------------------------------------------------------
// All write the fitted model into *d_top (device) and OR failure bits into d_aux->status.
// `scratch` must hold at least top_scratch_bytes() bytes.
size_t top_scratch_bytes(u64 num_leaves);
// Returns host-detected StatusBits (0 = launched); device-detected ones land in d_aux->status.
// d_sample: null, or where the key sample goes when top_fit_writes_sample(kind, exact).
void histogram_bins(u64 n, u64 num_leaves, u64* num_bins, u64* items_per_bin);
template <class T>
unsigned fit_top_model(const Launch& L, const T* keys, u64 n, int kind, int table_bits, u64 num_leaves, bool exact,
                       TopModel* d_top, BuildAux* d_aux, void* scratch, u32* d_table32, u64* d_pivots,
                       u64* d_radix_index, T* d_sample);

// Sortedness of a key array (verified once per dataset): *d_flag |= 1 if out of order.
template <class T> void check_sorted(const Launch& L, const T* keys, u64 n, u64 i0, u64 i1, unsigned* d_flag);

// ---- leaf layer (kernels_leaf.cu) ----------------------------------------------------------
// S[j] = first index whose clamped top prediction is >= j, for j in [0, N]; also verifies
// sortedness and monotonicity and derives the split (two_layer.rs:131-175).
// d_sample: the key sample fit_top_model left (null if none); when the boundaries are searched, the search starts in
// it, and afterwards its L2 lines are discarded (its contents are undefined from then on).
template <class T>
void compute_leaf_bounds(const Launch& L, const T* keys, u64 n, int top_kind, const TopModel* d_top, u64 num_leaves,
                         u64* d_S, BuildAux* d_aux, bool allow_search, const T* d_sample);
// Fused per-leaf pass: closed-form fit (build_models_from), empty-leaf constants, forward
// pass / max error, lower-bound widening (two_layer.rs:20-99, :186-259,
// lower_bound_correction.rs:91-137).  Writes N x ppm params, N errors, N counts.
template <class T>
void fit_leaves(const Launch& L, const T* keys, const Shard<T>& shard, int leaf_kind, u64 num_leaves, const u64* d_S,
                BuildAux* d_aux, double* d_params, u64* d_errors, u64* d_counts);
// After fit_leaves with L.copy set: makes L.stream wait until every slice's results are on the host.
void leaf_copy_join(const Launch& L);
// Summary statistics over the N leaves (two_layer.rs:267-284) into d_aux.
void leaf_statistics(const Launch& L, u64 n, u64 num_leaves, const u64* d_errors, const u64* d_counts,
                     BuildAux* d_aux, void* scratch);
size_t stats_scratch_bytes(u64 num_leaves);

// ---- error pass over given leaf tables (kernels_eval.cu, rmi_evaluate) ---------------------------
// fit_leaves's forward pass and widening without the fit and without the empty-leaf constants: from the boundaries
// d_S (compute_leaf_bounds) and N x ppm given parameters, writes N error bounds and N key counts.  no_dups: the keys
// hold no two equal ones (the run tracking is skipped).  d_scratch: 2 x N u64.  Three launches.
template <class T>
void evaluate_leaves(const Launch& L, const T* keys, u64 n, bool no_dups, int leaf_kind, u64 N, const u64* d_S,
                     const double* d_params, u64* d_scratch, u64* d_errors, u64* d_counts);

// ---- error pass over given leaf tables on a range-partitioned key array (kernels_shard_eval.cu, DESIGN.md section 15)
// This rank's contributions, from the global boundaries d_S, into d_part = part_err | part_run (2 x N u64, zeroed
// here): the per-key errors and the runs that end on this slab, and the widening terms whose key this slab holds.
// is_first: the first non-empty rank; has_next / next_key: the first key of the next non-empty rank.  sh.no_dups
// (identical on every rank) skips the run tracking.  After an all-reduce MAX of d_part (its first N words suffice when
// sh.no_dups), shard_evaluate_finish writes the N error bounds and key counts rmi_evaluate gives on the whole keys.
template <class T>
void shard_evaluate_partials(const Launch& L, const T* keys, const Shard<T>& sh, int is_first, int has_next, T next_key,
                             int leaf_kind, u64 N, const u64* d_S, const double* d_params, u64* d_part);
void shard_evaluate_finish(const Launch& L, u64 n, u64 N, bool no_dups, const u64* d_S, const u64* d_part, u64* d_errors,
                           u64* d_counts);

// ---- cross-rank pieces of a range-partitioned build (kernels_leaf.cu) --------------------------
// d_off[r] = first leaf owned by rank r, d_off[world] = N (d_bases: global index of every rank's first key,
// world + 1 entries; r_last: last rank that holds keys).  One tiny kernel, no host involvement.
void shard_owner_offsets(const Launch& L, const u64* d_S, u64 N, const u64* d_bases, int world, int r_last, u64* d_off);
// Summary statistics of the leaves this rank owns, as one partial record (stats_partial_bytes()) at d_part_out;
// after an all-gather of the partials, leaf_statistics_merge() finishes them into d_aux on every rank.
size_t stats_partial_bytes();
void leaf_statistics_owned(const Launch& L, u64 n, u64 N, const u64* d_errors, const u64* d_counts, const u64* d_off, int rank,
                           int world, void* d_part_out, void* scratch);
void leaf_statistics_merge(const Launch& L, const void* d_parts, int world, BuildAux* d_aux);

// ---- batched lookups on a trained index (kernels_lookup.cu, kernels_lookup_range.cu) ------------------------------
// The model groups the lookup kernels are instantiated for (-1: not a top / leaf model): the linear family shares
// one group, as in compute_leaf_bounds.
inline int lookup_top_group(int kind) {
  if (kind == M_LINEAR || kind == M_ROBUST_LINEAR || kind == M_LINEAR_SPLINE) return M_LINEAR;
  return kind >= M_LINEAR && kind <= M_HISTOGRAM ? kind : -1;
}
inline int lookup_leaf_group(int kind) {
  if (kind == M_LINEAR || kind == M_ROBUST_LINEAR || kind == M_LINEAR_SPLINE) return M_LINEAR;
  return kind >= M_CUBIC && kind <= M_LOGNORMAL ? kind : -1;
}
template <int K> using Kind = std::integral_constant<int, K>;
// f(Kind<TOP>, Kind<LEAF>) for the kernel group of the given top and leaf model kinds.
template <class F> void with_groups(int top_kind, int leaf_kind, F&& f) {
  auto leaf = [&](auto top) {
    switch (lookup_leaf_group(leaf_kind)) {
      case M_LINEAR: f(top, Kind<M_LINEAR>{}); break;
      case M_CUBIC: f(top, Kind<M_CUBIC>{}); break;
      case M_LOGLINEAR: f(top, Kind<M_LOGLINEAR>{}); break;
      case M_NORMAL: f(top, Kind<M_NORMAL>{}); break;
      default: f(top, Kind<M_LOGNORMAL>{}); break;
    }
  };
  switch (lookup_top_group(top_kind)) {
    case M_LINEAR: leaf(Kind<M_LINEAR>{}); break;
    case M_CUBIC: leaf(Kind<M_CUBIC>{}); break;
    case M_LOGLINEAR: leaf(Kind<M_LOGLINEAR>{}); break;
    case M_NORMAL: leaf(Kind<M_NORMAL>{}); break;
    case M_LOGNORMAL: leaf(Kind<M_LOGNORMAL>{}); break;
    case M_RADIX: leaf(Kind<M_RADIX>{}); break;
    case M_RADIX_TABLE: leaf(Kind<M_RADIX_TABLE>{}); break;
    case M_BRADIX: leaf(Kind<M_BRADIX>{}); break;
    default: leaf(Kind<M_HISTOGRAM>{}); break;
  }
}
// One packed record per leaf: its parameters in Model::params() order, then its error bound.
__host__ __device__ constexpr int lookup_record_bytes(int leaf_kind) { return leaf_kind == M_CUBIC ? 64 : 32; }
// N records (N x lookup_record_bytes bytes at `out`, host memory) from N x ppm parameters and N errors.
void pack_leaf_records(int leaf_kind, const double* params, const u64* errors, u64 N, void* out);
// What a lookup computes, and into which of its two outputs:
//   LOOKUP_PREDICT      out = position estimates, out2 (may be null) = the leaves' error bounds
//   LOOKUP_LOWER        out = exact lower bounds (the number of keys < q)
//   LOOKUP_UPPER        out = exact upper bounds (the number of keys <= q; 0 for NaN)
//   LOOKUP_EQUAL_RANGE  out = lower bounds, out2 = upper bounds, from one window per query
enum LookupMode { LOOKUP_PREDICT, LOOKUP_LOWER, LOOKUP_UPPER, LOOKUP_EQUAL_RANGE };
// One kernel launch on L.stream (none for nq == 0) over keys[0, n); last = keys[n-1], and the upper bound of a query
// >= it is n without a search.  *fallbacks (may be null) grows by the number of queries whose window missed (either
// end).  `top` is passed by value; its table pointers (t32, pivots) are device memory.
template <class T>
void lookup_batch(const Launch& L, LookupMode mode, const TopModel& top, int leaf_kind, const void* d_records, u64 N,
                  const T* keys, u64 n, T last, const T* d_queries, u64 nq, u64* d_out, u64* d_out2, u64* d_fallbacks);
// The same for a bounded (cache-fix) index over u64 keys: the RMI (d_records, N leaves) predicts one of the K knots
// at d_knots (K x {key, offset}, 16 bytes each), the spline step gives the key's line of line_size keys, and the
// bounds are searched in that line.  A prediction's error bound is line_size.
void lookup_bounded_batch(const Launch& L, LookupMode mode, const TopModel& top, int leaf_kind, const void* d_records,
                          u64 N, const void* d_knots, u64 K, u64 line_size, const u64* keys, u64 n, u64 last,
                          const u64* d_queries, u64 nq, u64* d_out, u64* d_out2, u64* d_fallbacks);

// ---- the sorted delta of an updatable index (kernels_delta.cu, DESIGN.md section 19) -----------------------------
// out[0, na + nb) = the stable merge of the sorted arrays a and b (a's key first on equal keys, compared by value).
// d_status (may be null) receives DELTA_ST_NAN if b holds a NaN.  One launch (none for na + nb == 0).
constexpr unsigned DELTA_ST_NAN = 1u;
template <class T> void delta_merge(const Launch& L, const T* a, u64 na, const T* b, u64 nb, T* out, unsigned* d_status);
// Adds, per query, the number of the m sorted delta keys d with d < q (DELTA_LOWER, into out_first), d <= q
// (DELTA_UPPER, into out_last) or both (DELTA_BOTH) to the answers already there.  One launch (none for m == 0 or
// nq == 0).
enum DeltaCountMode { DELTA_LOWER, DELTA_UPPER, DELTA_BOTH };
template <class T>
void delta_count(const Launch& L, DeltaCountMode mode, const T* delta, u64 m, const T* d_queries, u64 nq,
                 u64* out_first, u64* out_last);
// As delta_count for a delta with t > 0 removed keys: adds #{inserted keys before q} (m may be 0) and subtracts
// #{removed keys before q}, "before" as mode says.  One launch (none for t == 0 or nq == 0).
template <class T>
void delta_adjust(const Launch& L, DeltaCountMode mode, const T* ins, u64 m, const T* rem, u64 t, const T* d_queries,
                  u64 nq, u64* out_first, u64* out_last);
// For a sorted batch of removals, with [first[j], last[j]) the equal range of batch[j] over the logical key set:
// d_status receives DELTA_ST_NAN if the batch holds a NaN and DELTA_ST_MISSING if it holds more copies of a value than
// the key set does (multiset_diff.cuh).  One launch (none for n == 0).
constexpr unsigned DELTA_ST_MISSING = 2u;
template <class T>
void delta_check_remove(const Launch& L, const T* batch, u64 n, const u64* first, const u64* last, unsigned* d_status);
// out[0, nm - t) = the sorted keys M[0, nm) minus the t sorted removed keys, each removal taking the first copy of its
// value's run still there; requires rem ⊆ M as a multiset.  One launch (none for nm == 0).
template <class T> void delta_subtract(const Launch& L, const T* M, u64 nm, const T* rem, u64 t, T* out);

// ---- lookups over a range-partitioned data set (kernels_shard_lookup.cu, DESIGN.md section 14) -------------------
// A query goes to the last non-empty rank whose first key is < q (the first non-empty rank if none is).
constexpr int SHARD_ROUTE_MAX = 64;
template <class T> struct ShardRoute {
  T first[SHARD_ROUTE_MAX];                // first key of every non-empty rank, in rank order (non-decreasing)
  unsigned char rank[SHARD_ROUTE_MAX];     // that rank
  int count;                               // non-empty ranks, >= 1
};
// Per-block counts per rank of the route: d_block_counts holds world x shard_route_blocks(n) u32, d_block_offsets as
// many u64.
u64 shard_route_blocks(u64 n);
// Three launches (none for n == 0, where d_send_counts is zeroed): d_send receives the n queries in per-rank segments
// in rank order, d_send_counts[r] the length of rank r's segment, d_slot[i] the position of query i in d_send.
// upper: route by <= (the last non-empty rank whose first key is <= q), for upper bounds.
template <class T>
void shard_route(const Launch& L, const ShardRoute<T>& route, int world, const T* d_q, u64 n, u32* d_block_counts,
                 u64* d_block_offsets, T* d_send, u64* d_slot, u64* d_send_counts, bool upper = false);
// Exact global lower bounds of m queries routed to this rank (slab keys[0, n_local) at global index base), from the
// predictions d_pos / d_err of lookup_batch (predict, n = n_global).  One launch; *d_fallbacks (may be null) grows by
// the number of windows that missed.  n_local >= 1.  upper: exact global upper bounds of queries routed by <= instead;
// last = keys[n_local - 1] (queries >= it get base + n_local without a search).
template <class T>
void shard_search(const Launch& L, const T* keys, u64 n_local, u64 base, u64 n_global, const T* d_q, u64 m,
                  const u64* d_pos, const u64* d_err, u64* d_out, u64* d_fallbacks, bool upper = false, T last = T());
// d_out[i] = d_returned[d_slot[i]].  One launch (none for n == 0).
void shard_gather(const Launch& L, const u64* d_slot, const u64* d_returned, u64 n, u64* d_out);

// ---- `--bounded` lookups over a range-partitioned data set (kernels_shard_bounded.cu, DESIGN.md section 17) --------
// A rank's knots: global knots [k_lo, k_lo + k_len) at `knots` ({key, offset} pairs), its own knot slab [a0, a1) among
// them, K knots in all, line_size `line`.
struct BoundedKnotSlab {
  const void* knots;
  u64 k_lo, k_len, K, a0, a1, line;
};
// One launch (none for m == 0).  lower_bound = true: exact global lower bounds of m queries routed to this rank by key
// (slab keys[0, n_local) at global index base, n_local >= 1); *d_fallbacks (may be null) grows by the far queries and
// by the others whose global line missed.  lower_bound = false: the single-GPU bounded pos of m queries routed to this
// rank by knot index.  The RMI (d_records, N leaves, `top` by value) runs over the K knots.
// upper (with lower_bound): upper bounds of queries routed to this rank by key with <=; last = keys[n_local - 1].
void shard_bounded_search(const Launch& L, const TopModel& top, int leaf_kind, const void* d_records, u64 N,
                          const BoundedKnotSlab& ks, const u64* keys, u64 n_local, u64 base, u64 n_global,
                          const u64* d_queries, u64 m, u64* d_out, u64* d_fallbacks, bool lower_bound,
                          bool upper = false, u64 last = 0);
// d_out[i] = max(d_pos[i] - d_err[i], 0) + 1 (d_out may be d_pos): the value shard_route<u64> routes by knot index
// (a route whose "first keys" are the knot bases of the ranks that hold knots).  One launch (none for n == 0).
void shard_knot_route_keys(const Launch& L, const u64* d_pos, const u64* d_err, u64 n, u64* d_out);
// d_send[d_slot[i]] = d_q[i].  One launch (none for n == 0).
void shard_scatter_queries(const Launch& L, const u64* d_q, const u64* d_slot, u64 n, u64* d_send);
// d_out[i] = value.  One launch (none for n == 0).
void shard_fill(const Launch& L, u64 value, u64 n, u64* d_out);

// ---- the `--bounded` cache-fix scan (kernels_cachefix.cu, DESIGN.md section 12) ----------------------------------
// Key indices per speculation chunk, and how many of a chunk's speculative knots the stitch can join.
// (DESIGN.md section 12.3 gives the sweep.)
constexpr u64 CACHEFIX_CHUNK = 256;
constexpr int CACHEFIX_TARGETS = 16;
enum CacheFixStat { CF_STAT_POINTS = 0, CF_STAT_STITCH_SEGMENTS = 1, CF_STAT_FALLBACK_POINTS = 2, CF_STAT_EVALS = 3,
                    CF_NUM_STATS = 4 };
// Device scratch of one scan, nch = ceil(n / chunk) chunks: O(nch) words.
struct CacheFixScratch {
  u64* targets;       // nch x CACHEFIX_TARGETS: pids of the first knots of each chunk's speculative chain
  u64* spec_count;    // nch: knots the speculative chain starts inside its chunk
  u64* spec_exit;     // nch: its first knot at or past the chunk's end
  u64* stitch_exit;   // nch: the chunk's exit as the stitch found it
  u32* stitch_ok;     // nch
  u64* entry;         // nch: the chunk's first true knot (pid; may lie past the chunk)
  u64* count;         // nch: true knots inside the chunk
  u64* offsets;       // nch + 1: exclusive scan of count; offsets[nch] = knots before finish()'s last point
  u64* last_knot;     // 2: the point finish() appends
  u64* stats;         // CF_NUM_STATS counters, zeroed by the caller
};
// count / speculate / stitch / resolve: four launches on L.stream; s.offsets[nch] then holds the knot count - 1.
void cache_fix_scan(const Launch& L, const u64* keys, u64 n, u64 line, u64 chunk, const CacheFixScratch& s);
// One launch: writes the offsets[nch] + 1 knots as {key, offset} pairs to d_out.
void cache_fix_emit(const Launch& L, const u64* keys, u64 n, u64 line, u64 chunk, const CacheFixScratch& s,
                    void* d_out);

// ---- the cache-fix scan over one rank's slab of range-partitioned keys (kernels_shard_cachefix.cu, section 16) ----
// The keys a rank's walks read: its own keys [0, n_local), then the halo up to n_avail.  Point ids are global.
struct CacheFixSlab {
  const u64* keys;
  u64 base;        // global index of local key 0
  u64 n_local;     // the slab's own keys (> 0)
  u64 n_avail;     // own keys + halo keys
  u64 prev_key;    // the last key of the previous non-empty rank; 0 when there is none
  int has_prev;
  int at_end;      // base + n_avail is the end of the data
};
// Device scratch of one rank's scan, nch = ceil(n_local / chunk) chunks.
struct ShardCacheFixScratch {
  u64* targets;       // nch x CACHEFIX_TARGETS
  u64* spec_count;    // nch
  u64* spec_exit;     // nch
  u64* stitch_exit;   // nch
  u32* stitch_ok;     // nch
  u64* st_entry;      // 2 x nch: the stitch's entries | counts (kept across scans: they do not depend on the entry)
  u64* entry;         // 2 x nch: the resolved entries | counts of the last scan
  u64* offsets;       // nch + 1
  u64* res;           // 4: exit pid, knots in the slab, status (1: halo too small), global index the walk lacked
};
// Speculation of every chunk (once per slab and line size).
void shard_cache_fix_speculate(const Launch& L, const CacheFixSlab& S, u64 line, u64 chunk, const ShardCacheFixScratch& s);
// Stitch (every chunk, or chunk 0 alone when the other chunks' stitches are in s.st_entry already) from entry_pid
// (a pid in the slab: the chain starts at the first point at or after it), then the resolve; fills s.res.
void shard_cache_fix_join(const Launch& L, const CacheFixSlab& S, u64 line, u64 chunk, u64 entry_pid, bool chunk0_only,
                          const ShardCacheFixScratch& s);
// Writes the res[1] knots of the last join to d_out as {key, offset} pairs.
void shard_cache_fix_emit(const Launch& L, const CacheFixSlab& S, u64 line, u64 chunk, const ShardCacheFixScratch& s,
                          void* d_out);

// ---- range-partitioned build phases (kernels_shard.cu) ---------------------------------------
size_t shard_scratch_bytes();
// d_bradix_counts: bradix's 4 x N u32 per-bin counts (null for the other tops), merged by an all-reduce SUM between
// shard_top_local and shard_top_finish.
template <class T>
unsigned shard_top_local(const Launch& L, const T* keys, const Shard<T>& sh, int kind, u64 N, double px, double py,
                         T first_key, T last_key, u64 last_F, void* scratch, double* d_sums, TopModel* d_top,
                         BuildAux* d_aux, u32* d_bradix_counts);
template <class T>
void shard_top_mid(const Launch& L, const T* keys, const Shard<T>& sh, int kind, u64 N, T first_key, T last_key,
                   void* scratch, double* d_sums, BuildAux* d_aux);
template <class T>
void shard_top_finish(const Launch& L, const Shard<T>& sh, int kind, u64 N, double px, double py, const double* d_sums,
                      T first_key, T last_key, u64 last_F, const void* scratch, const u32* d_bradix_counts,
                      TopModel* d_top, BuildAux* d_aux);
// bradix over a range-partitioned array (kernels_top.cu).  shard_bradix_count: zero d_counts (4 x N u32), then count
// this rank's keys per bin for all four candidates in one pass (the scalars in d_top / d_aux already set).
// shard_bradix_decide: chi2 of every candidate over the merged counts, the strict minimum in candidate order, commit
// (k_bradix_pick / k_bradix_commit); scratch holds shard_bradix_scratch_bytes().
template <class T>
void shard_bradix_count(const Launch& L, const T* keys, const Shard<T>& sh, u64 N, const TopModel* d_top, BuildAux* d_aux,
                        u32* d_counts);
void shard_bradix_decide(const Launch& L, u64 n, u64 N, const u32* d_counts, void* scratch, TopModel* d_top,
                         BuildAux* d_aux);
size_t shard_bradix_scratch_bytes();
template <class T>
void shard_bounds(const Launch& L, const T* keys, const Shard<T>& sh, int kind, const TopModel* d_top, u64 N, u64* d_S,
                  BuildAux* d_aux);
// The streaming boundary pass for every top group (a given top model, not known to be monotone): S_local, n_global
// where no local key reaches a leaf, ST_NOT_SORTED / ST_NON_MONOTONE also across the cut before the slab.
template <class T>
void shard_bounds_given(const Launch& L, const T* keys, const Shard<T>& sh, int kind, const TopModel* d_top, u64 N,
                        u64* d_S, BuildAux* d_aux);
template <class T>
void shard_split(const Launch& L, const T* keys, const Shard<T>& sh, int kind, const TopModel* d_top, u64 N,
                 const u64* d_S, BuildAux* d_aux);
// Table tops (radix8..28, histogram): every rank fills the entries its slab decides (zero elsewhere; hint entries as
// value + 1), the caller all-reduces the table with MAX, then shard_table_decode / hist_radix_index finish it.
template <class T>
void shard_table_local(const Launch& L, const T* keys, const Shard<T>& sh, int kind, int table_bits, u64 N, T first_key,
                       T last_key, BuildAux* d_aux, u32* d_table32, u64* d_pivots, u64 num_bins, u64 items_per_bin);
void shard_table_decode(const Launch& L, int table_bits, u32* d_table32);
void hist_radix_index(const Launch& L, const u64* d_pivots, u64 num_bins, u64* d_radix_index);   // kernels_top.cu
void shard_copy_status(const Launch& L, const BuildAux* d_aux, unsigned* d_out);
// {status word, could_not_replace != 0} of this rank, for the cross-rank gather (two_layer.rs:199-203 warns if ANY leaf could not be replaced)
void shard_copy_flags(const Launch& L, const BuildAux* d_aux, unsigned* d_out2);

}  // namespace rmi
