/* rmi_b200.h — C ABI of the H100-native two-layer RMI trainer (librmi_b200.so).
 *
 * Drop-in boundary for the reference's `rmi_lib::train`
 *   pub fn train<T: TrainingKey>(data: &RMITrainingData<T>, model_spec: &str,
 *                                branch_factor: u64) -> TrainedRMI
 * (reference rmi_lib/src/train/mod.rs:100-126, re-exported rmi_lib/src/lib.rs:10; callers
 * src/main.rs:203,276, rmi_lib/src/optimizer.rs:227, train/mod.rs:146,174).  The reference
 * has no FFI layer of its own; a Rust `rmi_lib` would bind these symbols with `extern "C"`
 * in place of `two_layer::train_two_layer` (train/two_layer.rs:101) — INTEGRATION.md shows
 * the stub.  Plain pointers and sizes only; no C++ or torch types cross this boundary.
 *
 * Conventions (mirroring the reference's):
 *   - input  : an immutable, shareable key set (RMITrainingData, models/mod.rs:233-317).
 *              Here: `rmi_dataset`, device-resident, read-only, may be used by concurrent
 *              rmi_train calls (the optimizer does that, optimizer.rs:224).
 *   - output : an owned TrainedRMI (train/mod.rs:18-33).  Here: `rmi_result`, host memory
 *              owned by the library, released with rmi_result_free.
 *   - errors : the reference panics (process abort).  Here every entry point returns an
 *              rmi_status; rmi_last_error() gives the message the reference would have
 *              printed.  The library never calls exit/abort.
 * Keys must be sorted ascending (the reference's file format requires it, README.md:26-31);
 * an unsorted array is reported as RMI_ERR_PANIC ("keys are not sorted").
 */
#ifndef RMI_B200_H_
#define RMI_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* reference src/load.rs:15-19 DataType / rmi_lib/src/models/mod.rs:41-43 KeyType */
typedef enum { RMI_KEY_U64 = 0, RMI_KEY_U32 = 1, RMI_KEY_F64 = 2 } rmi_key_type;

typedef enum {
  RMI_OK = 0,
  RMI_ERR_PANIC = 1,        /* the reference would have panicked (assert!/unwrap/panic!) */
  RMI_ERR_INVALID = 2,      /* bad argument at this boundary (null pointer, bad enum, ...) */
  RMI_ERR_CUDA = 3,         /* CUDA runtime / driver failure, or no usable device */
  RMI_ERR_UNSUPPORTED = 4   /* valid in the reference, not offered by this build */
} rmi_status;

/* Model identifiers (reference train/mod.rs:37-54 train_model name table).  RADIX_TABLE
 * covers radix8/18/22/26/28 (table bits in rmi_result.l0_table_bits); BRADIX reports its
 * clamp-high / clamp-low variant in rmi_result.l0_bradix_high. */
typedef enum {
  RMI_MODEL_LINEAR = 0, RMI_MODEL_ROBUST_LINEAR = 1, RMI_MODEL_LINEAR_SPLINE = 2, RMI_MODEL_CUBIC = 3,
  RMI_MODEL_LOGLINEAR = 4, RMI_MODEL_NORMAL = 5, RMI_MODEL_LOGNORMAL = 6, RMI_MODEL_RADIX = 7,
  RMI_MODEL_RADIX_TABLE = 8, RMI_MODEL_BRADIX = 9, RMI_MODEL_HISTOGRAM = 10
} rmi_model_id;

/* rmi_train flags */
enum {
  RMI_FLAG_STATS_ONLY = 1u,     /* do not copy leaf parameters/errors to the host (optimizer use:
                                   only the statistics are consumed, optimizer.rs:163-171) */
  RMI_FLAG_TOP_FIT_EXACT = 2u,  /* fit linear/robust_linear/loglinear/normal TOP models with the
                                   reference's order-dependent serial chain (linear.rs:12-59,
                                   normal.rs:28-50) on one device warp, or on a host core for
                                   linear/robust_linear/normal at 2^20 keys and more: bit-identical
                                   to the reference, seconds at 200 M keys.  Default is the parallel
                                   fit (tree reduction, coefficients equal within 1e-9 relative).
                                   lognormal, cubic and the integer tops ignore the flag;
                                   rmi_result.top_fit_exact says whether it took effect. */
  RMI_FLAG_NO_ERRORS = 4u,      /* reserved for --no-errors (main.rs:84-86); errors are still computed */
  RMI_FLAG_LEAF_COUNTS = 8u,    /* also return l1_counts (keys per leaf as the error pass counts them,
                                   two_layer.rs:207-217); not part of TrainedRMI, used by parity checks */
  RMI_FLAG_SHARD_ROOT_ONLY = 16u /* rmi_shard_train: only rank 0 receives the leaf tables in host memory (every rank still
                                   holds them on its device and gets the top model and the statistics).  When all ranks
                                   run on one node, each rank copies the records of the leaves it owns straight into a
                                   host region the ranks share (POSIX shared memory registered with CUDA): world PCIe
                                   links in parallel.  Rank 0's l1_* pointers then point into that region, which has two
                                   halves used alternately: they stay valid until the NEXT-BUT-ONE rmi_shard_train with
                                   this flag on the same communicator (copy them if they must live longer). */
};

/* A device-resident sorted key set.  Replaces src/load.rs:132-157 load_data + the mmap
 * slice adapters (load.rs:21-95): same content (n packed little-endian keys), in HBM. */
typedef struct rmi_dataset rmi_dataset;

/* Copy n host keys to `device` (cudaMemcpyAsync from the caller's buffer; pinned buffers
 * transfer at full PCIe rate).  host_keys must stay valid until the call returns. */
int rmi_dataset_create(const void* host_keys, uint64_t n, rmi_key_type key_type, int device,
                       rmi_dataset** out);
/* Borrow keys that already live in device memory on `device` (no copy, caller keeps ownership
 * and must keep them alive and unmodified while the dataset exists).  device_keys must be
 * 16-byte aligned and readable up to the next 16-byte boundary after the last key (always the
 * case for a buffer that starts a CUDA allocation: those are at least 256-byte granular). */
int rmi_dataset_wrap_device(const void* device_keys, uint64_t n, rmi_key_type key_type, int device,
                            rmi_dataset** out);
/* Read a reference-format key file (u64 LE count + packed keys, README.md:26-31; key type from
 * the file-name suffix as src/main.rs:122-132 does when key_type < 0) straight into HBM through
 * a double-buffered pinned staging ring. */
int rmi_dataset_load_file(const char* path, int key_type_or_negative, int device, rmi_dataset** out);
/* A replica of `src` on another device: one device-to-device copy (NVLink peer copy when the two
 * GPUs are peers, staged by the driver otherwise; a plain copy when device == src's device).
 * Sortedness / duplicate-freeness are inherited, not re-verified.  This is how an --optimize
 * sweep spreads over the GPUs of a node (SURVEY.md section 8(e): replicas, zero communication per
 * configuration) after the key file has been read once. */
int rmi_dataset_replicate(const rmi_dataset* src, int device, rmi_dataset** out);
uint64_t rmi_dataset_len(const rmi_dataset* ds);
/* Copies the rmi_dataset_len(ds) keys to host_keys, synchronously (for example the keys rmi_delta_merge made). */
int rmi_dataset_copy_to_host(const rmi_dataset* ds, void* host_keys);
int rmi_dataset_key_type(const rmi_dataset* ds);
void rmi_dataset_destroy(rmi_dataset* ds);

/* Mirror of TrainedRMI (reference train/mod.rs:18-33).  All pointers are host memory owned
 * by the result; they stay valid until rmi_result_free. */
typedef struct {
  uint64_t num_rmi_rows;        /* TrainedRMI.num_rmi_rows  */
  uint64_t num_data_rows;       /* TrainedRMI.num_data_rows */
  uint64_t branching_factor;    /* TrainedRMI.branching_factor */
  double model_avg_error;       /* two_layer.rs:274-275 */
  double model_avg_l2_error;    /* two_layer.rs:277-279 */
  double model_avg_log2_error;  /* two_layer.rs:281-282 */
  double model_max_log2_error;  /* two_layer.rs:284 */
  uint64_t model_max_error;     /* two_layer.rs:267-271 */
  uint64_t model_max_error_idx;
  uint64_t build_time_ns;       /* wall clock of the rmi_train call (train/mod.rs:103,114-118) */
  uint64_t device_time_ns;      /* CUDA-event time of the kernels of this build */
  uint64_t phase_device_ns[4];  /* CUDA-event time per phase: [0] top-model fit, [1] leaf boundaries,
                                   [2] fused leaf fit + forward/error pass, [3] statistics */

  /* layer 0: TrainedRMI.rmi[0][0] */
  uint32_t l0_model_id;         /* rmi_model_id */
  uint32_t l0_bradix_high;      /* bradix: 1 = bradix_clamp_high, 0 = bradix_clamp_low */
  uint32_t l0_table_bits;       /* radix table: 8/18/22/26/28 */
  uint32_t l0_num_fparams;      /* float parameters in Model::params() order */
  double l0_fparams[4];
  uint32_t l0_num_iparams;      /* integer parameters in Model::params() order */
  uint32_t _pad0;
  uint64_t l0_iparams[4];
  uint64_t l0_table32_len;      /* radix table: hint table (ModelParam::Int32Array) */
  const uint32_t* l0_table32;
  uint64_t l0_array1_len;       /* histogram: radix index (ModelParam::IntArray) */
  const uint64_t* l0_array1;
  uint64_t l0_array2_len;       /* histogram: pivots (ModelParam::IntArray) */
  const uint64_t* l0_array2;

  /* layer 1: TrainedRMI.rmi[1][0..N] and TrainedRMI.last_layer_max_l1s */
  uint32_t l1_model_id;
  uint32_t l1_params_per_model;
  const double* l1_params;      /* N x params_per_model, leaf order; NULL with STATS_ONLY */
  const uint64_t* l1_errors;    /* N; NULL with STATS_ONLY */
  const uint64_t* l1_counts;    /* N keys-per-leaf as counted by two_layer.rs:207-217; only with RMI_FLAG_LEAF_COUNTS */
  uint32_t could_not_replace;   /* two_layer.rs:199-202 warning condition */
  uint32_t top_fit_exact;       /* 1 if the top model came from the serial recurrence */
} rmi_result;

/* rmi_lib::train.  model_spec is "top,leaf" (train/mod.rs:104-109); only two-layer specs are
 * accepted, as in the reference (train/mod.rs:123-125). */
int rmi_train(const rmi_dataset* ds, const char* model_spec, uint64_t branch_factor, uint32_t flags,
              rmi_result** out);
/* As rmi_train, but the top model's float parameters are given instead of fitted (linear,
 * robust_linear, linear_spline: alpha,beta; cubic: a,b,c,d; normal/lognormal: mean,stdev,scale). */
int rmi_train_with_top(const rmi_dataset* ds, const char* model_spec, uint64_t branch_factor, uint32_t flags,
                       const double* l0_fparams, uint32_t n_fparams, rmi_result** out);
void rmi_result_free(rmi_result* r);
/* The calls that take a given trained result (rmi_evaluate, rmi_index_create, rmi_index_create_bounded,
 * rmi_shard_index_create, rmi_shard_eval_create) first check it the same way, before they read a dataset, and refuse it with the same code
 * and the message "<function>: <reason>":
 *   RMI_ERR_INVALID      no l1_params, or (the indexes, which serve the error bounds) no l1_errors: "the result holds
 *                        no leaf tables ..." (RMI_FLAG_STATS_ONLY, or a rank other than 0 of an
 *                        RMI_FLAG_SHARD_ROOT_ONLY build);
 *   RMI_ERR_INVALID      a top or leaf model id that rmi_train does not offer there (radix tables: radix8, 18, 22, 26,
 *                        28 only; radix, bradix and histogram only as the top): "unknown model id";
 *   RMI_ERR_UNSUPPORTED  a radix-table leaf, with rmi_train's message;
 *   RMI_ERR_INVALID      l1_params_per_model not the leaf model's; a radix table absent or not of 2^l0_table_bits
 *                        entries; histogram pivots absent or empty; l0_array1_len > 0 with no l0_array1. */
/* The reference's error pass, lower-bound widening and statistics (two_layer.rs:205-284) of r's top and leaf tables
 * over ds's keys.  Parameters are never refitted or replaced: the returned result holds r's tables bit for bit,
 * with l1_errors, (with RMI_FLAG_LEAF_COUNTS) l1_counts and the summary statistics measured on ds, and
 * num_rmi_rows = num_data_rows = rmi_dataset_len(ds).  Flags: RMI_FLAG_STATS_ONLY, RMI_FLAG_LEAF_COUNTS.
 * A top model that is not monotone on ds is RMI_ERR_PANIC with the training's message (two_layer.rs:50).
 * phase_device_ns: [0] upload of the tables, [1] leaf boundaries, [2] error pass, [3] statistics. */
int rmi_evaluate(const rmi_dataset* ds, const rmi_result* r, uint32_t flags, rmi_result** out);

/* The optimizer's unit of work (optimizer.rs:110-125 enumerates every leaf type for each (top, branching factor)):
 * `num_leaf_models` configurations "top,leaf_k" with the SAME top model and branching factor in one call.  The top
 * model is fitted once and the leaf boundaries are derived once — one pass over the keys each instead of one per
 * configuration — then the fused leaf kernel runs once per leaf type.  Statistics only (as RMI_FLAG_STATS_ONLY): out[k]
 * receives configuration k's result (release each with rmi_result_free); a configuration the reference would panic on
 * fails the whole call, as it aborts the reference's sweep. */
int rmi_train_stats_batch(const rmi_dataset* ds, const char* top_model, const char* const* leaf_models, int num_leaf_models,
                          uint64_t branch_factor, uint32_t flags, rmi_result** out);

/* ---- Batched lookups on the GPU ------------------------------------------------------------------
 * A trained RMI bound to the device-resident keys it was trained on.  For a query q of the dataset's key type:
 *   predict      pos = the generated code's lookup(q, &err) (codegen.rs:612-718): t = min(N-1, top(q)),
 *                pos = min(n-1, leaf[t](q)), err = the error bound of leaf t; a NaN prediction maps to 0.
 *   lower_bound  the number of keys k with k < q (std::lower_bound; n past the last key, 0 for a NaN query),
 *                always exact: a binary search over [pos-err, pos+err], confirmed by the keys just outside that
 *                window, and a galloping search outward when the window misses (never, for a key of the data set). */
typedef struct rmi_index rmi_index;
/* One knot of a `--bounded` RMI's cache-fix spline (rmi_cache_fix below): a key and its first-occurrence offset. */
typedef struct { uint64_t key, offset; } rmi_spline_point;
/* Upload r's top model (incl. radix table / histogram pivots) and its leaf tables, packed, to ds's device and
 * bind them to ds's keys.  r must pass the checks of a given result (above, before rmi_evaluate) and r->num_rmi_rows
 * must equal rmi_dataset_len(ds); ds must outlive the index.  Immutable: concurrent calls on different streams are
 * fine. */
int rmi_index_create(const rmi_result* r, const rmi_dataset* ds, rmi_index** out);
/* A `--bounded` RMI (train_bounded, below): r is the RMI over the K knots of the cache-fix spline
 * (r->num_rmi_rows == num_knots), knots are those K {key, offset} points (the _L2_PARAMETERS layout, keys strictly
 * increasing, offsets non-decreasing and < n), ds holds the n u64 keys the spline was fitted to.  The knots are
 * copied to the device (the caller's array need not outlive the call); ds must outlive the index.  Refused (before
 * any device work): every result rmi_index_create refuses, then a non-u64 dataset, line_size 0, no knots, knots out
 * of order or past the keys.  The other rmi_index_* calls take either kind of index; on a bounded one:
 *   predict      the generated spline lookup(q, &err) (codegen.rs:410-437): (start, e) = the RMI's predict over the
 *                knots; res = the first knot in [start-e, min(start+e, K)) whose key is not < q (that upper end if
 *                none); res == K: pos = n-1; res == 0: pos = 0 (the generated code reads knots[-1] there);
 *                otherwise t = (double)(q - knots[res-1].key) / (double)(knots[res].key - knots[res-1].key) (wrapping
 *                u64 subtraction), pos = (sat_u64(fma(1-t, offset[res-1], t * offset[res])) / line_size) * line_size
 *                (sat_u64: Rust's saturating `as u64`, NaN -> 0); err = line_size.
 *   lower_bound  exact, as for a plain index: a search of [pos, pos + line_size] (clamped to [0, n]), confirmed by
 *                the keys just outside it when the search ends on an edge, and the galloping fallback (counted)
 *                when it misses — never, for a key of the data set; wrong knots cost fallbacks, not answers. */
int rmi_index_create_bounded(const rmi_result* r, const rmi_spline_point* knots, uint64_t num_knots,
                             uint64_t line_size, const rmi_dataset* ds, rmi_index** out);
void rmi_index_destroy(rmi_index* idx);
/* n queries (ds's key type) in device memory on the index's device; enqueued on cuda_stream, no host sync.
 * One kernel launch per call (n == 0: none).  d_err may be NULL. */
int rmi_index_predict(const rmi_index* idx, const void* d_queries, uint64_t n, uint64_t* d_pos, uint64_t* d_err,
                      void* cuda_stream);
/* Exact lower bounds; *d_fallbacks (may be NULL) is incremented by the number of queries whose window missed. */
int rmi_index_lower_bound(const rmi_index* idx, const void* d_queries, uint64_t n, uint64_t* d_out,
                          uint64_t* d_fallbacks, void* cuda_stream);
/* The same on host arrays, synchronously: copies the queries to the device, runs predict (lower_bound == 0; host_err
 * may be NULL) or lower_bound (*fallbacks, may be NULL, is SET to the fallback count) and copies the results back. */
int rmi_index_lookup_host(const rmi_index* idx, const void* host_queries, uint64_t n, int lower_bound,
                          uint64_t* host_out, uint64_t* host_err, uint64_t* fallbacks);
/* Upper bounds and equal ranges (DESIGN.md section 18), on either kind of index:
 *   upper_bound  the number of keys k with k <= q (std::upper_bound for every non-NaN q; n for q >= the last key).  A
 *                NaN query gives 0, so that equal_range(NaN) is the empty range [0, 0), as lower_bound(NaN) = 0.  Keys
 *                compare by value: -0.0 <= 0.0.  The search runs in the same window as lower_bound's: the model's
 *                error bounds cover the runs of equal keys (the reference widens each leaf's bound by its longest
 *                run), so for a key of the data set the window holds both ends of its run; a query >= the last key
 *                gets n without a search, because the data set's final run is the one no bound records.
 *   equal_range  (lower_bound(q), upper_bound(q)), half-open, in two arrays, from one model evaluation and one window;
 *                d_first is bit-equal to what rmi_index_lower_bound returns.
 * Always exact: a window that misses takes the galloping fallback.  *d_fallbacks (may be NULL) is incremented by the
 * number of queries whose window missed (for equal_range, a query counts once if either end missed); never, for a key
 * of the data set on a plain index.  One kernel launch per call (n == 0: none), enqueued on cuda_stream. */
int rmi_index_upper_bound(const rmi_index* idx, const void* d_queries, uint64_t n, uint64_t* d_out,
                          uint64_t* d_fallbacks, void* cuda_stream);
int rmi_index_equal_range(const rmi_index* idx, const void* d_queries, uint64_t n, uint64_t* d_first,
                          uint64_t* d_last, uint64_t* d_fallbacks, void* cuda_stream);
/* The same on host arrays, synchronously: upper bounds into host_last, and with host_first non-NULL the equal range
 * (lower bounds into host_first).  *fallbacks (may be NULL) is SET to the fallback count. */
int rmi_index_range_host(const rmi_index* idx, const void* host_queries, uint64_t n, uint64_t* host_first,
                         uint64_t* host_last, uint64_t* fallbacks);

/* ---- Updatable indexes: lookups over inserted and removed keys (DESIGN.md section 19) -----------------------------
 * An rmi_delta wraps an rmi_index, plain or bounded, and two device-resident sorted arrays: the keys inserted since
 * that index was built (m keys) and the keys removed since (t keys).  Its logical key set is the multiset
 * base keys ⊎ inserted keys ⊖ removed keys, and every answer is exact over it:
 *   lower_bound(q) = the base index's lower_bound(q) + #{inserted keys < q} - #{removed keys < q}; upper_bound likewise
 *   with <=; equal_range(q) = both.  A NaN query gives [0, 0), as on the base index.  The fallback counts are the base
 *   index's: the delta's part is an exact search and adds none.  The subtraction never drops below 0: every accepted
 *   removal keeps the removed keys a sub-multiset of the base and inserted keys.
 * There is no predict: the model's positions refer to the base keys only.
 * Equal keys keep one order everywhere: base keys before equal inserted keys, earlier inserts before later ones, keys
 * compared by value (-0.0 == 0.0).  A removal of value v takes away the first copy of v's run in that order.  So
 * rmi_delta_merge's keys are the stable sort of the base keys followed by every inserted batch, with the first c(v)
 * copies of every value v dropped, c(v) being how often v was removed.
 * Concurrency: lookups on one rmi_delta may run concurrently on several streams.  rmi_delta_insert, rmi_delta_remove
 * and rmi_delta_destroy must not overlap any other call on the same handle, lookups still in flight on other streams
 * included.  The base index is unchanged and immutable; base (and its dataset) must outlive the rmi_delta. */
typedef struct rmi_delta rmi_delta;
int rmi_delta_create(const rmi_index* base, rmi_delta** out);
void rmi_delta_destroy(rmi_delta* d);
/* Merges a batch into the delta, synchronously: on the calling thread's stream (cudaStreamPerThread), returning when
 * the merge has finished.  The batch must be a sorted data set (batch->sorted, as rmi_dataset_create and
 * rmi_dataset_wrap_device find it) of the base's key type on the base's device; duplicates, of any key, are fine.
 * Refused with RMI_ERR_INVALID: a null argument, another key type or device, an unsorted batch, and (after the merge,
 * which finds it) a float64 batch that holds a NaN.  A refused batch leaves the delta unchanged.  The delta's storage
 * is two device buffers that trade places at every insert; a buffer that is too small is replaced by one of twice
 * the larger capacity (at least the keys it has to hold). */
int rmi_delta_insert(rmi_delta* d, const rmi_dataset* batch);
/* Keys inserted so far (m). */
uint64_t rmi_delta_len(const rmi_delta* d);
/* Removes a batch of keys, synchronously, on the calling thread's stream (cudaStreamPerThread): each key of the batch
 * removes one copy of its value from the logical key set.  The batch must be a sorted data set of the base's key type
 * on the base's device, hold no NaN, and hold no value more often than the logical key set does at the time of the
 * call (values compared by value, so -0.0 == 0.0): a key that is not there, one copy too many, or a copy already
 * removed is refused.  Refused with RMI_ERR_INVALID: a null argument, another key type or device, an unsorted batch,
 * a NaN ("holds a NaN") and too many copies ("does not hold").  A refused batch changes nothing.  The removed keys
 * are stored as the inserted keys are, in two buffers that trade places. */
int rmi_delta_remove(rmi_delta* d, const rmi_dataset* batch);
/* Keys removed so far (t). */
uint64_t rmi_delta_removed_len(const rmi_delta* d);
/* As rmi_index_lower_bound / _upper_bound / _equal_range over the logical key set: the base index's launch, then, on
 * the same stream, one launch that adds the delta's counts to the outputs (none when m == 0 and t == 0, so the
 * answers and the launch count are then the base index's; none at all for n == 0). */
int rmi_delta_lower_bound(const rmi_delta* d, const void* d_queries, uint64_t n, uint64_t* d_out,
                          uint64_t* d_fallbacks, void* cuda_stream);
int rmi_delta_upper_bound(const rmi_delta* d, const void* d_queries, uint64_t n, uint64_t* d_out,
                          uint64_t* d_fallbacks, void* cuda_stream);
int rmi_delta_equal_range(const rmi_delta* d, const void* d_queries, uint64_t n, uint64_t* d_first,
                          uint64_t* d_last, uint64_t* d_fallbacks, void* cuda_stream);
/* The same on host arrays, synchronously: lower bounds into host_first, upper bounds into host_last; either may be
 * NULL, not both.  *fallbacks (may be NULL) is SET to the fallback count. */
int rmi_delta_range_host(const rmi_delta* d, const void* host_queries, uint64_t n, uint64_t* host_first,
                         uint64_t* host_last, uint64_t* fallbacks);
/* A new, owned data set of the n + m - t logical keys on the base's device (the base keys alone for an empty delta;
 * possibly no key at all when every key was removed), in the order given above, with
 * its sorted and no_dups flags found by the same check as rmi_dataset_create's.  Release it with
 * rmi_dataset_destroy.  Compaction trains or evaluates an index over it (rmi_train, rmi_evaluate,
 * rmi_cache_fix_device) and wraps that index in a new rmi_delta. */
int rmi_delta_merge(const rmi_delta* d, rmi_dataset** out);

/* ---- Range-partitioned (multi-GPU) build ----------------------------------------------------
 * One process per GPU; rank r holds the r-th contiguous slab of the globally sorted key array
 * in an rmi_dataset.  The leaf fits are independent once the top model and the leaf boundaries
 * are global, so a build is a sequence of local phases separated by three small collectives
 * that the HOST issues on the buffers below (rmi_b200/sharded.py does it with
 * torch.distributed over NCCL):
 *     RMI_PHASE_TOP_LOCAL   -> first top-model collective  (see rmi_shard_top_rounds)
 *    [RMI_PHASE_TOP_MID     -> second top-model collective; two-round tops only]
 *     RMI_PHASE_TOP_FINISH, RMI_PHASE_BOUNDS
 *                           -> all-reduce MIN  of buffers.S      ((N+1) u64)
 *     RMI_PHASE_SPLIT       -> halo: copy the keys of this rank's last leaf that live on the
 *                              following rank(s) behind the local keys, rmi_shard_set_halo()
 *     RMI_PHASE_LEAF        -> all-reduce SUM  of params / errors / counts (zero where not owned,
 *                              summed as 64-bit integers), all-reduce MAX of buffers.status
 *     RMI_PHASE_STATS, rmi_shard_finish()
 * All phases are enqueued on the caller's CUDA stream and do not synchronise.  The result is
 * identical on every rank and equal to a single-GPU build of the concatenated array (same
 * tolerance rules).  Offered for every top model: linear, robust_linear, linear_spline, cubic,
 * loglinear, normal, lognormal, radix, radix8..28, bradix and histogram (RMI_FLAG_TOP_FIT_EXACT, a
 * serial chain, is single-GPU only). */
typedef struct {          /* what a rank publishes about its slab (host struct) */
  uint64_t first_key_bits, last_key_bits;  /* raw key bits (u32 zero-extended, f64 bit pattern) */
  uint64_t last_run_start;                 /* local index of the first key equal to the last key */
  uint64_t n_local;
  uint64_t no_dups;                        /* 1 if no two LOCAL keys are equal (found when the dataset was created) */
} rmi_shard_ends;
int rmi_shard_ends_get(const rmi_dataset* ds, rmi_shard_ends* out);

typedef struct {          /* device buffers owned by the caller (the collectives run on them) */
  void* sums;             /* 16 x 8 bytes: [0,8) f64 sums (SUM rounds), [8,16) i64 slots (MIN round) */
  void* S;                /* (N+1) x u64 */
  void* params;           /* N x params_per_model x f64 */
  void* errors;           /* N x u64 */
  void* counts;           /* N x u64 */
  void* status;           /* 1 x u32 */
} rmi_shard_buffers;

enum { RMI_PHASE_TOP_LOCAL = 0, RMI_PHASE_TOP_FINISH = 1, RMI_PHASE_BOUNDS = 2, RMI_PHASE_SPLIT = 3,
       RMI_PHASE_LEAF = 4, RMI_PHASE_STATS = 5, RMI_PHASE_TOP_MID = 6, RMI_NUM_PHASES = 7 };

/* Which collectives the top-model fit of a range-partitioned build needs (the host issues them):
 *   -1  this top model is not offered for range-partitioned builds (no model name gives -1 today but unknown ones)
 *    0  none:  TOP_LOCAL, TOP_FINISH                                   (linear_spline, radix:
 *       O(1) functions of the global end keys, cubic_spline.rs / radix.rs need no pass)
 *    1  TOP_LOCAL -> all-reduce SUM of sums[0,8) as f64 -> TOP_FINISH  (linear, robust_linear, loglinear)
 *    2  TOP_LOCAL -> SUM f64 sums[0,8) -> TOP_MID -> SUM f64 sums[0,8) -> TOP_FINISH
 *                                                                       (normal, lognormal)
 *    3  TOP_LOCAL -> all-reduce MIN of sums[8,12) as SIGNED 64-bit integers -> TOP_MID
 *                 -> SUM f64 sums[0,8) -> TOP_FINISH                    (cubic)
 *    4  TOP_LOCAL -> all-reduce of the top model's table, as rmi_shard_top_table describes it -> TOP_FINISH
 *                 radix8..28: MAX of the 2^bits u32 hints; histogram: MAX of the u64 pivots (every entry has one
 *                 writer, the others hold 0); bradix: SUM, wrapping mod 2^32, of the 4 x N u32 per-bin key counts
 *                 of its four candidates (every rank counts its own keys) */
int rmi_shard_top_rounds(const char* top_model_name);

/* rmi_shard_build_create: one rank's build object.  ends_all holds every rank's rmi_shard_ends (rmi_shard_ends_get,
 * gathered over the ranks), as for rmi_shard_index_create; the library derives from it this rank's base, the key before
 * its slab and that key's run start, the global first and last keys and whether the whole key set is duplicate-free.
 * halo_capacity: keys of room behind the local keys in local's device array (rmi_shard_set_halo may fill up to that).
 * Refused before any device work, in this order: a null argument (RMI_ERR_INVALID); the model spec as rmi_train
 * refuses it; a top model not offered here (RMI_ERR_UNSUPPORTED); the ends-table checks of rmi_shard_index_create
 * (world / rank, ends_all[rank] not describing local, slabs out of key order); then rmi_train's checks of the
 * concatenated keys (branching factor 0, no keys, a local dataset that is not sorted: RMI_ERR_PANIC).  The object may
 * run any number of builds with these arguments; local and the buffers must outlive it. */
typedef struct rmi_shard_build rmi_shard_build;
int rmi_shard_build_create(const rmi_dataset* local, const rmi_shard_ends* ends_all, int world, int rank,
                           const char* model_spec, uint64_t branch_factor, uint64_t halo_capacity,
                           const rmi_shard_buffers* buffers, void* cuda_stream, rmi_shard_build** out);
int rmi_shard_phase(rmi_shard_build* b, int phase);
int rmi_shard_set_halo(rmi_shard_build* b, uint64_t halo_keys);

/* The table a code-4 top model (rmi_shard_top_rounds) merges between RMI_PHASE_TOP_LOCAL and RMI_PHASE_TOP_FINISH:
 * `entries` entries of `entry_bytes` bytes (4: u32, 8: u64) at the device pointer `table`, which the host-driven flow
 * all-reduces in place with `op` over the ranks.  The entries are unsigned: a host that reduces them as signed
 * integers must keep the unsigned order (MAX) and the wrap-around mod 2^32 (SUM).  entries == 0 for the top models
 * without a table.  The pointer stays valid for the build object's life. */
enum { RMI_TABLE_REDUCE_MAX = 0, RMI_TABLE_REDUCE_SUM = 1 };
typedef struct {
  void* table;
  uint64_t entries;
  uint32_t entry_bytes;
  uint32_t op;            /* RMI_TABLE_REDUCE_* */
} rmi_shard_top_table_info;
int rmi_shard_top_table(const rmi_shard_build* b, rmi_shard_top_table_info* out);
int rmi_shard_finish(rmi_shard_build* b, uint32_t flags, rmi_result** out);
void rmi_shard_build_destroy(rmi_shard_build* b);
uint32_t rmi_params_per_model(const char* leaf_model_name);

/* The same build in ONE call: all phases and every collective are enqueued on the build's CUDA stream by the
 * library itself (NCCL, bound at run time from libnccl.so.2), with no host round trip between the first kernel
 * and the result copy except one 8 x (world+1)-byte read of the leaf-ownership ranges that overlaps the leaf kernel.
 *     top model      all-reduce SUM of 8 doubles / MIN of 4 x i64 (rmi_shard_top_rounds)
 *     boundaries     all-reduce MIN of (N+1) u64
 *     leaf records   all-gather by ownership range: rank r owns the contiguous leaf range whose first key index
 *                    S[j] lies in its slab and broadcasts exactly that range (north_star: "a single NCCL allgather
 *                    of leaf parameters"); nothing is zero-filled or summed
 *     statistics     each rank reduces the leaves it owns, all-gather of one 40-byte partial per rank
 *     status         all-gather of every rank's status word, OR-ed on the host (a halo that is too small, or a
 *                    panic on any rank, fails the call on EVERY rank with the same message)
 * Setup per communicator: rank 0 calls rmi_shard_comm_unique_id and ships the 128 bytes to the other ranks by any
 * means (rmi_b200/sharded.py: torch.distributed broadcast); every rank then calls rmi_shard_comm_create (collective).
 * Setup per build object: rmi_shard_set_halo, as for the phases; c must have the build's world and rank.  The
 * host-driven rmi_shard_phase flow above remains (CPU tests drive it over gloo). */
typedef struct rmi_shard_comm rmi_shard_comm;
int rmi_shard_comm_unique_id(void* out_id128);
int rmi_shard_comm_create(const void* id128, int world, int rank, int device, rmi_shard_comm** out);
void rmi_shard_comm_destroy(rmi_shard_comm* c);
int rmi_shard_train(rmi_shard_build* b, rmi_shard_comm* c, uint32_t flags, rmi_result** out);

/* ---- The configuration search's unit of work over a range-partitioned data set (DESIGN.md section 9) ------------
 * rmi_train_stats_batch over the slabs: the configurations "top,leaf_k" (k < num_leaf_models) of ONE top model and
 * branching factor, statistics only.  The top model is fitted once and the leaf boundaries derived once, with the
 * collectives of rmi_shard_train; then, for every leaf type, the fused leaf kernel runs over the leaves this rank owns
 * and reduces them to one statistics partial.  One all-gather carries every rank's K RECORDS
 * (RMI_SHARD_STATS_RECORD_BYTES each: the 40-byte partial, then the u32 status word and the u32 "could not replace"
 * flag) and every rank merges them in rank order: the results are identical on every rank, and no leaf record leaves
 * the rank that owns it.  out[k] follows the statistics of rmi_train_stats_batch on the concatenated keys (avg_l2 and
 * avg_log2 are summed over a different tree); it holds no leaf tables.  Release each with rmi_result_free.
 *
 * rmi_shard_stats_batch_create refuses, before any device work, in this order: a null argument or num_leaf_models < 1
 * (RMI_ERR_INVALID); an unknown top or leaf model (RMI_ERR_PANIC); a radix-table leaf (RMI_ERR_UNSUPPORTED); then
 * whatever rmi_shard_build_create refuses (the ends-table checks, the keys).  It returns a build object whose phases
 * RMI_PHASE_TOP_LOCAL .. RMI_PHASE_SPLIT, rmi_shard_top_table and rmi_shard_set_halo work as for a build;
 * RMI_PHASE_LEAF / RMI_PHASE_STATS are refused (RMI_ERR_INVALID).  Of `buffers` it reads sums, S, errors, counts and
 * status (N entries each, whatever the leaf types); params is not used: the leaf parameters go to the batch's own
 * scratch.  Release with rmi_shard_build_destroy.
 *
 * Host-driven form (rmi_b200/sharded.py drives it over gloo): the phases and collectives of a build up to and including
 * RMI_PHASE_SPLIT and the halo, then for k = 0 .. K-1 rmi_shard_stats_leaf, which writes this rank's record of leaf
 * type k at d_record (device memory), then an all-gather of the K records of every rank (world x K records, rank by
 * rank) and rmi_shard_stats_finish over them.  The leaf calls are enqueued on the build's stream without a host
 * synchronisation.
 * One-call form: rmi_shard_train_stats_batch runs all of it on the build's stream over c (NCCL), with no host
 * synchronisation but the final one.
 * A status bit on any rank fails the call on EVERY rank with the same message, prefixed "top,leaf: " of the first leaf
 * type that has one; a leaf that reaches past the halo is reported as by rmi_shard_train ("... past the halo ..."), and
 * the caller may grow the halo and measure again.  flags: none is read (the batch is statistics only).  device_time_ns: the batch's device time shared out evenly
 * (one call: the whole stream, collectives included; host-driven: the sum of the phases). */
#define RMI_SHARD_STATS_RECORD_BYTES 48
int rmi_shard_stats_batch_create(const rmi_dataset* local, const rmi_shard_ends* ends_all, int world, int rank,
                                 const char* top_model, const char* const* leaf_models, int num_leaf_models,
                                 uint64_t branch_factor, uint64_t halo_capacity, const rmi_shard_buffers* buffers,
                                 void* cuda_stream, rmi_shard_build** out);
int rmi_shard_stats_leaf(rmi_shard_build* b, int k, void* d_record);
int rmi_shard_stats_finish(rmi_shard_build* b, const void* d_records, uint32_t flags, rmi_result** out);
int rmi_shard_train_stats_batch(rmi_shard_build* b, rmi_shard_comm* c, uint32_t flags, rmi_result** out);

/* ---- Lookups over a range-partitioned data set (DESIGN.md section 14) ------------------------------------------
 * Every rank holds the whole model and its own slab of the keys; together the slabs are the key set the model was
 * trained on (or evaluated on).  Query q is answered by the last non-empty rank whose first key is < q (the first
 * non-empty rank if none is, a NaN query included): every key before its slab is < q and every key after it is not,
 * so the global lower bound is the slab's base + the lower bound inside the slab, exactly, with no key of another rank
 * read.  predict is local (the model alone); lower_bound moves the queries (4 or 8 bytes each) to their ranks and the
 * 8-byte answers back.
 *
 * rmi_shard_index_create uploads r's tables as rmi_index_create does and binds them to `local`.  ends_all holds every
 * rank's rmi_shard_ends (rmi_shard_ends_get, gathered over the ranks).  Refused before any device work, in this
 * order: a null argument (RMI_ERR_INVALID); every result rmi_index_create refuses (the checks of a given result,
 * before rmi_evaluate); then with RMI_ERR_INVALID: rank / world out of range (1 <= world <= 63);
 * ends_all[rank].n_local != rmi_dataset_len(local); non-empty slabs out of key order (a slab's last key above the
 * next one's first); r->num_rmi_rows != the sum of n_local.  local must outlive the index. */
typedef struct rmi_shard_index rmi_shard_index;
int rmi_shard_index_create(const rmi_result* r, const rmi_dataset* local, const rmi_shard_ends* ends_all, int world,
                           int rank, rmi_shard_index** out);
void rmi_shard_index_destroy(rmi_shard_index* idx);
/* rmi_index_predict over the whole key set (n = the sum of n_local): local, no communication. */
int rmi_shard_index_predict(const rmi_shard_index* idx, const void* d_queries, uint64_t n, uint64_t* d_pos,
                            uint64_t* d_err, void* cuda_stream);
/* The lower bound in phases; the caller exchanges the buffers between them (rmi_b200/sharded.py does it with
 * torch.distributed):
 *   route    d_send (n keys) receives the n queries grouped by rank in rank order, d_send_counts (world u64) the size
 *            of each group, d_slot (n u64) the position of query i in d_send.  Three kernel launches (n == 0: none,
 *            d_send_counts is zeroed).
 *            -> every rank sends group p to rank p; the groups received are concatenated in source-rank order
 *   search   exact global lower bounds of the m received queries, in received order; *d_fallbacks (may be NULL) grows by
 *            the number of those queries whose window missed.  Two launches (the predict kernel, then the window search
 *            over the slab; none for m == 0).  A rank without keys receives no queries (m > 0 there is refused).
 *            -> every rank returns the answers of each source's group to that source, received in rank order
 *   gather   d_out[i] = d_returned[d_slot[i]].  One launch.
 * All calls are enqueued on cuda_stream without a host synchronisation; scratch comes from the stream-ordered pool. */
int rmi_shard_index_route(const rmi_shard_index* idx, const void* d_queries, uint64_t n, void* d_send, uint64_t* d_slot,
                          uint64_t* d_send_counts, void* cuda_stream);
int rmi_shard_index_search(const rmi_shard_index* idx, const void* d_received, uint64_t m, uint64_t* d_answers,
                           uint64_t* d_fallbacks, void* cuda_stream);
int rmi_shard_index_gather(const rmi_shard_index* idx, const uint64_t* d_slot, const uint64_t* d_returned, uint64_t n,
                           uint64_t* d_out, void* cuda_stream);
/* The whole lower bound in one call, collective over c (every rank calls it, n = 0 allowed): route; all-gather of the
 * world x world counts on the stream; one host read of them; grouped ncclSend / ncclRecv of the queries (a rank's own
 * group included); search; grouped send / receive of the answers; gather.  c must have the index's world and rank.
 * Returns after the exchanges are enqueued; the answers are in d_out when cuda_stream reaches them. */
int rmi_shard_index_lower_bound(rmi_shard_index* idx, rmi_shard_comm* c, const void* d_queries, uint64_t n,
                                uint64_t* d_out, uint64_t* d_fallbacks, void* cuda_stream);
/* Upper bounds over the slabs (DESIGN.md section 18), as the lower bound above but routed by <=: query q goes to the last
 * non-empty rank whose first key is <= q (the first non-empty rank if none is, a NaN query included).  Every key
 * before that rank's slab is <= q and every key after it is > q, so the global upper bound (the number of keys <= q;
 * 0 for NaN) is the slab's base + the upper bound inside the slab; the routing differs from the lower bound's only
 * for a query equal to some slab's first key.  route_upper and search_upper are the phases (launches as for route and
 * search; rmi_shard_index_gather completes them), and on a bounded index search_upper searches the key line as
 * lower_bound does (section 18 shows the halo of section 17 still covers its reads).  A query >= the last key of the
 * slab it reaches gets base + n_local without a search, and is not counted.  rmi_shard_index_upper_bound is the
 * one-call form over c, with the exchange code of rmi_shard_index_lower_bound.  All take plain and bounded indexes,
 * with the checks of the lower-bound calls.  An equal range over the slabs is a lower_bound and an upper_bound. */
int rmi_shard_index_route_upper(const rmi_shard_index* idx, const void* d_queries, uint64_t n, void* d_send,
                                uint64_t* d_slot, uint64_t* d_send_counts, void* cuda_stream);
int rmi_shard_index_search_upper(const rmi_shard_index* idx, const void* d_received, uint64_t m, uint64_t* d_answers,
                                 uint64_t* d_fallbacks, void* cuda_stream);
int rmi_shard_index_upper_bound(rmi_shard_index* idx, rmi_shard_comm* c, const void* d_queries, uint64_t n,
                                uint64_t* d_out, uint64_t* d_fallbacks, void* cuda_stream);
/* What the last one-call lookup on this index (rmi_shard_index_lower_bound, rmi_shard_index_upper_bound or, on a
 * bounded index, rmi_shard_index_predict_collective) did (waits for it to finish).  phase_ms: CUDA-event times of
 * route, count exchange with the host read, query exchange, search, answer exchange, gather. */
typedef struct {
  float phase_ms[6];
  uint64_t queries_routed;     /* n: this rank's queries */
  uint64_t queries_searched;   /* m: the queries this rank received and searched, its own included */
  uint64_t queries_kept;       /* of the n, those this rank answered itself */
} rmi_shard_lookup_stats;
int rmi_shard_index_last_stats(const rmi_shard_index* idx, rmi_shard_lookup_stats* out);

/* ---- `--bounded` lookups over a range-partitioned data set (DESIGN.md section 17) ----------------------------------
 * r is the RMI over the K knots of a `--bounded` RMI's cache-fix spline (train_bounded, or the range-partitioned
 * build); every rank holds its slab `local` of the u64 keys and its KNOT SLAB: the knots whose key routes to it by the
 * rule above (the last non-empty rank whose first key is < the knot's key, or the first non-empty rank), global knots
 * [a0, a1) with a0 = the sum of knot_counts over the earlier ranks.  `knots` (num_knots of them) is that slab with a halo:
 * halo_before knots before it and num_knots - halo_before - (a1 - a0) after it, each at least h = 2 e_max + 2 knots or
 * up to the end of the knots, where e_max is r's largest leaf error bound.  The knots are copied to the device.
 *
 * rmi_shard_index_create_bounded returns an rmi_shard_index: rmi_shard_index_route, _search, _gather, the one-call
 * rmi_shard_index_lower_bound and rmi_shard_index_last_stats take it as they take a plain one; rmi_shard_index_predict
 * refuses it (RMI_ERR_INVALID), because no rank holds every knot.  Refused before any device work, in this order: a
 * null argument (RMI_ERR_INVALID); every result rmi_index_create refuses; a dataset that is not u64, line_size 0,
 * num_knots 0; the ends-table checks of rmi_shard_index_create; a rank holding knots but no keys, more ranks holding
 * knots than the route takes; the sum of knot_counts != r->num_rmi_rows; a slab and halo that do not fit knot_counts, a
 * halo below h on a side; knots out of order (keys strictly increasing, offsets non-decreasing) or with offsets past
 * the keys of all slabs; slab knots whose keys route to another rank.  local must outlive the index.
 *
 * lower_bound (routed by key, as for a plain index): the owner evaluates the knot RMI, (start, e), and the knot window
 *              [lower, upper) of rmi_index_create_bounded's predict.  If the closed range [lower, upper] meets
 *              [a0, a1], the answer knot lies in the slab or is the first knot after it and the window lies in the
 *              halo: pos is the single-GPU one, bit for bit, and the line [pos, pos + line_size] is searched inside the
 *              slab.  Otherwise the query is FAR: its answer knot is the window's edge, which may lie past the halo, so
 *              the owner does not evaluate the spline; it searches its whole slab, exactly, and counts the query as a
 *              fallback.  *d_fallbacks grows by the far queries and by the others whose line [pos, pos + line_size]
 *              does not hold their lower bound (the single-GPU count).  Always exact.
 * predict      collective, routed by KNOT INDEX: the querying rank evaluates the knot RMI (start, e) and sends the query
 *              to the rank whose knot slab holds knot max(start - e, 0); that rank holds the whole window and the knot
 *              before it, so d_pos receives rmi_index_predict of the single-GPU bounded index, bit for bit, for every
 *              query, and d_err (may be NULL) line_size.  Phases, with the exchanges of rmi_shard_index_route's:
 *   predict_route   as rmi_shard_index_route, grouped by knot index (five kernel launches; none for n == 0, where
 *                   d_send_counts is zeroed)
 *   predict_search  pos of the m received queries, in received order (one launch; none for m == 0; a rank without
 *                   knots receives none, m > 0 there is refused)
 *   rmi_shard_index_gather
 * rmi_shard_index_predict_collective: the whole predict in one call over c, as rmi_shard_index_lower_bound (phase times
 * in rmi_shard_index_last_stats, which reports the last one-call form of either kind).  The phase calls and the
 * predict calls refuse a plain index (RMI_ERR_INVALID). */
int rmi_shard_index_create_bounded(const rmi_result* r, const rmi_spline_point* knots, uint64_t num_knots,
                                   uint64_t halo_before, const uint64_t* knot_counts, uint64_t line_size,
                                   const rmi_dataset* local, const rmi_shard_ends* ends_all, int world, int rank,
                                   rmi_shard_index** out);
int rmi_shard_index_predict_route(const rmi_shard_index* idx, const uint64_t* d_queries, uint64_t n, uint64_t* d_send,
                                  uint64_t* d_slot, uint64_t* d_send_counts, void* cuda_stream);
int rmi_shard_index_predict_search(const rmi_shard_index* idx, const uint64_t* d_received, uint64_t m, uint64_t* d_pos,
                                   void* cuda_stream);
int rmi_shard_index_predict_collective(rmi_shard_index* idx, rmi_shard_comm* c, const uint64_t* d_queries, uint64_t n,
                                       uint64_t* d_pos, uint64_t* d_err, void* cuda_stream);

/* ---- rmi_evaluate over a range-partitioned data set (DESIGN.md section 15) ----------------------------------------
 * Every rank holds the whole model r and its own slab `local`; the result is rmi_evaluate(concatenation of the slabs, r),
 * bit for bit in every field but the timings, on every rank.  Each rank reads only its own keys: the per-key errors,
 * the runs of equal keys that end on its slab and the widening terms whose key it holds are MAXima of contributions,
 * combined by one all-reduce MAX.  A top model that is not monotone on the keys (across a cut included) fails the
 * evaluation on EVERY rank with rmi_evaluate's message (RMI_ERR_PANIC).
 *
 * rmi_shard_eval_create refuses, before any device work, in this order: a null argument (RMI_ERR_INVALID); every result
 * rmi_evaluate refuses (the checks of a given result, above); the ends-table checks of rmi_shard_index_create (world /
 * rank, ends_all[rank] not describing local, slabs out of key order); then rmi_evaluate's checks of the concatenated
 * keys (branching factor 0, no keys, a local dataset that is not sorted: RMI_ERR_PANIC).  It derives every rank's
 * base, the key before its slab and that key's run start, the next slab's first key and whether the whole key set is
 * duplicate-free from ends_all, and allocates the device buffers of one evaluation.  r and local must outlive the
 * evaluator; r's tables are read again at every evaluation.
 *
 * Phase form (the caller issues the collectives between the calls, rmi_b200/sharded.py does it with torch.distributed):
 *   bounds   uploads r's tables, then the streaming boundary pass over the local keys into d_S ((N+1) u64, n_global
 *            where no local key reaches a leaf)               -> all-reduce MIN of d_S
 *   keys     this rank's contributions into d_partial (2N u64, part_err | part_run) and its status word into *d_status
 *                                                              -> all-reduce MAX of the first rmi_shard_eval_partial_words
 *                                                                 words of d_partial (N when the key set holds no two
 *                                                                 equal keys, else 2N); OR of every rank's status word
 *   finish   error bounds, counts and statistics from d_S and d_partial; waits for the stream of the last call and
 *            returns the result (status: the OR of the ranks' words).
 * bounds and keys are enqueued on cuda_stream without a host synchronisation.
 * rmi_shard_evaluate: the same in one call, the collectives on the evaluator's own stream over c (which must have the
 * evaluator's world and rank).  Flags: RMI_FLAG_STATS_ONLY, RMI_FLAG_LEAF_COUNTS.  num_rmi_rows = num_data_rows = the
 * keys of all slabs.  phase_device_ns: [0] upload, [1] boundaries with their all-reduce, [2] error pass with its
 * all-reduce, [3] statistics; device_time_ns is their sum. */
typedef struct rmi_shard_eval rmi_shard_eval;
int rmi_shard_eval_create(const rmi_result* r, const rmi_dataset* local, const rmi_shard_ends* ends_all, int world,
                          int rank, rmi_shard_eval** out);
void rmi_shard_eval_destroy(rmi_shard_eval* e);
uint64_t rmi_shard_eval_partial_words(const rmi_shard_eval* e);
int rmi_shard_eval_bounds(rmi_shard_eval* e, uint64_t* d_S, void* cuda_stream);
int rmi_shard_eval_keys(rmi_shard_eval* e, const uint64_t* d_S, uint64_t* d_partial, uint32_t* d_status, void* cuda_stream);
int rmi_shard_eval_finish(rmi_shard_eval* e, const uint64_t* d_S, const uint64_t* d_partial, uint32_t status,
                          uint32_t flags, rmi_result** out);
int rmi_shard_evaluate(rmi_shard_eval* e, rmi_shard_comm* c, uint32_t flags, rmi_result** out);

/* ---- `--bounded` support: rmi_lib::cache_fix (reference rmi_lib/src/cache_fix.rs:106-150) ----------
 * The error-bounded spline over key -> first-occurrence offset whose interpolation always lands in
 * the key's line (offset / line_size).  train_bounded (train/mod.rs:156-184) is then
 *     knots = rmi_cache_fix_device(ds);  kds = rmi_dataset_create(knot keys);  rmi_train(kds, ...)
 * — the knots' offsets are 0, 1, 2, ..., i.e. the knot keys are an ordinary sorted duplicate-free
 * data set.  Two forms with the same output, knot for knot:
 *   rmi_cache_fix         the reference's greedy scan on one host core (no device work), over n sorted u64
 *                         host_keys;
 *   rmi_cache_fix_device  the same spline fitted on the device from ds's resident keys, with no host copy of the
 *                         keys (DESIGN.md section 12 gives the method and its speed).
 * *out_points (rmi_spline_point, declared with the lookups above) is owned by the library: release with
 * rmi_spline_free.  Both report the reference's panics as RMI_ERR_PANIC with its messages (fewer keys than the
 * line size, line size 0, a first key of 0). */
int rmi_cache_fix(const uint64_t* host_keys, uint64_t n, uint64_t line_size, rmi_spline_point** out_points,
                  uint64_t* out_count);
/* What a device scan did (rmi_cache_fix_device's optional last argument). */
typedef struct {
  uint64_t chunk_keys;        /* key indices per speculation chunk */
  uint64_t chunks;            /* ceil(n / chunk_keys) */
  uint64_t points;            /* points in the spline's input stream (distinct keys and their key - 1 points) */
  uint64_t stitch_segments;   /* segments the stitch walked to join neighbouring chunks' chains */
  uint64_t fallback_points;   /* points the sequential fallback walked where speculation did not join */
  uint64_t evaluations;       /* spline predictions, all passes */
} rmi_cache_fix_stats;
/* ds: a u64 dataset ("Can only construct a bounded RMI on u64 data", src/main.rs:285-286; other key types and null
 * arguments are RMI_ERR_INVALID, before any device work).  Runs on the calling thread's CUDA stream (as rmi_train),
 * so concurrent calls from several host threads are safe; its device scratch is O(n / chunk_keys) words plus the
 * knots, from the stream-ordered pool, released before return.  Five kernel launches.  stats may be NULL. */
int rmi_cache_fix_device(const rmi_dataset* ds, uint64_t line_size, rmi_spline_point** out_points,
                         uint64_t* out_count, rmi_cache_fix_stats* stats);
void rmi_spline_free(rmi_spline_point* points);

/* ---- rmi_cache_fix_device over a range-partitioned data set (DESIGN.md section 16: method, measured cost) ---------
 * Every rank holds its slab `local` (u64 keys) and, behind it in the same device array, the first halo_keys keys of
 * the following ranks.  The knots of all ranks, in rank order, are rmi_cache_fix_device(concatenation of the slabs),
 * knot for knot.  The point stream is section 12's with global indices: point (global key index g, sub) has pid
 * 2g + sub (sub 0: (key - 1, g), sub 1: (key, g), both at the first index of a run of equal keys only).  A rank's
 * chain starts at an ENTRY pid E: the first point at or after E.  Its EXIT X(E) is the first knot of that chain at or
 * past 2 x (the next rank's base), RMI_SHARD_CACHE_FIX_PID_END when the last segment stays open to the end of the
 * data.  An entry at or past the slab's end, or an empty slab, passes straight through: no knots, X = E, no key read.
 *
 * rmi_shard_cache_fix_create refuses, before any device work, in this order: a null argument (RMI_ERR_INVALID); the
 * ends-table checks of rmi_shard_index_create (world / rank, ends_all[rank] not describing local, slabs out of key
 * order); a dataset that is not u64 and a halo that reaches past the end of the data (RMI_ERR_INVALID); then
 * rmi_cache_fix_device's panics with its messages, decided from ends_all so that every rank fails alike: fewer keys in
 * all slabs than the line size, line size 0, a local dataset that is not sorted, a first key of 0 (RMI_ERR_PANIC).
 * local must outlive the object; its device scratch is about 24 words per 256 local keys.
 *
 * Joining the ranks (the caller issues the collectives; rmi_b200/sharded.py cache_fix_sharded does it with
 * torch.distributed):
 *   1. every rank scans with E = 2 x its base (its own first point); rank 0's entry is the true first knot;
 *   2. all-gather every rank's (E, X, status);
 *   3. every rank r >= 1 whose E differs from X of rank r - 1 scans again with E = that X;
 *   4. repeat 2 and 3 until no entry changes (at most world - 1 more rounds: after round k, ranks 0..k have true
 *      entries);
 *   5. every rank emits its num_knots knots; the counts give the offsets of a gather.
 * scan runs on cuda_stream and waits for it (its result is read on the host).  The first scan runs the speculation
 * and every chunk's stitch; a later one re-runs only the stitch of the slab's first chunk and the resolve.  Status
 * RMI_SHARD_CACHE_FIX_HALO_TOO_SMALL: the chain needs keys past the halo, which does not reach the end of the data;
 * reach is the global index of the first key it could not read.  Nothing may be emitted then: build a new object
 * over a larger halo and start again.  emit writes the knots of the last scan's chain whose pids lie in the slab,
 * then, on the last non-empty rank, finish()'s point (the last key and the global index of its run's first key), to
 * d_out (device memory, num_knots entries), enqueued on cuda_stream without a host synchronisation. */
#define RMI_SHARD_CACHE_FIX_PID_END 0xFFFFFFFFFFFFFFFFull
#define RMI_SHARD_CACHE_FIX_HALO_TOO_SMALL 1u
typedef struct {
  uint64_t exit_pid;    /* X(E) */
  uint64_t num_knots;   /* knots emit writes for this entry, finish()'s point included */
  uint64_t reach;       /* with RMI_SHARD_CACHE_FIX_HALO_TOO_SMALL: the global index of the first key the walk lacked */
  uint32_t status;      /* 0 or RMI_SHARD_CACHE_FIX_HALO_TOO_SMALL */
  uint32_t _pad;
} rmi_shard_cache_fix_scan_result;
typedef struct rmi_shard_cache_fix rmi_shard_cache_fix;
int rmi_shard_cache_fix_create(const rmi_dataset* local, const rmi_shard_ends* ends_all, int world, int rank,
                               uint64_t line_size, uint64_t halo_keys, void* cuda_stream, rmi_shard_cache_fix** out);
int rmi_shard_cache_fix_scan(rmi_shard_cache_fix* cf, uint64_t entry_pid, rmi_shard_cache_fix_scan_result* out);
int rmi_shard_cache_fix_emit(rmi_shard_cache_fix* cf, rmi_spline_point* d_out);
void rmi_shard_cache_fix_destroy(rmi_shard_cache_fix* cf);

/* ---- The rest of rmi_lib's public surface (host-side code, no device work of their own) ---------
 * rmi_lib::rmi_size (codegen.rs:375-394): bytes of the model's parameters (+ 8 per leaf with the
 * last-layer errors, + 16 per spline knot of a bounded RMI). */
uint64_t rmi_model_size(const rmi_result* r, int include_errors, uint64_t num_spline_points);

/* rmi_lib::output_rmi (codegen.rs:757-788): writes <out_dir>/<ns>.cpp, <ns>.h, <ns>_data.h and the
 * parameter blobs <data_dir>/<ns>_L{i}_PARAMETERS, byte for byte in the reference's layouts.
 * key_type: the KeyType handed to codegen (src/main.rs:122-132: uint32 FILES keep RMI_KEY_U64).
 * knots != NULL: a `--bounded` RMI (TrainedRMI.cache_fix = (line_size, knots); num_data_rows = the
 * length of the ORIGINAL data set, train/mod.rs:175-176).  `r` must hold the leaf tables (not
 * RMI_FLAG_STATS_ONLY). */
int rmi_output_rmi(const char* ns, const rmi_result* r, const char* data_dir, const char* out_dir, int key_type,
                   int include_errors, uint64_t build_time_ns, const rmi_spline_point* knots, uint64_t num_knots,
                   uint64_t line_size, uint64_t num_data_rows);

/* What rmi_load_rmi found in an artefact besides the model. */
typedef struct {
  int key_type;            /* RMI_KEY_U64 or RMI_KEY_F64: the lookup signature's key type */
  int has_errors;          /* 0: a --no-errors artefact; the result's l1_errors is NULL */
  uint64_t line_size;      /* --bounded: the cache-fix line size; 0 otherwise */
  uint64_t num_knots;      /* --bounded: knots returned in *knots (free with rmi_spline_free); 0 otherwise */
  uint64_t num_data_rows;  /* --bounded: total_keys; otherwise num_rmi_rows */
  uint64_t build_time_ns;  /* BUILD_TIME_NS */
} rmi_artefact_info;
/* The inverse of rmi_output_rmi (host code, no device work): reads <out_dir>/<ns>.cpp, <ns>.h, <ns>_data.h and the
 * blobs under data_dir, in the forms the reference's code generator writes, and rebuilds the two-layer model as a
 * result (release with rmi_result_free).  linear, robust_linear and linear_spline generate the same code and load as
 * RMI_MODEL_LINEAR.  The artefact holds no statistics: the model_avg_* / model_max_log2_error fields are NaN and
 * model_max_error(_idx) 0; rmi_evaluate measures them.  build_time_ns = BUILD_TIME_NS, the timings are 0.  *knots is
 * NULL unless the artefact is --bounded.  A malformed artefact (missing or truncated blob, wrong namespace, unknown
 * function, bad constant, sizes that disagree, RMI_SIZE included) is RMI_ERR_INVALID with the file named in
 * rmi_last_error(); a --bounded artefact without errors, whose generated code does not compile, RMI_ERR_UNSUPPORTED. */
int rmi_load_rmi(const char* ns, const char* out_dir, const char* data_dir, rmi_result** out, rmi_spline_point** knots,
                 rmi_artefact_info* info);

/* optimizer::find_pareto_efficient_configs (optimizer.rs:233-249): the two-phase search over
 * (models, branching factor); every candidate is one stats-only build.  `replicas` are
 * rmi_datasets holding the SAME keys on one or more devices (rmi_dataset_replicate): the
 * independent builds are spread over them, one host thread per replica.  RMI_OPTIMIZER_PROFILE
 * (fast | memory | disk) selects the grid as in the reference (optimizer.rs:15-57).  At most
 * `capacity` entries are written, sorted by average log2 error; *out_count = size of the front. */
typedef struct {
  char models[64];
  uint64_t branching_factor;
  double average_log2_error, max_log2_error;
  uint64_t size;
} rmi_config_stats;
int rmi_find_pareto_efficient_configs(const rmi_dataset* const* replicas, int num_replicas, uint64_t restrict_to,
                                      uint32_t flags, rmi_config_stats* out, uint64_t capacity, uint64_t* out_count);
/* The same search with the caller's measuring step: measure(ctx, top, bf, leaves, K, flags, out) fills out[k]'s
 * average_log2_error, max_log2_error and size (rmi_model_size(r, 1, 0) of a result) for the configurations
 * "top,leaves[k]" at branching factor bf, and returns 0; any other value stops the search, which then fails with
 * RMI_ERR_PANIC and the message the callback left in rmi_last_error() (if any).  The callback runs on the calling thread,
 * once per (top, branching factor) group of each phase, every group whole, smallest branching factor first (the order of
 * the replicas' sweep).  rmi_b200/sharded.py measures range-partitioned slabs with it. */
typedef int (*rmi_measure_group_fn)(void* ctx, const char* top_model, uint64_t branch_factor, const char* const* leaf_models,
                                    int num_leaf_models, uint32_t flags, rmi_config_stats* out);
int rmi_find_pareto_efficient_configs_with(rmi_measure_group_fn measure, void* ctx, uint64_t restrict_to, uint32_t flags,
                                           rmi_config_stats* out, uint64_t capacity, uint64_t* out_count);

/* rmi_train keeps one CUDA stream set and one device scratch buffer per host thread and device (created on first use,
 * grown to the largest build and reused by later builds; results never live in it).  A worker thread that will not
 * build again releases them with this call before it exits (the optimizer's per-replica workers do); the main
 * thread's are reclaimed at process exit. */
void rmi_thread_release(void);

/* Message of the last failure on the calling thread ("" if none). */
const char* rmi_last_error(void);
/* Number of kernels this library has launched in this process (bench.py's gpu_launches). */
uint64_t rmi_kernel_launch_count(void);
/* Library / build identification, e.g. "rmi_b200 0.1 (sm_90a)". */
const char* rmi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* RMI_B200_H_ */
