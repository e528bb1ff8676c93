// api.cu — the C ABI of librmi_b200.so (include/rmi_b200.h): datasets in HBM, the
// rmi_lib::train replacement, result marshalling, error text.
//
// One rmi_train call = the calling thread's build stream and device scratch (BuildContext,
// reused by that thread's later calls); the dataset is read-only and may be shared by
// concurrent calls (reference optimizer.rs:224 trains many configurations on one shared
// RMITrainingData).  No host synchronisation happens between the first kernel and the final
// result copy, and a call synchronises once.
#include <algorithm>
#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>
#include <atomic>
#include <chrono>
#include <cstdlib>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/rmi_b200.h"
#include "kernels.h"
#include "nccl_dl.h"
#include "../../host/cache_fix.hpp"
#include "../../host/artefact_load.hpp"
#include "../../host/codegen.hpp"
#include "../../host/optimizer.hpp"
#include "../../host/slab_layout.hpp"

using namespace rmi;

namespace {

thread_local std::string g_last_error;
std::atomic<uint64_t> g_launches{0};

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}
#define CUDA_TRY(expr)                                                                             \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      return fail(RMI_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));               \
  } while (0)

size_t key_bytes(int kt) { return kt == RMI_KEY_U32 ? 4 : 8; }

struct DeviceInfo { int num_sms = 0; };
int device_info(int device, DeviceInfo* out) {
  static std::mutex mu;
  static std::vector<DeviceInfo> cache;
  std::lock_guard<std::mutex> lk(mu);
  if ((int)cache.size() <= device) cache.resize(device + 1);
  if (cache[device].num_sms == 0) {
    int sms = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    cache[device].num_sms = sms;
    // keep the stream-ordered scratch pool's memory mapped between builds instead of
    // returning it to the driver at every synchronisation
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
      unsigned long long keep = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
  }
  *out = cache[device];
  return RMI_OK;
}

// fparams / iparams: how many of TopModel::f / ::ip the model uses as a top model (models.cuh: TopModel).
// root_only: the model may only be the root (train/mod.rs:59-85).
// shard_rounds: rmi_shard_top_rounds (include/rmi_b200.h); -1 where range-partitioned builds do not offer the top.
struct ModelName { const char* name; int kind; int table_bits; int fparams, iparams; bool root_only; int shard_rounds; };
const ModelName kModels[] = {   // reference train/mod.rs:37-54
    {"linear", M_LINEAR, 0, 2, 0, false, 1},          {"robust_linear", M_ROBUST_LINEAR, 0, 2, 0, false, 1},
    {"linear_spline", M_LINEAR_SPLINE, 0, 2, 0, false, 0}, {"cubic", M_CUBIC, 0, 4, 0, false, 3},
    {"loglinear", M_LOGLINEAR, 0, 2, 0, false, 1},   {"normal", M_NORMAL, 0, 3, 0, false, 2},
    {"lognormal", M_LOGNORMAL, 0, 3, 0, false, 2},    {"radix", M_RADIX, 0, 0, 2, true, 0},
    {"radix8", M_RADIX_TABLE, 8, 0, 1, false, 4},     {"radix18", M_RADIX_TABLE, 18, 0, 1, false, 4},
    {"radix22", M_RADIX_TABLE, 22, 0, 1, false, 4},   {"radix26", M_RADIX_TABLE, 26, 0, 1, false, 4},
    {"radix28", M_RADIX_TABLE, 28, 0, 1, false, 4},   {"bradix", M_BRADIX, 0, 0, 3, true, 4},
    {"histogram", M_HISTOGRAM, 0, 0, 1, true, 4}};

const ModelName* find_model(const std::string& s) {
  for (const auto& m : kModels) if (s == m.name) return &m;
  return nullptr;
}

// The model table entry of a result's model id: a radix table by its table bits, except for a leaf, whose width a
// result does not record (any radix table matches, and check_leaf refuses it).
const ModelName* model_of(uint32_t kind, uint32_t table_bits, bool leaf) {
  for (const auto& m : kModels)
    if (m.kind == (int)kind && (kind != M_RADIX_TABLE || leaf || m.table_bits == (int)table_bits)) return &m;
  return nullptr;
}

// ---- the reference's checks of a model spec and of a build's arguments, in rmi_train's order ----------------
int find_layer(const std::string& name, bool is_root, const ModelName** out) {
  const ModelName* m = find_model(name);
  if (!m) return fail(RMI_ERR_PANIC, "Unknown model type: " + name);
  if (m->root_only && !is_root) return fail(RMI_ERR_PANIC, "if used, model type " + name + " must be the root model");
  *out = m;
  return RMI_OK;
}

// who: what the message starts with ("" for a build)
int check_leaf(const ModelName* leaf, const std::string& who = "") {
  if (leaf->kind == M_RADIX_TABLE)
    return fail(RMI_ERR_UNSUPPORTED, who + "radix tables are only offered as the top model in this build");
  return RMI_OK;
}

// train/mod.rs:104-125: split the spec on ',', validate every layer, then insist on two layers
int parse_two_layer(const char* spec, const ModelName** top, const ModelName** leaf) {
  std::vector<const ModelName*> models;
  std::string s(spec);
  for (size_t pos = 0;;) {
    const size_t c = s.find(',', pos);
    const ModelName* m = nullptr;
    if (int rc = find_layer(s.substr(pos, c == std::string::npos ? std::string::npos : c - pos), models.empty(), &m)) return rc;
    models.push_back(m);
    if (c == std::string::npos) break;
    pos = c + 1;
  }
  if (models.size() != 2)   // train/mod.rs:123-125 panic!() for anything but two layers
    return fail(RMI_ERR_PANIC, "only two-layer RMIs can be trained (the reference panics on other depths)");
  *top = models[0];
  *leaf = models[1];
  return check_leaf(*leaf);
}

int check_build(uint64_t n, uint64_t N, bool sorted) {
  if (N < 1) return fail(RMI_ERR_PANIC, "branching factor must be at least 1");
  if (n == 0) return fail(RMI_ERR_PANIC, "start index was 0 but end index was 0");
  if (!sorted) return fail(RMI_ERR_PANIC, "keys are not sorted in ascending order");
  return RMI_OK;
}

// The check of a given trained result that rmi_evaluate and the indexes make first, before they read a dataset: the
// leaf tables (with the error bounds if the caller serves them), models of the model table with a leaf model that is
// not root-only, and the top model's tables.  Every (kind, table bits) it accepts has a lookup kernel
// (lookup_top_group / lookup_leaf_group).  *top / *leaf (may be null) receive r's models.  Messages name fn.
int check_result(const rmi_result* r, bool needs_errors, const std::string& fn, const ModelName** top = nullptr,
                 const ModelName** leaf = nullptr) {
  if (!r->l1_params || (needs_errors && !r->l1_errors))
    return fail(RMI_ERR_INVALID, fn + ": the result holds no leaf tables (RMI_FLAG_STATS_ONLY, or a rank other than 0 "
                                      "of an RMI_FLAG_SHARD_ROOT_ONLY build)");
  const ModelName* t = model_of(r->l0_model_id, r->l0_table_bits, false);
  const ModelName* l = model_of(r->l1_model_id, 0, true);
  if (!t || !l || l->root_only)
    return fail(RMI_ERR_INVALID, fn + ": unknown model id (top " + std::to_string(r->l0_model_id) + ", leaf " +
                                     std::to_string(r->l1_model_id) + ")");
  if (int rc = check_leaf(l, fn + ": ")) return rc;
  if (r->l1_params_per_model != (uint32_t)leaf_params_per_model(l->kind))
    return fail(RMI_ERR_INVALID, fn + ": wrong number of leaf parameters");
  if (t->kind == M_RADIX_TABLE && (!r->l0_table32 || r->l0_table32_len != ((uint64_t)1 << t->table_bits)))
    return fail(RMI_ERR_INVALID, fn + ": radix table missing or of the wrong size");
  if (t->kind == M_HISTOGRAM && (!r->l0_array2 || !r->l0_array2_len))
    return fail(RMI_ERR_INVALID, fn + ": histogram pivots missing");
  if (t->kind == M_HISTOGRAM && r->l0_array1_len && !r->l0_array1)
    return fail(RMI_ERR_INVALID, fn + ": histogram radix index missing");
  if (top) *top = t;
  if (leaf) *leaf = l;
  return RMI_OK;
}

// f(T()) with T the C++ type of an rmi_key_type
template <class F> auto with_key_type(int key_type, F&& f) {
  switch (key_type) {
    case RMI_KEY_U64: return f(u64());
    case RMI_KEY_U32: return f(u32());
    default: return f(double());
  }
}

std::string status_text(unsigned st) {
  struct { unsigned bit; const char* text; } table[] = {
      {ST_NOT_SORTED, "keys are not sorted in ascending order"},
      {ST_NON_MONOTONE, "assertion failed: target >= last_target (top model is not monotonic on this data)"},
      {ST_SPLIT_AT_ZERO, "start index was 0 but end index was 0"},
      {ST_SPLIT_AT_END, "start index was n but end index was n (split at the last key)"},
      {ST_TOP_OUT_OF_BOUNDS, "Top model gave an index which is out of bounds"},
      {ST_NUM_BITS, "assertion failed: nbits >= 1"},
      {ST_CUBIC_UNWRAP, "called `Option::unwrap()` on a `None` value (cubic: no interior point)"},
      {ST_ROBUST_TOO_SMALL, "assertion failed: bnd * 2 + 1 < data.len()"},
      {ST_HIST_BINS, "not enough items for equidepth histogram"},
      {ST_NEG_VARIANCE, "variance of model was negative"},
      {ST_BRADIX_OOB, "index out of bounds (bradix chi2 counts)"},
      {ST_RADIX_TABLE_OOB, "assertion failed: current_radix < hint_table.len()"}};
  std::string out;
  for (auto& e : table)
    if (st & e.bit) { if (!out.empty()) out += "; "; out += e.text; }
  return out;
}

}  // namespace

namespace rmi {
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
}  // namespace rmi

struct rmi_dataset {
  void* d_keys = nullptr;
  uint64_t n = 0;
  int key_type = 0;
  int device = 0;
  bool owned = false;
  bool pooled = false;  // d_keys came from the stream-ordered pool (cudaMallocAsync)
  bool sorted = true;   // verified once, when the dataset is created (the data is immutable)
  bool no_dups = false; // found at the same time: no two keys are equal (kernels drop the duplicate tracking)
};

namespace {
// The reference requires sorted input (README.md:26-31) and otherwise trips over its own
// monotonicity assertion (two_layer.rs:50).  The check is one streaming pass, done once per
// dataset instead of once per build; every build on an unsorted dataset then fails fast.
int verify_sorted(rmi_dataset* ds) {
  if (ds->n < 2) return RMI_OK;
  if ((reinterpret_cast<uintptr_t>(ds->d_keys) & 15u) != 0)
    return fail(RMI_ERR_INVALID, "device key arrays must be 16-byte aligned");
  DeviceInfo di;
  if (int rc = device_info(ds->device, &di)) return rc;
  unsigned* d_flag = nullptr;
  CUDA_TRY(cudaMalloc(&d_flag, sizeof(unsigned)));
  cudaMemset(d_flag, 0, sizeof(unsigned));
  Launch L{nullptr, di.num_sms};
  with_key_type(ds->key_type, [&](auto k) {
    using T = decltype(k);
    check_sorted<T>(L, (const T*)ds->d_keys, ds->n, 0, ds->n, d_flag);
  });
  unsigned h = 0;
  cudaError_t e = cudaMemcpy(&h, d_flag, sizeof(unsigned), cudaMemcpyDeviceToHost);
  cudaFree(d_flag);
  if (e != cudaSuccess) return fail(RMI_ERR_CUDA, std::string("sortedness check: ") + cudaGetErrorString(e));
  ds->sorted = (h & 1u) == 0;
  ds->no_dups = (h & 2u) == 0;
  return RMI_OK;
}
}  // namespace

// Page-locked host buffers for results: D2H copies land directly in the memory the caller
// reads (no pageable staging), and freed buffers are recycled because cudaMallocHost /
// cudaFreeHost cost far more than a build.
class PinnedCache {
 public:
  void* get(size_t bytes) {
    if (bytes == 0) return nullptr;
    {
      std::lock_guard<std::mutex> lk(mu_);
      size_t best = free_.size();
      for (size_t i = 0; i < free_.size(); ++i)
        if (free_[i].second >= bytes && (best == free_.size() || free_[i].second < free_[best].second)) best = i;
      if (best != free_.size() && free_[best].second <= 2 * bytes + 4096) {
        auto e = free_[best];
        free_.erase(free_.begin() + best);
        live_.push_back(e);
        return e.first;
      }
    }
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr;
    std::lock_guard<std::mutex> lk(mu_);
    live_.push_back({p, bytes});
    return p;
  }
  void put(void* p) {
    if (!p) return;
    std::lock_guard<std::mutex> lk(mu_);
    for (size_t i = 0; i < live_.size(); ++i)
      if (live_[i].first == p) {
        free_.push_back(live_[i]);
        live_.erase(live_.begin() + i);
        break;
      }
    // keep at most 16 buffers AND at most 256 MiB of page-locked memory in the free list (a radix26/28 or histogram
    // sweep would otherwise pin gigabytes for good)
    size_t bytes = 0;
    for (auto& e : free_) bytes += e.second;
    while (!free_.empty() && (free_.size() > 16 || bytes > ((size_t)256 << 20))) {
      bytes -= free_.front().second;
      cudaFreeHost(free_.front().first);
      free_.erase(free_.begin());
    }
  }
 private:
  std::mutex mu_;
  std::vector<std::pair<void*, size_t>> free_, live_;
};
PinnedCache g_pinned;

template <class P> struct PinnedArray {
  P* ptr = nullptr;
  size_t count = 0;
  bool resize(size_t n) {
    g_pinned.put(ptr);
    ptr = (P*)g_pinned.get(n * sizeof(P));
    count = ptr ? n : 0;
    return n == 0 || ptr != nullptr;
  }
  P* data() { return ptr; }
  size_t size() const { return count; }
  bool empty() const { return count == 0; }
  ~PinnedArray() { g_pinned.put(ptr); }
};

// The allocation behind an rmi_result: the public struct first, then the owned buffers.
struct ResultBox {
  rmi_result pub;
  PinnedArray<double> l1_params;
  PinnedArray<uint64_t> l1_errors, l1_counts;
  PinnedArray<uint32_t> table32;
  PinnedArray<uint64_t> arr1, arr2;
  PinnedArray<char> scalars;   // BuildAux + TopModel read-back
  std::unique_ptr<rmihost::LoadedArtefact> loaded;   // rmi_load_rmi: owns the tables (host memory, no device needed)
};

namespace {

// An Alloc for TopTables that outlive the call (rmi_index, rmi_shard_build): null if cudaMalloc failed.
void* device_alloc(size_t bytes) {
  void* p = nullptr;
  return cudaMalloc(&p, bytes) == cudaSuccess ? p : nullptr;
}

// The device tables of a table top: radix8..28's hint table, the histogram's pivots and, in a build, its radix index;
// in a range-partitioned build, bradix's per-bin counts (not part of any result).
struct TopTables {
  u32* t32 = nullptr;
  u64* pivots = nullptr;        // hist_bins (+ 1 in a build)
  u64* radix_index = nullptr;   // ri_len; a build's output only: no kernel reads it through TopModel
  u32* bradix_counts = nullptr; // bradix_len = 4 x N: every candidate's count of keys per bin (shard_bradix_count)
  u64 t32_len = 0, ri_len = 0;
  u64 hist_bins = 0, hist_ipb = 0;
  u64 bradix_len = 0;

  // alloc(bytes) returns device memory or null; false if an allocation failed
  template <class Alloc> bool allocate(const ModelName& top, uint64_t n, uint64_t N, Alloc&& alloc) {
    if (top.kind == M_RADIX_TABLE) {
      t32_len = (u64)1 << top.table_bits;
      t32 = (u32*)alloc(sizeof(u32) * t32_len);
      return t32 != nullptr;
    }
    if (top.kind == M_HISTOGRAM) {
      histogram_bins(n, N, &hist_bins, &hist_ipb);
      ri_len = ((u64)1 << 20) + 1;
      pivots = (u64*)alloc(sizeof(u64) * (hist_bins + 1));
      radix_index = (u64*)alloc(sizeof(u64) * ri_len);
      return pivots && radix_index;
    }
    return true;
  }

  // A range-partitioned build's bradix counts (the single-GPU fit takes bin boundaries from its scratch instead).
  template <class Alloc> bool allocate_shard_counts(const ModelName& top, uint64_t N, Alloc&& alloc) {
    if (top.kind != M_BRADIX) return true;
    bradix_len = 4 * (u64)N;
    bradix_counts = (u32*)alloc(sizeof(u32) * bradix_len);
    return bradix_counts != nullptr;
  }

  // The tables of a given result's top model (check_result passed), allocated with alloc and copied on st: the first
  // CUDA error, cudaErrorMemoryAllocation where alloc returned null.  Of the histogram's radix index only the length
  // is kept: the lookups and the error pass read the pivots alone.
  template <class Alloc> cudaError_t upload(const rmi_result& r, cudaStream_t st, Alloc&& alloc) {
    if (r.l0_model_id == M_RADIX_TABLE) {
      t32_len = r.l0_table32_len;
      t32 = (u32*)alloc(sizeof(u32) * t32_len);
      if (!t32) return cudaErrorMemoryAllocation;
      return cudaMemcpyAsync(t32, r.l0_table32, sizeof(u32) * t32_len, cudaMemcpyHostToDevice, st);
    }
    if (r.l0_model_id == M_HISTOGRAM) {
      hist_bins = r.l0_array2_len;
      ri_len = r.l0_array1_len;
      pivots = (u64*)alloc(sizeof(u64) * hist_bins);
      if (!pivots) return cudaErrorMemoryAllocation;
      return cudaMemcpyAsync(pivots, r.l0_array2, sizeof(u64) * hist_bins, cudaMemcpyHostToDevice, st);
    }
    return cudaSuccess;
  }

  // The TopModel of a given result, pointing at the tables upload() placed.
  TopModel given(const rmi_result& r) const {
    TopModel h;
    memset(&h, 0, sizeof(h));
    h.kind = (int)r.l0_model_id;
    h.high = (int)r.l0_bradix_high;
    h.table_bits = (int)r.l0_table_bits;
    for (int q = 0; q < 4; ++q) { h.f[q] = r.l0_fparams[q]; h.ip[q] = r.l0_iparams[q]; }
    h.t32 = t32;
    h.pivots = pivots;
    h.npivots = hist_bins;
    return h;
  }

  // Frees tables placed with device_alloc.
  void free_device() {
    cudaFree(t32);
    cudaFree(pivots);
    cudaFree(radix_index);
    cudaFree(bradix_counts);
  }

  // The TopModel a build starts from; f: nf injected top parameters, or null.
  TopModel initial(const ModelName& top, const double* f = nullptr, uint32_t nf = 0) const {
    TopModel h;
    memset(&h, 0, sizeof(h));
    h.kind = top.kind;
    h.high = 1;
    h.table_bits = top.table_bits;
    h.t32 = t32;
    h.pivots = pivots;
    h.npivots = hist_bins;
    if (top.kind == M_HISTOGRAM) h.ip[0] = hist_bins;
    for (uint32_t q = 0; f && q < nf && q < 4; ++q) h.f[q] = f[q];
    return h;
  }
};

// Takes the pinned buffers a build's result is copied into: the scalars, the leaf tables if `leaves` (and the key
// counts if `counts`), and the top model's tables if `tables` is given.  False if page-locked memory ran out.
bool reserve_result(ResultBox* box, const TopTables* tables, uint64_t N, int ppm, bool leaves, bool counts) {
  bool ok = box->scalars.resize(sizeof(BuildAux) + sizeof(TopModel));
  if (ok) memset(box->scalars.data(), 0, sizeof(BuildAux) + sizeof(TopModel));
  if (leaves) ok = ok && box->l1_params.resize((size_t)N * ppm) && box->l1_errors.resize(N);
  if (leaves && counts) ok = ok && box->l1_counts.resize(N);
  if (tables && tables->t32_len) ok = ok && box->table32.resize(tables->t32_len);
  if (tables && tables->ri_len) ok = ok && box->arr1.resize(tables->ri_len);
  if (tables && tables->hist_bins) ok = ok && box->arr2.resize(tables->hist_bins);
  return ok;
}
const char* const kPinnedFailed = "pinned host allocation for the results failed";

// Issues the copies into the buffers reserve_result took: BuildAux and TopModel, then the leaf tables (params null:
// none, or already copied; counts null: none), then the top model's tables (tables null: none).
void copy_result_to_host(ResultBox* box, const TopTables* tables, const BuildAux* d_aux, const TopModel* d_top,
                         const double* params, const u64* errors, const u64* counts, cudaStream_t st) {
  cudaMemcpyAsync(box->scalars.data(), d_aux, sizeof(BuildAux), cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(box->scalars.data() + sizeof(BuildAux), d_top, sizeof(TopModel), cudaMemcpyDeviceToHost, st);
  if (params) {
    cudaMemcpyAsync(box->l1_params.data(), params, sizeof(double) * box->l1_params.size(), cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(box->l1_errors.data(), errors, sizeof(u64) * box->l1_errors.size(), cudaMemcpyDeviceToHost, st);
    if (counts) cudaMemcpyAsync(box->l1_counts.data(), counts, sizeof(u64) * box->l1_counts.size(), cudaMemcpyDeviceToHost, st);
  }
  if (tables && tables->t32_len)
    cudaMemcpyAsync(box->table32.data(), tables->t32, sizeof(u32) * tables->t32_len, cudaMemcpyDeviceToHost, st);
  if (tables && tables->ri_len) {
    cudaMemcpyAsync(box->arr1.data(), tables->radix_index, sizeof(u64) * tables->ri_len, cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(box->arr2.data(), tables->pivots, sizeof(u64) * tables->hist_bins, cudaMemcpyDeviceToHost, st);
  }
}

const BuildAux& result_aux(const ResultBox* box) { return *reinterpret_cast<const BuildAux*>(box->scalars.ptr); }

// The public struct from what copy_result_to_host brought back (the stream synchronised): the statistics
// (two_layer.rs:267-284), the top model, the leaf model and the tables the box holds.  The top tables' lengths are
// filled in even where the tables stay on the device: rmi_model_size reads them.
void fill_result(ResultBox* box, const ModelName& top, const ModelName& leaf, const TopTables& tables, uint64_t n,
                 uint64_t N) {
  const BuildAux& a = result_aux(box);
  const TopModel& t = *reinterpret_cast<const TopModel*>(box->scalars.ptr + sizeof(BuildAux));
  rmi_result& R = box->pub;
  memset(&R, 0, sizeof(R));
  R.num_rmi_rows = n; R.num_data_rows = n; R.branching_factor = N;
  R.model_max_error = a.max_error;
  R.model_max_error_idx = a.max_error_idx;
  R.model_avg_error = (double)a.sum_n_err / (double)n;
  R.model_avg_l2_error = a.sum_l2;
  R.model_avg_log2_error = a.sum_log2 / (double)n;
  R.model_max_log2_error = std::log2((double)a.max_error);
  R.l0_model_id = top.kind;
  R.l0_bradix_high = t.high;
  R.l0_table_bits = top.table_bits;
  R.l0_num_fparams = top.fparams;
  R.l0_num_iparams = top.iparams;
  for (int q = 0; q < 4; ++q) { R.l0_fparams[q] = t.f[q]; R.l0_iparams[q] = t.ip[q]; }
  R.l0_table32_len = tables.t32_len;
  R.l0_table32 = box->table32.empty() ? nullptr : box->table32.data();
  R.l0_array1_len = tables.ri_len;
  R.l0_array1 = box->arr1.empty() ? nullptr : box->arr1.data();
  R.l0_array2_len = tables.hist_bins;
  R.l0_array2 = box->arr2.empty() ? nullptr : box->arr2.data();
  R.l1_model_id = leaf.kind;
  R.l1_params_per_model = leaf_params_per_model(leaf.kind);
  R.l1_params = box->l1_params.empty() ? nullptr : box->l1_params.data();
  R.l1_errors = box->l1_errors.empty() ? nullptr : box->l1_errors.data();
  R.l1_counts = box->l1_counts.empty() ? nullptr : box->l1_counts.data();
  R.could_not_replace = a.could_not_replace ? 1 : 0;
}

uint64_t elapsed_ns(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0.f;
  cudaEventElapsedTime(&ms, a, b);
  return (uint64_t)((double)ms * 1e6);
}

}  // namespace

extern "C" {

const char* rmi_last_error(void) { return g_last_error.c_str(); }
uint64_t rmi_kernel_launch_count(void) { return g_launches.load(); }
const char* rmi_version(void) { return "rmi_b200 0.1 (sm_90a)"; }

int rmi_dataset_create(const void* host_keys, uint64_t n, rmi_key_type key_type, int device, rmi_dataset** out) {
  if (!out || (!host_keys && n) || (int)key_type < 0 || (int)key_type > 2)
    return fail(RMI_ERR_INVALID, "rmi_dataset_create: bad argument");
  CUDA_TRY(cudaSetDevice(device));
  DeviceInfo di;
  if (int rc = device_info(device, &di)) return rc;   // also pins the pool's release threshold
  auto* ds = new rmi_dataset();
  ds->n = n; ds->key_type = key_type; ds->device = device; ds->owned = true; ds->pooled = true;
  const size_t kb = key_bytes(key_type), bytes = (size_t)n * kb;
  if (bytes == 0) { *out = ds; return RMI_OK; }
  // The key array comes from the stream-ordered pool (a re-created dataset of the same size
  // costs no driver allocation), the copy runs in 64 MiB pieces and the sortedness check of
  // piece c runs behind the copy of piece c+1.
  cudaStream_t st = nullptr;
  unsigned* d_flag = nullptr;
  cudaError_t e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMallocAsync(&ds->d_keys, (bytes + 15) & ~(size_t)15, st);
  if (e == cudaSuccess) e = cudaMallocAsync((void**)&d_flag, sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_flag, 0, sizeof(unsigned), st);
  unsigned h_flag = 0;
  if (e == cudaSuccess) {
    const uint64_t CH = ((uint64_t)64 << 20) / kb;   // keys per piece (multiple of 4)
    Launch L{st, di.num_sms};
    for (uint64_t i0 = 0; i0 < n && e == cudaSuccess; i0 += CH) {
      const uint64_t i1 = std::min<uint64_t>(n, i0 + CH);
      e = cudaMemcpyAsync((char*)ds->d_keys + i0 * kb, (const char*)host_keys + i0 * kb, (i1 - i0) * kb,
                          cudaMemcpyHostToDevice, st);
      with_key_type(key_type, [&](auto k) {
        using T = decltype(k);
        check_sorted<T>(L, (const T*)ds->d_keys, i1, i0, i1, d_flag);
      });
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&h_flag, d_flag, sizeof(unsigned), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  }
  if (d_flag) cudaFreeAsync(d_flag, st);
  if (e != cudaSuccess) {
    if (ds->d_keys) cudaFreeAsync(ds->d_keys, st);
    if (st) { cudaStreamSynchronize(st); cudaStreamDestroy(st); }
    delete ds;
    return fail(RMI_ERR_CUDA, std::string("rmi_dataset_create: ") + cudaGetErrorString(e));
  }
  cudaStreamSynchronize(st);
  cudaStreamDestroy(st);
  ds->sorted = (h_flag & 1u) == 0;
  ds->no_dups = (h_flag & 2u) == 0;
  *out = ds;
  return RMI_OK;
}

int rmi_dataset_wrap_device(const void* device_keys, uint64_t n, rmi_key_type key_type, int device, rmi_dataset** out) {
  if (!out || (!device_keys && n) || (int)key_type < 0 || (int)key_type > 2)
    return fail(RMI_ERR_INVALID, "rmi_dataset_wrap_device: bad argument");
  auto* ds = new rmi_dataset();
  ds->d_keys = const_cast<void*>(device_keys);
  ds->n = n; ds->key_type = key_type; ds->device = device; ds->owned = false;
  if (cudaSetDevice(device) != cudaSuccess) { delete ds; return fail(RMI_ERR_CUDA, "cudaSetDevice failed"); }
  if (int rc = verify_sorted(ds)) { delete ds; return rc; }
  *out = ds;
  return RMI_OK;
}

int rmi_dataset_load_file(const char* path, int key_type_or_negative, int device, rmi_dataset** out) {
  if (!path || !out) return fail(RMI_ERR_INVALID, "rmi_dataset_load_file: bad argument");
  int kt = key_type_or_negative;
  if (kt < 0) {   // src/main.rs:122-132: type from the file-name suffix
    std::string p(path);
    auto ends = [&](const char* s) { size_t l = strlen(s); return p.size() >= l && p.compare(p.size() - l, l, s) == 0; };
    if (ends("uint64")) kt = RMI_KEY_U64;
    else if (ends("uint32")) kt = RMI_KEY_U32;
    else if (ends("f64")) kt = RMI_KEY_F64;
    else return fail(RMI_ERR_PANIC, "Data file must end in .uint64, .uint32, or .f64");
  }
  if (kt > 2) return fail(RMI_ERR_INVALID, "rmi_dataset_load_file: bad key type");
  FILE* f = fopen(path, "rb");
  if (!f) return fail(RMI_ERR_PANIC, std::string("Unable to open data file at ") + path);
  uint64_t n = 0;
  if (fread(&n, 8, 1, f) != 1) { fclose(f); return fail(RMI_ERR_PANIC, "data file too short for its header"); }
  if (cudaSetDevice(device) != cudaSuccess) { fclose(f); return fail(RMI_ERR_CUDA, "cudaSetDevice failed"); }
  auto* ds = new rmi_dataset();
  ds->n = n; ds->key_type = kt; ds->device = device; ds->owned = true;
  size_t kb = key_bytes(kt), bytes = (size_t)n * kb;
  cudaStream_t st = nullptr;
  void* stage[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
  const size_t CHUNK = (size_t)64 << 20;
  int rc = RMI_OK;
  auto cleanup = [&]() {
    for (int b = 0; b < 2; ++b) { if (stage[b]) cudaFreeHost(stage[b]); if (ev[b]) cudaEventDestroy(ev[b]); }
    if (st) cudaStreamDestroy(st);
    fclose(f);
  };
  if (bytes) {
    if (cudaMalloc(&ds->d_keys, (bytes + 15) & ~(size_t)15) != cudaSuccess || cudaStreamCreate(&st) != cudaSuccess ||
        cudaMallocHost(&stage[0], CHUNK) != cudaSuccess || cudaMallocHost(&stage[1], CHUNK) != cudaSuccess ||
        cudaEventCreate(&ev[0]) != cudaSuccess || cudaEventCreate(&ev[1]) != cudaSuccess) {
      rc = fail(RMI_ERR_CUDA, "rmi_dataset_load_file: allocation failed");
    } else {
      // double-buffered: fread into one pinned buffer while the other is in flight to HBM
      size_t off = 0; int b = 0;
      while (off < bytes) {
        size_t len = std::min(CHUNK, bytes - off);
        cudaEventSynchronize(ev[b]);
        if (fread(stage[b], 1, len, f) != len) { rc = fail(RMI_ERR_PANIC, "data file shorter than its header says"); break; }
        cudaMemcpyAsync((char*)ds->d_keys + off, stage[b], len, cudaMemcpyHostToDevice, st);
        cudaEventRecord(ev[b], st);
        off += len; b ^= 1;
      }
      if (cudaStreamSynchronize(st) != cudaSuccess && rc == RMI_OK) rc = fail(RMI_ERR_CUDA, "H2D copy failed");
    }
  }
  cleanup();
  if (rc == RMI_OK) rc = verify_sorted(ds);
  if (rc != RMI_OK) { if (ds->d_keys) cudaFree(ds->d_keys); delete ds; return rc; }
  *out = ds;
  return RMI_OK;
}

int rmi_cache_fix(const uint64_t* host_keys, uint64_t n, uint64_t line_size, rmi_spline_point** out_points,
                  uint64_t* out_count) {
  g_last_error.clear();
  if (!host_keys || !out_points || !out_count) return fail(RMI_ERR_INVALID, "rmi_cache_fix: null argument");
  try {
    std::vector<rmihost::SplinePoint> sp = rmihost::cache_fix(host_keys, n, line_size);
    auto* p = static_cast<rmi_spline_point*>(std::malloc(std::max<size_t>(sp.size(), 1) * sizeof(rmi_spline_point)));
    if (!p) return fail(RMI_ERR_INVALID, "rmi_cache_fix: out of host memory");
    for (size_t i = 0; i < sp.size(); ++i) { p[i].key = sp[i].first; p[i].offset = sp[i].second; }
    *out_points = p;
    *out_count = sp.size();
    return RMI_OK;
  } catch (const std::exception& e) {
    return fail(RMI_ERR_PANIC, e.what());   // the reference's assert! messages (cache_fix.rs)
  }
}
void rmi_spline_free(rmi_spline_point* points) { std::free(points); }

uint64_t rmi_model_size(const rmi_result* r, int include_errors, uint64_t num_spline_points) {
  if (!r) return 0;
  return rmihost::rmi_size(*r, include_errors != 0, nullptr) + 16 * num_spline_points;
}

int rmi_output_rmi(const char* ns, const rmi_result* r, const char* data_dir, const char* out_dir, int key_type,
                   int include_errors, uint64_t build_time_ns, const rmi_spline_point* knots, uint64_t num_knots,
                   uint64_t line_size, uint64_t num_data_rows) {
  g_last_error.clear();
  if (!ns || !r || !data_dir || !out_dir) return fail(RMI_ERR_INVALID, "rmi_output_rmi: null argument");
  try {
    std::vector<rmihost::SplinePoint> sp;
    rmihost::CacheFixInfo cf;
    if (knots) {
      sp.reserve(num_knots);
      for (uint64_t i = 0; i < num_knots; ++i) sp.emplace_back(knots[i].key, knots[i].offset);
      cf.line_size = line_size; cf.spline = &sp; cf.num_data_rows = num_data_rows;
    }
    rmihost::output_rmi(ns, *r, data_dir, key_type, include_errors != 0, build_time_ns, out_dir, knots ? &cf : nullptr);
    return RMI_OK;
  } catch (const std::exception& e) {
    return fail(RMI_ERR_PANIC, e.what());
  }
}

int rmi_load_rmi(const char* ns, const char* out_dir, const char* data_dir, rmi_result** out, rmi_spline_point** knots,
                 rmi_artefact_info* info) {
  g_last_error.clear();
  if (!ns || !out_dir || !data_dir || !out || !knots || !info) return fail(RMI_ERR_INVALID, "rmi_load_rmi: null argument");
  auto a = std::make_unique<rmihost::LoadedArtefact>();
  try {
    rmihost::load_rmi(ns, out_dir, data_dir, a.get());
  } catch (const rmihost::LoadError& e) {
    return fail(e.code, e.what());
  } catch (const std::exception& e) {
    return fail(RMI_ERR_INVALID, std::string("rmi_load_rmi: ") + e.what());
  }
  rmi_spline_point* pts = nullptr;
  if (!a->knots.empty()) {
    pts = static_cast<rmi_spline_point*>(std::malloc(a->knots.size() * sizeof(rmi_spline_point)));
    if (!pts) return fail(RMI_ERR_INVALID, "rmi_load_rmi: out of host memory");
    for (size_t k = 0; k < a->knots.size(); ++k) { pts[k].key = a->knots[k].first; pts[k].offset = a->knots[k].second; }
  }
  auto box = new ResultBox();
  box->pub = a->r;
  *out = &box->pub;
  *knots = pts;
  info->key_type = a->key_type;
  info->has_errors = a->has_errors ? 1 : 0;
  info->line_size = a->line_size;
  info->num_knots = a->knots.size();
  info->num_data_rows = a->r.num_data_rows;
  info->build_time_ns = a->build_time_ns;
  box->loaded = std::move(a);   // the result's tables live in the loaded artefact
  return RMI_OK;
}

int rmi_find_pareto_efficient_configs(const rmi_dataset* const* replicas, int num_replicas, uint64_t restrict_to,
                                      uint32_t flags, rmi_config_stats* out, uint64_t capacity, uint64_t* out_count) {
  g_last_error.clear();
  if (!replicas || num_replicas < 1 || !out_count || (capacity && !out))
    return fail(RMI_ERR_INVALID, "rmi_find_pareto_efficient_configs: bad argument");
  try {
    std::vector<const rmi_dataset*> reps(replicas, replicas + num_replicas);
    std::vector<rmihost::RMIStatistics> front = rmihost::find_pareto_efficient_configs(reps, (size_t)restrict_to, flags, false);
    *out_count = front.size();
    for (size_t i = 0; i < front.size() && i < capacity; ++i) {
      std::snprintf(out[i].models, sizeof out[i].models, "%s", front[i].models.c_str());
      out[i].branching_factor = front[i].branching_factor;
      out[i].average_log2_error = front[i].average_log2_error;
      out[i].max_log2_error = front[i].max_log2_error;
      out[i].size = front[i].size;
    }
    return RMI_OK;
  } catch (const std::exception& e) {
    return fail(RMI_ERR_PANIC, e.what());
  }
}

int rmi_find_pareto_efficient_configs_with(rmi_measure_group_fn measure, void* ctx, uint64_t restrict_to, uint32_t flags,
                                           rmi_config_stats* out, uint64_t capacity, uint64_t* out_count) {
  g_last_error.clear();
  if (!measure || !out_count || (capacity && !out))
    return fail(RMI_ERR_INVALID, "rmi_find_pareto_efficient_configs_with: bad argument");
  try {
    rmihost::MeasureStep step;   // one thread, and every (top, branching factor) group whole
    step.measure = [&](size_t, const rmihost::MeasureGroup& g) {
      std::vector<const char*> names;
      for (auto& l : g.leaves) names.push_back(l.c_str());
      std::vector<rmi_config_stats> res(g.leaves.size());
      memset(res.data(), 0, sizeof(rmi_config_stats) * res.size());
      g_last_error.clear();
      const int rc = measure(ctx, g.top.c_str(), g.bf, names.data(), (int)names.size(), flags, res.data());
      if (rc != 0) {
        std::string msg = rmi_last_error();
        throw std::runtime_error(msg.empty() ? "the measuring callback returned " + std::to_string(rc) : msg);
      }
      std::vector<rmihost::RMIStatistics> v(res.size());
      for (size_t k = 0; k < res.size(); ++k) {
        v[k].average_log2_error = res[k].average_log2_error;
        v[k].max_log2_error = res[k].max_log2_error;
        v[k].size = res[k].size;
      }
      return v;
    };
    std::vector<rmihost::RMIStatistics> front = rmihost::find_pareto_efficient_configs(step, (size_t)restrict_to);
    g_last_error.clear();
    *out_count = front.size();
    for (size_t i = 0; i < front.size() && i < capacity; ++i) {
      std::snprintf(out[i].models, sizeof out[i].models, "%s", front[i].models.c_str());
      out[i].branching_factor = front[i].branching_factor;
      out[i].average_log2_error = front[i].average_log2_error;
      out[i].max_log2_error = front[i].max_log2_error;
      out[i].size = front[i].size;
    }
    return RMI_OK;
  } catch (const std::exception& e) {
    return fail(RMI_ERR_PANIC, e.what());
  }
}

int rmi_dataset_replicate(const rmi_dataset* src, int device, rmi_dataset** out) {
  g_last_error.clear();
  if (!src || !out) return fail(RMI_ERR_INVALID, "rmi_dataset_replicate: null argument");
  const size_t ksz = src->key_type == RMI_KEY_U32 ? 4 : 8;
  const size_t bytes = ((size_t)src->n * ksz + 15) & ~(size_t)15;   // readable up to the next 16-byte boundary
  CUDA_TRY(cudaSetDevice(device));
  void* d = nullptr;
  CUDA_TRY(cudaMalloc(&d, bytes ? bytes : 16));
  cudaError_t e = cudaSuccess;
  if (src->n) {
    if (device != src->device) {
      int can = 0;
      cudaDeviceCanAccessPeer(&can, device, src->device);
      if (can) { cudaError_t pe = cudaDeviceEnablePeerAccess(src->device, 0); if (pe != cudaSuccess) cudaGetLastError(); }
    }
    e = cudaMemcpyPeer(d, device, src->d_keys, src->device, (size_t)src->n * ksz);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
  }
  if (e != cudaSuccess) { cudaFree(d); return fail(RMI_ERR_CUDA, std::string("rmi_dataset_replicate: ") + cudaGetErrorString(e)); }
  auto* ds = new rmi_dataset();
  ds->d_keys = d; ds->n = src->n; ds->key_type = src->key_type; ds->device = device;
  ds->owned = true; ds->pooled = false; ds->sorted = src->sorted; ds->no_dups = src->no_dups;
  *out = ds;
  return RMI_OK;
}

uint64_t rmi_dataset_len(const rmi_dataset* ds) { return ds ? ds->n : 0; }
int rmi_dataset_copy_to_host(const rmi_dataset* ds, void* host_keys) {
  if (!ds || (!host_keys && ds->n)) return fail(RMI_ERR_INVALID, "rmi_dataset_copy_to_host: null argument");
  if (ds->n == 0) return RMI_OK;
  CUDA_TRY(cudaSetDevice(ds->device));
  CUDA_TRY(cudaMemcpy(host_keys, ds->d_keys, (size_t)ds->n * key_bytes(ds->key_type), cudaMemcpyDeviceToHost));
  return RMI_OK;
}
int rmi_dataset_key_type(const rmi_dataset* ds) { return ds ? ds->key_type : -1; }
void rmi_dataset_destroy(rmi_dataset* ds) {
  if (!ds) return;
  if (ds->owned && ds->d_keys) {
    cudaSetDevice(ds->device);
    if (ds->pooled) cudaFreeAsync(ds->d_keys, nullptr); else cudaFree(ds->d_keys);
  }
  delete ds;
}

void rmi_result_free(rmi_result* r) { delete reinterpret_cast<ResultBox*>(r); }

}  // extern "C"

// A trained RMI bound to the device-resident keys it was trained on: the top model by value (its tables in device
// memory) and one packed record per leaf (kernels.h: lookup_record_bytes).  Immutable after creation.
struct rmi_index {
  const rmi_dataset* ds = nullptr;
  TopTables tables;          // the top model's tables, on the device
  TopModel top;              // points at `tables`
  int leaf_kind = 0;
  uint64_t N = 0;
  // the positions the model predicts over: ds->n, or the whole key set's size for the index inside an
  // rmi_shard_index, which only predicts (shard_search turns the predictions into lower bounds in the slab)
  uint64_t n = 0;
  void* d_records = nullptr;
  int num_sms = 0;
  // a bounded (cache-fix) index: the RMI above runs over K knots; null / 0 for a plain index
  void* d_knots = nullptr;   // K x rmi_spline_point
  uint64_t K = 0;
  uint64_t line_size = 0;
  uint64_t last_key_bits = 0;   // ds's last key (raw bits, u32 zero-extended): upper bounds of queries >= it are n
};

namespace {
void index_free_device(rmi_index* idx) {
  idx->tables.free_device();
  cudaFree(idx->d_records);
  cudaFree(idx->d_knots);
}

int index_check_call(const rmi_index* idx, const void* d_queries, uint64_t n, const void* d_out, const char* fn) {
  if (!idx) return fail(RMI_ERR_INVALID, std::string(fn) + ": null index");
  if (n && (!d_queries || !d_out)) return fail(RMI_ERR_INVALID, std::string(fn) + ": null query or output pointer");
  return RMI_OK;
}

// One launch of `mode` (kernels.h: LookupMode) into d_out and d_out2, none for n == 0.
int index_launch(const rmi_index* idx, LookupMode mode, const void* d_queries, uint64_t n, uint64_t* d_out,
                 uint64_t* d_out2, uint64_t* d_fallbacks, void* cuda_stream) {
  if (n == 0) return RMI_OK;
  const rmi_dataset* ds = idx->ds;
  CUDA_TRY(cudaSetDevice(ds->device));
  Launch L{(cudaStream_t)cuda_stream, idx->num_sms};
  if (idx->d_knots) {
    lookup_bounded_batch(L, mode, idx->top, idx->leaf_kind, idx->d_records, idx->N, idx->d_knots, idx->K,
                         idx->line_size, (const u64*)ds->d_keys, idx->n, idx->last_key_bits, (const u64*)d_queries, n,
                         (u64*)d_out, (u64*)d_out2, (u64*)d_fallbacks);
  } else {
    with_key_type(ds->key_type, [&](auto k) {
      using T = decltype(k);
      lookup_batch<T>(L, mode, idx->top, idx->leaf_kind, idx->d_records, idx->N, (const T*)ds->d_keys, idx->n,
                      rmihost::key_from_bits<T>(idx->last_key_bits), (const T*)d_queries, n, (u64*)d_out,
                      (u64*)d_out2, (u64*)d_fallbacks);
    });
  }
  CUDA_TRY(cudaGetLastError());
  return RMI_OK;
}

// The host-array form of a lookup, synchronously on a stream of its own: copies the n queries to the device, runs
// launch(d_q, d_a, d_b, d_fallbacks, stream) (d_b null when host_b is; *d_fallbacks starts at 0) and copies d_a to
// host_a, d_b to host_b and the fallback count to *fallbacks where those are given.
template <class Launch_>
int index_host_call(const rmi_index* idx, const void* host_queries, uint64_t n, uint64_t* host_a, uint64_t* host_b,
                    uint64_t* fallbacks, const char* fn, Launch_&& launch) {
  if (n == 0) return RMI_OK;
  CUDA_TRY(cudaSetDevice(idx->ds->device));
  const size_t qb = (size_t)n * key_bytes(idx->ds->key_type), ob = (size_t)n * sizeof(uint64_t);
  cudaStream_t st = nullptr;
  char* d = nullptr;   // queries | a | b | fallback counter
  cudaError_t e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMallocAsync((void**)&d, qb + 2 * ob + 8 + 8, st);
  int rc = RMI_OK;
  if (e == cudaSuccess) {
    char* d_q = d;
    uint64_t* d_a = (uint64_t*)(d + ((qb + 7) & ~(size_t)7));
    uint64_t* d_b = d_a + n;
    uint64_t* d_fb = d_b + n;
    e = cudaMemcpyAsync(d_q, host_queries, qb, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_fb, 0, sizeof(u64), st);
    if (e == cudaSuccess) rc = launch(d_q, d_a, host_b ? d_b : nullptr, d_fb, st);
    if (e == cudaSuccess && rc == RMI_OK) e = cudaMemcpyAsync(host_a, d_a, ob, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && rc == RMI_OK && host_b) e = cudaMemcpyAsync(host_b, d_b, ob, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && rc == RMI_OK && fallbacks)
      e = cudaMemcpyAsync(fallbacks, d_fb, sizeof(u64), cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(d, st);
  }
  if (st) {
    cudaError_t es = cudaStreamSynchronize(st);
    if (e == cudaSuccess) e = es;
    cudaStreamDestroy(st);
  }
  if (rc != RMI_OK) return rc;
  if (e != cudaSuccess) return fail(RMI_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e));
  return RMI_OK;
}

// After check_result, the checks every kind of index shares: r must have been trained on `rows` rows (the dataset's
// keys, the knots of a bounded index, or the keys of all slabs of a range-partitioned one), which `holder` names in
// the message; `keys` is the number of keys the index searches (0: an empty index).  Messages name `fn`.
int index_check_tables(const rmi_result* r, uint64_t rows, const char* holder, uint64_t keys, const std::string& fn) {
  if (r->num_rmi_rows != rows)
    return fail(RMI_ERR_INVALID, fn + ": the result was trained on " + std::to_string(r->num_rmi_rows) + " keys, " +
                                     holder + std::to_string(rows));
  if (keys == 0 || r->branching_factor == 0) return fail(RMI_ERR_INVALID, fn + ": empty index");
  return RMI_OK;
}

// Builds the index on ds's device, predicting over n positions; knots (K of them, may be null) make it a bounded one.
int index_upload(const rmi_result* r, const rmi_dataset* ds, uint64_t n, const rmi_spline_point* knots, uint64_t K,
                 uint64_t line_size, const std::string& fn, rmi_index** out) {
  CUDA_TRY(cudaSetDevice(ds->device));
  DeviceInfo di;
  if (int rc = device_info(ds->device, &di)) return rc;
  auto* idx = new rmi_index();
  idx->ds = ds;
  idx->leaf_kind = (int)r->l1_model_id;
  idx->N = r->branching_factor;
  idx->n = n;
  idx->num_sms = di.num_sms;
  std::vector<char> packed((size_t)idx->N * lookup_record_bytes(idx->leaf_kind));
  pack_leaf_records(idx->leaf_kind, r->l1_params, (const u64*)r->l1_errors, idx->N, packed.data());
  cudaError_t e = idx->tables.upload(*r, nullptr, device_alloc);
  idx->top = idx->tables.given(*r);
  if (e == cudaSuccess) e = cudaMalloc(&idx->d_records, packed.size());
  if (e == cudaSuccess) e = cudaMemcpy(idx->d_records, packed.data(), packed.size(), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && ds->n > 0) {
    const size_t kb = key_bytes(ds->key_type);
    e = cudaMemcpy(&idx->last_key_bits, (const char*)ds->d_keys + (ds->n - 1) * kb, kb, cudaMemcpyDeviceToHost);
  }
  if (e == cudaSuccess && knots) {
    e = cudaMalloc(&idx->d_knots, sizeof(rmi_spline_point) * K);
    if (e == cudaSuccess) e = cudaMemcpy(idx->d_knots, knots, sizeof(rmi_spline_point) * K, cudaMemcpyHostToDevice);
    idx->K = K;
    idx->line_size = line_size;
  }
  // the table copies are asynchronous: r's host tables may be released once this returns
  if (e == cudaSuccess) e = cudaStreamSynchronize(nullptr);
  if (e != cudaSuccess) {
    index_free_device(idx);
    delete idx;
    return fail(RMI_ERR_CUDA, fn + ": " + cudaGetErrorString(e));
  }
  *out = idx;
  return RMI_OK;
}


}  // namespace

extern "C" {

int rmi_index_create(const rmi_result* r, const rmi_dataset* ds, rmi_index** out) {
  const std::string fn = "rmi_index_create";
  if (!r || !ds || !out) return fail(RMI_ERR_INVALID, fn + ": null argument");
  if (int rc = check_result(r, true, fn)) return rc;
  if (int rc = index_check_tables(r, ds->n, "the dataset holds ", ds->n, fn)) return rc;
  return index_upload(r, ds, ds->n, nullptr, 0, 0, fn, out);
}

int rmi_index_create_bounded(const rmi_result* r, const rmi_spline_point* knots, uint64_t num_knots,
                             uint64_t line_size, const rmi_dataset* ds, rmi_index** out) {
  const std::string fn = "rmi_index_create_bounded";
  if (!r || !knots || !ds || !out) return fail(RMI_ERR_INVALID, fn + ": null argument");
  if (int rc = check_result(r, true, fn)) return rc;
  if (ds->key_type != RMI_KEY_U64) return fail(RMI_ERR_INVALID, fn + ": Can only construct a bounded RMI on u64 data");
  if (line_size == 0) return fail(RMI_ERR_INVALID, fn + ": line size 0");
  if (num_knots == 0) return fail(RMI_ERR_INVALID, fn + ": no spline knots");
  if (int rc = index_check_tables(r, num_knots, "the spline has ", ds->n, fn)) return rc;
  for (uint64_t i = 0; i < num_knots; ++i) {
    if (knots[i].offset >= ds->n)
      return fail(RMI_ERR_INVALID, fn + ": knot " + std::to_string(i) + " has offset " + std::to_string(knots[i].offset) +
                                       ", the dataset holds " + std::to_string(ds->n) + " keys");
    if (i && !(knots[i - 1].key < knots[i].key && knots[i - 1].offset <= knots[i].offset))
      return fail(RMI_ERR_INVALID, fn + ": knots " + std::to_string(i - 1) + " and " + std::to_string(i) +
                                       " are out of order (keys must increase strictly, offsets must not decrease)");
  }
  return index_upload(r, ds, ds->n, knots, num_knots, line_size, fn, out);
}

void rmi_index_destroy(rmi_index* idx) {
  if (!idx) return;
  cudaSetDevice(idx->ds->device);
  index_free_device(idx);
  delete idx;
}

int rmi_index_predict(const rmi_index* idx, const void* d_queries, uint64_t n, uint64_t* d_pos, uint64_t* d_err,
                      void* cuda_stream) {
  if (int rc = index_check_call(idx, d_queries, n, d_pos, "rmi_index_predict")) return rc;
  return index_launch(idx, LOOKUP_PREDICT, d_queries, n, d_pos, d_err, nullptr, cuda_stream);
}

int rmi_index_lower_bound(const rmi_index* idx, const void* d_queries, uint64_t n, uint64_t* d_out,
                          uint64_t* d_fallbacks, void* cuda_stream) {
  if (int rc = index_check_call(idx, d_queries, n, d_out, "rmi_index_lower_bound")) return rc;
  return index_launch(idx, LOOKUP_LOWER, d_queries, n, d_out, nullptr, d_fallbacks, cuda_stream);
}

int rmi_index_upper_bound(const rmi_index* idx, const void* d_queries, uint64_t n, uint64_t* d_out,
                          uint64_t* d_fallbacks, void* cuda_stream) {
  if (int rc = index_check_call(idx, d_queries, n, d_out, "rmi_index_upper_bound")) return rc;
  return index_launch(idx, LOOKUP_UPPER, d_queries, n, d_out, nullptr, d_fallbacks, cuda_stream);
}

int rmi_index_equal_range(const rmi_index* idx, const void* d_queries, uint64_t n, uint64_t* d_first, uint64_t* d_last,
                          uint64_t* d_fallbacks, void* cuda_stream) {
  if (int rc = index_check_call(idx, d_queries, n, d_last, "rmi_index_equal_range")) return rc;
  if (n && !d_first) return fail(RMI_ERR_INVALID, "rmi_index_equal_range: null query or output pointer");
  return index_launch(idx, LOOKUP_EQUAL_RANGE, d_queries, n, d_first, d_last, d_fallbacks, cuda_stream);
}

int rmi_index_range_host(const rmi_index* idx, const void* host_queries, uint64_t n, uint64_t* host_first,
                         uint64_t* host_last, uint64_t* fallbacks) {
  if (int rc = index_check_call(idx, host_queries, n, host_last, "rmi_index_range_host")) return rc;
  if (fallbacks) *fallbacks = 0;
  return index_host_call(idx, host_queries, n, host_last, host_first, fallbacks, "rmi_index_range_host",
                         [&](const void* d_q, uint64_t* d_last, uint64_t* d_first, uint64_t* d_fb, cudaStream_t st) {
                           return d_first ? index_launch(idx, LOOKUP_EQUAL_RANGE, d_q, n, d_first, d_last, d_fb, st)
                                         : index_launch(idx, LOOKUP_UPPER, d_q, n, d_last, nullptr, d_fb, st);
                         });
}

int rmi_index_lookup_host(const rmi_index* idx, const void* host_queries, uint64_t n, int lower_bound,
                          uint64_t* host_out, uint64_t* host_err, uint64_t* fallbacks) {
  if (int rc = index_check_call(idx, host_queries, n, host_out, "rmi_index_lookup_host")) return rc;
  return index_host_call(idx, host_queries, n, host_out, lower_bound ? nullptr : host_err,
                         lower_bound ? fallbacks : nullptr, "rmi_index_lookup_host",
                         [&](const void* d_q, uint64_t* d_out, uint64_t* d_err, uint64_t* d_fb, cudaStream_t st) {
                           return lower_bound ? index_launch(idx, LOOKUP_LOWER, d_q, n, d_out, nullptr, d_fb, st)
                                              : index_launch(idx, LOOKUP_PREDICT, d_q, n, d_out, d_err, nullptr, st);
                         });
}

}  // extern "C"

// A sorted device array of keys in one of two buffers: an update merges the array and a batch into the other one,
// which then holds the array.
struct DeltaKeys {
  void* buf[2] = {nullptr, nullptr};
  uint64_t cap[2] = {0, 0};   // keys each buffer holds room for
  int cur = 0;                // buf[cur] holds the len keys
  uint64_t len = 0;
  const void* keys() const { return buf[cur]; }
  void* spare() const { return buf[1 - cur]; }
  // Makes the spare buffer hold `need` keys: one of twice the larger capacity (at least `need`, at least 1024 keys)
  // when it is too small.
  int reserve_spare(uint64_t need, size_t key_bytes, const std::string& fn) {
    const int s = 1 - cur;
    if (cap[s] >= need) return RMI_OK;
    const uint64_t c = std::max<uint64_t>({need, 2 * std::max(cap[0], cap[1]), 1024});
    void* p = nullptr;
    if (cudaMalloc(&p, (size_t)c * key_bytes) != cudaSuccess) {
      cudaGetLastError();
      return fail(RMI_ERR_CUDA, fn + ": device allocation of " + std::to_string(c) + " keys failed");
    }
    cudaFree(buf[s]);
    buf[s] = p;
    cap[s] = c;
    return RMI_OK;
  }
  // The spare buffer, holding n keys, becomes the array.
  void swap_in(uint64_t n) { cur = 1 - cur; len = n; }
  void release() { cudaFree(buf[0]); cudaFree(buf[1]); }
};

// An updatable index (DESIGN.md section 19): a base index, the sorted keys inserted since it was built (m) and the
// sorted keys removed since (t).  The logical key set is base ⊎ inserted ⊖ removed.
struct rmi_delta {
  const rmi_index* base = nullptr;
  DeltaKeys ins, rem;
  unsigned* d_status = nullptr;
};

namespace {

int delta_check_call(const rmi_delta* d, const void* d_queries, uint64_t n, const void* d_out, const char* fn) {
  if (!d) return fail(RMI_ERR_INVALID, std::string(fn) + ": null delta index");
  if (n && (!d_queries || !d_out)) return fail(RMI_ERR_INVALID, std::string(fn) + ": null query or output pointer");
  return RMI_OK;
}

// The base index's launch of `mode`, then, on the same stream, the delta's share added to its answers: k_delta_count
// over the inserted keys while nothing has been removed (no launch for an empty delta), k_delta_adjust otherwise.
int delta_launch(const rmi_delta* d, LookupMode mode, const void* d_queries, uint64_t n, uint64_t* d_first,
                 uint64_t* d_last, uint64_t* d_fallbacks, void* cuda_stream) {
  if (n == 0) return RMI_OK;
  uint64_t* out = mode == LOOKUP_UPPER ? d_last : d_first;
  if (int rc = index_launch(d->base, mode, d_queries, n, out, mode == LOOKUP_EQUAL_RANGE ? d_last : nullptr, d_fallbacks,
                            cuda_stream))
    return rc;
  if (d->ins.len == 0 && d->rem.len == 0) return RMI_OK;
  const DeltaCountMode cm = mode == LOOKUP_LOWER ? DELTA_LOWER : mode == LOOKUP_UPPER ? DELTA_UPPER : DELTA_BOTH;
  Launch L{(cudaStream_t)cuda_stream, d->base->num_sms};
  with_key_type(d->base->ds->key_type, [&](auto k) {
    using T = decltype(k);
    if (d->rem.len == 0)
      delta_count<T>(L, cm, (const T*)d->ins.keys(), d->ins.len, (const T*)d_queries, n, (u64*)d_first, (u64*)d_last);
    else
      delta_adjust<T>(L, cm, (const T*)d->ins.keys(), d->ins.len, (const T*)d->rem.keys(), d->rem.len,
                      (const T*)d_queries, n, (u64*)d_first, (u64*)d_last);
  });
  CUDA_TRY(cudaGetLastError());
  return RMI_OK;
}

// a (na keys) and b (nb keys) merged into out on the calling thread's stream, synchronously; *status receives the
// merge's status word (DELTA_ST_NAN) when d_status is given.
int delta_merge_sync(const rmi_delta* d, const void* a, uint64_t na, const void* b, uint64_t nb, void* out,
                     unsigned* d_status, unsigned* status, const char* fn) {
  const cudaStream_t st = cudaStreamPerThread;
  if (d_status) CUDA_TRY(cudaMemsetAsync(d_status, 0, sizeof(unsigned), st));
  Launch L{st, d->base->num_sms};
  with_key_type(d->base->ds->key_type, [&](auto k) {
    using T = decltype(k);
    delta_merge<T>(L, (const T*)a, na, (const T*)b, nb, (T*)out, d_status);
  });
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess && d_status) e = cudaMemcpyAsync(status, d_status, sizeof(unsigned), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(RMI_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e));
  return RMI_OK;
}

}  // namespace

extern "C" {

int rmi_delta_create(const rmi_index* base, rmi_delta** out) {
  if (!base || !out) return fail(RMI_ERR_INVALID, "rmi_delta_create: null argument");
  CUDA_TRY(cudaSetDevice(base->ds->device));
  auto* d = new rmi_delta();
  d->base = base;
  if (cudaMalloc(&d->d_status, sizeof(unsigned)) != cudaSuccess) {
    delete d;
    return fail(RMI_ERR_CUDA, "rmi_delta_create: device allocation failed");
  }
  *out = d;
  return RMI_OK;
}

void rmi_delta_destroy(rmi_delta* d) {
  if (!d) return;
  cudaSetDevice(d->base->ds->device);
  d->ins.release();
  d->rem.release();
  cudaFree(d->d_status);
  delete d;
}

uint64_t rmi_delta_len(const rmi_delta* d) { return d ? d->ins.len : 0; }

uint64_t rmi_delta_removed_len(const rmi_delta* d) { return d ? d->rem.len : 0; }

int rmi_delta_insert(rmi_delta* d, const rmi_dataset* batch) {
  const std::string fn = "rmi_delta_insert";
  if (!d || !batch) return fail(RMI_ERR_INVALID, fn + ": null argument");
  const rmi_dataset* ds = d->base->ds;
  if (batch->key_type != ds->key_type) return fail(RMI_ERR_INVALID, fn + ": the batch's key type differs from the index's");
  if (batch->device != ds->device) return fail(RMI_ERR_INVALID, fn + ": the batch is on another device than the index");
  if (!batch->sorted) return fail(RMI_ERR_INVALID, fn + ": the batch is not sorted in ascending order");
  if (batch->n == 0) return RMI_OK;
  CUDA_TRY(cudaSetDevice(ds->device));
  const uint64_t need = d->ins.len + batch->n;
  if (int rc = d->ins.reserve_spare(need, key_bytes(ds->key_type), fn)) return rc;
  unsigned status = 0;
  if (int rc = delta_merge_sync(d, d->ins.keys(), d->ins.len, batch->d_keys, batch->n, d->ins.spare(), d->d_status,
                                &status, fn.c_str()))
    return rc;
  if (status & DELTA_ST_NAN) return fail(RMI_ERR_INVALID, fn + ": the batch holds a NaN");
  d->ins.swap_in(need);
  return RMI_OK;
}

int rmi_delta_remove(rmi_delta* d, const rmi_dataset* batch) {
  const std::string fn = "rmi_delta_remove";
  if (!d || !batch) return fail(RMI_ERR_INVALID, fn + ": null argument");
  const rmi_dataset* ds = d->base->ds;
  if (batch->key_type != ds->key_type) return fail(RMI_ERR_INVALID, fn + ": the batch's key type differs from the index's");
  if (batch->device != ds->device) return fail(RMI_ERR_INVALID, fn + ": the batch is on another device than the index");
  if (!batch->sorted) return fail(RMI_ERR_INVALID, fn + ": the batch is not sorted in ascending order");
  const uint64_t n = batch->n;
  if (n == 0) return RMI_OK;
  CUDA_TRY(cudaSetDevice(ds->device));
  // c(v) for every batch key: its equal range over the logical key set, from the lookup path itself
  const cudaStream_t st = cudaStreamPerThread;
  uint64_t* d_range = nullptr;   // first | last
  CUDA_TRY(cudaMallocAsync((void**)&d_range, (size_t)2 * n * sizeof(u64), st));
  int rc = delta_launch(d, LOOKUP_EQUAL_RANGE, batch->d_keys, n, d_range, d_range + n, nullptr, st);
  unsigned status = 0;
  cudaError_t e = cudaMemsetAsync(d->d_status, 0, sizeof(unsigned), st);
  if (rc == RMI_OK && e == cudaSuccess) {
    Launch L{st, d->base->num_sms};
    with_key_type(ds->key_type, [&](auto k) {
      using T = decltype(k);
      delta_check_remove<T>(L, (const T*)batch->d_keys, n, (const u64*)d_range, (const u64*)d_range + n, d->d_status);
    });
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(&status, d->d_status, sizeof(unsigned), cudaMemcpyDeviceToHost, st);
    const cudaError_t ef = cudaFreeAsync(d_range, st);
    if (e == cudaSuccess) e = ef;
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  } else {
    cudaFreeAsync(d_range, st);
  }
  if (rc != RMI_OK) return rc;
  if (e != cudaSuccess) return fail(RMI_ERR_CUDA, fn + ": " + cudaGetErrorString(e));
  if (status & DELTA_ST_NAN) return fail(RMI_ERR_INVALID, fn + ": the batch holds a NaN");
  if (status & DELTA_ST_MISSING)
    return fail(RMI_ERR_INVALID, fn + ": the index does not hold every key of the batch (as many copies of each value)");
  const uint64_t need = d->rem.len + n;
  if ((rc = d->rem.reserve_spare(need, key_bytes(ds->key_type), fn))) return rc;
  if ((rc = delta_merge_sync(d, d->rem.keys(), d->rem.len, batch->d_keys, n, d->rem.spare(), nullptr, nullptr,
                             fn.c_str())))
    return rc;
  d->rem.swap_in(need);
  return RMI_OK;
}

int rmi_delta_lower_bound(const rmi_delta* d, const void* d_queries, uint64_t n, uint64_t* d_out,
                          uint64_t* d_fallbacks, void* cuda_stream) {
  if (int rc = delta_check_call(d, d_queries, n, d_out, "rmi_delta_lower_bound")) return rc;
  return delta_launch(d, LOOKUP_LOWER, d_queries, n, d_out, nullptr, d_fallbacks, cuda_stream);
}

int rmi_delta_upper_bound(const rmi_delta* d, const void* d_queries, uint64_t n, uint64_t* d_out,
                          uint64_t* d_fallbacks, void* cuda_stream) {
  if (int rc = delta_check_call(d, d_queries, n, d_out, "rmi_delta_upper_bound")) return rc;
  return delta_launch(d, LOOKUP_UPPER, d_queries, n, nullptr, d_out, d_fallbacks, cuda_stream);
}

int rmi_delta_equal_range(const rmi_delta* d, const void* d_queries, uint64_t n, uint64_t* d_first, uint64_t* d_last,
                          uint64_t* d_fallbacks, void* cuda_stream) {
  if (int rc = delta_check_call(d, d_queries, n, d_last, "rmi_delta_equal_range")) return rc;
  if (n && !d_first) return fail(RMI_ERR_INVALID, "rmi_delta_equal_range: null query or output pointer");
  return delta_launch(d, LOOKUP_EQUAL_RANGE, d_queries, n, d_first, d_last, d_fallbacks, cuda_stream);
}

int rmi_delta_range_host(const rmi_delta* d, const void* host_queries, uint64_t n, uint64_t* host_first,
                         uint64_t* host_last, uint64_t* fallbacks) {
  const char* fn = "rmi_delta_range_host";
  if (int rc = delta_check_call(d, host_queries, n, host_first ? (const void*)host_first : host_last, fn)) return rc;
  if (fallbacks) *fallbacks = 0;
  if (n == 0) return RMI_OK;
  // index_host_call fills host_a always and host_b when given: the lower bounds go first whenever they are asked for
  uint64_t* host_a = host_first ? host_first : host_last;
  uint64_t* host_b = host_first ? host_last : nullptr;
  const LookupMode mode = !host_first ? LOOKUP_UPPER : host_last ? LOOKUP_EQUAL_RANGE : LOOKUP_LOWER;
  return index_host_call(d->base, host_queries, n, host_a, host_b, fallbacks, fn,
                         [&](const void* d_q, uint64_t* d_a, uint64_t* d_b, uint64_t* d_fb, cudaStream_t st) {
                           return mode == LOOKUP_UPPER ? delta_launch(d, mode, d_q, n, nullptr, d_a, d_fb, st)
                                                       : delta_launch(d, mode, d_q, n, d_a, d_b, d_fb, st);
                         });
}

int rmi_delta_merge(const rmi_delta* d, rmi_dataset** out) {
  const std::string fn = "rmi_delta_merge";
  if (!d || !out) return fail(RMI_ERR_INVALID, fn + ": null argument");
  const rmi_dataset* base = d->base->ds;
  CUDA_TRY(cudaSetDevice(base->device));
  const uint64_t m = d->ins.len, t = d->rem.len;
  const uint64_t n = base->n + m - t;   // t <= base->n + m: every removal was checked against the key set
  void* keys = nullptr;
  // readable up to the next 16-byte boundary, as every dataset the library allocates
  if (cudaMalloc(&keys, std::max<size_t>(16, ((size_t)n * key_bytes(base->key_type) + 15) & ~(size_t)15)) != cudaSuccess) {
    cudaGetLastError();
    return fail(RMI_ERR_CUDA, fn + ": device allocation of " + std::to_string(n) + " keys failed");
  }
  auto* ds = new rmi_dataset();
  ds->d_keys = keys; ds->n = n; ds->key_type = base->key_type; ds->device = base->device;
  ds->owned = true; ds->pooled = false;
  int rc = RMI_OK;
  if (t == 0) {
    rc = delta_merge_sync(d, base->d_keys, base->n, d->ins.keys(), m, keys, nullptr, nullptr, fn.c_str());
  } else {
    // base and inserted keys merged into scratch, then the removed keys subtracted into the data set
    const cudaStream_t st = cudaStreamPerThread;
    void* merged = nullptr;
    cudaError_t e = cudaMallocAsync(&merged, std::max<size_t>(16, (size_t)(base->n + m) * key_bytes(base->key_type)), st);
    if (e == cudaSuccess) {
      rc = delta_merge_sync(d, base->d_keys, base->n, d->ins.keys(), m, merged, nullptr, nullptr, fn.c_str());
      if (rc == RMI_OK) {
        Launch L{st, d->base->num_sms};
        with_key_type(base->key_type, [&](auto k) {
          using T = decltype(k);
          delta_subtract<T>(L, (const T*)merged, base->n + m, (const T*)d->rem.keys(), t, (T*)keys);
        });
        e = cudaGetLastError();
      }
      const cudaError_t ef = cudaFreeAsync(merged, st);
      if (e == cudaSuccess) e = ef;
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    } else {
      cudaGetLastError();
    }
    if (rc == RMI_OK && e != cudaSuccess) rc = fail(RMI_ERR_CUDA, fn + ": " + cudaGetErrorString(e));
  }
  if (rc == RMI_OK) rc = verify_sorted(ds);
  if (rc != RMI_OK) { rmi_dataset_destroy(ds); return rc; }
  *out = ds;
  return RMI_OK;
}

}  // extern "C"

namespace {

// Streams / events of the sliced leaf launch (kernels.h: LeafCopyOut), created once per host
// thread and device and reused by every rmi_train call of that thread.  Slice c's stream has a
// higher priority than slice c + 1's (below the long-leaf side stream's): the block scheduler
// then hands out the slices' blocks in slice order, so the small slices at the end of the taper
// are the last to finish (at equal priorities it picks among the pending slices in no fixed
// order, and a full-size slice, whose copy is then exposed, often runs last).
struct SliceResources {
  int device = -1;
  LeafCopyOut co;
  void release() {
    if (device < 0) return;
    for (int c = 0; c < LEAF_SLICES; ++c) {
      if (co.streams[c]) cudaStreamDestroy(co.streams[c]);
      if (co.ev_kernel[c]) cudaEventDestroy(co.ev_kernel[c]);
      if (co.ev_copied[c]) cudaEventDestroy(co.ev_copied[c]);
    }
    if (co.ev_ready) cudaEventDestroy(co.ev_ready);
    co = LeafCopyOut();
    device = -1;
  }
  LeafCopyOut* get(int dev) {
    if (device == dev) return &co;
    release();
    int least = 0, greatest = 0;   // numerically: greatest <= least
    cudaDeviceGetStreamPriorityRange(&least, &greatest);
    bool ok = cudaEventCreateWithFlags(&co.ev_ready, cudaEventDisableTiming) == cudaSuccess;
    for (int c = 0; c < LEAF_SLICES && ok; ++c)
      ok = cudaStreamCreateWithPriority(&co.streams[c], cudaStreamNonBlocking, std::min(least, greatest + 1 + c)) == cudaSuccess &&
           cudaEventCreateWithFlags(&co.ev_kernel[c], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&co.ev_copied[c], cudaEventDisableTiming) == cudaSuccess;
    device = dev;
    if (!ok) { release(); cudaGetLastError(); return nullptr; }
    return &co;
  }
  ~SliceResources() {}   // process exit: the driver reclaims them (destroying here could run after CUDA shut down)
};
thread_local SliceResources t_slices;

// The build's own stream, the high-priority side stream of the long-leaf kernel and the timing
// events, likewise kept per host thread and device (creating and destroying two streams and
// seven events per call cost more host time than the launches of a small build).  Also the
// device scratch of the thread's builds (BuildScratch) and the pinned slot a build's initial
// TopModel and zeroed BuildAux are uploaded from.
struct BuildContext {
  int device = -1;
  cudaStream_t st = nullptr, side = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, evp[3] = {nullptr, nullptr, nullptr}, ev_fork = nullptr, ev_join = nullptr;
  char* scratch = nullptr;   // device, scratch_cap bytes
  size_t scratch_cap = 0;
  char* h_init = nullptr;    // pinned, kInitBytes
  static constexpr size_t kInitBytes = sizeof(TopModel) + sizeof(BuildAux);
  // builds that need more scratch than this take the excess from the pool per call rather than keep it for the thread
  static constexpr size_t kScratchKeepMax = (size_t)1 << 30;
  void release() {
    if (device < 0) return;
    if (scratch) cudaFree(scratch);   // builds are synchronous: nothing in flight still uses it
    if (h_init) cudaFreeHost(h_init);
    if (st) cudaStreamDestroy(st);
    if (side) cudaStreamDestroy(side);
    for (cudaEvent_t e : {ev0, ev1, evp[0], evp[1], evp[2], ev_fork, ev_join}) if (e) cudaEventDestroy(e);
    *this = BuildContext();
  }
  BuildContext* get(int dev) {
    if (device == dev) return this;
    release();
    int lo_prio = 0, hi_prio = 0;
    cudaDeviceGetStreamPriorityRange(&lo_prio, &hi_prio);
    bool ok = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) == cudaSuccess &&
              cudaEventCreate(&ev0) == cudaSuccess && cudaEventCreate(&ev1) == cudaSuccess &&
              cudaEventCreate(&evp[0]) == cudaSuccess && cudaEventCreate(&evp[1]) == cudaSuccess &&
              cudaEventCreate(&evp[2]) == cudaSuccess &&
              cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming) == cudaSuccess &&
              cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming) == cudaSuccess &&
              cudaMallocHost((void**)&h_init, kInitBytes) == cudaSuccess;
    if (ok && cudaStreamCreateWithPriority(&side, cudaStreamNonBlocking, hi_prio) != cudaSuccess) { side = nullptr; cudaGetLastError(); }
    device = dev;
    if (!ok) { release(); cudaGetLastError(); return nullptr; }
    return this;
  }
  // Issues the upload of a build's starting state on st: top to d_init[0, sizeof(TopModel)), a zeroed BuildAux after
  // it.  One copy from page-locked memory (a pageable copy stages through the driver on the calling thread).  The slot
  // is rewritten only by the next build of this thread, which starts after this one has synchronised.
  void upload_init(void* d_init, const TopModel& top) {
    memcpy(h_init, &top, sizeof(TopModel));
    memset(h_init + sizeof(TopModel), 0, sizeof(BuildAux));
    cudaMemcpyAsync(d_init, h_init, kInitBytes, cudaMemcpyHostToDevice, st);
  }
  // After a build that needed `bytes` of scratch (its stream synchronised): a larger buffer for the next ones.
  void grow_scratch(size_t bytes) {
    if (bytes <= scratch_cap || bytes > kScratchKeepMax) return;
    if (scratch) cudaFreeAsync(scratch, st);
    scratch = nullptr;
    scratch_cap = 0;
    if (cudaMallocAsync((void**)&scratch, bytes, st) == cudaSuccess) scratch_cap = bytes;
    else { scratch = nullptr; cudaGetLastError(); }
  }
};
thread_local BuildContext t_build_ctx;
static_assert(sizeof(TopModel) % alignof(BuildAux) == 0, "the BuildAux after a TopModel in one upload must be aligned");

// A build's device scratch, carved from its thread's BuildContext buffer: once that buffer has grown to the largest
// build the thread runs, a build allocates and frees nothing on the device.  A build that needs more takes the excess
// from the stream-ordered pool for itself, and once it has synchronised the buffer grows to what it needed.  Reuse is
// safe because builds are synchronous: every stream a build uses is joined into bc->st before the build's one
// synchronisation, so nothing of a build is in flight when the next build of the same thread carves the buffer again.
// Results never live here: they go to pinned host buffers of their own (ResultBox).
struct BuildScratch {
  BuildContext* bc;
  size_t used = 0;
  std::vector<void*> extra;   // the excess of a build larger than the buffer
  cudaError_t err = cudaSuccess;
  explicit BuildScratch(BuildContext* c) : bc(c) {}
  template <class P> P* get(size_t count) {
    const size_t bytes = (std::max<size_t>(count * sizeof(P), 16) + 255) & ~(size_t)255;   // cudaMallocAsync's alignment
    used += bytes;
    if (used <= bc->scratch_cap) return (P*)(bc->scratch + used - bytes);
    void* p = nullptr;
    cudaError_t e = cudaMallocAsync(&p, bytes, bc->st);
    if (e != cudaSuccess) { err = e; return nullptr; }
    extra.push_back(p);
    return (P*)p;
  }
  ~BuildScratch() {   // runs after the build's synchronisation (or before anything was launched)
    for (void* p : extra) cudaFreeAsync(p, bc->st);
    if (err == cudaSuccess) bc->grow_scratch(used);
  }
};

struct Arena {   // stream-ordered scratch; everything is released when the call ends
  cudaStream_t st;
  std::vector<void*> ptrs;
  cudaError_t err = cudaSuccess;
  explicit Arena(cudaStream_t s) : st(s) {}
  template <class P> P* get(size_t count) {
    void* p = nullptr;
    cudaError_t e = cudaMallocAsync(&p, std::max<size_t>(count * sizeof(P), 16), st);
    if (e != cudaSuccess) { err = e; return nullptr; }
    ptrs.push_back(p);
    return (P*)p;
  }
  ~Arena() { for (void* p : ptrs) cudaFreeAsync(p, st); }
};

// ---- RMI_FLAG_TOP_FIT_EXACT for linear / robust_linear / normal tops: the reference's serial recurrence on a HOST core ----
// slr() (linear.rs:12-59) is a loop-carried chain — sub, div, add per item on mean_x — that no parallel schedule can
// reproduce bit for bit.  A CPU core runs that chain at ~20 cycles per item (the division's latency); one GPU warp
// needs ~300.  So the exact mode streams the keys back to pinned host memory (64 MiB pieces on a side stream, the copy
// of piece c+1 behind the arithmetic on piece c: the copy is far shorter than the chain) and runs the recurrence there, exactly as the reference does; the coefficients are then injected like
// rmi_train_with_top's.  Returns StatusBits (0 = ok).
template <class T> inline double host_as_float(T k) { return (double)k; }
inline uint64_t host_scale(uint64_t off, double sf, bool use_sf) { return use_sf ? (uint64_t)((double)off * sf) : off; }

template <class T>
unsigned host_exact_top(const rmi_dataset* ds, int kind, uint64_t N, double* out_f) {
  const uint64_t n = ds->n;
  const T* d_keys = (const T*)ds->d_keys;
  const double sf = (double)N / (double)n;
  const bool use_sf = std::fabs(sf - 1.0) > DBL_EPSILON;
  uint64_t i0 = 0, i1 = n;
  bool repeat = true;
  if (kind == M_ROBUST_LINEAR) {   // linear.rs:239-256: skip(bnd).take(len - 2 * bnd), never drained
    uint64_t bnd = (uint64_t)((double)n * 0.0001);
    if (bnd < 1) bnd = 1;
    if (!(bnd * 2 + 1 < n)) return ST_ROBUST_TOO_SMALL;
    i0 = bnd; i1 = n - bnd; repeat = false;
  }
  const size_t PIECE = ((size_t)64 << 20) / sizeof(T);
  T* stage[2] = {(T*)g_pinned.get(PIECE * sizeof(T)), (T*)g_pinned.get(PIECE * sizeof(T))};
  cudaStream_t cs = nullptr;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  bool ok = stage[0] && stage[1] && cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking) == cudaSuccess &&
            cudaEventCreateWithFlags(&ev[0], cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&ev[1], cudaEventDisableTiming) == cudaSuccess;
  unsigned status = 0;
  if (ok) {
    const int passes = kind == M_NORMAL ? 2 : 1;
    double mean_x = 0.0, mean_y = 0.0, c = 0.0, m2 = 0.0;   // slr state
    uint64_t cnt = 0;
    double nmean = 0.0, nstd = 0.0;                          // normal.rs:28-50 state
    const double nf = (double)n;
    T last_key = T();
    uint64_t last_F = 0;
    for (int pass = 0; pass < passes && ok; ++pass) {
      auto issue = [&](uint64_t piece) {
        const uint64_t a = piece * PIECE, b = std::min<uint64_t>(n, a + PIECE);
        cudaMemcpyAsync(stage[piece & 1], d_keys + a, (b - a) * sizeof(T), cudaMemcpyDeviceToHost, cs);
        cudaEventRecord(ev[piece & 1], cs);
      };
      const uint64_t npieces = (n + PIECE - 1) / PIECE;
      if (npieces) issue(0);
      uint64_t F = 0;
      T prev = T();
      for (uint64_t piece = 0; piece < npieces && ok; ++piece) {
        if (cudaEventSynchronize(ev[piece & 1]) != cudaSuccess) { ok = false; break; }
        if (piece + 1 < npieces) issue(piece + 1);
        const T* kb = stage[piece & 1];
        const uint64_t a = piece * PIECE, b = std::min<uint64_t>(n, a + PIECE);
        for (uint64_t i = a; i < b; ++i) {
          const T k = kb[i - a];
          if (i == 0 || k != prev) F = i;     // FixDupsIter: offset of the first key of the run (models/mod.rs:154-185)
          prev = k;
          if (kind == M_NORMAL) {
            const double x = host_as_float(k);
            if (pass == 0) nmean = nmean + x / nf;
            else { const double d = x - nmean; nstd = nstd + d * d; }
          } else if (i >= i0 && i < i1) {
            const double x = host_as_float(k), y = (double)host_scale(F, sf, use_sf);
            cnt += 1;
            const double dx = x - mean_x;
            const double cf = (double)cnt;
            mean_x = mean_x + dx / cf;
            mean_y = mean_y + (y - mean_y) / cf;
            c = c + dx * (y - mean_y);
            const double dx2 = x - mean_x;
            m2 = m2 + dx * dx2;
          }
        }
        if (b == n && n > 0) { last_key = prev; last_F = F; }
      }
      if (!ok) break;
      // the drained iterator repeats its final item (models/mod.rs:180)
      if (n > 0) {
        const double x = host_as_float(last_key);
        if (kind == M_NORMAL) {
          if (pass == 0) nmean = nmean + x / nf;
          else { const double d = x - nmean; nstd = nstd + d * d; }
        } else if (repeat) {
          const double y = (double)host_scale(last_F, sf, use_sf);
          cnt += 1;
          const double dx = x - mean_x;
          const double cf = (double)cnt;
          mean_x = mean_x + dx / cf;
          mean_y = mean_y + (y - mean_y) / cf;
          c = c + dx * (y - mean_y);
          const double dx2 = x - mean_x;
          m2 = m2 + dx * dx2;
        }
      }
    }
    if (ok) {
      if (kind == M_NORMAL) {
        out_f[0] = nmean;
        out_f[1] = std::sqrt(nstd / nf);
        out_f[2] = n > 0 ? std::fmax(-INFINITY, (double)host_scale(last_F, sf, use_sf)) : -INFINITY;
      } else {   // linear.rs:36-58
        double alpha, beta;
        if (cnt == 0) { alpha = 0.0; beta = 0.0; }
        else if (cnt == 1) { alpha = mean_y; beta = 0.0; }
        else {
          const double nm1 = (double)(cnt - 1);
          const double cov = c / nm1, var = m2 / nm1;
          if (!(var >= 0.0)) { status |= ST_NEG_VARIANCE; alpha = 0.0; beta = 0.0; }
          else if (var == 0.0) { alpha = mean_y; beta = 0.0; }
          else { beta = cov / var; alpha = mean_y - beta * mean_x; }
        }
        out_f[0] = alpha; out_f[1] = beta;
      }
    }
  }
  if (cs) { cudaStreamSynchronize(cs); cudaStreamDestroy(cs); }
  for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
  g_pinned.put(stage[0]); g_pinned.put(stage[1]);
  if (!ok) return 0x80000000u;   // CUDA failure marker (decoded by the caller)
  return status;
}
inline bool serial_top_kind(int kind) {
  return kind == M_LINEAR || kind == M_ROBUST_LINEAR || kind == M_LOGLINEAR || kind == M_NORMAL;
}
inline bool host_exact_kind(int kind) { return kind == M_LINEAR || kind == M_ROBUST_LINEAR || kind == M_NORMAL; }
// exact serial tops on at least this many keys run on a host core (host_exact_top); smaller sets keep the one-warp
// device chain (no PCIe round trip, and the CPU tests of the chain itself stay meaningful)
constexpr uint64_t HOST_EXACT_MIN = (uint64_t)1 << 20;

template <class T>
int train_typed(const rmi_dataset* ds, const ModelName& top, const ModelName& leaf, uint64_t N, uint32_t flags,
                const double* l0_over, uint32_t n_over, rmi_result** out) {
  auto t_start = std::chrono::steady_clock::now();
  const uint64_t n = ds->n;
  const T* keys = (const T*)ds->d_keys;
  CUDA_TRY(cudaSetDevice(ds->device));
  DeviceInfo di;
  if (int rc = device_info(ds->device, &di)) return rc;

  // stream + events of a build: created once per host thread and device, reused by later calls
  BuildContext* bc = t_build_ctx.get(ds->device);
  if (!bc) return fail(RMI_ERR_CUDA, "could not create the build's CUDA streams / events");
  cudaStream_t st = bc->st;
  cudaEvent_t ev0 = bc->ev0, ev1 = bc->ev1, *evp = bc->evp;
  int rc = RMI_OK;
  auto box = new ResultBox();
  {
    BuildScratch A(bc);
    Launch L{st, di.num_sms};
    L.side = bc->side; L.ev_fork = bc->ev_fork; L.ev_join = bc->ev_join;
    L.d_long = A.get<u32>(LONG_LEAF_CAP + 1);
    const int ppm = leaf_params_per_model(leaf.kind);
    char* d_init = A.get<char>(BuildContext::kInitBytes);   // TopModel, then BuildAux (BuildContext::upload_init)
    TopModel* d_top = reinterpret_cast<TopModel*>(d_init);
    BuildAux* d_aux = reinterpret_cast<BuildAux*>(d_init + sizeof(TopModel));
    u64* d_S = A.get<u64>(N + 1);
    double* d_params = A.get<double>(N * ppm);
    u64* d_errors = A.get<u64>(N);
    u64* d_counts = A.get<u64>(N);
    void* d_scratch = A.get<char>(top_scratch_bytes(N));
    void* d_stats = A.get<char>(stats_scratch_bytes(N));
    // the key sample the top fit leaves for the boundary search (kernels.h); not with injected top parameters
    T* d_sample = !l0_over && top_fit_writes_sample(top.kind, (flags & RMI_FLAG_TOP_FIT_EXACT) != 0)
                      ? bounds_sample_at<T>(A.get<char>(bounds_sample_bytes(n, sizeof(T)))) : nullptr;
    TopTables tables;
    tables.allocate(top, n, N, [&](size_t bytes) -> void* { return A.get<char>(bytes); });
    // pinned host buffers the results are copied into (and that the caller then reads)
    const bool stats_only = (flags & RMI_FLAG_STATS_ONLY) != 0;
    const bool want_counts = !stats_only && (flags & RMI_FLAG_LEAF_COUNTS) != 0;
    const bool host_ok = reserve_result(box, &tables, N, ppm, !stats_only, want_counts);
    if (A.err != cudaSuccess) {
      rc = fail(RMI_ERR_CUDA, std::string("scratch allocation: ") + cudaGetErrorString(A.err));
    } else if (!host_ok) {
      rc = fail(RMI_ERR_CUDA, kPinnedFailed);
    } else {
      TopModel h_top = tables.initial(top, l0_over, n_over);
      cudaEventRecord(ev0, st);
      unsigned host_status = 0;
      bool exact = (flags & RMI_FLAG_TOP_FIT_EXACT) != 0;
      bool host_top = false;
      if (exact && !l0_over && host_exact_kind(top.kind) && n >= HOST_EXACT_MIN) {
        cudaEventSynchronize(ev0);
        unsigned hs = host_exact_top<T>(ds, top.kind, N, h_top.f);
        if (hs == 0x80000000u) rc = fail(RMI_ERR_CUDA, "exact top fit: copying the keys back to the host failed");
        else { host_status |= hs; host_top = true; }
      }
      bc->upload_init(d_init, h_top);
      bool leaf_results_copied = false;
      if (!l0_over && !host_top && rc == RMI_OK)
        host_status |= fit_top_model<T>(L, keys, n, top.kind, top.table_bits, N, exact, d_top, d_aux, d_scratch, tables.t32,
                                        tables.pivots, tables.radix_index, d_sample);
      cudaEventRecord(evp[0], st);
      if (host_status == 0 && rc == RMI_OK) {
        // injected top parameters are not known to be monotone: take the streaming pass, which checks
        compute_leaf_bounds<T>(L, keys, n, top.kind, d_top, N, d_S, d_aux, /*allow_search=*/l0_over == nullptr, d_sample);
        cudaEventRecord(evp[1], st);
        {
          Shard<T> whole = whole_array<T>(n);
          whole.no_dups = ds->no_dups ? 1 : 0;
          // leaf results go to the host slice by slice while later slices compute (kernels.h: LeafCopyOut)
          LeafCopyOut* co = stats_only ? nullptr : t_slices.get(ds->device);
          if (co) {
            co->h_params = box->l1_params.data(); co->h_errors = reinterpret_cast<u64*>(box->l1_errors.data());
            co->h_counts = want_counts ? reinterpret_cast<u64*>(box->l1_counts.data()) : nullptr;
            co->used = 0;
            L.copy = co;
            leaf_results_copied = true;
          }
          fit_leaves<T>(L, keys, whole, leaf.kind, N, d_S, d_aux, d_params, d_errors, d_counts);
        }
        cudaEventRecord(evp[2], st);
        leaf_statistics(L, n, N, d_errors, d_counts, d_aux, d_stats);
      } else {
        cudaEventRecord(evp[1], st);
        cudaEventRecord(evp[2], st);
      }
      cudaEventRecord(ev1, st);
      // ---- results to the host --------------------------------------------------------------
      leaf_copy_join(L);   // slice copies issued by fit_leaves
      const bool fitted = host_status == 0;
      copy_result_to_host(box, fitted ? &tables : nullptr, d_aux, d_top,
                          fitted && !stats_only && !leaf_results_copied ? d_params : nullptr, d_errors,
                          want_counts ? d_counts : nullptr, st);
      cudaError_t e = cudaStreamSynchronize(st);
      if (rc != RMI_OK) {
        // (the exact top fit's key read-back failed: reported above)
      } else if (e != cudaSuccess) {
        rc = fail(RMI_ERR_CUDA, std::string("rmi_train: ") + cudaGetErrorString(e));
      } else if (host_status | result_aux(box).status) {
        rc = fail(RMI_ERR_PANIC, status_text(host_status | result_aux(box).status));
      } else {
        fill_result(box, top, leaf, tables, n, N);
        rmi_result& R = box->pub;
        R.device_time_ns = elapsed_ns(ev0, ev1);
        cudaEvent_t seq[5] = {ev0, evp[0], evp[1], evp[2], ev1};
        for (int q = 0; q < 4; ++q) R.phase_device_ns[q] = elapsed_ns(seq[q], seq[q + 1]);
        // only the tops the flag switches to a serial chain (k_slr_exact, k_normal_exact or host_exact_top) were fitted
        // bit for bit as the reference fits them; lognormal, cubic and the integer tops ignore the flag
        R.top_fit_exact = (exact && !l0_over && serial_top_kind(top.kind)) ? 1 : 0;
      }
    }
  }
  if (rc != RMI_OK) { cudaStreamSynchronize(st); delete box; return rc; }
  box->pub.build_time_ns =
      (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t_start).count();
  *out = &box->pub;
  return RMI_OK;
}

// Several configurations that share the top model and the branching factor (the optimizer's grid enumerates every
// leaf type for each (top, branching factor), optimizer.rs:110-125): ONE top-model fit and ONE boundary pass over the
// keys, then the fused leaf kernel once per leaf type.  Statistics only (what the search consumes, optimizer.rs:163-171).
template <class T>
int train_batch_typed(const rmi_dataset* ds, const ModelName& top, const std::vector<const ModelName*>& leaves, uint64_t N,
                      uint32_t flags, rmi_result** out) {
  auto t_start = std::chrono::steady_clock::now();
  const uint64_t n = ds->n;
  const T* keys = (const T*)ds->d_keys;
  CUDA_TRY(cudaSetDevice(ds->device));
  DeviceInfo di;
  if (int rc = device_info(ds->device, &di)) return rc;
  BuildContext* bc = t_build_ctx.get(ds->device);
  if (!bc) return fail(RMI_ERR_CUDA, "could not create the build's CUDA streams / events");
  cudaStream_t st = bc->st;
  const size_t K = leaves.size();
  std::vector<ResultBox*> boxes(K, nullptr);
  int rc = RMI_OK;
  {
    BuildScratch A(bc);
    Launch L{st, di.num_sms};
    L.side = bc->side; L.ev_fork = bc->ev_fork; L.ev_join = bc->ev_join;
    L.d_long = A.get<u32>(LONG_LEAF_CAP + 1);
    int max_ppm = 2;
    for (auto* lf : leaves) max_ppm = std::max(max_ppm, leaf_params_per_model(lf->kind));
    char* d_init = A.get<char>(BuildContext::kInitBytes);   // TopModel, then BuildAux (BuildContext::upload_init)
    TopModel* d_top = reinterpret_cast<TopModel*>(d_init);
    BuildAux* d_aux0 = reinterpret_cast<BuildAux*>(d_init + sizeof(TopModel));
    BuildAux* d_auxk = A.get<BuildAux>(K);
    u64* d_S = A.get<u64>(N + 1);
    double* d_params = A.get<double>(N * max_ppm);
    u64* d_errors = A.get<u64>(N);
    u64* d_counts = A.get<u64>(N);
    void* d_scratch = A.get<char>(top_scratch_bytes(N));
    void* d_stats = A.get<char>(stats_scratch_bytes(N));
    T* d_sample = top_fit_writes_sample(top.kind, (flags & RMI_FLAG_TOP_FIT_EXACT) != 0)
                      ? bounds_sample_at<T>(A.get<char>(bounds_sample_bytes(n, sizeof(T)))) : nullptr;
    TopTables tables;
    tables.allocate(top, n, N, [&](size_t bytes) -> void* { return A.get<char>(bytes); });
    bool host_ok = true;
    for (size_t k = 0; k < K; ++k) {
      boxes[k] = new ResultBox();
      host_ok = host_ok && reserve_result(boxes[k], nullptr, N, 0, false, false);
    }
    if (A.err != cudaSuccess) rc = fail(RMI_ERR_CUDA, std::string("scratch allocation: ") + cudaGetErrorString(A.err));
    else if (!host_ok) rc = fail(RMI_ERR_CUDA, kPinnedFailed);
    else {
      const TopModel h_top = tables.initial(top);
      cudaEventRecord(bc->ev0, st);
      bc->upload_init(d_init, h_top);
      const bool exact = (flags & RMI_FLAG_TOP_FIT_EXACT) != 0;
      unsigned host_status = fit_top_model<T>(L, keys, n, top.kind, top.table_bits, N, exact, d_top, d_aux0, d_scratch,
                                              tables.t32, tables.pivots, tables.radix_index, d_sample);
      if (host_status == 0) {
        compute_leaf_bounds<T>(L, keys, n, top.kind, d_top, N, d_S, d_aux0, /*allow_search=*/true, d_sample);
        Shard<T> whole = whole_array<T>(n);
        whole.no_dups = ds->no_dups ? 1 : 0;
        for (size_t k = 0; k < K; ++k) {
          BuildAux* d_aux = d_auxk + k;   // own status word, replacement counter and statistics per configuration
          cudaMemcpyAsync(d_aux, d_aux0, sizeof(BuildAux), cudaMemcpyDeviceToDevice, st);
          fit_leaves<T>(L, keys, whole, leaves[k]->kind, N, d_S, d_aux, d_params, d_errors, d_counts);
          leaf_statistics(L, n, N, d_errors, d_counts, d_aux, d_stats);
          copy_result_to_host(boxes[k], nullptr, d_aux, d_top, nullptr, nullptr, nullptr, st);
        }
      }
      cudaEventRecord(bc->ev1, st);
      cudaError_t e = cudaStreamSynchronize(st);
      if (e != cudaSuccess) rc = fail(RMI_ERR_CUDA, std::string("rmi_train_stats_batch: ") + cudaGetErrorString(e));
      else if (host_status) rc = fail(RMI_ERR_PANIC, status_text(host_status));
      else {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, bc->ev0, bc->ev1);
        for (size_t k = 0; k < K && rc == RMI_OK; ++k) {
          const unsigned status = result_aux(boxes[k]).status;
          if (status) { rc = fail(RMI_ERR_PANIC, std::string(top.name) + "," + leaves[k]->name + ": " + status_text(status)); break; }
          // the top tables stay on the device: the result holds their lengths (rmi_model_size) without them
          fill_result(boxes[k], top, *leaves[k], tables, n, N);
          boxes[k]->pub.device_time_ns = (uint64_t)((double)ms * 1e6 / (double)K);   // the batch's device time, shared out evenly
          boxes[k]->pub.top_fit_exact = exact && serial_top_kind(top.kind) ? 1 : 0;
        }
      }
    }
  }
  if (rc != RMI_OK) { cudaStreamSynchronize(st); for (auto* b : boxes) delete b; return rc; }
  const uint64_t wall = (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t_start).count();
  for (size_t k = 0; k < K; ++k) { boxes[k]->pub.build_time_ns = wall / K; out[k] = &boxes[k]->pub; }
  return RMI_OK;
}

int train_entry(const rmi_dataset* ds, const char* model_spec, uint64_t N, uint32_t flags, const double* l0_over,
                uint32_t n_over, rmi_result** out) {
  g_last_error.clear();
  if (!ds || !model_spec || !out) return fail(RMI_ERR_INVALID, "rmi_train: null argument");
  const ModelName *top = nullptr, *leaf = nullptr;
  if (int rc = parse_two_layer(model_spec, &top, &leaf)) return rc;
  if (int rc = check_build(ds->n, N, ds->sorted)) return rc;
  if (l0_over && (top->fparams == 0 || n_over != (uint32_t)top->fparams))
    return fail(RMI_ERR_INVALID, "rmi_train_with_top: top model has no float parameters or wrong count");
  return with_key_type(ds->key_type, [&](auto k) {
    return train_typed<decltype(k)>(ds, *top, *leaf, N, flags, l0_over, n_over, out);
  });
}

// The statuses of the boundary pass that concern a given top model: the error pass clamps the top's prediction to
// N - 1 (two_layer.rs:210-211) and fits nothing, so only the order checks of two_layer.rs:50 remain.
constexpr unsigned kEvaluateStatus = ST_NOT_SORTED | ST_NON_MONOTONE;

// The public struct of an evaluation of r over n keys, from what reserve_result / copy_result_to_host brought back (the
// error bounds and counts included, the stream synchronised): r's tables as given (the device copies were only read),
// the statistics measured.
void fill_given_result(ResultBox* box, const rmi_result* r, const ModelName& top, const ModelName& leaf,
                       const TopTables& tables, uint64_t n, bool stats_only) {
  const uint64_t N = r->branching_factor;
  if (!stats_only) memcpy(box->l1_params.data(), r->l1_params, sizeof(double) * N * leaf_params_per_model(leaf.kind));
  if (tables.t32_len) memcpy(box->table32.data(), r->l0_table32, sizeof(u32) * tables.t32_len);
  if (tables.ri_len) memcpy(box->arr1.data(), r->l0_array1, sizeof(u64) * tables.ri_len);
  if (tables.hist_bins) memcpy(box->arr2.data(), r->l0_array2, sizeof(u64) * tables.hist_bins);
  fill_result(box, top, leaf, tables, n, N);
  rmi_result& R = box->pub;
  R.l0_num_fparams = r->l0_num_fparams;
  R.l0_num_iparams = r->l0_num_iparams;
  R.top_fit_exact = r->top_fit_exact;
}

template <class T>
int evaluate_typed(const rmi_dataset* ds, const rmi_result* r, const ModelName& top, const ModelName& leaf, uint32_t flags,
                   rmi_result** out) {
  auto t_start = std::chrono::steady_clock::now();
  const uint64_t n = ds->n, N = r->branching_factor;
  const T* keys = (const T*)ds->d_keys;
  CUDA_TRY(cudaSetDevice(ds->device));
  DeviceInfo di;
  if (int rc = device_info(ds->device, &di)) return rc;
  BuildContext* bc = t_build_ctx.get(ds->device);
  if (!bc) return fail(RMI_ERR_CUDA, "could not create the build's CUDA streams / events");
  cudaStream_t st = bc->st;
  cudaEvent_t ev0 = bc->ev0, ev1 = bc->ev1, *evp = bc->evp;
  const int ppm = leaf_params_per_model(leaf.kind);
  const bool stats_only = (flags & RMI_FLAG_STATS_ONLY) != 0;
  const bool want_counts = !stats_only && (flags & RMI_FLAG_LEAF_COUNTS) != 0;
  int rc = RMI_OK;
  auto box = new ResultBox();
  {
    BuildScratch A(bc);
    Launch L{st, di.num_sms};
    char* d_init = A.get<char>(BuildContext::kInitBytes);   // TopModel, then BuildAux (BuildContext::upload_init)
    TopModel* d_top = reinterpret_cast<TopModel*>(d_init);
    BuildAux* d_aux = reinterpret_cast<BuildAux*>(d_init + sizeof(TopModel));
    u64* d_S = A.get<u64>(N + 1);
    double* d_params = A.get<double>(N * ppm);
    u64* d_errors = A.get<u64>(N);
    u64* d_counts = A.get<u64>(N);
    u64* d_scratch = A.get<u64>(2 * N);
    void* d_stats = A.get<char>(stats_scratch_bytes(N));
    TopTables tables;
    cudaEventRecord(ev0, st);
    const cudaError_t te = tables.upload(*r, st, [&](size_t bytes) -> void* { return A.get<char>(bytes); });
    const bool host_ok = reserve_result(box, &tables, N, ppm, !stats_only, want_counts);
    if (A.err != cudaSuccess) {
      rc = fail(RMI_ERR_CUDA, std::string("scratch allocation: ") + cudaGetErrorString(A.err));
    } else if (te != cudaSuccess) {
      rc = fail(RMI_ERR_CUDA, std::string("rmi_evaluate: ") + cudaGetErrorString(te));
    } else if (!host_ok) {
      rc = fail(RMI_ERR_CUDA, kPinnedFailed);
    } else {
      const TopModel h_top = tables.given(*r);
      bc->upload_init(d_init, h_top);
      cudaMemcpyAsync(d_params, r->l1_params, sizeof(double) * N * ppm, cudaMemcpyHostToDevice, st);
      cudaEventRecord(evp[0], st);
      // the streaming pass: the given top is not known to be monotone on these keys
      compute_leaf_bounds<T>(L, keys, n, top.kind, d_top, N, d_S, d_aux, /*allow_search=*/false, nullptr);
      cudaEventRecord(evp[1], st);
      evaluate_leaves<T>(L, keys, n, ds->no_dups, leaf.kind, N, d_S, d_params, d_scratch, d_errors, d_counts);
      cudaEventRecord(evp[2], st);
      leaf_statistics(L, n, N, d_errors, d_counts, d_aux, d_stats);
      cudaEventRecord(ev1, st);
      copy_result_to_host(box, nullptr, d_aux, d_top, nullptr, nullptr, nullptr, st);
      if (!stats_only) {
        cudaMemcpyAsync(box->l1_errors.data(), d_errors, sizeof(u64) * N, cudaMemcpyDeviceToHost, st);
        if (want_counts) cudaMemcpyAsync(box->l1_counts.data(), d_counts, sizeof(u64) * N, cudaMemcpyDeviceToHost, st);
      }
      cudaError_t e = cudaStreamSynchronize(st);
      const unsigned status = e == cudaSuccess ? result_aux(box).status & kEvaluateStatus : 0;
      if (e != cudaSuccess) {
        rc = fail(RMI_ERR_CUDA, std::string("rmi_evaluate: ") + cudaGetErrorString(e));
      } else if (status) {
        rc = fail(RMI_ERR_PANIC, status_text(status));
      } else {
        fill_given_result(box, r, top, leaf, tables, n, stats_only);
        rmi_result& R = box->pub;
        R.device_time_ns = elapsed_ns(ev0, ev1);
        cudaEvent_t seq[5] = {ev0, evp[0], evp[1], evp[2], ev1};
        for (int q = 0; q < 4; ++q) R.phase_device_ns[q] = elapsed_ns(seq[q], seq[q + 1]);
      }
    }
  }
  if (rc != RMI_OK) { cudaStreamSynchronize(st); delete box; return rc; }
  box->pub.build_time_ns =
      (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t_start).count();
  *out = &box->pub;
  return RMI_OK;
}

}  // namespace

extern "C" {

void rmi_thread_release(void) {
  // streams / events this host thread created for its builds (kept per thread and device so that repeated builds do
  // not re-create them): a worker thread that is about to exit hands them back here
  t_build_ctx.release();
  t_slices.release();
}

int rmi_train(const rmi_dataset* ds, const char* model_spec, uint64_t branch_factor, uint32_t flags, rmi_result** out) {
  return train_entry(ds, model_spec, branch_factor, flags, nullptr, 0, out);
}
int rmi_train_stats_batch(const rmi_dataset* ds, const char* top_model, const char* const* leaf_models, int num_leaf_models,
                          uint64_t branch_factor, uint32_t flags, rmi_result** out) {
  g_last_error.clear();
  if (!ds || !top_model || !leaf_models || num_leaf_models < 1 || !out) return fail(RMI_ERR_INVALID, "rmi_train_stats_batch: bad argument");
  const ModelName* top = nullptr;
  if (int rc = find_layer(top_model, true, &top)) return rc;
  std::vector<const ModelName*> leaves(num_leaf_models);
  for (int k = 0; k < num_leaf_models; ++k) {
    if (int rc = find_layer(leaf_models[k] ? leaf_models[k] : "(null)", false, &leaves[k])) return rc;
    if (int rc = check_leaf(leaves[k])) return rc;
  }
  if (int rc = check_build(ds->n, branch_factor, ds->sorted)) return rc;
  return with_key_type(ds->key_type, [&](auto k) {
    return train_batch_typed<decltype(k)>(ds, *top, leaves, branch_factor, flags, out);
  });
}
int rmi_train_with_top(const rmi_dataset* ds, const char* model_spec, uint64_t branch_factor, uint32_t flags,
                       const double* l0_fparams, uint32_t n_fparams, rmi_result** out) {
  if (!l0_fparams) return fail(RMI_ERR_INVALID, "rmi_train_with_top: null parameters");
  return train_entry(ds, model_spec, branch_factor, flags, l0_fparams, n_fparams, out);
}

int rmi_evaluate(const rmi_dataset* ds, const rmi_result* r, uint32_t flags, rmi_result** out) {
  g_last_error.clear();
  const std::string fn = "rmi_evaluate";
  if (!ds || !r || !out) return fail(RMI_ERR_INVALID, fn + ": null argument");
  const ModelName *top = nullptr, *leaf = nullptr;
  if (int rc = check_result(r, false, fn, &top, &leaf)) return rc;
  if (int rc = check_build(ds->n, r->branching_factor, ds->sorted)) return rc;
  return with_key_type(ds->key_type, [&](auto k) { return evaluate_typed<decltype(k)>(ds, r, *top, *leaf, flags, out); });
}

int rmi_cache_fix_device(const rmi_dataset* ds, uint64_t line_size, rmi_spline_point** out_points, uint64_t* out_count,
                         rmi_cache_fix_stats* stats) {
  g_last_error.clear();
  const std::string fn = "rmi_cache_fix_device";
  if (!ds || !out_points || !out_count) return fail(RMI_ERR_INVALID, fn + ": null argument");
  if (ds->key_type != RMI_KEY_U64) return fail(RMI_ERR_INVALID, fn + ": Can only construct a bounded RMI on u64 data");
  // The host scan's panics, in its order (cache_fix.hpp).  Nothing else can fire on sorted keys: along the point
  // stream x strictly increases (a key's minus point is emitted only when it differs from the previous key, and
  // key - 1 >= previous key for distinct sorted keys), so minus_epsilon's and add_point's ordering asserts hold, and
  // offsets never decrease, so dest.1 >= from_y holds.  The one exception is key 0: its minus point wraps to
  // 2^64 - 1 and with_new_dest then refuses the following point (0, 0).
  const uint64_t n = ds->n;
  if (!(n > line_size)) return fail(RMI_ERR_PANIC, "Cannot apply a cachefix with fewer items than the line size");
  if (line_size == 0) return fail(RMI_ERR_PANIC, "attempt to divide by zero");
  if (!ds->sorted) return fail(RMI_ERR_PANIC, "keys are not sorted in ascending order");
  CUDA_TRY(cudaSetDevice(ds->device));
  DeviceInfo di;
  if (int rc = device_info(ds->device, &di)) return rc;
  BuildContext* bc = t_build_ctx.get(ds->device);
  if (!bc) return fail(RMI_ERR_CUDA, fn + ": could not create the CUDA stream");
  cudaStream_t st = bc->st;
  const u64* keys = (const u64*)ds->d_keys;
  uint64_t first = 0;
  CUDA_TRY(cudaMemcpyAsync(&first, keys, sizeof(u64), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (first == 0) return fail(RMI_ERR_PANIC, "When source x is 18446744073709551615, cannot set dest x to 0");

  const u64 chunk = CACHEFIX_CHUNK, nch = (n + chunk - 1) / chunk;
  u64 h_stats[CF_NUM_STATS] = {};
  rmi_spline_point* host = nullptr;
  u64 total = 0;
  cudaError_t e = cudaSuccess;
  {
    Arena A(st);
    CacheFixScratch s;
    s.targets = A.get<u64>(nch * CACHEFIX_TARGETS);
    s.spec_count = A.get<u64>(nch);
    s.spec_exit = A.get<u64>(nch);
    s.stitch_exit = A.get<u64>(nch);
    s.stitch_ok = A.get<u32>(nch);
    s.entry = A.get<u64>(nch);
    s.count = A.get<u64>(nch);
    s.offsets = A.get<u64>(nch + 1);
    s.last_knot = A.get<u64>(2);
    s.stats = A.get<u64>(CF_NUM_STATS);
    e = A.err;
    if (e == cudaSuccess) e = cudaMemsetAsync(s.stats, 0, sizeof(u64) * CF_NUM_STATS, st);
    Launch L{st, di.num_sms};
    if (e == cudaSuccess) {
      cache_fix_scan(L, keys, n, line_size, chunk, s);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&total, s.offsets + nch, sizeof(u64), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    ++total;   // finish()'s last point
    u64* d_out = e == cudaSuccess ? A.get<u64>(2 * total) : nullptr;
    if (e == cudaSuccess) e = A.err;
    if (e == cudaSuccess) {
      cache_fix_emit(L, keys, n, line_size, chunk, s, d_out);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_stats, s.stats, sizeof h_stats, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) {
      host = static_cast<rmi_spline_point*>(std::malloc(total * sizeof(rmi_spline_point)));
      if (!host) return fail(RMI_ERR_INVALID, fn + ": out of host memory");
      e = cudaMemcpyAsync(host, d_out, total * sizeof(rmi_spline_point), cudaMemcpyDeviceToHost, st);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);   // the scratch is back in the pool
  if (e != cudaSuccess) {
    std::free(host);
    return fail(RMI_ERR_CUDA, fn + ": " + cudaGetErrorString(e));
  }
  *out_points = host;
  *out_count = total;
  if (stats) {
    stats->chunk_keys = chunk;
    stats->chunks = nch;
    stats->points = h_stats[CF_STAT_POINTS];
    stats->stitch_segments = h_stats[CF_STAT_STITCH_SEGMENTS];
    stats->fallback_points = h_stats[CF_STAT_FALLBACK_POINTS];
    stats->evaluations = h_stats[CF_STAT_EVALS];
  }
  return RMI_OK;
}

}  // extern "C"

// ===========================================================================================
// Range-partitioned build (include/rmi_b200.h, "Range-partitioned (multi-GPU) build")
// ===========================================================================================
using rmihost::bits_from_key;
using rmihost::key_from_bits;
using rmihost::SlabLayout;

struct rmi_shard_build {
  const rmi_dataset* ds = nullptr;
  SlabLayout lay;
  uint64_t halo_capacity = 0;           // keys of room behind the local keys in the device array
  rmi_shard_buffers buf{};
  const ModelName* top = nullptr;
  const ModelName* leaf = nullptr;
  uint64_t N = 0;
  uint64_t halo = 0;
  cudaStream_t st = nullptr;
  int num_sms = 0;
  TopModel* d_top = nullptr;
  BuildAux* d_aux = nullptr;
  void* d_scratch = nullptr;
  void* d_stats = nullptr;
  unsigned host_status = 0;
  std::chrono::steady_clock::time_point t_start;
  cudaStream_t side = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  u32* d_long = nullptr;
  cudaEvent_t ev_begin[RMI_NUM_PHASES] = {};
  cudaEvent_t ev_end[RMI_NUM_PHASES] = {};
  bool ran[RMI_NUM_PHASES] = {};
  // rmi_shard_train: the partition of the key array over the ranks and the exchange scratch
  int world = 0, rank = 0, r_last = 0;  // r_last: the last rank that holds keys
  u64* d_bases = nullptr;               // world + 1: global index of every rank's first key
  u64* d_off = nullptr;                 // world + 1: first leaf owned by every rank
  u64* h_off = nullptr;                 // pinned mirror
  void* d_parts = nullptr;              // world x statistics partials
  unsigned* d_flags_mine = nullptr;     // {status, could_not_replace != 0}
  unsigned* d_flags_all = nullptr;      // world x 2
  unsigned* h_flags_all = nullptr;      // pinned mirror
  bool gather_mode = false;             // rmi_shard_train: owners broadcast their leaf ranges, nothing is zero-filled
  const LeafCopyOut* leaf_copy = nullptr;   // rmi_shard_train with a shared result region: sliced launch of the owned leaf window,
  u64 leaf_lo = 0, leaf_hi = 0;             //   each slice's records copied to the host while the next slice computes
  // table tops (radix8..28, histogram): the table every rank fills its part of, merged by an all-reduce MAX
  TopTables tables;
  cudaEvent_t ev_off = nullptr, ev_t0 = nullptr, ev_t1 = nullptr;
  // statistics-only batches (rmi_shard_stats_batch_create): the K leaf types and scratch of the batch's own
  std::vector<const ModelName*> batch;       // empty: an ordinary build object
  double* d_batch_params = nullptr;          // N x the largest params-per-model of the batch
  BuildAux* d_batch_aux = nullptr;           // K: every leaf type's status, replacement flag and statistics
  char* d_batch_recs = nullptr;              // world x K records (rmi_shard_train_stats_batch gathers into it)
  char* d_batch_parts = nullptr;             // K x world statistics partials, leaf type by leaf type
  unsigned char* h_batch_recs = nullptr;     // pinned: world x K records
};

struct rmi_shard_comm {
  ncclComm_t comm = nullptr;
  int world = 0, rank = 0, device = 0;
  // Node-local shared result memory (RMI_FLAG_SHARD_ROOT_ONLY): a POSIX shared-memory region every rank maps and
  // registers with CUDA, so that each rank copies the leaf records IT OWNS straight to the host buffer rank 0 reads —
  // world PCIe links in parallel instead of rank 0 pulling all N records through its own.  Two halves, used alternately.
  bool single_node = false;
  uint32_t uid_hash = 0;
  int shm_gen = 0;
  unsigned char* shm = nullptr;
  size_t shm_half = 0;            // bytes of one half
  int parity = 0;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_leaf_done = nullptr, ev_copy_done = nullptr;
  unsigned* d_token = nullptr;    // 4 bytes: the payload of the "copies have landed" all-reduce
};

namespace {

// The kernels' view of a rank's slab: its place among the others, its own keys and the halo keys readable behind them.
template <class T> Shard<T> shard_of(const SlabLayout& lay, uint64_t n_local, uint64_t n_avail) {
  Shard<T> s;
  s.base = lay.base;
  s.n_global = lay.n_global;
  s.n_local = n_local;
  s.n_avail = n_avail;
  s.has_prev = lay.has_prev;
  s.is_last = lay.is_last;
  s.prev_key = key_from_bits<T>(lay.prev_key_bits);
  s.prev_F = lay.prev_F;
  s.no_dups = lay.no_dups ? 1 : 0;   // global: no rank has equal keys and none straddle a cut
  return s;
}

template <class T> int shard_ends_typed(const rmi_dataset* ds, rmi_shard_ends* out) {
  out->n_local = ds->n;
  out->no_dups = ds->no_dups ? 1 : 0;
  out->first_key_bits = out->last_key_bits = out->last_run_start = 0;
  if (ds->n == 0) return RMI_OK;
  const T* keys = (const T*)ds->d_keys;
  T first, last;
  CUDA_TRY(cudaMemcpy(&first, keys, sizeof(T), cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(&last, keys + (ds->n - 1), sizeof(T), cudaMemcpyDeviceToHost));
  out->first_key_bits = bits_from_key<T>(first);
  out->last_key_bits = bits_from_key<T>(last);
  // first index whose key equals the last key: host-driven binary search (a handful of 8-byte reads)
  uint64_t lo = 0, hi = ds->n - 1;
  while (lo < hi) {
    uint64_t mid = lo + (hi - lo) / 2;
    T v;
    CUDA_TRY(cudaMemcpy(&v, keys + mid, sizeof(T), cudaMemcpyDeviceToHost));
    if (v == last) hi = mid; else lo = mid + 1;
  }
  out->last_run_start = lo;
  return RMI_OK;
}

template <class T> int shard_phase_typed(rmi_shard_build* b, int phase) {
  const T* keys = (const T*)b->ds->d_keys;
  Shard<T> sh = shard_of<T>(b->lay, b->ds->n, b->ds->n + b->halo);
  Launch L{b->st, b->num_sms};
  L.side = b->side; L.ev_fork = b->ev_fork; L.ev_join = b->ev_join; L.d_long = b->d_long;
  const int ppm = leaf_params_per_model(b->leaf->kind);
  if (phase >= 0 && phase < RMI_NUM_PHASES) { cudaEventRecord(b->ev_begin[phase], b->st); b->ran[phase] = true; }
  if (phase == RMI_PHASE_TOP_LOCAL) {   // a build object may be reused for many builds
    b->t_start = std::chrono::steady_clock::now();
    b->host_status = 0;
    for (int q = 1; q < RMI_NUM_PHASES; ++q) b->ran[q] = false;
  }
  const T first_key = key_from_bits<T>(b->lay.first_key_bits), last_key = key_from_bits<T>(b->lay.last_key_bits);
  const TopTables& tt = b->tables;
  switch (phase) {
    case RMI_PHASE_TOP_LOCAL:
      cudaMemsetAsync(b->d_aux, 0, sizeof(BuildAux), b->st);
      {
        const TopModel h = tt.initial(*b->top);
        cudaMemcpyAsync(b->d_top, &h, sizeof(h), cudaMemcpyHostToDevice, b->st);
      }
      if (b->top->kind == M_HISTOGRAM && (tt.hist_bins == 0 || tt.hist_ipb < 1)) b->host_status |= ST_HIST_BINS;   // histogram.rs:25-27
      b->host_status |= shard_top_local<T>(L, keys, sh, b->top->kind, b->N, b->lay.pivot_x, b->lay.pivot_y, first_key,
                                           last_key, b->lay.last_F, b->d_scratch, (double*)b->buf.sums, b->d_top,
                                           b->d_aux, tt.bradix_counts);
      if ((b->top->kind == M_RADIX_TABLE || b->top->kind == M_HISTOGRAM) && b->host_status == 0)
        shard_table_local<T>(L, keys, sh, b->top->kind, b->top->table_bits, b->N, first_key, last_key, b->d_aux, tt.t32,
                             tt.pivots, tt.hist_bins, tt.hist_ipb);
      break;
    case RMI_PHASE_TOP_MID:
      shard_top_mid<T>(L, keys, sh, b->top->kind, b->N, first_key, last_key, b->d_scratch, (double*)b->buf.sums, b->d_aux);
      break;
    case RMI_PHASE_TOP_FINISH:
      shard_top_finish<T>(L, sh, b->top->kind, b->N, b->lay.pivot_x, b->lay.pivot_y, (const double*)b->buf.sums,
                          first_key, last_key, b->lay.last_F, b->d_scratch, tt.bradix_counts, b->d_top, b->d_aux);
      if (b->top->kind == M_RADIX_TABLE && b->host_status == 0) shard_table_decode(L, b->top->table_bits, tt.t32);
      if (b->top->kind == M_HISTOGRAM && b->host_status == 0) hist_radix_index(L, tt.pivots, tt.hist_bins, tt.radix_index);
      break;
    case RMI_PHASE_BOUNDS:
      shard_bounds<T>(L, keys, sh, b->top->kind, b->d_top, b->N, (u64*)b->buf.S, b->d_aux);
      break;
    case RMI_PHASE_SPLIT:
      shard_split<T>(L, keys, sh, b->top->kind, b->d_top, b->N, (const u64*)b->buf.S, b->d_aux);
      break;
    case RMI_PHASE_LEAF:
      if (!b->gather_mode) {   // host-driven flow: the leaf records are combined by an all-reduce SUM of zero-filled arrays
        cudaMemsetAsync(b->buf.params, 0, sizeof(double) * b->N * ppm, b->st);
        cudaMemsetAsync(b->buf.errors, 0, sizeof(u64) * b->N, b->st);
        cudaMemsetAsync(b->buf.counts, 0, sizeof(u64) * b->N, b->st);
      }
      L.copy = b->leaf_copy; L.leaf_lo = b->leaf_lo; L.leaf_hi = b->leaf_hi;
      fit_leaves<T>(L, keys, sh, b->leaf->kind, b->N, (const u64*)b->buf.S, b->d_aux, (double*)b->buf.params,
                    (u64*)b->buf.errors, (u64*)b->buf.counts);
      L.copy = nullptr; L.leaf_lo = L.leaf_hi = 0;
      shard_copy_status(L, b->d_aux, (unsigned*)b->buf.status);
      break;
    case RMI_PHASE_STATS:
      leaf_statistics(L, b->lay.n_global, b->N, (const u64*)b->buf.errors, (const u64*)b->buf.counts, b->d_aux, b->d_stats);
      break;
    default:
      return fail(RMI_ERR_INVALID, "rmi_shard_phase: unknown phase");
  }
  if (phase >= 0 && phase < RMI_NUM_PHASES) cudaEventRecord(b->ev_end[phase], b->st);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(RMI_ERR_CUDA, std::string("rmi_shard_phase: ") + cudaGetErrorString(e));
  return RMI_OK;
}

// The checks of a gathered ends table that the consumers of range-partitioned keys (rmi_shard_build_create,
// rmi_shard_index_create, rmi_shard_eval_create) make before any device work, with RMI_ERR_INVALID and messages naming
// fn: world and rank in range, ends_all[rank] describing `local`, the non-empty slabs in key order.  *base / *total:
// this rank's global index of its first key and the keys of all slabs.
int check_slabs(const std::string& fn, const rmi_dataset* local, const rmi_shard_ends* ends_all, int world, int rank,
                uint64_t* base, uint64_t* total) {
  if (world < 1 || world > SHARD_ROUTE_MAX - 1 || rank < 0 || rank >= world)
    return fail(RMI_ERR_INVALID, fn + ": bad world or rank (0 <= rank < world <= 63)");
  if (ends_all[rank].n_local != local->n)
    return fail(RMI_ERR_INVALID, fn + ": ends_all[" + std::to_string(rank) + "] describes " +
                                     std::to_string(ends_all[rank].n_local) + " keys, the local dataset holds " +
                                     std::to_string(local->n));
  *total = 0;
  for (int p = 0; p < world; ++p) {
    if (p == rank) *base = *total;
    *total += ends_all[p].n_local;
  }
  // the non-empty slabs must follow each other in key order: no slab's last key above the next one's first
  int prev = -1;
  const int bad = with_key_type(local->key_type, [&](auto k) {
    using T = decltype(k);
    for (int p = 0; p < world; ++p) {
      if (!ends_all[p].n_local) continue;
      if (prev >= 0 && key_from_bits<T>(ends_all[p].first_key_bits) < key_from_bits<T>(ends_all[prev].last_key_bits))
        return p;
      prev = p;
    }
    return -1;
  });
  if (bad >= 0)
    return fail(RMI_ERR_INVALID, fn + ": the slabs are out of order (rank " + std::to_string(bad) +
                                     "'s first key is below the last key of rank " + std::to_string(prev) + ")");
  return RMI_OK;
}

}  // namespace

extern "C" {

uint32_t rmi_params_per_model(const char* leaf_model_name) {
  const ModelName* m = leaf_model_name ? find_model(leaf_model_name) : nullptr;
  return m ? (uint32_t)leaf_params_per_model(m->kind) : 0;
}

int rmi_shard_top_rounds(const char* top_model_name) {
  const ModelName* m = top_model_name ? find_model(top_model_name) : nullptr;
  return m ? m->shard_rounds : -1;
}

int rmi_shard_ends_get(const rmi_dataset* ds, rmi_shard_ends* out) {
  if (!ds || !out) return fail(RMI_ERR_INVALID, "rmi_shard_ends_get: null argument");
  CUDA_TRY(cudaSetDevice(ds->device));
  return with_key_type(ds->key_type, [&](auto k) { return shard_ends_typed<decltype(k)>(ds, out); });
}

int rmi_shard_build_create(const rmi_dataset* local, const rmi_shard_ends* ends_all, int world, int rank,
                           const char* model_spec, uint64_t branch_factor, uint64_t halo_capacity,
                           const rmi_shard_buffers* buffers, void* cuda_stream, rmi_shard_build** out) {
  const std::string fn = "rmi_shard_build_create";
  g_last_error.clear();
  if (!local || !ends_all || !model_spec || !buffers || !out) return fail(RMI_ERR_INVALID, fn + ": null argument");
  const ModelName *top = nullptr, *leaf = nullptr;
  if (int rc = parse_two_layer(model_spec, &top, &leaf)) return rc;
  if (top->shard_rounds < 0)   // every top model of the table is offered now; the check stays for the table's contract
    return fail(RMI_ERR_UNSUPPORTED, "range-partitioned builds do not offer the top model " + std::string(top->name));
  uint64_t total = 0, base = 0;
  if (int rc = check_slabs(fn, local, ends_all, world, rank, &base, &total)) return rc;
  if (int rc = check_build(total, branch_factor, local->sorted)) return rc;
  CUDA_TRY(cudaSetDevice(local->device));
  DeviceInfo di;
  if (int rc = device_info(local->device, &di)) return rc;
  auto* b = new rmi_shard_build();
  b->ds = local; b->buf = *buffers; b->top = top; b->leaf = leaf; b->N = branch_factor;
  b->st = (cudaStream_t)cuda_stream; b->num_sms = di.num_sms; b->halo = 0; b->halo_capacity = halo_capacity;
  b->t_start = std::chrono::steady_clock::now();
  b->lay = with_key_type(local->key_type, [&](auto k) {
    return rmihost::slab_layout<decltype(k)>(ends_all, world, rank, branch_factor);
  });
  b->world = world; b->rank = rank;
  std::vector<uint64_t> bases(world + 1, 0);
  for (int r = 0; r < world; ++r) {
    bases[r + 1] = bases[r] + ends_all[r].n_local;
    if (ends_all[r].n_local) b->r_last = r;
  }
  bool ok = cudaMalloc(&b->d_top, sizeof(TopModel)) == cudaSuccess && cudaMalloc(&b->d_aux, sizeof(BuildAux)) == cudaSuccess &&
            cudaMalloc(&b->d_scratch, shard_scratch_bytes()) == cudaSuccess &&
            cudaMalloc(&b->d_stats, stats_scratch_bytes(branch_factor)) == cudaSuccess;
  for (int q = 0; q < RMI_NUM_PHASES; ++q) ok = ok && cudaEventCreate(&b->ev_begin[q]) == cudaSuccess && cudaEventCreate(&b->ev_end[q]) == cudaSuccess;
  {
    int lo_prio = 0, hi_prio = 0;
    cudaDeviceGetStreamPriorityRange(&lo_prio, &hi_prio);
    ok = ok && cudaStreamCreateWithPriority(&b->side, cudaStreamNonBlocking, hi_prio) == cudaSuccess &&
         cudaEventCreateWithFlags(&b->ev_fork, cudaEventDisableTiming) == cudaSuccess &&
         cudaEventCreateWithFlags(&b->ev_join, cudaEventDisableTiming) == cudaSuccess &&
         cudaMalloc((void**)&b->d_long, sizeof(u32) * (LONG_LEAF_CAP + 1)) == cudaSuccess;
  }
  ok = ok && b->tables.allocate(*top, total, branch_factor, device_alloc) &&
       b->tables.allocate_shard_counts(*top, branch_factor, device_alloc);
  // rmi_shard_train's exchange: leaf ownership, statistics partials and status words of every rank
  ok = ok && cudaMalloc((void**)&b->d_bases, sizeof(u64) * (world + 1)) == cudaSuccess &&
       cudaMalloc((void**)&b->d_off, sizeof(u64) * (world + 1)) == cudaSuccess &&
       cudaMalloc(&b->d_parts, stats_partial_bytes() * world) == cudaSuccess &&
       cudaMalloc((void**)&b->d_flags_mine, 2 * sizeof(unsigned)) == cudaSuccess &&
       cudaMalloc((void**)&b->d_flags_all, 2 * sizeof(unsigned) * world) == cudaSuccess &&
       cudaMallocHost((void**)&b->h_off, sizeof(u64) * (world + 1)) == cudaSuccess &&
       cudaMallocHost((void**)&b->h_flags_all, 2 * sizeof(unsigned) * world) == cudaSuccess &&
       cudaEventCreateWithFlags(&b->ev_off, cudaEventDisableTiming) == cudaSuccess &&
       cudaEventCreate(&b->ev_t0) == cudaSuccess && cudaEventCreate(&b->ev_t1) == cudaSuccess &&
       cudaMemcpy(b->d_bases, bases.data(), sizeof(u64) * (world + 1), cudaMemcpyHostToDevice) == cudaSuccess;
  if (!ok) { rmi_shard_build_destroy(b); return fail(RMI_ERR_CUDA, fn + ": device allocation failed"); }
  *out = b;
  return RMI_OK;
}

int rmi_shard_top_table(const rmi_shard_build* b, rmi_shard_top_table_info* out) {
  if (!b || !out) return fail(RMI_ERR_INVALID, "rmi_shard_top_table: null argument");
  const TopTables& tt = b->tables;
  *out = rmi_shard_top_table_info{};
  if (b->top->kind == M_RADIX_TABLE) {
    *out = {tt.t32, tt.t32_len, (uint32_t)sizeof(u32), RMI_TABLE_REDUCE_MAX};
  } else if (b->top->kind == M_HISTOGRAM) {
    *out = {tt.pivots, tt.hist_bins, (uint32_t)sizeof(u64), RMI_TABLE_REDUCE_MAX};
  } else if (b->top->kind == M_BRADIX) {
    *out = {tt.bradix_counts, tt.bradix_len, (uint32_t)sizeof(u32), RMI_TABLE_REDUCE_SUM};
  }
  return RMI_OK;
}

int rmi_shard_phase(rmi_shard_build* b, int phase) {
  if (!b) return fail(RMI_ERR_INVALID, "rmi_shard_phase: null build");
  if (!b->batch.empty() && (phase == RMI_PHASE_LEAF || phase == RMI_PHASE_STATS))
    return fail(RMI_ERR_INVALID, "rmi_shard_phase: a statistics batch runs its leaves with rmi_shard_stats_leaf");
  b->gather_mode = false;   // host-driven flow: the caller combines the leaf records with an all-reduce SUM of zero-filled arrays
  CUDA_TRY(cudaSetDevice(b->ds->device));
  return with_key_type(b->ds->key_type, [&](auto k) { return shard_phase_typed<decltype(k)>(b, phase); });
}

int rmi_shard_set_halo(rmi_shard_build* b, uint64_t halo_keys) {
  if (!b) return fail(RMI_ERR_INVALID, "rmi_shard_set_halo: null build");
  if (halo_keys > b->halo_capacity) return fail(RMI_ERR_INVALID, "rmi_shard_set_halo: halo exceeds the capacity behind the local keys");
  b->halo = halo_keys;
  return RMI_OK;
}

}  // extern "C"

// The public result from what copy_result_to_host brought back (after the stream has been synchronised).
// st_all: OR of every rank's status word; cnr: some rank could not replace an empty leaf.
static int shard_result(rmi_shard_build* b, ResultBox* box, unsigned st_all, bool cnr, const uint64_t* total_device_ns,
                        rmi_result** out, const ModelName* leaf = nullptr) {
  if (st_all) {
    std::string msg = status_text((b->host_status | result_aux(box).status | st_all) & ~ST_HALO_TOO_SMALL);
    if (st_all & ST_HALO_TOO_SMALL) msg += (msg.empty() ? "" : "; ") + std::string("a leaf reaches past the halo copied from the next rank");
    if (msg.empty()) msg = "another rank reported a failure";
    delete box;
    return fail(RMI_ERR_PANIC, msg);
  }
  fill_result(box, *b->top, leaf ? *leaf : *b->leaf, b->tables, b->lay.n_global, b->N);
  rmi_result& R = box->pub;
  {   // device time of this rank's phases (collectives between them are not included)
    const int map[RMI_NUM_PHASES] = {0, 0, 1, 1, 2, 3, 0};
    for (int q = 0; q < RMI_NUM_PHASES; ++q) {
      if (!b->ran[q]) continue;
      const uint64_t ns = elapsed_ns(b->ev_begin[q], b->ev_end[q]);
      R.phase_device_ns[map[q]] += ns;
      R.device_time_ns += ns;
    }
  }
  if (total_device_ns) R.device_time_ns = *total_device_ns;   // whole build on the stream, collectives included
  R.could_not_replace = cnr ? 1 : 0;   // two_layer.rs:199-203: ANY leaf, on any rank
  R.build_time_ns = (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - b->t_start).count();
  *out = &box->pub;
  return RMI_OK;
}

extern "C" {

int rmi_shard_finish(rmi_shard_build* b, uint32_t flags, rmi_result** out) {
  if (!b || !out) return fail(RMI_ERR_INVALID, "rmi_shard_finish: null argument");
  CUDA_TRY(cudaSetDevice(b->ds->device));
  const bool stats_only = (flags & RMI_FLAG_STATS_ONLY) != 0;
  const bool want_counts = !stats_only && (flags & RMI_FLAG_LEAF_COUNTS) != 0;
  auto box = new ResultBox();
  if (!reserve_result(box, &b->tables, b->N, leaf_params_per_model(b->leaf->kind), !stats_only, want_counts)) {
    delete box;
    return fail(RMI_ERR_CUDA, kPinnedFailed);
  }
  copy_result_to_host(box, &b->tables, b->d_aux, b->d_top, stats_only ? nullptr : (const double*)b->buf.params,
                      (const u64*)b->buf.errors, want_counts ? (const u64*)b->buf.counts : nullptr, b->st);
  unsigned h_status = 0;
  cudaError_t e = cudaStreamSynchronize(b->st);
  if (e == cudaSuccess) e = cudaMemcpy(&h_status, b->buf.status, sizeof(unsigned), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) { delete box; return fail(RMI_ERR_CUDA, std::string("rmi_shard_finish: ") + cudaGetErrorString(e)); }
  // host-driven flow: buffers.status holds whatever the caller combined over the ranks (sharded.py: a bitwise OR)
  const BuildAux& h_aux = result_aux(box);
  return shard_result(b, box, b->host_status | h_aux.status | h_status, h_aux.could_not_replace != 0, nullptr, out);
}

// ---- the whole range-partitioned build in one call, collectives issued on the build's stream ----------
#define NCCL_TRY(expr)                                                                                          \
  do {                                                                                                          \
    ncclResult_t _r = (expr);                                                                                   \
    if (_r != ncclSuccess) return fail(RMI_ERR_CUDA, std::string(#expr) + ": " + nccl_api().GetErrorString(_r)); \
  } while (0)

int rmi_shard_comm_unique_id(void* out_id128) {
  g_last_error.clear();
  if (!out_id128) return fail(RMI_ERR_INVALID, "rmi_shard_comm_unique_id: null argument");
  const NcclApi& nc = nccl_api();
  if (!nc.ok) return fail(RMI_ERR_UNSUPPORTED, nc.error);
  ncclUniqueId id;
  NCCL_TRY(nc.GetUniqueId(&id));
  static_assert(sizeof(id) == 128, "ncclUniqueId is 128 bytes");
  memcpy(out_id128, &id, sizeof(id));
  return RMI_OK;
}

int rmi_shard_comm_create(const void* id128, int world, int rank, int device, rmi_shard_comm** out) {
  g_last_error.clear();
  if (!id128 || !out || world < 1 || world > 63 || rank < 0 || rank >= world)
    return fail(RMI_ERR_INVALID, "rmi_shard_comm_create: bad argument (1 <= world <= 63)");
  const NcclApi& nc = nccl_api();
  if (!nc.ok) return fail(RMI_ERR_UNSUPPORTED, nc.error);
  CUDA_TRY(cudaSetDevice(device));
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  auto* c = new rmi_shard_comm();
  c->world = world; c->rank = rank; c->device = device;
  ncclResult_t r = nc.CommInitRank(&c->comm, world, id, rank);
  if (r != ncclSuccess) { delete c; return fail(RMI_ERR_CUDA, std::string("ncclCommInitRank: ") + nc.GetErrorString(r)); }
  for (size_t i = 0; i < sizeof(id); ++i) c->uid_hash = c->uid_hash * 16777619u ^ (unsigned char)id.internal[i];
  // are all ranks on this host?  (all-gather of a host-name hash; the shared result region needs one node)
  {
    char host[256] = {0};
    gethostname(host, sizeof(host) - 1);
    unsigned long long hh = 1469598103934665603ull;
    for (const char* p = host; *p; ++p) hh = (hh ^ (unsigned char)*p) * 1099511628211ull;
    unsigned long long* d_h = nullptr;
    std::vector<unsigned long long> all(world, 0);
    bool ok = cudaMalloc((void**)&d_h, sizeof(unsigned long long) * world) == cudaSuccess &&
              cudaMemcpy(d_h + rank, &hh, sizeof(hh), cudaMemcpyHostToDevice) == cudaSuccess &&
              nc.AllGather(d_h + rank, d_h, 1, ncclUint64, c->comm, nullptr) == ncclSuccess &&
              cudaDeviceSynchronize() == cudaSuccess &&
              cudaMemcpy(all.data(), d_h, sizeof(unsigned long long) * world, cudaMemcpyDeviceToHost) == cudaSuccess;
    cudaFree(d_h);
    c->single_node = ok;
    for (int q = 0; q < world && ok; ++q) if (all[q] != hh) c->single_node = false;
    ok = cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking) == cudaSuccess &&
         cudaEventCreateWithFlags(&c->ev_leaf_done, cudaEventDisableTiming) == cudaSuccess &&
         cudaEventCreateWithFlags(&c->ev_copy_done, cudaEventDisableTiming) == cudaSuccess &&
         cudaMalloc((void**)&c->d_token, sizeof(unsigned)) == cudaSuccess && cudaMemset(c->d_token, 0, sizeof(unsigned)) == cudaSuccess;
    if (!ok) { c->single_node = false; cudaGetLastError(); }
  }
  *out = c;
  return RMI_OK;
}

static void comm_release_shared(rmi_shard_comm* c) {
  if (c->shm) {
    cudaHostUnregister(c->shm);
    munmap(c->shm, 2 * c->shm_half);
    c->shm = nullptr; c->shm_half = 0;
  }
}

// Collective over the communicator: make sure a shared, CUDA-registered host region of 2 x `half` bytes exists.
static int comm_ensure_shared(rmi_shard_comm* c, size_t half, cudaStream_t st) {
  if (c->shm && c->shm_half >= half) return RMI_OK;
  const NcclApi& nc = nccl_api();
  comm_release_shared(c);
  half = (half + 4095) & ~(size_t)4095;
  char name[64];
  std::snprintf(name, sizeof name, "/rmi_b200_%08x_%d", c->uid_hash, ++c->shm_gen);
  auto barrier = [&]() -> bool {
    return nc.AllReduce(c->d_token, c->d_token, 1, ncclUint32, ncclMax, c->comm, st) == ncclSuccess && cudaStreamSynchronize(st) == cudaSuccess;
  };
  void* base = MAP_FAILED;
  bool ok = true;
  if (c->rank == 0) {
    shm_unlink(name);
    int fd = shm_open(name, O_CREAT | O_EXCL | O_RDWR, 0600);
    ok = fd >= 0 && ftruncate(fd, (off_t)(2 * half)) == 0;
    if (ok) base = mmap(nullptr, 2 * half, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    if (fd >= 0) close(fd);
    ok = ok && base != MAP_FAILED;
  }
  if (!barrier()) ok = false;          // the region exists (or rank 0 failed: found out below)
  if (c->rank != 0) {
    int fd = shm_open(name, O_RDWR, 0600);
    ok = fd >= 0;
    if (ok) base = mmap(nullptr, 2 * half, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    if (fd >= 0) close(fd);
    ok = ok && base != MAP_FAILED;
  }
  if (!barrier()) ok = false;          // everyone has mapped it: the name can go
  if (c->rank == 0) shm_unlink(name);
  if (ok && cudaHostRegister(base, 2 * half, cudaHostRegisterPortable) != cudaSuccess) { cudaGetLastError(); ok = false; }
  // agree on the outcome (a rank that failed must not leave the others copying into a region it cannot see)
  unsigned mine = ok ? 0u : 1u, any = 1u;
  if (cudaMemcpy(c->d_token, &mine, sizeof(mine), cudaMemcpyHostToDevice) == cudaSuccess && barrier() &&
      cudaMemcpy(&any, c->d_token, sizeof(any), cudaMemcpyDeviceToHost) == cudaSuccess) {
    unsigned zero = 0;
    cudaMemcpy(c->d_token, &zero, sizeof(zero), cudaMemcpyHostToDevice);
  }
  if (any != 0) {
    if (ok) cudaHostUnregister(base);
    if (base != MAP_FAILED) munmap(base, 2 * half);
    c->single_node = false;   // fall back for good: rank 0 pulls the whole result through its own link
    return RMI_OK;
  }
  c->shm = (unsigned char*)base;
  c->shm_half = half;
  return RMI_OK;
}

void rmi_shard_comm_destroy(rmi_shard_comm* c) {
  if (!c) return;
  comm_release_shared(c);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  if (c->ev_leaf_done) cudaEventDestroy(c->ev_leaf_done);
  if (c->ev_copy_done) cudaEventDestroy(c->ev_copy_done);
  cudaFree(c->d_token);
  if (c->comm && nccl_api().ok) nccl_api().CommDestroy(c->comm);
  delete c;
}

}  // extern "C"

// The top model and the leaf boundaries of a one-call build (rmi_shard_train, rmi_shard_train_stats_batch): phases
// RMI_PHASE_TOP_LOCAL to RMI_PHASE_SPLIT and their collectives, enqueued on the build's stream.  mark(what): a trace
// point after each step.
template <class T, class Mark>
static int shard_top_and_bounds(rmi_shard_build* b, rmi_shard_comm* c, Mark&& mark) {
  const NcclApi& nc = nccl_api();
  const uint64_t N = b->N;
  const int W = b->world;
  cudaStream_t st = b->st;
  ncclComm_t comm = c->comm;
  double* sums = (double*)b->buf.sums;
  int rc = RMI_OK;
  auto phase = [&](int ph) { if (rc == RMI_OK) rc = shard_phase_typed<T>(b, ph); };
  auto nccl = [&](ncclResult_t r, const char* what) {
    if (rc == RMI_OK && r != ncclSuccess) rc = fail(RMI_ERR_CUDA, std::string(what) + ": " + nc.GetErrorString(r));
  };
  // ---- top model: local part, 0-2 tiny all-reduces, closed form (identical on every rank) -----------------
  phase(RMI_PHASE_TOP_LOCAL);
  mark("top local");
  const int rounds = b->top->shard_rounds;
  if (W > 1 && rc == RMI_OK) {
    if (rounds == 1 || rounds == 2) nccl(nc.AllReduce(sums, sums, 8, ncclFloat64, ncclSum, comm, st), "ncclAllReduce(top sums)");
    if (rounds == 3) nccl(nc.AllReduce(sums + 8, sums + 8, 4, ncclInt64, ncclMin, comm, st), "ncclAllReduce(cubic interior points)");
    if (rounds == 4 && b->host_status == 0) {   // table tops: merge the ranks' partial tables (rmi_shard_top_table)
      const TopTables& tt = b->tables;
      if (b->top->kind == M_RADIX_TABLE)
        nccl(nc.AllReduce(tt.t32, tt.t32, tt.t32_len, ncclUint32, ncclMax, comm, st), "ncclAllReduce(radix table)");
      else if (b->top->kind == M_BRADIX)
        nccl(nc.AllReduce(tt.bradix_counts, tt.bradix_counts, tt.bradix_len, ncclUint32, ncclSum, comm, st),
             "ncclAllReduce(bradix counts)");
      else
        nccl(nc.AllReduce(tt.pivots, tt.pivots, tt.hist_bins, ncclUint64, ncclMax, comm, st), "ncclAllReduce(histogram pivots)");
    }
  }
  if (rounds >= 2) {
    phase(RMI_PHASE_TOP_MID);
    if (W > 1 && rc == RMI_OK) nccl(nc.AllReduce(sums, sums, 8, ncclFloat64, ncclSum, comm, st), "ncclAllReduce(top sums, round 2)");
  }
  mark("top all-reduces");
  phase(RMI_PHASE_TOP_FINISH);
  mark("top finish");
  // ---- leaf boundaries: local lower bounds -> all-reduce MIN; split; who owns which leaves -----------------
  phase(RMI_PHASE_BOUNDS);
  mark("bounds");
  if (W > 1 && rc == RMI_OK) nccl(nc.AllReduce(b->buf.S, b->buf.S, N + 1, ncclUint64, ncclMin, comm, st), "ncclAllReduce(leaf boundaries)");
  mark("bounds all-reduce");
  phase(RMI_PHASE_SPLIT);
  return rc;
}

template <class T>
static int shard_train_typed(rmi_shard_build* b, rmi_shard_comm* c, uint32_t flags, rmi_result** out) {
  const NcclApi& nc = nccl_api();
  const uint64_t N = b->N;
  const int ppm = leaf_params_per_model(b->leaf->kind);
  const int W = b->world, rank = b->rank;
  const bool stats_only = (flags & RMI_FLAG_STATS_ONLY) != 0;
  const bool want_counts = !stats_only && (flags & RMI_FLAG_LEAF_COUNTS) != 0;
  cudaStream_t st = b->st;
  ncclComm_t comm = c->comm;
  // RMI_FLAG_SHARD_ROOT_ONLY on one node: every rank copies the records of the leaves it owns into a host region all
  // ranks share (comm_ensure_shared) — rank 0's result points into it — instead of rank 0 copying all N records itself
  bool shared = !stats_only && (flags & RMI_FLAG_SHARD_ROOT_ONLY) != 0 && W > 1 && c->single_node;
  const size_t shared_bytes = sizeof(double) * N * ppm + sizeof(u64) * N * (want_counts ? 2 : 1);
  if (shared) {
    if (int rcs = comm_ensure_shared(c, shared_bytes, st)) return rcs;
    shared = c->single_node && c->shm != nullptr;
  }
  unsigned char* const region = shared ? c->shm + (size_t)c->parity * c->shm_half : nullptr;
  double* const sh_params = (double*)region;
  u64* const sh_errors = shared ? (u64*)(region + sizeof(double) * N * ppm) : nullptr;
  u64* const sh_counts = (shared && want_counts) ? sh_errors + N : nullptr;
  const bool leaves_to_host = !shared && !stats_only && (rank == 0 || (flags & RMI_FLAG_SHARD_ROOT_ONLY) == 0);
  Launch L{st, b->num_sms};
  // pinned host memory for the results first (nothing below waits for the host except the owner offsets)
  auto box = new ResultBox();
  if (!reserve_result(box, &b->tables, N, ppm, leaves_to_host, want_counts)) { delete box; return fail(RMI_ERR_CUDA, kPinnedFailed); }
  b->gather_mode = true;
  int rc = RMI_OK;
  auto phase = [&](int ph) { if (rc == RMI_OK) rc = shard_phase_typed<T>(b, ph); };
  auto nccl = [&](ncclResult_t r, const char* what) {
    if (rc == RMI_OK && r != ncclSuccess) rc = fail(RMI_ERR_CUDA, std::string(what) + ": " + nc.GetErrorString(r));
  };
  // RMI_DEV_SHARD_TRACE=1: device time between the marks below, printed per build by every rank (developer probe)
  static const bool trace = [] { const char* e = getenv("RMI_DEV_SHARD_TRACE"); return e && e[0] == '1'; }();
  struct Mark { const char* what; cudaEvent_t ev; };
  static thread_local std::vector<Mark> marks;
  size_t n_marks = 0;
  auto mark = [&](const char* what) {
    if (!trace) return;
    if (n_marks == marks.size()) { Mark m{what, nullptr}; cudaEventCreate(&m.ev); marks.push_back(m); }
    marks[n_marks].what = what;
    cudaEventRecord(marks[n_marks++].ev, st);
  };
  cudaEventRecord(b->ev_t0, st);
  mark("start");
  rc = shard_top_and_bounds<T>(b, c, mark);
  if (rc == RMI_OK) {
    shard_owner_offsets(L, (const u64*)b->buf.S, N, b->d_bases, W, b->r_last, b->d_off);
    cudaMemcpyAsync(b->h_off, b->d_off, sizeof(u64) * (W + 1), cudaMemcpyDeviceToHost, st);
    cudaEventRecord(b->ev_off, st);
  }
  mark("split + owner offsets");
  // ---- leaves owned by this rank ---------------------------------------------------------------------------------
  // With a shared result region the host waits for the ownership ranges first (a few microseconds of idle GPU) and
  // launches only the owned leaf window, in slices whose records cross PCIe while the next slice computes — after the
  // kernel that copy would be exposed.  Otherwise the whole leaf range is launched at
  // once (blocks without an owned leaf return immediately) and the host learns the ranges while it runs.
  LeafCopyOut* co = nullptr;
  if (shared && rc == RMI_OK) {
    cudaError_t e = cudaEventSynchronize(b->ev_off);
    if (e != cudaSuccess) rc = fail(RMI_ERR_CUDA, std::string("rmi_shard_train: ") + cudaGetErrorString(e));
    co = rc == RMI_OK ? t_slices.get(b->ds->device) : nullptr;
    if (co) {
      co->h_params = sh_params; co->h_errors = sh_errors; co->h_counts = sh_counts;
      co->used = 0;
      b->leaf_copy = co;
      b->leaf_lo = b->h_off[rank]; b->leaf_hi = b->h_off[rank + 1];
      if (b->leaf_hi == 0) b->leaf_lo = b->leaf_hi = N;   // owns nothing (0 would mean "no window")
    }
  }
  phase(RMI_PHASE_LEAF);
  mark("leaf (incl. host wait for the offsets)");
  b->leaf_copy = nullptr; b->leaf_lo = b->leaf_hi = 0;
  if (rc == RMI_OK) {
    shard_copy_flags(L, b->d_aux, b->d_flags_mine);
    // statistics of the owned leaves (needs only local results), gathered below
    leaf_statistics_owned(L, b->lay.n_global, N, (const u64*)b->buf.errors, (const u64*)b->buf.counts, b->d_off, rank, W,
                          (char*)b->d_parts + stats_partial_bytes() * rank, b->d_stats);
    if (shared && !co) cudaEventRecord(c->ev_leaf_done, st);
    if (!shared) {
      cudaError_t e = cudaEventSynchronize(b->ev_off);
      if (e != cudaSuccess) rc = fail(RMI_ERR_CUDA, std::string("rmi_shard_train: ") + cudaGetErrorString(e));
    }
    if (shared && !co && rc == RMI_OK) {
      // (no slice streams: copy the owned range after the kernel, on the communicator's side stream)
      const uint64_t j0 = b->h_off[rank], cnt = b->h_off[rank + 1] - b->h_off[rank];
      cudaStreamWaitEvent(c->copy_stream, c->ev_leaf_done, 0);
      if (cnt) {
        cudaMemcpyAsync(sh_params + j0 * ppm, (double*)b->buf.params + j0 * ppm, sizeof(double) * cnt * ppm, cudaMemcpyDeviceToHost, c->copy_stream);
        cudaMemcpyAsync(sh_errors + j0, (u64*)b->buf.errors + j0, sizeof(u64) * cnt, cudaMemcpyDeviceToHost, c->copy_stream);
        if (sh_counts) cudaMemcpyAsync(sh_counts + j0, (u64*)b->buf.counts + j0, sizeof(u64) * cnt, cudaMemcpyDeviceToHost, c->copy_stream);
      }
      cudaEventRecord(c->ev_copy_done, c->copy_stream);
    }
  }
  mark("flags + owned statistics");
  // ---- every owner publishes its leaf range: an all-gather with per-rank counts (grouped broadcasts) ----------
  // Not when the records go to the host region all ranks share: each owner has just sent its own range there, nobody
  // reads another rank's records on the device, and 2-3 broadcasts per rank are the longest part of the exchange.
  if (rc == RMI_OK && W > 1) {
    nccl(nc.GroupStart(), "ncclGroupStart");
    for (int r = 0; r < W && rc == RMI_OK && !shared; ++r) {
      const uint64_t j0 = b->h_off[r], cnt = b->h_off[r + 1] - b->h_off[r];
      if (cnt == 0) continue;
      double* pp = (double*)b->buf.params + j0 * ppm;
      u64* pe = (u64*)b->buf.errors + j0;
      nccl(nc.Broadcast(pp, pp, cnt * ppm, ncclFloat64, r, comm, st), "ncclBroadcast(leaf parameters)");
      nccl(nc.Broadcast(pe, pe, cnt, ncclUint64, r, comm, st), "ncclBroadcast(leaf error bounds)");
      if (want_counts) {
        u64* pc = (u64*)b->buf.counts + j0;
        nccl(nc.Broadcast(pc, pc, cnt, ncclUint64, r, comm, st), "ncclBroadcast(leaf key counts)");
      }
    }
    nccl(nc.AllGather(b->d_flags_mine, b->d_flags_all, 2, ncclUint32, comm, st), "ncclAllGather(status)");
    nccl(nc.AllGather((char*)b->d_parts + stats_partial_bytes() * rank, b->d_parts, stats_partial_bytes(), ncclChar, comm, st),
         "ncclAllGather(statistics)");
    nccl(nc.GroupEnd(), "ncclGroupEnd");
  } else if (rc == RMI_OK) {
    cudaMemcpyAsync(b->d_flags_all, b->d_flags_mine, 2 * sizeof(unsigned), cudaMemcpyDeviceToDevice, st);
  }
  mark("gather group");
  if (rc == RMI_OK) {
    if (b->ran[RMI_PHASE_STATS] == false) { cudaEventRecord(b->ev_begin[RMI_PHASE_STATS], st); b->ran[RMI_PHASE_STATS] = true; }
    leaf_statistics_merge(L, b->d_parts, W, b->d_aux);
    cudaEventRecord(b->ev_end[RMI_PHASE_STATS], st);
    mark("statistics merge");
    if (shared) {
      // "every rank's copy has landed": an all-reduce each rank enqueues behind its own copy (or slice copies)
      if (co) for (int q = 0; q < co->used; ++q) cudaStreamWaitEvent(st, co->ev_copied[q], 0);
      else cudaStreamWaitEvent(st, c->ev_copy_done, 0);
      nccl(nc.AllReduce(c->d_token, c->d_token, 1, ncclUint32, ncclMax, comm, st), "ncclAllReduce(result copies landed)");
    }
  }
  mark("copies landed + barrier");
  cudaEventRecord(b->ev_t1, st);
  if (rc != RMI_OK) { cudaStreamSynchronize(st); delete box; return rc; }
  // ---- results to the host ------------------------------------------------------------------------------------
  copy_result_to_host(box, &b->tables, b->d_aux, b->d_top, leaves_to_host ? (const double*)b->buf.params : nullptr,
                      (const u64*)b->buf.errors, want_counts ? (const u64*)b->buf.counts : nullptr, st);
  cudaMemcpyAsync(b->h_flags_all, b->d_flags_all, 2 * sizeof(unsigned) * W, cudaMemcpyDeviceToHost, st);
  cudaError_t e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { delete box; return fail(RMI_ERR_CUDA, std::string("rmi_shard_train: ") + cudaGetErrorString(e)); }
  if (trace && n_marks > 1) {
    std::string line = "[rmi_b200 shard trace] rank " + std::to_string(rank) + ":";
    char buf[96];
    for (size_t q = 1; q < n_marks; ++q) {
      float dt = 0.f;
      cudaEventElapsedTime(&dt, marks[q - 1].ev, marks[q].ev);
      std::snprintf(buf, sizeof buf, " | %s %.3f", marks[q].what, dt);
      line += buf;
    }
    std::fprintf(stderr, "%s\n", line.c_str());
  }
  unsigned st_all = b->host_status;
  bool cnr = false;
  for (int r = 0; r < W; ++r) { st_all |= b->h_flags_all[2 * r]; cnr = cnr || b->h_flags_all[2 * r + 1] != 0; }
  float ms = 0.f;
  cudaEventElapsedTime(&ms, b->ev_t0, b->ev_t1);
  const uint64_t total_ns = (uint64_t)((double)ms * 1e6);
  int rcf = shard_result(b, box, st_all, cnr, &total_ns, out);
  if (rcf == RMI_OK && shared) {
    if (rank == 0) {   // the leaf tables live in the shared region (valid until the next-but-one call, see the header)
      rmi_result* R = *out;
      R->l1_params = sh_params;
      R->l1_errors = reinterpret_cast<const uint64_t*>(sh_errors);
      R->l1_counts = reinterpret_cast<const uint64_t*>(sh_counts);
    }
    c->parity ^= 1;
  }
  return rcf;
}

// ---- statistics-only batches over the slabs (rmi_shard_stats_batch_create) ---------------------------------------
// A record: this rank's statistics partial of the leaves it owns, then {status word, could_not_replace != 0}.
static size_t stats_record_bytes() { return stats_partial_bytes() + 2 * sizeof(unsigned); }

// Leaf type k of the batch over the leaves this rank owns, after RMI_PHASE_SPLIT: the fused leaf kernel into the
// batch's own parameter scratch, then this rank's record at d_rec.  The owner offsets are derived again here (one
// tiny kernel) so that the host-driven flow needs no extra call.
template <class T> static int shard_stats_leaf_typed(rmi_shard_build* b, int k, char* d_rec) {
  const T* keys = (const T*)b->ds->d_keys;
  Shard<T> sh = shard_of<T>(b->lay, b->ds->n, b->ds->n + b->halo);
  Launch L{b->st, b->num_sms};
  L.side = b->side; L.ev_fork = b->ev_fork; L.ev_join = b->ev_join; L.d_long = b->d_long;
  if (k == 0) {
    cudaEventRecord(b->ev_begin[RMI_PHASE_LEAF], b->st);
    b->ran[RMI_PHASE_LEAF] = true;
    shard_owner_offsets(L, (const u64*)b->buf.S, b->N, b->d_bases, b->world, b->r_last, b->d_off);
  }
  BuildAux* a = b->d_batch_aux + k;   // starts from the state the top model and the boundaries left
  cudaMemcpyAsync(a, b->d_aux, sizeof(BuildAux), cudaMemcpyDeviceToDevice, b->st);
  fit_leaves<T>(L, keys, sh, b->batch[k]->kind, b->N, (const u64*)b->buf.S, a, b->d_batch_params, (u64*)b->buf.errors,
                (u64*)b->buf.counts);
  leaf_statistics_owned(L, b->lay.n_global, b->N, (const u64*)b->buf.errors, (const u64*)b->buf.counts, b->d_off, b->rank,
                        b->world, d_rec, b->d_stats);
  shard_copy_flags(L, a, (unsigned*)(d_rec + stats_partial_bytes()));
  cudaEventRecord(b->ev_end[RMI_PHASE_LEAF], b->st);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(RMI_ERR_CUDA, std::string("rmi_shard_stats_leaf: ") + cudaGetErrorString(e));
  return RMI_OK;
}

// The K results from every rank's records (d_recs: world x K records in device memory, rank by rank): the partials of
// each leaf type are merged in rank order into its BuildAux, the status words and replacement flags OR-ed over the
// ranks.  The batch's device time is shared out evenly: with one_call, the whole stream from the first phase to the
// merge (collectives included), otherwise the sum of the phases.
static int shard_stats_results(rmi_shard_build* b, const char* d_recs, bool one_call, rmi_result** out) {
  const int K = (int)b->batch.size(), W = b->world;
  const size_t rec = stats_record_bytes(), part = stats_partial_bytes();
  cudaStream_t st = b->st;
  Launch L{st, b->num_sms};
  std::vector<ResultBox*> boxes(K, nullptr);
  bool ok = true;
  for (int k = 0; k < K; ++k) {
    boxes[k] = new ResultBox();
    ok = ok && reserve_result(boxes[k], &b->tables, b->N, 0, false, false);
  }
  if (!ok) { for (auto* x : boxes) delete x; return fail(RMI_ERR_CUDA, kPinnedFailed); }
  if (!b->ran[RMI_PHASE_STATS]) { cudaEventRecord(b->ev_begin[RMI_PHASE_STATS], st); b->ran[RMI_PHASE_STATS] = true; }
  for (int k = 0; k < K; ++k) {
    char* parts = b->d_batch_parts + part * W * k;   // leaf type k's partials of ranks 0..W-1, contiguous
    cudaMemcpy2DAsync(parts, part, d_recs + rec * k, rec * K, part, W, cudaMemcpyDeviceToDevice, st);
    leaf_statistics_merge(L, parts, W, b->d_batch_aux + k);
    copy_result_to_host(boxes[k], &b->tables, b->d_batch_aux + k, b->d_top, nullptr, nullptr, nullptr, st);
  }
  cudaEventRecord(b->ev_end[RMI_PHASE_STATS], st);
  cudaMemcpyAsync(b->h_batch_recs, d_recs, rec * K * W, cudaMemcpyDeviceToHost, st);
  cudaError_t e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { for (auto* x : boxes) delete x; return fail(RMI_ERR_CUDA, std::string("rmi_shard_stats_finish: ") + cudaGetErrorString(e)); }
  uint64_t device_ns = 0;
  if (one_call) device_ns = elapsed_ns(b->ev_t0, b->ev_end[RMI_PHASE_STATS]);
  else for (int q = 0; q < RMI_NUM_PHASES; ++q) if (b->ran[q]) device_ns += elapsed_ns(b->ev_begin[q], b->ev_end[q]);
  int rc = RMI_OK;
  for (int k = 0; k < K; ++k) {
    unsigned st_all = b->host_status;
    bool cnr = false;
    for (int r = 0; r < W; ++r) {
      const unsigned* f = (const unsigned*)(b->h_batch_recs + rec * ((size_t)r * K + k) + part);
      st_all |= f[0];
      cnr = cnr || f[1] != 0;
    }
    const uint64_t share = device_ns / (uint64_t)K;
    if (rc == RMI_OK) {
      rc = shard_result(b, boxes[k], st_all, cnr, &share, &out[k], b->batch[k]);   // deletes the box on failure
      if (rc != RMI_OK) {
        const std::string msg = std::string(b->top->name) + "," + b->batch[k]->name + ": " + rmi_last_error();
        for (int q = 0; q < k; ++q) rmi_result_free(out[q]);
        rc = fail(rc, msg);
      }
    } else {
      delete boxes[k];
    }
  }
  if (rc != RMI_OK) return rc;
  for (int k = 0; k < K; ++k) out[k]->build_time_ns /= (uint64_t)K;   // the batch's wall time, shared out evenly
  return RMI_OK;
}

template <class T>
static int shard_stats_batch_typed(rmi_shard_build* b, rmi_shard_comm* c, rmi_result** out) {
  const int K = (int)b->batch.size(), W = b->world;
  const size_t rec = stats_record_bytes();
  cudaStream_t st = b->st;
  b->gather_mode = true;
  cudaEventRecord(b->ev_t0, st);
  int rc = shard_top_and_bounds<T>(b, c, [](const char*) {});
  char* mine = b->d_batch_recs + rec * K * b->rank;
  for (int k = 0; k < K && rc == RMI_OK; ++k) rc = shard_stats_leaf_typed<T>(b, k, mine + rec * k);
  // one all-gather carries every leaf type's partial and status words: K records per rank
  if (rc == RMI_OK && W > 1) {
    ncclResult_t r = nccl_api().AllGather(mine, b->d_batch_recs, rec * K, ncclChar, c->comm, st);
    if (r != ncclSuccess) rc = fail(RMI_ERR_CUDA, std::string("ncclAllGather(statistics records): ") + nccl_api().GetErrorString(r));
  }
  if (rc != RMI_OK) { cudaStreamSynchronize(st); return rc; }
  // the records are merged on the stream behind the gather
  return shard_stats_results(b, b->d_batch_recs, true, out);
}

extern "C" {

int rmi_shard_train(rmi_shard_build* b, rmi_shard_comm* c, uint32_t flags, rmi_result** out) {
  g_last_error.clear();
  if (!b || !c || !out) return fail(RMI_ERR_INVALID, "rmi_shard_train: null argument");
  if (c->world != b->world || c->rank != b->rank)
    return fail(RMI_ERR_INVALID, "rmi_shard_train: the communicator is rank " + std::to_string(c->rank) + " of " +
                                     std::to_string(c->world) + ", the build rank " + std::to_string(b->rank) + " of " +
                                     std::to_string(b->world));
  if (!nccl_api().ok) return fail(RMI_ERR_UNSUPPORTED, nccl_api().error);
  CUDA_TRY(cudaSetDevice(b->ds->device));
  return with_key_type(b->ds->key_type, [&](auto k) { return shard_train_typed<decltype(k)>(b, c, flags, out); });
}

int rmi_shard_stats_batch_create(const rmi_dataset* local, const rmi_shard_ends* ends_all, int world, int rank,
                                 const char* top_model, const char* const* leaf_models, int num_leaf_models,
                                 uint64_t branch_factor, uint64_t halo_capacity, const rmi_shard_buffers* buffers,
                                 void* cuda_stream, rmi_shard_build** out) {
  const std::string fn = "rmi_shard_stats_batch_create";
  g_last_error.clear();
  if (!local || !ends_all || !top_model || !leaf_models || num_leaf_models < 1 || !buffers || !out)
    return fail(RMI_ERR_INVALID, fn + ": bad argument");
  // rmi_train_stats_batch's checks of the model names first, then rmi_shard_build_create's (the ends table and the keys)
  const ModelName* top = nullptr;
  if (int rc = find_layer(top_model, true, &top)) return rc;
  std::vector<const ModelName*> leaves(num_leaf_models);
  for (int k = 0; k < num_leaf_models; ++k) {
    if (int rc = find_layer(leaf_models[k] ? leaf_models[k] : "(null)", false, &leaves[k])) return rc;
    if (int rc = check_leaf(leaves[k])) return rc;
  }
  const std::string spec = std::string(top->name) + "," + leaves[0]->name;
  rmi_shard_build* b = nullptr;
  if (int rc = rmi_shard_build_create(local, ends_all, world, rank, spec.c_str(), branch_factor, halo_capacity, buffers,
                                      cuda_stream, &b)) {
    std::string msg = rmi_last_error();
    if (msg.rfind("rmi_shard_build_create", 0) == 0) msg = fn + msg.substr(strlen("rmi_shard_build_create"));
    return fail(rc, msg);
  }
  b->batch = leaves;
  int max_ppm = 2;
  for (auto* lf : leaves) max_ppm = std::max(max_ppm, leaf_params_per_model(lf->kind));
  const size_t rec = stats_record_bytes(), K = leaves.size();
  bool ok = rec == RMI_SHARD_STATS_RECORD_BYTES &&
            cudaMalloc((void**)&b->d_batch_params, sizeof(double) * branch_factor * max_ppm) == cudaSuccess &&
            cudaMalloc((void**)&b->d_batch_aux, sizeof(BuildAux) * K) == cudaSuccess &&
            cudaMalloc((void**)&b->d_batch_recs, rec * K * world) == cudaSuccess &&
            cudaMalloc((void**)&b->d_batch_parts, stats_partial_bytes() * K * world) == cudaSuccess &&
            cudaMallocHost((void**)&b->h_batch_recs, rec * K * world) == cudaSuccess;
  if (!ok) { rmi_shard_build_destroy(b); return fail(RMI_ERR_CUDA, fn + ": device allocation failed"); }
  *out = b;
  return RMI_OK;
}

int rmi_shard_stats_leaf(rmi_shard_build* b, int k, void* d_record) {
  if (!b || !d_record) return fail(RMI_ERR_INVALID, "rmi_shard_stats_leaf: null argument");
  if (b->batch.empty() || k < 0 || k >= (int)b->batch.size())
    return fail(RMI_ERR_INVALID, "rmi_shard_stats_leaf: not a leaf type of this statistics batch");
  b->gather_mode = false;
  CUDA_TRY(cudaSetDevice(b->ds->device));
  return with_key_type(b->ds->key_type, [&](auto t) { return shard_stats_leaf_typed<decltype(t)>(b, k, (char*)d_record); });
}

int rmi_shard_stats_finish(rmi_shard_build* b, const void* d_records, uint32_t flags, rmi_result** out) {
  (void)flags;
  if (!b || !d_records || !out) return fail(RMI_ERR_INVALID, "rmi_shard_stats_finish: null argument");
  if (b->batch.empty()) return fail(RMI_ERR_INVALID, "rmi_shard_stats_finish: not a statistics batch");
  CUDA_TRY(cudaSetDevice(b->ds->device));
  return shard_stats_results(b, (const char*)d_records, false, out);
}

int rmi_shard_train_stats_batch(rmi_shard_build* b, rmi_shard_comm* c, uint32_t flags, rmi_result** out) {
  (void)flags;
  g_last_error.clear();
  if (!b || !c || !out) return fail(RMI_ERR_INVALID, "rmi_shard_train_stats_batch: null argument");
  if (b->batch.empty()) return fail(RMI_ERR_INVALID, "rmi_shard_train_stats_batch: not a statistics batch");
  if (c->world != b->world || c->rank != b->rank)
    return fail(RMI_ERR_INVALID, "rmi_shard_train_stats_batch: the communicator is rank " + std::to_string(c->rank) + " of " +
                                     std::to_string(c->world) + ", the build rank " + std::to_string(b->rank) + " of " +
                                     std::to_string(b->world));
  if (!nccl_api().ok) return fail(RMI_ERR_UNSUPPORTED, nccl_api().error);
  CUDA_TRY(cudaSetDevice(b->ds->device));
  return with_key_type(b->ds->key_type, [&](auto t) { return shard_stats_batch_typed<decltype(t)>(b, c, out); });
}

void rmi_shard_build_destroy(rmi_shard_build* b) {
  if (!b) return;
  cudaFree(b->d_top); cudaFree(b->d_aux); cudaFree(b->d_scratch); cudaFree(b->d_stats);
  for (int q = 0; q < RMI_NUM_PHASES; ++q) { if (b->ev_begin[q]) cudaEventDestroy(b->ev_begin[q]); if (b->ev_end[q]) cudaEventDestroy(b->ev_end[q]); }
  if (b->ev_fork) cudaEventDestroy(b->ev_fork);
  if (b->ev_join) cudaEventDestroy(b->ev_join);
  if (b->side) cudaStreamDestroy(b->side);
  cudaFree(b->d_long);
  b->tables.free_device();
  cudaFree(b->d_bases); cudaFree(b->d_off); cudaFree(b->d_parts); cudaFree(b->d_flags_mine); cudaFree(b->d_flags_all);
  if (b->h_off) cudaFreeHost(b->h_off);
  if (b->h_flags_all) cudaFreeHost(b->h_flags_all);
  for (cudaEvent_t e : {b->ev_off, b->ev_t0, b->ev_t1}) if (e) cudaEventDestroy(e);
  cudaFree(b->d_batch_params); cudaFree(b->d_batch_aux); cudaFree(b->d_batch_recs); cudaFree(b->d_batch_parts);
  if (b->h_batch_recs) cudaFreeHost(b->h_batch_recs);
  delete b;
}

}  // extern "C"

// ---- lookups over a range-partitioned data set (DESIGN.md section 14) ----------------------------------------------
constexpr int SHARD_LOOKUP_EVENTS = 7;   // around route, count exchange, query exchange, search, answer exchange, gather

struct rmi_shard_index {
  rmi_index* idx = nullptr;       // the tables, bound to this rank's slab
  int world = 0, rank = 0;
  uint64_t base = 0, n_global = 0;
  // the route (kernels.h ShardRoute), as raw key bits
  uint64_t first_bits[SHARD_ROUTE_MAX] = {};
  unsigned char route_rank[SHARD_ROUTE_MAX] = {};
  int route_count = 0;
  uint64_t* h_counts = nullptr;   // world x world, pinned: the one host read of the one-call forms
  cudaEvent_t ev[SHARD_LOOKUP_EVENTS] = {};
  rmi_shard_lookup_stats last = {};
  bool ran = false;
  // a bounded index (rmi_shard_index_create_bounded, DESIGN.md section 17): idx is the RMI over the knots (predicting
  // over K positions), ks this rank's knot slab with its halo (ks.knots: device memory owned here); the route by knot
  // index holds the knot base of every rank that holds knots.  Null / 0 for a plain index.
  void* d_knots = nullptr;
  BoundedKnotSlab ks = {};
  uint64_t knot_first[SHARD_ROUTE_MAX] = {};
  unsigned char knot_rank[SHARD_ROUTE_MAX] = {};
  int knot_route_count = 0;
};

namespace {

template <class T> ShardRoute<T> shard_route_of(const rmi_shard_index* si) {
  ShardRoute<T> r;
  memset(&r, 0, sizeof(r));
  for (int k = 0; k < si->route_count; ++k) {
    r.first[k] = key_from_bits<T>(si->first_bits[k]);
    r.rank[k] = si->route_rank[k];
  }
  r.count = si->route_count;
  return r;
}

// Frees a stream-ordered allocation when the scope ends (also on an early error return).
struct PoolScratch {
  void* p = nullptr;
  cudaStream_t st = nullptr;
  ~PoolScratch() { if (p) cudaFreeAsync(p, st); }
};

size_t round8(size_t b) { return (b + 7) & ~(size_t)7; }

// upper: route by <= for upper bounds (DESIGN §18)
template <class T>
int shard_lookup_route(const rmi_shard_index* si, const T* d_q, uint64_t n, T* d_send, u64* d_slot, u64* d_counts,
                       cudaStream_t st, bool upper) {
  const u64 nb = shard_route_blocks(n), W = (u64)si->world;
  PoolScratch s{nullptr, st};
  if (n) CUDA_TRY(cudaMallocAsync(&s.p, nb * W * (sizeof(u64) + sizeof(u32)), st));
  Launch L{st, si->idx->num_sms};
  shard_route<T>(L, shard_route_of<T>(si), si->world, d_q, n, (u32*)((u64*)s.p + nb * W), (u64*)s.p, d_send, d_slot,
                 d_counts, upper);
  CUDA_TRY(cudaGetLastError());
  return RMI_OK;
}

// upper: upper bounds of queries routed by <=
template <class T>
int shard_lookup_search(const rmi_shard_index* si, const T* d_recv, uint64_t m, u64* d_answers, u64* d_fallbacks,
                        cudaStream_t st, bool upper) {
  if (m == 0) return RMI_OK;
  const rmi_index* idx = si->idx;
  const rmi_dataset* ds = idx->ds;
  if (ds->n == 0)
    return fail(RMI_ERR_INVALID, std::string(upper ? "rmi_shard_index_search_upper" : "rmi_shard_index_search") +
                                     ": this rank holds no keys, so no query is routed to it");
  if constexpr (std::is_same<T, u64>::value) {
    if (si->d_knots) {
      Launch L{st, idx->num_sms};
      shard_bounded_search(L, idx->top, idx->leaf_kind, idx->d_records, idx->N, si->ks, (const u64*)ds->d_keys, ds->n,
                           si->base, si->n_global, d_recv, m, d_answers, d_fallbacks, true, upper, idx->last_key_bits);
      CUDA_TRY(cudaGetLastError());
      return RMI_OK;
    }
  }
  PoolScratch s{nullptr, st};
  CUDA_TRY(cudaMallocAsync(&s.p, 2 * sizeof(u64) * m, st));
  uint64_t* pos = (uint64_t*)s.p;   // m predictions, then their error bounds
  if (int rc = index_launch(idx, LOOKUP_PREDICT, d_recv, m, pos, pos + m, nullptr, st)) return rc;
  Launch L{st, idx->num_sms};
  shard_search<T>(L, (const T*)ds->d_keys, ds->n, si->base, si->n_global, d_recv, m, (const u64*)pos,
                  (const u64*)pos + m, d_answers, d_fallbacks, upper, rmihost::key_from_bits<T>(idx->last_key_bits));
  CUDA_TRY(cudaGetLastError());
  return RMI_OK;
}

// The bounded index's predict route: the knot RMI's (start, e) per query, the route by knot index over lower + 1
// (written over start in place), then the queries themselves into the route's positions (over the routed values).
int shard_predict_route(const rmi_shard_index* si, const u64* d_q, uint64_t n, u64* d_send, u64* d_slot, u64* d_counts,
                        cudaStream_t st) {
  PoolScratch s{nullptr, st};
  if (n) CUDA_TRY(cudaMallocAsync(&s.p, 2 * sizeof(u64) * n, st));
  uint64_t* pos = (uint64_t*)s.p;   // n predictions, then their error bounds
  if (int rc = index_launch(si->idx, LOOKUP_PREDICT, d_q, n, pos, pos + n, nullptr, st)) return rc;
  Launch L{st, si->idx->num_sms};
  shard_knot_route_keys(L, (const u64*)pos, (const u64*)pos + n, n, (u64*)pos);
  ShardRoute<u64> route;
  memset(&route, 0, sizeof(route));
  for (int k = 0; k < si->knot_route_count; ++k) {
    route.first[k] = si->knot_first[k];
    route.rank[k] = si->knot_rank[k];
  }
  route.count = si->knot_route_count;
  const u64 nb = shard_route_blocks(n), W = (u64)si->world;
  PoolScratch s2{nullptr, st};
  if (n) CUDA_TRY(cudaMallocAsync(&s2.p, nb * W * (sizeof(u64) + sizeof(u32)), st));
  shard_route<u64>(L, route, si->world, (const u64*)pos, n, (u32*)((u64*)s2.p + nb * W), (u64*)s2.p, d_send, d_slot,
                   d_counts, false);
  shard_scatter_queries(L, d_q, d_slot, n, d_send);
  CUDA_TRY(cudaGetLastError());
  return RMI_OK;
}

int shard_predict_search(const rmi_shard_index* si, const u64* d_recv, uint64_t m, u64* d_pos, cudaStream_t st) {
  if (m == 0) return RMI_OK;
  const rmi_index* idx = si->idx;
  if (si->ks.a1 == si->ks.a0)
    return fail(RMI_ERR_INVALID, "rmi_shard_index_predict_search: this rank holds no knots, so no query is routed to it");
  Launch L{st, idx->num_sms};
  shard_bounded_search(L, idx->top, idx->leaf_kind, idx->d_records, idx->N, si->ks, (const u64*)idx->ds->d_keys,
                       idx->ds->n, si->base, si->n_global, d_recv, m, d_pos, nullptr, false);
  CUDA_TRY(cudaGetLastError());
  return RMI_OK;
}

// The one-call exchange of rmi_shard_index_lower_bound and rmi_shard_index_predict_collective: route(d_send, d_slot,
// d_counts) groups the n queries by destination; the world x world counts are all-gathered and read once on the host;
// the queries go to their ranks, search(d_recv, m, d_ans) answers the m received ones, the answers come back and are
// gathered into d_out.  Events around every phase for rmi_shard_index_last_stats.
template <class T, class Route, class Search>
int shard_one_call(rmi_shard_index* si, rmi_shard_comm* c, uint64_t n, u64* d_out, cudaStream_t st, const char* fn,
                   Route&& route, Search&& search) {
  const NcclApi& nc = nccl_api();
  const int W = si->world, me = si->rank;
  const size_t kb = sizeof(T);
  // send | slot | count matrix
  PoolScratch s1{nullptr, st};
  const size_t send_b = round8(n * kb), slot_b = n * sizeof(u64), mat_b = (size_t)W * W * sizeof(u64);
  CUDA_TRY(cudaMallocAsync(&s1.p, send_b + slot_b + mat_b, st));
  T* d_send = (T*)s1.p;
  u64* d_slot = (u64*)((char*)s1.p + send_b);
  u64* d_mat = (u64*)((char*)s1.p + send_b + slot_b);
  cudaEventRecord(si->ev[0], st);
  if (int rc = route(d_send, d_slot, d_mat + (size_t)me * W)) return rc;
  cudaEventRecord(si->ev[1], st);
  NCCL_TRY(nc.AllGather(d_mat + (size_t)me * W, d_mat, W, ncclUint64, c->comm, st));
  CUDA_TRY(cudaMemcpyAsync(si->h_counts, d_mat, mat_b, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  cudaEventRecord(si->ev[2], st);
  // row r of the matrix: what rank r sends to every rank
  std::vector<u64> scount(W), rcount(W), soff(W + 1, 0), roff(W + 1, 0);
  for (int p = 0; p < W; ++p) {
    scount[p] = si->h_counts[(size_t)me * W + p];
    rcount[p] = si->h_counts[(size_t)p * W + me];
    soff[p + 1] = soff[p] + scount[p];
    roff[p + 1] = roff[p] + rcount[p];
  }
  if (soff[W] != n) return fail(RMI_ERR_CUDA, std::string(fn) + ": the route's counts do not add up to the queries");
  const u64 m = roff[W];
  // received queries | their answers | the answers returned to this rank
  PoolScratch s2{nullptr, st};
  const size_t recv_b = round8(m * kb);
  CUDA_TRY(cudaMallocAsync(&s2.p, recv_b + (m + n) * sizeof(u64) + 8, st));
  T* d_recv = (T*)s2.p;
  u64* d_ans = (u64*)((char*)s2.p + recv_b);
  u64* d_ret = d_ans + m;
  NCCL_TRY(nc.GroupStart());
  for (int p = 0; p < W; ++p) {
    if (scount[p]) NCCL_TRY(nc.Send(d_send + soff[p], scount[p] * kb, ncclUint8, p, c->comm, st));
    if (rcount[p]) NCCL_TRY(nc.Recv(d_recv + roff[p], rcount[p] * kb, ncclUint8, p, c->comm, st));
  }
  NCCL_TRY(nc.GroupEnd());
  cudaEventRecord(si->ev[3], st);
  if (int rc = search((const T*)d_recv, m, d_ans)) return rc;
  cudaEventRecord(si->ev[4], st);
  NCCL_TRY(nc.GroupStart());
  for (int p = 0; p < W; ++p) {
    if (rcount[p]) NCCL_TRY(nc.Send(d_ans + roff[p], rcount[p], ncclUint64, p, c->comm, st));
    if (scount[p]) NCCL_TRY(nc.Recv(d_ret + soff[p], scount[p], ncclUint64, p, c->comm, st));
  }
  NCCL_TRY(nc.GroupEnd());
  cudaEventRecord(si->ev[5], st);
  Launch L{st, si->idx->num_sms};
  shard_gather(L, d_slot, d_ret, n, d_out);
  CUDA_TRY(cudaGetLastError());
  cudaEventRecord(si->ev[6], st);
  si->last.queries_routed = n;
  si->last.queries_searched = m;
  si->last.queries_kept = scount[me];
  si->ran = true;
  return RMI_OK;
}

template <class T>
int shard_lookup_one_call(rmi_shard_index* si, rmi_shard_comm* c, const T* d_q, uint64_t n, u64* d_out, u64* d_fallbacks,
                          cudaStream_t st, bool upper) {
  return shard_one_call<T>(
      si, c, n, d_out, st, upper ? "rmi_shard_index_upper_bound" : "rmi_shard_index_lower_bound",
      [&](T* d_send, u64* d_slot, u64* d_counts) {
        return shard_lookup_route<T>(si, d_q, n, d_send, d_slot, d_counts, st, upper);
      },
      [&](const T* d_recv, u64 m, u64* d_ans) {
        return shard_lookup_search<T>(si, d_recv, m, d_ans, d_fallbacks, st, upper);
      });
}

// The checks of a call that takes a communicator (the one-call forms).
int shard_check_comm(const rmi_shard_index* si, const rmi_shard_comm* c, const std::string& fn) {
  if (c->world != si->world || c->rank != si->rank)
    return fail(RMI_ERR_INVALID, fn + ": the communicator is rank " + std::to_string(c->rank) + " of " +
                                     std::to_string(c->world) + ", the index rank " + std::to_string(si->rank) + " of " +
                                     std::to_string(si->world));
  const NcclApi& nc = nccl_api();
  if (!nc.ok) return fail(RMI_ERR_UNSUPPORTED, nc.error);
  return RMI_OK;
}

// The part of creating a shard index after its checks: binds the uploaded tables to the route of ends_all.
int shard_index_make(rmi_index* idx, const rmi_shard_ends* ends_all, int world, int rank, uint64_t base, uint64_t total,
                     const std::string& fn, rmi_shard_index** out) {
  auto* si = new rmi_shard_index();
  si->idx = idx;
  si->world = world;
  si->rank = rank;
  si->base = base;
  si->n_global = total;
  for (int p = 0; p < world; ++p) {
    if (!ends_all[p].n_local) continue;
    si->first_bits[si->route_count] = ends_all[p].first_key_bits;
    si->route_rank[si->route_count++] = (unsigned char)p;
  }
  bool ok = cudaMallocHost((void**)&si->h_counts, sizeof(u64) * world * world) == cudaSuccess;
  for (int q = 0; q < SHARD_LOOKUP_EVENTS; ++q) ok = ok && cudaEventCreate(&si->ev[q]) == cudaSuccess;
  if (!ok) {
    rmi_shard_index_destroy(si);
    return fail(RMI_ERR_CUDA, fn + ": allocation failed");
  }
  *out = si;
  return RMI_OK;
}

}  // namespace

extern "C" {

int rmi_shard_index_create(const rmi_result* r, const rmi_dataset* local, const rmi_shard_ends* ends_all, int world,
                           int rank, rmi_shard_index** out) {
  const std::string fn = "rmi_shard_index_create";
  g_last_error.clear();
  if (!r || !local || !ends_all || !out) return fail(RMI_ERR_INVALID, fn + ": null argument");
  if (int rc = check_result(r, true, fn)) return rc;
  uint64_t total = 0, base = 0;
  if (int rc = check_slabs(fn, local, ends_all, world, rank, &base, &total)) return rc;
  if (int rc = index_check_tables(r, total, "the slabs hold ", total, fn)) return rc;
  rmi_index* idx = nullptr;
  if (int rc = index_upload(r, local, total, nullptr, 0, 0, fn, &idx)) return rc;
  return shard_index_make(idx, ends_all, world, rank, base, total, fn, out);
}

void rmi_shard_index_destroy(rmi_shard_index* si) {
  if (!si) return;
  if (si->d_knots) {
    cudaSetDevice(si->idx->ds->device);
    cudaFree(si->d_knots);
  }
  rmi_index_destroy(si->idx);
  if (si->h_counts) cudaFreeHost(si->h_counts);
  for (cudaEvent_t e : si->ev) if (e) cudaEventDestroy(e);
  delete si;
}

int rmi_shard_index_predict(const rmi_shard_index* si, const void* d_queries, uint64_t n, uint64_t* d_pos,
                            uint64_t* d_err, void* cuda_stream) {
  if (!si) return fail(RMI_ERR_INVALID, "rmi_shard_index_predict: null index");
  if (si->d_knots)
    return fail(RMI_ERR_INVALID, "rmi_shard_index_predict: a bounded index predicts collectively "
                                 "(rmi_shard_index_predict_collective, or its phases)");
  if (int rc = index_check_call(si->idx, d_queries, n, d_pos, "rmi_shard_index_predict")) return rc;
  return index_launch(si->idx, LOOKUP_PREDICT, d_queries, n, d_pos, d_err, nullptr, cuda_stream);
}

}  // extern "C"

namespace {
int shard_route_call(const rmi_shard_index* si, const void* d_queries, uint64_t n, void* d_send, uint64_t* d_slot,
                     uint64_t* d_send_counts, void* cuda_stream, bool upper) {
  const char* fn = upper ? "rmi_shard_index_route_upper" : "rmi_shard_index_route";
  if (!si || !d_send_counts) return fail(RMI_ERR_INVALID, std::string(fn) + ": null index or count pointer");
  if (n && (!d_queries || !d_send || !d_slot)) return fail(RMI_ERR_INVALID, std::string(fn) + ": null query, send or slot pointer");
  CUDA_TRY(cudaSetDevice(si->idx->ds->device));
  return with_key_type(si->idx->ds->key_type, [&](auto k) {
    using T = decltype(k);
    return shard_lookup_route<T>(si, (const T*)d_queries, n, (T*)d_send, (u64*)d_slot, (u64*)d_send_counts,
                                 (cudaStream_t)cuda_stream, upper);
  });
}

int shard_search_call(const rmi_shard_index* si, const void* d_received, uint64_t m, uint64_t* d_answers,
                      uint64_t* d_fallbacks, void* cuda_stream, bool upper) {
  const char* fn = upper ? "rmi_shard_index_search_upper" : "rmi_shard_index_search";
  if (!si) return fail(RMI_ERR_INVALID, std::string(fn) + ": null index");
  if (int rc = index_check_call(si->idx, d_received, m, d_answers, fn)) return rc;
  CUDA_TRY(cudaSetDevice(si->idx->ds->device));
  return with_key_type(si->idx->ds->key_type, [&](auto k) {
    using T = decltype(k);
    return shard_lookup_search<T>(si, (const T*)d_received, m, (u64*)d_answers, (u64*)d_fallbacks,
                                  (cudaStream_t)cuda_stream, upper);
  });
}

int shard_bound_call(rmi_shard_index* si, rmi_shard_comm* c, const void* d_queries, uint64_t n, uint64_t* d_out,
                     uint64_t* d_fallbacks, void* cuda_stream, bool upper) {
  const char* fn = upper ? "rmi_shard_index_upper_bound" : "rmi_shard_index_lower_bound";
  g_last_error.clear();
  if (!si || !c) return fail(RMI_ERR_INVALID, std::string(fn) + ": null index or communicator");
  if (n && (!d_queries || !d_out)) return fail(RMI_ERR_INVALID, std::string(fn) + ": null query or output pointer");
  if (int rc = shard_check_comm(si, c, fn)) return rc;
  CUDA_TRY(cudaSetDevice(si->idx->ds->device));
  return with_key_type(si->idx->ds->key_type, [&](auto k) {
    using T = decltype(k);
    return shard_lookup_one_call<T>(si, c, (const T*)d_queries, n, (u64*)d_out, (u64*)d_fallbacks,
                                    (cudaStream_t)cuda_stream, upper);
  });
}
}  // namespace

extern "C" {

int rmi_shard_index_route(const rmi_shard_index* si, const void* d_queries, uint64_t n, void* d_send, uint64_t* d_slot,
                          uint64_t* d_send_counts, void* cuda_stream) {
  return shard_route_call(si, d_queries, n, d_send, d_slot, d_send_counts, cuda_stream, false);
}

int rmi_shard_index_route_upper(const rmi_shard_index* si, const void* d_queries, uint64_t n, void* d_send,
                                uint64_t* d_slot, uint64_t* d_send_counts, void* cuda_stream) {
  return shard_route_call(si, d_queries, n, d_send, d_slot, d_send_counts, cuda_stream, true);
}

int rmi_shard_index_search(const rmi_shard_index* si, const void* d_received, uint64_t m, uint64_t* d_answers,
                           uint64_t* d_fallbacks, void* cuda_stream) {
  return shard_search_call(si, d_received, m, d_answers, d_fallbacks, cuda_stream, false);
}

int rmi_shard_index_search_upper(const rmi_shard_index* si, const void* d_received, uint64_t m, uint64_t* d_answers,
                                 uint64_t* d_fallbacks, void* cuda_stream) {
  return shard_search_call(si, d_received, m, d_answers, d_fallbacks, cuda_stream, true);
}

int rmi_shard_index_gather(const rmi_shard_index* si, const uint64_t* d_slot, const uint64_t* d_returned, uint64_t n,
                           uint64_t* d_out, void* cuda_stream) {
  if (!si) return fail(RMI_ERR_INVALID, "rmi_shard_index_gather: null index");
  if (n && (!d_slot || !d_returned || !d_out)) return fail(RMI_ERR_INVALID, "rmi_shard_index_gather: null pointer");
  CUDA_TRY(cudaSetDevice(si->idx->ds->device));
  Launch L{(cudaStream_t)cuda_stream, si->idx->num_sms};
  shard_gather(L, (const u64*)d_slot, (const u64*)d_returned, n, (u64*)d_out);
  CUDA_TRY(cudaGetLastError());
  return RMI_OK;
}

int rmi_shard_index_lower_bound(rmi_shard_index* si, rmi_shard_comm* c, const void* d_queries, uint64_t n,
                                uint64_t* d_out, uint64_t* d_fallbacks, void* cuda_stream) {
  return shard_bound_call(si, c, d_queries, n, d_out, d_fallbacks, cuda_stream, false);
}

int rmi_shard_index_upper_bound(rmi_shard_index* si, rmi_shard_comm* c, const void* d_queries, uint64_t n,
                                uint64_t* d_out, uint64_t* d_fallbacks, void* cuda_stream) {
  return shard_bound_call(si, c, d_queries, n, d_out, d_fallbacks, cuda_stream, true);
}

int rmi_shard_index_last_stats(const rmi_shard_index* si, rmi_shard_lookup_stats* out) {
  if (!si || !out) return fail(RMI_ERR_INVALID, "rmi_shard_index_last_stats: null argument");
  if (!si->ran) return fail(RMI_ERR_INVALID, "rmi_shard_index_last_stats: no one-call lookup has run");
  CUDA_TRY(cudaEventSynchronize(si->ev[SHARD_LOOKUP_EVENTS - 1]));
  *out = si->last;
  for (int q = 0; q + 1 < SHARD_LOOKUP_EVENTS; ++q) CUDA_TRY(cudaEventElapsedTime(&out->phase_ms[q], si->ev[q], si->ev[q + 1]));
  return RMI_OK;
}

// ---- `--bounded` lookups over a range-partitioned data set (DESIGN.md section 17) ----------------------------------

int rmi_shard_index_create_bounded(const rmi_result* r, const rmi_spline_point* knots, uint64_t num_knots,
                                   uint64_t halo_before, const uint64_t* knot_counts, uint64_t line_size,
                                   const rmi_dataset* local, const rmi_shard_ends* ends_all, int world, int rank,
                                   rmi_shard_index** out) {
  const std::string fn = "rmi_shard_index_create_bounded";
  g_last_error.clear();
  if (!r || !knots || !knot_counts || !local || !ends_all || !out) return fail(RMI_ERR_INVALID, fn + ": null argument");
  if (int rc = check_result(r, true, fn)) return rc;
  if (local->key_type != RMI_KEY_U64) return fail(RMI_ERR_INVALID, fn + ": Can only construct a bounded RMI on u64 data");
  if (line_size == 0) return fail(RMI_ERR_INVALID, fn + ": line size 0");
  if (num_knots == 0) return fail(RMI_ERR_INVALID, fn + ": no spline knots");
  uint64_t total = 0, base = 0;
  if (int rc = check_slabs(fn, local, ends_all, world, rank, &base, &total)) return rc;
  // the knot slabs: rank p holds global knots [kbase[p], kbase[p] + knot_counts[p])
  std::vector<uint64_t> kbase(world + 1, 0);
  int knot_ranks = 0;
  for (int p = 0; p < world; ++p) {
    if (knot_counts[p] && !ends_all[p].n_local)
      return fail(RMI_ERR_INVALID, fn + ": rank " + std::to_string(p) + " holds " + std::to_string(knot_counts[p]) +
                                       " knots and no keys (a knot goes to the rank its key routes to)");
    knot_ranks += knot_counts[p] ? 1 : 0;
    kbase[p + 1] = kbase[p] + knot_counts[p];
  }
  if (knot_ranks > SHARD_ROUTE_MAX)
    return fail(RMI_ERR_INVALID, fn + ": more ranks hold knots than the route takes (" + std::to_string(SHARD_ROUTE_MAX) + ")");
  const uint64_t K = kbase[world], a0 = kbase[rank], a1 = kbase[rank + 1];
  if (int rc = index_check_tables(r, K, "the knot slabs hold ", total, fn)) return rc;
  // the slab and its halo: halo_before knots before it, the rest after it, each at least h = 2 e_max + 2 knots (or up
  // to the end of the knots), so that every window the lookups search lies inside (DESIGN.md section 17)
  uint64_t e_max = 0;
  for (uint64_t j = 0; j < r->branching_factor; ++j) e_max = std::max<uint64_t>(e_max, ((const uint64_t*)r->l1_errors)[j]);
  const uint64_t h = e_max >= (UINT64_MAX - 2) / 2 ? UINT64_MAX : 2 * e_max + 2;
  if (halo_before > a0 || a1 - a0 > num_knots - std::min(num_knots, halo_before) ||
      num_knots - halo_before - (a1 - a0) > K - a1)
    return fail(RMI_ERR_INVALID, fn + ": " + std::to_string(num_knots) + " knots with " + std::to_string(halo_before) +
                                     " before the slab do not fit knot slab [" + std::to_string(a0) + ", " +
                                     std::to_string(a1) + ") of " + std::to_string(K));
  const uint64_t halo_after = num_knots - halo_before - (a1 - a0);
  if (halo_before < std::min(h, a0) || halo_after < std::min(h, K - a1))
    return fail(RMI_ERR_INVALID, fn + ": the halo (" + std::to_string(halo_before) + " knots before the slab, " +
                                     std::to_string(halo_after) + " after) is below 2 x the largest leaf error + 2 = " +
                                     std::to_string(h) + " knots on a side");
  for (uint64_t i = 0; i < num_knots; ++i) {
    if (knots[i].offset >= total)
      return fail(RMI_ERR_INVALID, fn + ": knot " + std::to_string(i) + " has offset " + std::to_string(knots[i].offset) +
                                       ", the slabs hold " + std::to_string(total) + " keys");
    if (i && !(knots[i - 1].key < knots[i].key && knots[i - 1].offset <= knots[i].offset))
      return fail(RMI_ERR_INVALID, fn + ": knots " + std::to_string(i - 1) + " and " + std::to_string(i) +
                                       " are out of order (keys must increase strictly, offsets must not decrease)");
  }
  // the slab's knots route to this rank: above its first key (unless it is the first rank with keys), not above the
  // next non-empty rank's first key
  if (a1 > a0) {
    int first_rank = 0, next = -1;
    while (!ends_all[first_rank].n_local) ++first_rank;
    for (int p = rank + 1; p < world && next < 0; ++p)
      if (ends_all[p].n_local) next = p;
    const uint64_t lo_key = knots[halo_before].key, hi_key = knots[halo_before + (a1 - a0) - 1].key;
    if ((rank != first_rank && !(lo_key > ends_all[rank].first_key_bits)) ||
        (next >= 0 && hi_key > ends_all[next].first_key_bits))
      return fail(RMI_ERR_INVALID, fn + ": the knot slab holds knots whose keys route to other ranks");
  }
  rmi_index* idx = nullptr;
  if (int rc = index_upload(r, local, K, nullptr, 0, 0, fn, &idx)) return rc;
  rmi_shard_index* si = nullptr;
  if (int rc = shard_index_make(idx, ends_all, world, rank, base, total, fn, &si)) return rc;
  for (int p = 0; p < world; ++p) {
    if (!knot_counts[p]) continue;
    si->knot_first[si->knot_route_count] = kbase[p];
    si->knot_rank[si->knot_route_count++] = (unsigned char)p;
  }
  cudaError_t e = cudaMalloc(&si->d_knots, sizeof(rmi_spline_point) * num_knots);
  if (e == cudaSuccess) e = cudaMemcpy(si->d_knots, knots, sizeof(rmi_spline_point) * num_knots, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    rmi_shard_index_destroy(si);
    return fail(RMI_ERR_CUDA, fn + ": " + cudaGetErrorString(e));
  }
  si->ks = BoundedKnotSlab{si->d_knots, a0 - halo_before, num_knots, K, a0, a1, line_size};
  *out = si;
  return RMI_OK;
}

static int shard_check_bounded(const rmi_shard_index* si, const char* fn) {
  if (!si) return fail(RMI_ERR_INVALID, std::string(fn) + ": null index");
  if (!si->d_knots)
    return fail(RMI_ERR_INVALID, std::string(fn) + ": not a bounded index (a plain index predicts locally: "
                                                   "rmi_shard_index_predict)");
  return RMI_OK;
}

int rmi_shard_index_predict_route(const rmi_shard_index* si, const uint64_t* d_queries, uint64_t n, uint64_t* d_send,
                                  uint64_t* d_slot, uint64_t* d_send_counts, void* cuda_stream) {
  const char* fn = "rmi_shard_index_predict_route";
  if (int rc = shard_check_bounded(si, fn)) return rc;
  if (!d_send_counts) return fail(RMI_ERR_INVALID, std::string(fn) + ": null count pointer");
  if (n && (!d_queries || !d_send || !d_slot)) return fail(RMI_ERR_INVALID, std::string(fn) + ": null query, send or slot pointer");
  CUDA_TRY(cudaSetDevice(si->idx->ds->device));
  return shard_predict_route(si, (const u64*)d_queries, n, (u64*)d_send, (u64*)d_slot, (u64*)d_send_counts,
                             (cudaStream_t)cuda_stream);
}

int rmi_shard_index_predict_search(const rmi_shard_index* si, const uint64_t* d_received, uint64_t m, uint64_t* d_pos,
                                   void* cuda_stream) {
  const char* fn = "rmi_shard_index_predict_search";
  if (int rc = shard_check_bounded(si, fn)) return rc;
  if (m && (!d_received || !d_pos)) return fail(RMI_ERR_INVALID, std::string(fn) + ": null query or output pointer");
  CUDA_TRY(cudaSetDevice(si->idx->ds->device));
  return shard_predict_search(si, (const u64*)d_received, m, (u64*)d_pos, (cudaStream_t)cuda_stream);
}

int rmi_shard_index_predict_collective(rmi_shard_index* si, rmi_shard_comm* c, const uint64_t* d_queries, uint64_t n,
                                       uint64_t* d_pos, uint64_t* d_err, void* cuda_stream) {
  const char* fn = "rmi_shard_index_predict_collective";
  g_last_error.clear();
  if (int rc = shard_check_bounded(si, fn)) return rc;
  if (!c) return fail(RMI_ERR_INVALID, std::string(fn) + ": null communicator");
  if (n && (!d_queries || !d_pos)) return fail(RMI_ERR_INVALID, std::string(fn) + ": null query or output pointer");
  if (int rc = shard_check_comm(si, c, fn)) return rc;
  CUDA_TRY(cudaSetDevice(si->idx->ds->device));
  const cudaStream_t st = (cudaStream_t)cuda_stream;
  const u64* d_q = (const u64*)d_queries;
  int rc = shard_one_call<u64>(
      si, c, n, (u64*)d_pos, st, fn,
      [&](u64* d_send, u64* d_slot, u64* d_counts) { return shard_predict_route(si, d_q, n, d_send, d_slot, d_counts, st); },
      [&](const u64* d_recv, u64 m, u64* d_ans) { return shard_predict_search(si, d_recv, m, d_ans, st); });
  if (rc == RMI_OK && d_err) {
    Launch L{st, si->idx->num_sms};
    shard_fill(L, si->ks.line, n, (u64*)d_err);
    CUDA_TRY(cudaGetLastError());
  }
  return rc;
}

}  // extern "C"

// ---- rmi_evaluate over a range-partitioned data set (DESIGN.md section 15) -----------------------------------------
constexpr int SHARD_EVAL_EVENTS = 5;   // upload | boundaries (+ all-reduce) | error pass (+ all-reduce) | statistics

struct rmi_shard_eval {
  const rmi_result* r = nullptr;   // the caller's: read at every evaluation
  const rmi_dataset* ds = nullptr;
  const ModelName* top = nullptr;
  const ModelName* leaf = nullptr;
  int world = 0, rank = 0, num_sms = 0;
  uint64_t N = 0;
  SlabLayout lay;
  TopTables tables;                // device copies of r's top tables (device_alloc)
  TopModel* d_top = nullptr;
  BuildAux* d_aux = nullptr;
  double* d_params = nullptr;
  u64* d_errors = nullptr;
  u64* d_counts = nullptr;
  void* d_stats = nullptr;
  // rmi_shard_evaluate: its own stream and the exchanged buffers
  cudaStream_t own = nullptr;
  u64* d_S = nullptr;              // N + 1
  u64* d_part = nullptr;           // 2 x N
  unsigned* d_status = nullptr;    // world: every rank's status word
  cudaStream_t st = nullptr;       // the stream of the evaluation under way
  cudaEvent_t ev[SHARD_EVAL_EVENTS] = {};
  std::chrono::steady_clock::time_point t_start;
};

namespace {

uint64_t eval_partial_words(const rmi_shard_eval* e) { return e->lay.no_dups ? e->N : 2 * e->N; }

int eval_bounds(rmi_shard_eval* e, u64* d_S, cudaStream_t st) {
  CUDA_TRY(cudaSetDevice(e->ds->device));
  e->st = st;
  e->t_start = std::chrono::steady_clock::now();
  const rmi_result& r = *e->r;
  cudaEventRecord(e->ev[0], st);
  const TopModel h_top = e->tables.given(r);
  cudaMemcpyAsync(e->d_top, &h_top, sizeof(h_top), cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(e->d_params, r.l1_params, sizeof(double) * e->N * leaf_params_per_model(e->leaf->kind),
                  cudaMemcpyHostToDevice, st);
  if (e->tables.t32_len) cudaMemcpyAsync(e->tables.t32, r.l0_table32, sizeof(u32) * e->tables.t32_len, cudaMemcpyHostToDevice, st);
  if (e->tables.hist_bins) cudaMemcpyAsync(e->tables.pivots, r.l0_array2, sizeof(u64) * e->tables.hist_bins, cudaMemcpyHostToDevice, st);
  cudaMemsetAsync(e->d_aux, 0, sizeof(BuildAux), st);
  cudaEventRecord(e->ev[1], st);
  Launch L{st, e->num_sms};
  with_key_type(e->ds->key_type, [&](auto k) {
    using T = decltype(k);
    shard_bounds_given<T>(L, (const T*)e->ds->d_keys, shard_of<T>(e->lay, e->ds->n, e->ds->n), e->top->kind, e->d_top,
                          e->N, d_S, e->d_aux);
  });
  CUDA_TRY(cudaGetLastError());
  return RMI_OK;
}

int eval_keys(rmi_shard_eval* e, const u64* d_S, u64* d_part, unsigned* d_status, cudaStream_t st) {
  CUDA_TRY(cudaSetDevice(e->ds->device));
  e->st = st;
  cudaEventRecord(e->ev[2], st);
  Launch L{st, e->num_sms};
  with_key_type(e->ds->key_type, [&](auto k) {
    using T = decltype(k);
    shard_evaluate_partials<T>(L, (const T*)e->ds->d_keys, shard_of<T>(e->lay, e->ds->n, e->ds->n), e->lay.is_first,
                               e->lay.has_next, key_from_bits<T>(e->lay.next_key_bits), e->leaf->kind, e->N, d_S,
                               e->d_params, d_part);
  });
  shard_copy_status(L, e->d_aux, d_status);
  CUDA_TRY(cudaGetLastError());
  return RMI_OK;
}

int eval_finish(rmi_shard_eval* e, const u64* d_S, const u64* d_part, unsigned status, uint32_t flags, const char* fn,
                rmi_result** out) {
  CUDA_TRY(cudaSetDevice(e->ds->device));
  cudaStream_t st = e->st;
  const uint64_t n = e->lay.n_global, N = e->N;
  const bool stats_only = (flags & RMI_FLAG_STATS_ONLY) != 0;
  const bool want_counts = !stats_only && (flags & RMI_FLAG_LEAF_COUNTS) != 0;
  Launch L{st, e->num_sms};
  cudaEventRecord(e->ev[3], st);
  shard_evaluate_finish(L, n, N, e->lay.no_dups, d_S, d_part, e->d_errors, e->d_counts);
  leaf_statistics(L, n, N, e->d_errors, e->d_counts, e->d_aux, e->d_stats);
  cudaEventRecord(e->ev[4], st);
  // the host buffers are taken while the kernels run
  auto box = new ResultBox();
  if (!reserve_result(box, &e->tables, N, leaf_params_per_model(e->leaf->kind), !stats_only, want_counts)) {
    cudaStreamSynchronize(st);
    delete box;
    return fail(RMI_ERR_CUDA, kPinnedFailed);
  }
  copy_result_to_host(box, nullptr, e->d_aux, e->d_top, nullptr, nullptr, nullptr, st);
  if (!stats_only) {
    cudaMemcpyAsync(box->l1_errors.data(), e->d_errors, sizeof(u64) * N, cudaMemcpyDeviceToHost, st);
    if (want_counts) cudaMemcpyAsync(box->l1_counts.data(), e->d_counts, sizeof(u64) * N, cudaMemcpyDeviceToHost, st);
  }
  const cudaError_t ce = cudaStreamSynchronize(st);
  if (ce != cudaSuccess) { delete box; return fail(RMI_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(ce)); }
  // status: the OR over every rank, so that all of them fail alike; this rank's own word is in it
  const unsigned bad = (status | result_aux(box).status) & kEvaluateStatus;
  if (bad) { delete box; return fail(RMI_ERR_PANIC, status_text(bad)); }
  fill_given_result(box, e->r, *e->top, *e->leaf, e->tables, n, stats_only);
  rmi_result& R = box->pub;
  for (int q = 0; q < 4; ++q) {
    R.phase_device_ns[q] = elapsed_ns(e->ev[q], e->ev[q + 1]);
    R.device_time_ns += R.phase_device_ns[q];
  }
  R.build_time_ns =
      (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - e->t_start).count();
  *out = &box->pub;
  return RMI_OK;
}

}  // namespace

extern "C" {

int rmi_shard_eval_create(const rmi_result* r, const rmi_dataset* local, const rmi_shard_ends* ends_all, int world,
                          int rank, rmi_shard_eval** out) {
  const std::string fn = "rmi_shard_eval_create";
  g_last_error.clear();
  if (!r || !local || !ends_all || !out) return fail(RMI_ERR_INVALID, fn + ": null argument");
  const ModelName *top = nullptr, *leaf = nullptr;
  if (int rc = check_result(r, false, fn, &top, &leaf)) return rc;
  uint64_t total = 0, base = 0;
  if (int rc = check_slabs(fn, local, ends_all, world, rank, &base, &total)) return rc;
  // rmi_evaluate's checks of the concatenated keys: leaves, no keys, this slab's order
  if (int rc = check_build(total, r->branching_factor, local->sorted)) return rc;
  CUDA_TRY(cudaSetDevice(local->device));
  DeviceInfo di;
  if (int rc = device_info(local->device, &di)) return rc;
  auto* e = new rmi_shard_eval();
  e->r = r; e->ds = local; e->top = top; e->leaf = leaf;
  e->world = world; e->rank = rank; e->num_sms = di.num_sms;
  e->N = r->branching_factor;
  e->lay = with_key_type(local->key_type, [&](auto k) {
    return rmihost::slab_layout<decltype(k)>(ends_all, world, rank, e->N);
  });
  const uint64_t N = e->N;
  bool ok = cudaStreamCreateWithFlags(&e->own, cudaStreamNonBlocking) == cudaSuccess;
  for (int q = 0; q < SHARD_EVAL_EVENTS; ++q) ok = ok && cudaEventCreate(&e->ev[q]) == cudaSuccess;
  ok = ok && (e->d_top = (TopModel*)device_alloc(sizeof(TopModel))) && (e->d_aux = (BuildAux*)device_alloc(sizeof(BuildAux))) &&
       (e->d_params = (double*)device_alloc(sizeof(double) * N * leaf_params_per_model(leaf->kind))) &&
       (e->d_errors = (u64*)device_alloc(sizeof(u64) * N)) && (e->d_counts = (u64*)device_alloc(sizeof(u64) * N)) &&
       (e->d_stats = device_alloc(stats_scratch_bytes(N))) && (e->d_S = (u64*)device_alloc(sizeof(u64) * (N + 1))) &&
       (e->d_part = (u64*)device_alloc(sizeof(u64) * 2 * N)) &&
       (e->d_status = (unsigned*)device_alloc(sizeof(unsigned) * world));
  // the top tables' device homes (their contents are copied again at every evaluation)
  ok = ok && e->tables.upload(*r, e->own, device_alloc) == cudaSuccess && cudaStreamSynchronize(e->own) == cudaSuccess;
  if (!ok) {
    cudaGetLastError();
    rmi_shard_eval_destroy(e);
    return fail(RMI_ERR_CUDA, fn + ": device allocation failed");
  }
  *out = e;
  return RMI_OK;
}

void rmi_shard_eval_destroy(rmi_shard_eval* e) {
  if (!e) return;
  e->tables.free_device();
  for (void* p : {(void*)e->d_top, (void*)e->d_aux, (void*)e->d_params, (void*)e->d_errors, (void*)e->d_counts, e->d_stats,
                  (void*)e->d_S, (void*)e->d_part, (void*)e->d_status})
    cudaFree(p);
  for (cudaEvent_t v : e->ev) if (v) cudaEventDestroy(v);
  if (e->own) cudaStreamDestroy(e->own);
  delete e;
}

uint64_t rmi_shard_eval_partial_words(const rmi_shard_eval* e) { return e ? eval_partial_words(e) : 0; }

int rmi_shard_eval_bounds(rmi_shard_eval* e, uint64_t* d_S, void* cuda_stream) {
  g_last_error.clear();
  if (!e || !d_S) return fail(RMI_ERR_INVALID, "rmi_shard_eval_bounds: null argument");
  return eval_bounds(e, (u64*)d_S, (cudaStream_t)cuda_stream);
}

int rmi_shard_eval_keys(rmi_shard_eval* e, const uint64_t* d_S, uint64_t* d_partial, uint32_t* d_status, void* cuda_stream) {
  g_last_error.clear();
  if (!e || !d_S || !d_partial || !d_status) return fail(RMI_ERR_INVALID, "rmi_shard_eval_keys: null argument");
  return eval_keys(e, (const u64*)d_S, (u64*)d_partial, (unsigned*)d_status, (cudaStream_t)cuda_stream);
}

int rmi_shard_eval_finish(rmi_shard_eval* e, const uint64_t* d_S, const uint64_t* d_partial, uint32_t status,
                          uint32_t flags, rmi_result** out) {
  g_last_error.clear();
  if (!e || !d_S || !d_partial || !out) return fail(RMI_ERR_INVALID, "rmi_shard_eval_finish: null argument");
  return eval_finish(e, (const u64*)d_S, (const u64*)d_partial, status, flags, "rmi_shard_eval_finish", out);
}

int rmi_shard_evaluate(rmi_shard_eval* e, rmi_shard_comm* c, uint32_t flags, rmi_result** out) {
  const char* fn = "rmi_shard_evaluate";
  g_last_error.clear();
  if (!e || !c || !out) return fail(RMI_ERR_INVALID, std::string(fn) + ": null argument");
  if (c->world != e->world || c->rank != e->rank)
    return fail(RMI_ERR_INVALID, std::string(fn) + ": the communicator is rank " + std::to_string(c->rank) + " of " +
                                     std::to_string(c->world) + ", the evaluator rank " + std::to_string(e->rank) + " of " +
                                     std::to_string(e->world));
  const NcclApi& nc = nccl_api();
  if (!nc.ok) return fail(RMI_ERR_UNSUPPORTED, nc.error);
  const int W = e->world;
  cudaStream_t st = e->own;
  if (int rc = eval_bounds(e, e->d_S, st)) return rc;
  if (W > 1) NCCL_TRY(nc.AllReduce(e->d_S, e->d_S, e->N + 1, ncclUint64, ncclMin, c->comm, st));
  if (int rc = eval_keys(e, e->d_S, e->d_part, e->d_status + e->rank, st)) return rc;
  if (W > 1) {
    NCCL_TRY(nc.GroupStart());
    NCCL_TRY(nc.AllReduce(e->d_part, e->d_part, eval_partial_words(e), ncclUint64, ncclMax, c->comm, st));
    NCCL_TRY(nc.AllGather(e->d_status + e->rank, e->d_status, 1, ncclUint32, c->comm, st));
    NCCL_TRY(nc.GroupEnd());
  }
  std::vector<unsigned> all(W, 0);
  CUDA_TRY(cudaMemcpyAsync(all.data(), e->d_status, sizeof(unsigned) * W, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  unsigned status = 0;
  for (unsigned s : all) status |= s;
  return eval_finish(e, e->d_S, e->d_part, status, flags, fn, out);
}

}  // extern "C"

// ---- the cache-fix spline over a range-partitioned data set (DESIGN.md section 16) ---------------------------------
struct rmi_shard_cache_fix {
  const rmi_dataset* ds = nullptr;
  CacheFixSlab slab{};
  uint64_t line = 0, nch = 0;
  int is_last = 0;
  rmi_spline_point finish{};       // finish()'s point, written by the last non-empty rank
  cudaStream_t st = nullptr;
  int num_sms = 0;
  void* d_mem = nullptr;
  ShardCacheFixScratch s{};
  bool speculated = false;         // speculation and the stitches of chunks 1.. are in s
  bool scanned = false, passed = false;
  uint64_t slab_knots = 0;         // knots of the last scan's chain inside the slab
};

extern "C" {

int rmi_shard_cache_fix_create(const rmi_dataset* local, const rmi_shard_ends* ends_all, int world, int rank,
                               uint64_t line_size, uint64_t halo_keys, void* cuda_stream, rmi_shard_cache_fix** out) {
  const std::string fn = "rmi_shard_cache_fix_create";
  g_last_error.clear();
  if (!local || !ends_all || !out) return fail(RMI_ERR_INVALID, fn + ": null argument");
  uint64_t total = 0, base = 0;
  if (int rc = check_slabs(fn, local, ends_all, world, rank, &base, &total)) return rc;
  if (local->key_type != RMI_KEY_U64) return fail(RMI_ERR_INVALID, fn + ": Can only construct a bounded RMI on u64 data");
  if (base + local->n + halo_keys > total)
    return fail(RMI_ERR_INVALID, fn + ": the halo reaches past the end of the data");
  // rmi_cache_fix_device's panics, in its order, decided from the ends table so that every rank fails alike
  if (!(total > line_size)) return fail(RMI_ERR_PANIC, "Cannot apply a cachefix with fewer items than the line size");
  if (line_size == 0) return fail(RMI_ERR_PANIC, "attempt to divide by zero");
  if (!local->sorted) return fail(RMI_ERR_PANIC, "keys are not sorted in ascending order");
  const SlabLayout lay = rmihost::slab_layout<uint64_t>(ends_all, world, rank, 1);
  if (lay.first_key_bits == 0) return fail(RMI_ERR_PANIC, "When source x is 18446744073709551615, cannot set dest x to 0");
  CUDA_TRY(cudaSetDevice(local->device));
  DeviceInfo di;
  if (int rc = device_info(local->device, &di)) return rc;
  auto* cf = new rmi_shard_cache_fix();
  cf->ds = local;
  cf->line = line_size;
  cf->st = (cudaStream_t)cuda_stream;
  cf->num_sms = di.num_sms;
  cf->is_last = lay.is_last;
  cf->finish = rmi_spline_point{lay.last_key_bits, lay.last_F};
  CacheFixSlab& S = cf->slab;
  S.keys = (const u64*)local->d_keys;
  S.base = base;
  S.n_local = local->n;
  S.n_avail = local->n + halo_keys;
  S.prev_key = lay.has_prev ? lay.prev_key_bits : 0;
  S.has_prev = lay.has_prev;
  S.at_end = base + S.n_avail == total;
  const u64 nch = cf->nch = (local->n + CACHEFIX_CHUNK - 1) / CACHEFIX_CHUNK;
  if (nch) {
    const size_t words = nch * CACHEFIX_TARGETS + 3 * nch + (nch + 1) / 2 + 4 * nch + (nch + 1) + 4;
    if (cudaMalloc(&cf->d_mem, sizeof(u64) * words) != cudaSuccess) {
      cudaGetLastError();
      delete cf;
      return fail(RMI_ERR_CUDA, fn + ": device allocation failed");
    }
    u64* p = (u64*)cf->d_mem;
    ShardCacheFixScratch& s = cf->s;
    s.targets = p; p += nch * CACHEFIX_TARGETS;
    s.spec_count = p; p += nch;
    s.spec_exit = p; p += nch;
    s.stitch_exit = p; p += nch;
    s.stitch_ok = (u32*)p; p += (nch + 1) / 2;
    s.st_entry = p; p += 2 * nch;
    s.entry = p; p += 2 * nch;
    s.offsets = p; p += nch + 1;
    s.res = p;
  }
  *out = cf;
  return RMI_OK;
}

void rmi_shard_cache_fix_destroy(rmi_shard_cache_fix* cf) {
  if (!cf) return;
  if (cf->d_mem) {
    cudaStreamSynchronize(cf->st);
    cudaFree(cf->d_mem);
  }
  delete cf;
}

int rmi_shard_cache_fix_scan(rmi_shard_cache_fix* cf, uint64_t entry_pid, rmi_shard_cache_fix_scan_result* out) {
  const std::string fn = "rmi_shard_cache_fix_scan";
  g_last_error.clear();
  if (!cf || !out) return fail(RMI_ERR_INVALID, fn + ": null argument");
  const CacheFixSlab& S = cf->slab;
  if (entry_pid < 2 * S.base)
    return fail(RMI_ERR_INVALID, fn + ": entry pid " + std::to_string(entry_pid) + " lies before the slab (first pid " +
                                     std::to_string(2 * S.base) + ")");
  *out = rmi_shard_cache_fix_scan_result{};
  cf->scanned = true;
  cf->passed = entry_pid >= 2 * (S.base + S.n_local);   // a segment spanning the whole slab, or an empty slab
  if (cf->passed) {
    cf->slab_knots = 0;
    out->exit_pid = entry_pid;
  } else {
    CUDA_TRY(cudaSetDevice(cf->ds->device));
    Launch L{cf->st, cf->num_sms};
    if (!cf->speculated) shard_cache_fix_speculate(L, S, cf->line, CACHEFIX_CHUNK, cf->s);
    shard_cache_fix_join(L, S, cf->line, CACHEFIX_CHUNK, entry_pid, cf->speculated, cf->s);
    u64 res[4] = {};
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(res, cf->s.res, sizeof res, cudaMemcpyDeviceToHost, cf->st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(cf->st);
    if (e != cudaSuccess) { cf->scanned = false; return fail(RMI_ERR_CUDA, fn + ": " + cudaGetErrorString(e)); }
    cf->speculated = true;
    cf->slab_knots = res[1];
    out->exit_pid = res[0];
    out->status = res[2] ? RMI_SHARD_CACHE_FIX_HALO_TOO_SMALL : 0;
    out->reach = res[3];
    if (out->status) cf->scanned = false;
  }
  out->num_knots = cf->slab_knots + (cf->is_last ? 1 : 0);
  return RMI_OK;
}

int rmi_shard_cache_fix_emit(rmi_shard_cache_fix* cf, rmi_spline_point* d_out) {
  const std::string fn = "rmi_shard_cache_fix_emit";
  g_last_error.clear();
  if (!cf) return fail(RMI_ERR_INVALID, fn + ": null argument");
  if (!cf->scanned) return fail(RMI_ERR_INVALID, fn + ": no complete scan to emit");
  const uint64_t total = cf->slab_knots + (cf->is_last ? 1 : 0);
  if (!total) return RMI_OK;
  if (!d_out) return fail(RMI_ERR_INVALID, fn + ": null output");
  CUDA_TRY(cudaSetDevice(cf->ds->device));
  if (!cf->passed && cf->slab_knots) {
    Launch L{cf->st, cf->num_sms};
    shard_cache_fix_emit(L, cf->slab, cf->line, CACHEFIX_CHUNK, cf->s, d_out);
    CUDA_TRY(cudaGetLastError());
  }
  // finish() (cache_fix.rs:91-93): from pageable memory, staged before the call returns
  if (cf->is_last) CUDA_TRY(cudaMemcpyAsync(d_out + cf->slab_knots, &cf->finish, sizeof(rmi_spline_point),
                                            cudaMemcpyHostToDevice, cf->st));
  return RMI_OK;
}

}  // extern "C"
