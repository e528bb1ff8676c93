// Checks rmi_b200/csrc/multiset_diff.cuh on the CPU against a std::map count of every value:
//   - the subtraction k_delta_subtract performs (each tile's window of removed keys, then every thread's walk over its
//     MERGE_ITEMS keys), which must drop the first c(v) copies of every value v removed c(v) times and place every
//     survivor at its position in the difference, bit for bit (so f64 -0.0 / 0.0 runs must lose their first copies);
//   - the removal check of k_delta_check_remove, which must flag exactly the batch keys beyond the copies the key set
//     holds.
// Prints one line per case, "case=<name> n_m=.. n_r=.. fail=<0|1>", and FAIL on a mismatch.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <random>
#include <string>
#include <vector>

#include "../../rmi_b200/csrc/multiset_diff.cuh"

using rmi::MERGE_ITEMS;
using rmi::MERGE_THREADS;
using rmi::MERGE_TILE;

template <class T> bool same_bits(const std::vector<T>& x, const std::vector<T>& y) {
  return x.size() == y.size() && (x.empty() || std::memcmp(x.data(), y.data(), x.size() * sizeof(T)) == 0);
}

template <class T> bool is_nan(const T& v) { return !(v == v); }

// std::map orders by <, so -0.0 and 0.0 share one entry: counts are by value.  NaN keys are never counted.
template <class T> std::map<T, uint64_t> counts(const std::vector<T>& a) {
  std::map<T, uint64_t> c;
  for (const T& v : a)
    if (!is_nan(v)) ++c[v];
  return c;
}

// M without the first c(v) copies of each value v, c(v) the copies of v in r.
template <class T> std::vector<T> oracle_diff(const std::vector<T>& M, const std::vector<T>& r) {
  std::map<T, uint64_t> left = counts(r);
  std::vector<T> out;
  for (const T& v : M) {
    if (!is_nan(v)) {
      auto it = left.find(v);
      if (it != left.end() && it->second) { --it->second; continue; }
    }
    out.push_back(v);
  }
  return out;
}

// The kernel's decomposition, sequentially; false when a destination is out of range or written twice.
template <class T> bool subtract_like_kernel(const std::vector<T>& M, const std::vector<T>& r, std::vector<T>& out) {
  const uint64_t nm = M.size(), t = r.size();
  if (t > nm) return false;
  out.assign(nm - t, T(0));
  std::vector<char> written(nm - t, 0);
  bool ok = true;
  uint64_t emitted = 0;
  for (uint64_t p0 = 0; p0 < nm; p0 += MERGE_TILE) {
    const uint64_t len = std::min<uint64_t>(MERGE_TILE, nm - p0);
    const uint64_t lo = rmi::diff_search<false>(r.data(), 0, t, M[p0]);
    const uint64_t hi = std::max(lo, rmi::diff_search<true>(r.data(), 0, t, M[p0 + len - 1]));
    for (int th = 0; th < MERGE_THREADS; ++th) {
      const uint64_t k0 = (uint64_t)th * MERGE_ITEMS;
      if (k0 >= len) break;
      const uint64_t kn = std::min<uint64_t>(MERGE_ITEMS, len - k0);
      rmi::subtract_keys(M.data() + p0 + k0, p0 + k0, kn, M.data(), r.data(), lo, hi, [&](uint64_t k, uint64_t dest) {
        if (dest >= nm - t || written[dest]) { ok = false; return; }
        written[dest] = 1;
        out[dest] = M[p0 + k0 + k];
        ++emitted;
      });
    }
  }
  return ok && emitted == nm - t;
}

// The removal check: batch[j] is flagged when the batch holds more copies of its value up to j than the set holds.
template <class T> bool check_rule_matches(const std::vector<T>& set, const std::vector<T>& batch) {
  const std::map<T, uint64_t> held = counts(set);
  std::map<T, uint64_t> seen;
  for (uint64_t j = 0; j < batch.size(); ++j) {
    const T v = batch[j];
    auto it = held.find(v);
    const uint64_t c = is_nan(v) || it == held.end() ? 0 : it->second;
    const bool want_missing = is_nan(v) || seen[v]++ >= c;
    if (rmi::past_first_copies(batch.data(), j, c) != want_missing) return false;
  }
  return true;
}

int failures = 0;

template <class T> void check(const std::string& name, const std::vector<T>& M, const std::vector<T>& r) {
  std::vector<T> got;
  bool ok = subtract_like_kernel(M, r, got) && same_bits(got, oracle_diff(M, r));
  ok = ok && check_rule_matches(M, r);
  if (!ok) ++failures;
  std::printf("case=%s n_m=%zu n_r=%zu fail=%d%s\n", name.c_str(), M.size(), r.size(), ok ? 0 : 1, ok ? "" : " FAIL");
}

// A batch checked against a set that need not hold it (the check alone).
template <class T> void check_batch(const std::string& name, const std::vector<T>& set, const std::vector<T>& batch) {
  const bool ok = check_rule_matches(set, batch);
  if (!ok) ++failures;
  std::printf("case=%s n_m=%zu n_r=%zu fail=%d%s\n", name.c_str(), set.size(), batch.size(), ok ? 0 : 1,
              ok ? "" : " FAIL");
}

template <class T> std::vector<T> sorted_random(std::mt19937_64& rng, uint64_t n, uint64_t range) {
  std::vector<T> v(n);
  for (auto& x : v) x = (T)(rng() % range);
  std::sort(v.begin(), v.end());
  return v;
}

// A sorted sub-multiset of M: each key kept with probability 1 / every.
template <class T> std::vector<T> sample(std::mt19937_64& rng, const std::vector<T>& M, unsigned every) {
  std::vector<T> r;
  for (const T& v : M)
    if (!is_nan(v) && rng() % every == 0) r.push_back(v);
  return r;
}

template <class T> void cases(const std::string& ty, std::mt19937_64& rng) {
  const uint64_t tile = MERGE_TILE;
  check<T>(ty + "/both_empty", {}, {});
  check<T>(ty + "/removed_empty", sorted_random<T>(rng, 3000, 1000), {});
  {
    std::vector<T> M = sorted_random<T>(rng, 3000, 1000);
    check<T>(ty + "/remove_everything", M, M);
  }
  {
    std::vector<T> M(5000, (T)42);
    check<T>(ty + "/all_equal_some", M, std::vector<T>(1234, (T)42));
    check<T>(ty + "/all_equal_every", M, M);
    check<T>(ty + "/all_equal_one", M, std::vector<T>(1, (T)42));
  }
  {
    // runs that straddle tiles, some removed whole, some in part, some not at all
    std::vector<T> M, r;
    for (int k = 0; k < 6; ++k) {
      const uint64_t run = 2 * tile + 13 * k + (k % 2 ? tile / 2 : 0);
      M.insert(M.end(), run, (T)(10 * k));
      M.insert(M.end(), 7, (T)(10 * k + 5));
      const uint64_t gone = k % 3 == 0 ? run : k % 3 == 1 ? run / 2 + 1 : 0;
      r.insert(r.end(), gone, (T)(10 * k));
      if (k % 2) r.push_back((T)(10 * k + 5));
    }
    check<T>(ty + "/runs_across_tiles", M, r);
  }
  {
    // one tile's window far longer than the tile: a run of 5 tiles, all but its last key removed
    std::vector<T> M(5 * tile, (T)7);
    M.push_back((T)9);
    check<T>(ty + "/window_beyond_tile", M, std::vector<T>(5 * tile - 1, (T)7));
  }
  for (uint64_t total : {tile - 1, tile, tile + 1, 2 * tile + 1, 3 * tile + 7})
    for (unsigned every : {1u, 2u, 5u, 50u}) {
      std::vector<T> M = sorted_random<T>(rng, total, every % 2 ? 40 : 1000000);
      check<T>(ty + "/size_" + std::to_string(total) + "_every_" + std::to_string(every), M, sample(rng, M, every));
    }
  {
    std::vector<T> M = sorted_random<T>(rng, 200000, 1u << 16);
    check<T>(ty + "/random_large", M, sample(rng, M, 7));
  }
  {
    // the check alone: absent keys, one copy too many, a run held in full
    std::vector<T> set = {(T)1, (T)2, (T)2, (T)3, (T)3, (T)3, (T)9};
    check_batch<T>(ty + "/check_absent", set, {(T)1, (T)4});
    check_batch<T>(ty + "/check_one_too_many", set, {(T)2, (T)2, (T)2, (T)3});
    check_batch<T>(ty + "/check_full_runs", set, {(T)2, (T)2, (T)3, (T)3, (T)3});
    check_batch<T>(ty + "/check_empty_set", {}, {(T)0, (T)0});
  }
}

int main() {
  std::mt19937_64 rng(777);
  cases<uint32_t>("u32", rng);
  cases<uint64_t>("u64", rng);
  cases<double>("f64", rng);
  {
    // signed zeros compare equal: a removal takes the first copies of the zero run, whatever their sign
    std::vector<double> M = {-1.0};
    for (int i = 0; i < 3000; ++i) M.push_back(i % 3 ? -0.0 : 0.0);
    M.push_back(1.0);
    check<double>("f64/signed_zeros_some", M, std::vector<double>(1001, 0.0));
    check<double>("f64/signed_zeros_mixed_batch", M, {-1.0, -0.0, 0.0, -0.0, 1.0});
    check<double>("f64/signed_zeros_all", M, std::vector<double>(3000, -0.0));
    check_batch<double>("f64/check_signed_zeros", M, std::vector<double>(3001, 0.0));
  }
  {
    // NaNs at the end of M (merge_path.cuh's order): never removed, kept in place
    std::vector<double> M = sorted_random<double>(rng, 3 * MERGE_TILE, 500);
    std::vector<double> r = sample(rng, M, 3);
    M.insert(M.end(), 5, std::nan(""));
    check<double>("f64/nan_in_m", M, r);
    check_batch<double>("f64/check_nan", M, {1.0, std::nan("")});
  }
  std::printf("failures=%d\n", failures);
  return failures ? 1 : 0;
}
