// Checks rmi_b200/csrc/merge_path.cuh on the CPU: every co-rank, and the merge k_delta_merge performs (block co-ranks
// at tile boundaries, then per-thread co-ranks and tile merges inside the block's slices), against std::merge, which
// is stable with the first range first on equal keys.  Compared bit for bit, so f64 -0.0 / 0.0 ties must keep the
// first input's zero first.  Prints one line per case, "case=<name> n_a=.. n_b=.. fail=<0|1>", and FAIL on a mismatch.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../../rmi_b200/csrc/merge_path.cuh"

using rmi::MERGE_ITEMS;
using rmi::MERGE_THREADS;
using rmi::MERGE_TILE;

template <class T> bool same_bits(const std::vector<T>& x, const std::vector<T>& y) {
  return x.size() == y.size() && (x.empty() || std::memcmp(x.data(), y.data(), x.size() * sizeof(T)) == 0);
}

// The kernel's decomposition, sequentially.
template <class T> std::vector<T> merge_like_kernel(const std::vector<T>& a, const std::vector<T>& b) {
  const uint64_t na = a.size(), nb = b.size(), total = na + nb;
  std::vector<T> out(total);
  for (uint64_t d0 = 0; d0 < total; d0 += MERGE_TILE) {
    const uint64_t d1 = std::min(total, d0 + MERGE_TILE);
    const uint64_t i0 = rmi::merge_corank(a.data(), na, b.data(), nb, d0);
    uint64_t i1 = rmi::merge_corank(a.data(), na, b.data(), nb, d1);
    i1 = std::min(std::max(i1, i0), i0 + (d1 - d0));
    const uint64_t j0 = d0 - i0, la = i1 - i0, len = d1 - d0;
    std::vector<T> s_in(len);
    for (uint64_t t = 0; t < len; ++t) s_in[t] = t < la ? a[i0 + t] : b[j0 + t - la];
    for (int th = 0; th < MERGE_THREADS; ++th) {
      const uint64_t t0 = (uint64_t)th * MERGE_ITEMS;
      if (t0 < len)
        rmi::merge_tile(s_in.data(), la, s_in.data() + la, len - la, t0, std::min<uint64_t>(len, t0 + MERGE_ITEMS),
                        out.data() + d0 + t0);
    }
  }
  return out;
}

int failures = 0;

template <class T> void check(const std::string& name, std::vector<T> a, std::vector<T> b) {
  std::vector<T> want(a.size() + b.size());
  std::merge(a.begin(), a.end(), b.begin(), b.end(), want.begin());
  bool ok = same_bits(merge_like_kernel(a, b), want);
  // every co-rank: a's keys among the first d of the stable merge
  std::vector<int> from_a;   // 1 where want[k] came from a, in the stable merge's own order
  {
    uint64_t i = 0, j = 0;
    while (i < a.size() || j < b.size()) {
      const bool ta = j == b.size() || (i < a.size() && !(b[j] < a[i]));
      from_a.push_back(ta ? 1 : 0);
      ta ? ++i : ++j;
    }
  }
  uint64_t ia = 0;
  for (uint64_t d = 0; d <= want.size() && ok; ++d) {
    if (rmi::merge_corank(a.data(), a.size(), b.data(), b.size(), d) != ia) ok = false;
    if (d < want.size()) ia += from_a[d];
  }
  // one merge_tile over the whole range and over uneven pieces
  for (uint64_t piece : {(uint64_t)1, (uint64_t)7, MERGE_TILE - 1, MERGE_TILE + 1}) {
    std::vector<T> out(want.size());
    for (uint64_t d0 = 0; d0 < want.size(); d0 += piece)
      rmi::merge_tile(a.data(), a.size(), b.data(), b.size(), d0, std::min<uint64_t>(want.size(), d0 + piece),
                      out.data() + d0);
    ok = ok && same_bits(out, want);
  }
  if (!ok) ++failures;
  std::printf("case=%s n_a=%zu n_b=%zu fail=%d%s\n", name.c_str(), a.size(), b.size(), ok ? 0 : 1, ok ? "" : " FAIL");
}

template <class T> std::vector<T> sorted_random(std::mt19937_64& rng, uint64_t n, uint64_t range) {
  std::vector<T> v(n);
  for (auto& x : v) x = (T)(rng() % range);
  std::sort(v.begin(), v.end());
  return v;
}

template <class T> void cases(const std::string& ty, std::mt19937_64& rng) {
  const uint64_t tile = MERGE_TILE;
  check<T>(ty + "/both_empty", {}, {});
  check<T>(ty + "/a_empty", {}, sorted_random<T>(rng, 3000, 1000));
  check<T>(ty + "/b_empty", sorted_random<T>(rng, 3000, 1000), {});
  {
    std::vector<T> lo = sorted_random<T>(rng, 2500, 1000), hi = sorted_random<T>(rng, 1800, 1000);
    for (auto& x : hi) x = (T)(x + 5000);
    check<T>(ty + "/a_below_b", lo, hi);
    check<T>(ty + "/b_below_a", hi, lo);
  }
  check<T>(ty + "/all_equal", std::vector<T>(5000, (T)42), std::vector<T>(3000, (T)42));
  {
    // runs of one key that straddle several tiles, in both inputs
    std::vector<T> a, b;
    for (int r = 0; r < 4; ++r) {
      a.insert(a.end(), 3 * tile + 17 * r, (T)(10 * r));
      b.insert(b.end(), tile + 5 + 31 * r, (T)(10 * r));
      b.insert(b.end(), 11, (T)(10 * r + 5));
    }
    check<T>(ty + "/long_runs", a, b);
  }
  for (uint64_t total : {tile - 1, tile, tile + 1, 2 * tile - 1, 2 * tile, 2 * tile + 1, 3 * tile + 7})
    for (uint64_t na : {(uint64_t)0, (uint64_t)1, total / 3, total / 2, total - 1, total}) {
      const uint64_t range = (na % 2) ? 50 : 1000000;   // many ties, or few
      check<T>(ty + "/size_" + std::to_string(total) + "_" + std::to_string(na), sorted_random<T>(rng, na, range),
               sorted_random<T>(rng, total - na, range));
    }
  check<T>(ty + "/random_large", sorted_random<T>(rng, 100000, 1u << 20), sorted_random<T>(rng, 37000, 1u << 20));
}

int main() {
  std::mt19937_64 rng(12345);
  cases<uint32_t>("u32", rng);
  cases<uint64_t>("u64", rng);
  cases<double>("f64", rng);
  {
    // signed zeros compare equal: the first input's zero comes first, whatever its sign
    std::vector<double> a, b;
    for (int i = 0; i < 3000; ++i) a.push_back(i % 3 ? -0.0 : 0.0);
    for (int i = 0; i < 2500; ++i) b.push_back(i % 2 ? 0.0 : -0.0);
    std::vector<double> a2 = {-1.0}, b2 = {-1.0};
    a2.insert(a2.end(), a.begin(), a.end());
    a2.push_back(1.0);
    b2.insert(b2.end(), b.begin(), b.end());
    b2.push_back(1.0);
    check<double>("f64/signed_zeros", a2, b2);
    check<double>("f64/signed_zeros_swapped", b2, a2);
  }
  {
    // uint64 keys that collide as doubles stay distinct here: the merge compares the keys themselves
    std::vector<uint64_t> a, b;
    for (uint64_t i = 0; i < 3000; ++i) a.push_back((1ull << 60) + 2 * i);
    for (uint64_t i = 0; i < 3000; ++i) b.push_back((1ull << 60) + 2 * i + 1);
    check<uint64_t>("u64/interleaved_beyond_2e53", a, b);
  }
  std::printf("failures=%d\n", failures);
  return failures ? 1 : 0;
}
