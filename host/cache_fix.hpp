// cache_fix.hpp — the `--bounded <line_size>` pre-pass: an error-bounded linear spline over the
// key -> offset function whose prediction always lands in the correct cache line
// (line = offset / line_size).  CPU-side restatement of rmi_lib/src/cache_fix.rs
// (Spline :5-44, SplineFit :46-104, cache_fix :106-150) and of train_bounded
// (rmi_lib/src/train/mod.rs:156-184).  The fit is the reference's greedy scan on one host core
// (every accepted point is re-checked against the whole current segment): rmi_cache_fix's CPU
// path, and the reference the device scan (kernels_cachefix.cu, rmi_cache_fix_device) is
// tested against knot for knot.  The device scan rests on a property of this code: the knot
// after a knot depends on that knot alone (DESIGN.md section 12).  The output, the spline's
// knots, is a sorted duplicate-free key array that then goes through the ordinary GPU build
// (rmi_train) as the data set.
#pragma once
#include <cmath>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

namespace rmihost {

using SplinePoint = std::pair<uint64_t, uint64_t>;   // (key, offset)

namespace cachefix_detail {

// Rust's saturating `f64 as usize` (NaN -> 0)
inline uint64_t f64_to_usize(double v) {
  if (!(v == v) || v <= 0.0) return 0;
  if (v >= 18446744073709551615.0) return UINT64_MAX;
  return (uint64_t)v;
}

struct Spline {   // cache_fix.rs:5-44
  uint64_t from_x, from_y, to_x, to_y;
  uint64_t predict(uint64_t inp) const {   // :36-43 (release build: the subtraction wraps)
    double v0 = (double)from_y, v1 = (double)to_y;
    double t = (double)(inp - from_x) / (double)(to_x - from_x);
    return f64_to_usize(std::fma(1.0 - t, v0, t * v1));
  }
};

struct SplineFit {   // :46-104
  bool has = false;
  Spline spline{};
  std::vector<SplinePoint> curr;
  uint64_t line;
  explicit SplineFit(uint64_t line_size) : line(line_size) {}

  bool check(const Spline& s) const {   // :96-103
    for (const auto& pt : curr)
      if (s.predict(pt.first) / line != pt.second / line) return false;
    return true;
  }
  // returns true and sets `out` when a knot is emitted
  bool add_point(SplinePoint p, SplinePoint& out) {   // :62-88
    if (!has) { has = true; spline = Spline{p.first, p.second, p.first, p.second}; out = p; return true; }
    // with_new_dest (:23-30) asserts the destination is not before the segment's start
    if (p.first < spline.from_x)
      throw std::runtime_error("When source x is " + std::to_string(spline.from_x) + ", cannot set dest x to " + std::to_string(p.first));
    if (p.second < spline.from_y) throw std::runtime_error("assertion failed: dest.1 >= self.from_y");
    Spline proposed{spline.from_x, spline.from_y, p.first, p.second};
    curr.emplace_back(spline.to_x, spline.to_y);
    if (check(proposed)) { spline = proposed; return false; }
    SplinePoint prev{spline.to_x, spline.to_y};
    if (!(p.first > prev.first)) throw std::runtime_error("new point does not advance past the previous point");   // :79-81
    spline = Spline{prev.first, prev.second, p.first, p.second};
    curr.clear();
    curr.push_back(p);
    out = prev;
    return true;
  }
};

}  // namespace cachefix_detail

// cache_fix.rs:106-150 on a sorted u64 key array.  The stream is data.iter_unique()
// (models/mod.rs:187-231, :286-288): one (key, index of its first occurrence) per distinct key.
inline std::vector<SplinePoint> cache_fix(const uint64_t* keys, uint64_t n, uint64_t line_size) {
  using namespace cachefix_detail;
  if (!(n > line_size)) throw std::runtime_error("Cannot apply a cachefix with fewer items than the line size");
  if (line_size == 0) throw std::runtime_error("attempt to divide by zero");
  SplineFit fit(line_size);
  std::vector<SplinePoint> spline;
  SplinePoint knot;
  uint64_t last_key = 0;
  for (uint64_t i = 0; i < n; ++i) {
    if (i > 0 && keys[i] == keys[i - 1]) continue;   // DedupIter: the first item of each run of equal keys
    const uint64_t key = keys[i], off = i;
    const uint64_t km = key - 1;                     // minus_epsilon, wrapping in a release build
    if (!(km >= last_key))
      throw std::runtime_error("key: " + std::to_string(key) + " last key: " + std::to_string(last_key) + ", key - e: " + std::to_string(km));
    if (km != last_key && fit.add_point({km, off}, knot)) spline.push_back(knot);
    if (fit.add_point({key, off}, knot)) spline.push_back(knot);
    last_key = key;
  }
  if (fit.has) spline.emplace_back(fit.spline.to_x, fit.spline.to_y);   // finish(), :91-93
  return spline;
}

}  // namespace rmihost
