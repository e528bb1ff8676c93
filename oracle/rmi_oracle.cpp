// rmi_oracle.cpp — CPU restatement of learnedsystems/RMI's two-layer build.
//
// THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
// and bench.py's cpu_baseline / --impl reference legs may load this library; the product
// (rmi_b200/csrc, librmi_b200.so) never links, loads or calls anything in oracle/.
//
// Parity status: the reference (Rust) cannot be compiled in this environment (no cargo /
// rustc, no network), and it ships no golden vectors.  The oracle is pinned by
//   * the known-answer vectors of the reference's own (stale) unit tests
//     (tests/golden/reference_kats.json, citing models/*.rs line numbers), and
//   * the reference's integration-test property |lookup(k) - lower_bound(k)| <= err for
//     every key (tests/simple_model_wiki/main.cpp:26-42), checked on synthetic data.
// Byte-level parity of parameters against a run of the real binary is UNPINNED
// ("parity unpinned" for blobs; see DESIGN.md).
//
// Every function cites the reference file:line it restates (paths relative to
// the reference repository's rmi_lib/src/).  Release-build semantics are used throughout (the
// reference's tests build --release, tests/Makefile:20): wrapping integer arithmetic,
// masked shift amounts, saturating float->int `as` casts, no debug_assert, no FP
// contraction (compile with -ffp-contract=off), fused multiply-add only where the
// reference writes mul_add.
//
// Build: see oracle/Makefile  (g++ -O2 -std=c++17 -ffp-contract=off -shared -fPIC).

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <memory>
#include <string>
#include <thread>
#include <utility>
#include <vector>

namespace {

// A reference panic!/assert!/unwrap failure.  The C API turns it into a non-zero return.
struct Panic {
  std::string msg;
};
#define REF_ASSERT(cond, text)   \
  do {                           \
    if (!(cond)) throw Panic{text}; \
  } while (0)

// Rust `f64 as u64` / `as usize`: saturating, NaN -> 0.
inline uint64_t f64_to_u64(double v) {
  if (!(v > 0.0)) return 0;  // NaN, negatives, -0.0, 0.0
  if (v >= 18446744073709551616.0) return UINT64_MAX;
  return (uint64_t)v;
}
// ln at fit time (loglinear's ln y, lognormal's ln x).  Compiled with -DORACLE_FIT_LN_NOISE (a test-only variant,
// never the default build) it is moved by -1, 0 or +1 ulp, chosen by a hash of the argument: how far the fitted
// parameters move when two libms' ln disagree in the last place.
inline double fit_ln(double x) {
  double l = std::log(x);
#ifdef ORACLE_FIT_LN_NOISE
  if (std::isfinite(l) && l != 0.0) {
    uint64_t b;
    std::memcpy(&b, &x, sizeof b);
    const int step = (int)(((b * 0x9E3779B97F4A7C15ull) >> 40) % 3) - 1;
    if (step) l = std::nextafter(l, step > 0 ? INFINITY : -INFINITY);
  }
#endif
  return l;
}

// Rust f64::max(a, b): returns the non-NaN operand if one is NaN.
inline double rust_fmax(double a, double b) {
  if (std::isnan(a)) return b;
  if (std::isnan(b)) return a;
  return a > b ? a : b;
}
// Rust release-mode shifts mask the shift amount to the bit width (wrapping_shl/shr).
inline uint64_t shl64(uint64_t x, unsigned s) { return x << (s & 63u); }
inline uint64_t shr64(uint64_t x, unsigned s) { return x >> (s & 63u); }

// models/mod.rs:372-466  ModelInput
struct ModelInput {
  bool is_float;
  uint64_t i;
  double f;
  double as_float() const { return is_float ? f : (double)i; }          // mod.rs:421-426
  uint64_t as_int() const { return is_float ? f64_to_u64(f) : i; }       // mod.rs:428-433
};

// models/mod.rs:65-111  TrainingKey for u64 / u32 / f64
template <class T> struct KeyTraits;
template <> struct KeyTraits<uint64_t> {
  static uint64_t minus_epsilon(uint64_t k) { return k - 1; }   // wraps in release
  static uint64_t plus_epsilon(uint64_t k) { return k + 1; }
  static uint64_t zero_value() { return 0; }
  static uint64_t max_value() { return UINT64_MAX; }
  static double as_float(uint64_t k) { return (double)k; }
  static uint64_t as_uint(uint64_t k) { return k; }
  static ModelInput to_model_input(uint64_t k) { return ModelInput{false, k, 0.0}; }
};
template <> struct KeyTraits<uint32_t> {
  static uint32_t minus_epsilon(uint32_t k) { return (uint32_t)(k - 1u); }
  static uint32_t plus_epsilon(uint32_t k) { return (uint32_t)(k + 1u); }
  static uint32_t zero_value() { return 0; }
  static uint32_t max_value() { return UINT32_MAX; }
  static double as_float(uint32_t k) { return (double)k; }
  static uint64_t as_uint(uint32_t k) { return (uint64_t)k; }
  static ModelInput to_model_input(uint32_t k) { return ModelInput{false, (uint64_t)k, 0.0}; }
};
template <> struct KeyTraits<double> {
  static double minus_epsilon(double k) { return k - DBL_EPSILON; }
  static double plus_epsilon(double k) { return k + DBL_EPSILON; }
  static double zero_value() { return 0.0; }
  static double max_value() { return DBL_MAX; }
  static double as_float(double k) { return k; }
  static uint64_t as_uint(double k) { return f64_to_u64(k); }
  static ModelInput to_model_input(double k) { return ModelInput{true, 0, k}; }
};

// models/mod.rs:233-317  RMITrainingData: a provider of (key, offset) pairs plus `scale`.
// offs == nullptr means offset = index (the mmap adapters, src/load.rs:26-95).
template <class T> struct Data {
  const T* keys = nullptr;
  const uint64_t* offs = nullptr;
  size_t n = 0;
  double scale = 1.0;

  size_t len() const { return n; }
  size_t raw_off(size_t i) const { return offs ? (size_t)offs[i] : i; }
  // mod.rs:238-250  map_scale!
  size_t map_scale(size_t off) const {
    bool use_sf = std::fabs(scale - 1.0) > DBL_EPSILON;
    return use_sf ? (size_t)f64_to_u64((double)off * scale) : off;
  }
  // mod.rs:268-274  get / get_key: raw provider item, scaled, NOT duplicate-fixed.
  std::pair<T, size_t> get(size_t i) const { return {keys[i], map_scale(raw_off(i))}; }
  T get_key(size_t i) const { return keys[i]; }
};

// mod.rs:143-185 FixDupsIter wrapped by map_scale! (mod.rs:276-283 iter / iter_model_input).
// NB (mod.rs:180): when the inner iterator is exhausted the adaptor returns
// `self.last_item.take()`, i.e. it yields ONE EXTRA trailing item equal to the last
// distinct (key, first offset) pair before terminating.  Every consumer that drains the
// iterator therefore sees len()+1 items; consumers behind .take(k) do not.
// Test knob (default = today's reference behaviour).  With the repeat switched off the
// adaptor behaves like a plain duplicate-fixing iterator; the reference's stale unit tests
// predate FixDupsIter, and one of them (loglinear, linear.rs:217-224) only holds without it.
static bool g_trailing_repeat = true;

template <class T> struct FixDupsIter {
  const Data<T>& d;
  size_t i = 0;
  bool has_last = false;
  T last_key{};
  size_t last_off = 0;
  explicit FixDupsIter(const Data<T>& dd) : d(dd) {}
  bool next(T& k, size_t& y) {
    if (!has_last) {
      if (i >= d.n) return false;
      last_key = d.keys[i];
      last_off = d.raw_off(i);
      ++i;
      has_last = true;
      k = last_key;
      y = d.map_scale(last_off);
      return true;
    }
    if (i < d.n) {
      T ck = d.keys[i];
      size_t co = d.raw_off(i);
      ++i;
      if (ck == last_key) {
        k = ck;
        y = d.map_scale(last_off);
      } else {
        last_key = ck;
        last_off = co;
        k = ck;
        y = d.map_scale(co);
      }
      return true;
    }
    // inner iterator exhausted: last_item.take()
    if (!g_trailing_repeat) return false;
    has_last = false;
    k = last_key;
    y = d.map_scale(last_off);
    return true;
  }
};

// ---------------------------------------------------------------------------------------
// Models (models/mod.rs:730-764 Model trait)
// ---------------------------------------------------------------------------------------
enum Kind {
  K_LINEAR = 0,
  K_ROBUST_LINEAR = 1,
  K_LINEAR_SPLINE = 2,
  K_CUBIC = 3,
  K_LOGLINEAR = 4,
  K_NORMAL = 5,
  K_LOGNORMAL = 6,
  K_RADIX = 7,
  K_RADIX_TABLE = 8,
  K_BRADIX = 9,
  K_HISTOGRAM = 10
};

struct Model {
  Kind kind;
  std::vector<double> fp;      // float params, in params() order
  std::vector<uint64_t> ip;    // int params, in params() order
  std::vector<uint32_t> t32;   // RadixTable hint table
  std::vector<uint64_t> a1;    // histogram: radix index
  std::vector<uint64_t> a2;    // histogram: pivots
  bool high = true;            // bradix variant
  uint8_t table_bits = 0;      // RadixTable

  explicit Model(Kind k) : kind(k) {}

  // models/normal.rs:12-26, linear.rs:156-166
  static double exp1(double inp) {
    double x = inp;
    x = 1.0 + x / 64.0;
    x *= x; x *= x; x *= x; x *= x; x *= x; x *= x;
    return x;
  }
  static double phi(double x) { return 1.0 / (1.0 + exp1(-1.65451 * x)); }

  bool float_valued() const { return kind <= K_LOGNORMAL; }

  double predict_to_float(const ModelInput& in) const {
    switch (kind) {
      case K_LINEAR:          // linear.rs:87-90
      case K_ROBUST_LINEAR:   // linear.rs:264-267
      case K_LINEAR_SPLINE:   // linear_spline.rs:50-53
        return std::fma(fp[1], in.as_float(), fp[0]);
      case K_CUBIC: {         // cubic_spline.rs:140-151
        double val = in.as_float();
        double v1 = std::fma(fp[0], val, fp[1]);
        double v2 = std::fma(v1, val, fp[2]);
        return std::fma(v2, val, fp[3]);
      }
      case K_LOGLINEAR:       // linear.rs:177-180
        return exp1(std::fma(fp[1], in.as_float(), fp[0]));
      case K_NORMAL:          // normal.rs:89-92
        return phi((in.as_float() - fp[0]) / fp[1]) * fp[2];
      case K_LOGNORMAL: {     // normal.rs:163-167
        double data = in.as_float();
        return phi((rust_fmax(std::log(data), 0.0) - fp[0]) / fp[1]) * fp[2];
      }
      default:                // mod.rs:731-733
        return (double)predict_to_int(in);
    }
  }

  uint64_t predict_to_int(const ModelInput& in) const {
    switch (kind) {
      case K_RADIX: {         // radix.rs:43-50
        uint64_t as_int = in.as_int();
        return shr64(shl64(as_int, (unsigned)ip[0]), (unsigned)(uint8_t)(64 - (uint8_t)ip[1]));
      }
      case K_RADIX_TABLE: {   // radix.rs:123-132
        uint64_t as_int = in.as_int();
        uint8_t prefix = (uint8_t)ip[0];
        uint8_t bits = table_bits;
        uint8_t num_bits = (prefix + bits > 64) ? 0 : (uint8_t)(64 - (prefix + bits));
        uint64_t res = shr64(shr64(shl64(as_int, prefix), prefix), num_bits);
        return (uint64_t)t32[(size_t)res];
      }
      case K_BRADIX: {        // balanced_radix.rs:101-113
        uint64_t as_int = in.as_int();
        uint64_t res = shr64(shl64(as_int, (unsigned)ip[0]), (unsigned)(uint8_t)(64 - (uint8_t)ip[1]));
        uint64_t clamp = ip[2];
        if (high) return std::min(res, clamp);
        return res < clamp ? 0 : res - clamp;
      }
      case K_HISTOGRAM: {     // histogram.rs:57-61 (superslice upper_bound - 1, wrapping)
        uint64_t val = in.as_int();
        size_t ub = (size_t)(std::upper_bound(a2.begin(), a2.end(), val) - a2.begin());
        return (uint64_t)(ub - 1);
      }
      default:                // mod.rs:735-737
        return f64_to_u64(rust_fmax(0.0, std::floor(predict_to_float(in))));
    }
  }

  bool needs_bounds_check() const {
    // cubic_spline.rs:184, radix.rs:75,164, balanced_radix.rs:164, histogram.rs:103
    return !(kind == K_CUBIC || kind == K_RADIX || kind == K_RADIX_TABLE || kind == K_BRADIX ||
             kind == K_HISTOGRAM);
  }
  bool must_be_top() const {
    // radix.rs:78, balanced_radix.rs:167, histogram.rs:102 (RadixTable: None, radix.rs:167)
    return kind == K_RADIX || kind == K_BRADIX || kind == K_HISTOGRAM;
  }
  bool set_to_constant_model(uint64_t c) {
    switch (kind) {
      case K_LINEAR:          // linear.rs:116-119
      case K_ROBUST_LINEAR:   // linear.rs:293-296
      case K_LINEAR_SPLINE:   // linear_spline.rs:79-82
        fp[0] = (double)c; fp[1] = 0.0; return true;
      case K_CUBIC:           // cubic_spline.rs:188-191
        fp[0] = 0.0; fp[1] = 0.0; fp[2] = 0.0; fp[3] = (double)c; return true;
      default:                // mod.rs:761-763
        return false;
    }
  }
};

// models/linear.rs:12-59  slr over a stream of (x, y)
struct Slr {
  double mean_x = 0.0, mean_y = 0.0, c = 0.0, m2 = 0.0;
  uint64_t n = 0;
  uint64_t data_size = 0;
  inline void push(double x, double y) {
    n += 1;
    double dx = x - mean_x;
    mean_x += dx / (double)n;
    mean_y += (y - mean_y) / (double)n;
    c += dx * (y - mean_y);
    double dx2 = x - mean_x;
    m2 += dx * dx2;
    data_size += 1;
  }
  std::pair<double, double> finish() const {
    if (data_size == 0) return {0.0, 0.0};
    if (data_size == 1) return {mean_y, 0.0};
    double cov = c / (double)(n - 1);
    double var = m2 / (double)(n - 1);
    REF_ASSERT(var >= 0.0, "variance of model was negative");
    if (var == 0.0) return {mean_y, 0.0};
    double beta = cov / var;
    double alpha = mean_y - beta * mean_x;
    return {alpha, beta};
  }
};

// models/linear.rs:79-83  LinearModel::new
template <class T> Model linear_new(const Data<T>& data) {
  Slr s;
  FixDupsIter<T> it(data);
  T k; size_t y;
  while (it.next(k, y)) s.push(KeyTraits<T>::as_float(k), (double)y);
  auto p = s.finish();
  Model m(K_LINEAR);
  m.fp = {p.first, p.second};
  return m;
}

// models/linear.rs:239-260  RobustLinearModel::new
template <class T> Model robust_linear_new(const Data<T>& data) {
  Model m(K_ROBUST_LINEAR);
  size_t total_items = data.len();
  if (total_items == 0) { m.fp = {0.0, 0.0}; return m; }
  size_t bnd = std::max<size_t>(1, (size_t)f64_to_u64((double)total_items * 0.0001));
  REF_ASSERT(bnd * 2 + 1 < data.len(), "robust_linear: bnd*2+1 < data.len() failed");
  Slr s;
  FixDupsIter<T> it(data);
  T k; size_t y;
  size_t skip = bnd, take = data.len() - 2 * bnd;
  for (size_t j = 0; j < skip; ++j) if (!it.next(k, y)) break;
  for (size_t j = 0; j < take; ++j) {
    if (!it.next(k, y)) break;
    s.push(KeyTraits<T>::as_float(k), (double)y);
  }
  auto p = s.finish();
  m.fp = {p.first, p.second};
  return m;
}

// models/linear.rs:61-72, 169-173  loglinear_slr / LogLinearModel::new
template <class T> Model loglinear_new(const Data<T>& data) {
  Slr s;
  FixDupsIter<T> it(data);
  T k; size_t y;
  while (it.next(k, y)) {
    double ly = fit_ln((double)y);
    if (!std::isfinite(ly)) continue;
    s.push(KeyTraits<T>::as_float(k), ly);
  }
  auto p = s.finish();
  Model m(K_LOGLINEAR);
  m.fp = {p.first, p.second};
  return m;
}

// models/linear_spline.rs:13-35  linear_splines
template <class T> std::pair<double, double> linear_splines(const Data<T>& data) {
  if (data.len() == 0) return {0.0, 0.0};
  if (data.len() == 1) return {(double)data.get(0).second, 0.0};
  auto first_pt = data.get(0);
  auto last_pt = data.get(data.len() - 1);
  if (first_pt.first == last_pt.first) return {(double)data.get(0).second, 0.0};
  double slope = ((double)first_pt.second - (double)last_pt.second) /
                 (KeyTraits<T>::as_float(first_pt.first) - KeyTraits<T>::as_float(last_pt.first));
  double intercept = (double)first_pt.second - slope * KeyTraits<T>::as_float(first_pt.first);
  return {intercept, slope};
}
template <class T> Model linear_spline_new(const Data<T>& data) {
  Model m(K_LINEAR_SPLINE);
  auto p = linear_splines(data);
  m.fp = {p.first, p.second};
  return m;
}

// models/cubic_spline.rs:11-15 scale!
inline double scale3(double val, double mn, double mx) { return (val - mn) / (mx - mn); }

// models/cubic_spline.rs:18-101  cubic
template <class T> void cubic_params(const Data<T>& data, double out[4]) {
  if (data.len() == 0) { out[0] = 0.0; out[1] = 0.0; out[2] = 1.0; out[3] = 0.0; return; }
  if (data.len() == 1) { out[0] = out[1] = out[2] = 0.0; out[3] = (double)data.get(0).second; return; }
  {
    T candidate = data.get(0).first;
    bool uniq = false;
    FixDupsIter<T> it(data);
    T k; size_t y;
    while (it.next(k, y)) if (k != candidate) { uniq = true; break; }
    if (!uniq) { out[0] = out[1] = out[2] = 0.0; out[3] = (double)data.get(0).second; return; }
  }
  auto first_pt = data.get(0);
  auto last_pt = data.get(data.len() - 1);
  double xmin = KeyTraits<T>::as_float(first_pt.first), ymin = (double)first_pt.second;
  double xmax = KeyTraits<T>::as_float(last_pt.first), ymax = (double)last_pt.second;
  const double x1 = 0.0, y1 = 0.0, x2 = 1.0, y2 = 1.0;

  double m1;
  {
    FixDupsIter<T> it(data);
    T k; size_t y;
    bool found = false;
    while (it.next(k, y)) {
      if (scale3(KeyTraits<T>::as_float(k), xmin, xmax) > 0.0) { found = true; break; }
    }
    REF_ASSERT(found, "cubic: no point with scaled x > 0 (unwrap on None)");
    double sxn = scale3(KeyTraits<T>::as_float(k), xmin, xmax);
    double syn = scale3((double)y, ymin, ymax);
    m1 = (syn - y1) / (sxn - x1);
  }
  double m2;
  {
    bool found = false;
    std::pair<T, size_t> p{};
    for (size_t idx = data.len(); idx-- > 0;) {
      p = data.get(idx);
      if (scale3(KeyTraits<T>::as_float(p.first), xmin, xmax) < 1.0) { found = true; break; }
    }
    REF_ASSERT(found, "cubic: no point with scaled x < 1 (unwrap on None)");
    double sxp = scale3(KeyTraits<T>::as_float(p.first), xmin, xmax);
    double syp = scale3((double)p.second, ymin, ymax);
    m2 = (y2 - syp) / (x2 - sxp);
  }
  // powf(2.0) is lowered to x*x by LLVM; powf(3.0) stays a libm pow call.
  if (m1 * m1 + m2 * m2 > 9.0) {
    double tau = 3.0 / std::sqrt(m1 * m1 + m2 * m2);
    m1 *= tau;
    m2 *= tau;
  }
  double d3 = std::pow(xmax - xmin, 3.0);
  double a = (m1 + m2 - 2.0) / d3;
  double b = -(xmax * (2.0 * m1 + m2 - 3.0) + xmin * (m1 + 2.0 * m2 - 3.0)) / d3;
  double c = (m1 * (xmax * xmax) + m2 * (xmin * xmin) + xmax * xmin * (2.0 * m1 + 2.0 * m2 - 6.0)) / d3;
  double d = -xmin * (m1 * (xmax * xmax) + xmax * xmin * (m2 - 3.0) + (xmin * xmin)) / d3;
  a *= ymax - ymin;
  b *= ymax - ymin;
  c *= ymax - ymin;
  d *= ymax - ymin;
  d += ymin;
  out[0] = a; out[1] = b; out[2] = c; out[3] = d;
}

// models/cubic_spline.rs:108-136  CubicSplineModel::new
template <class T> Model cubic_new(const Data<T>& data) {
  Model cubic(K_CUBIC);
  cubic.fp.resize(4);
  cubic_params(data, cubic.fp.data());
  Model linear = linear_spline_new(data);
  double our_error = 0.0, lin_error = 0.0;
  FixDupsIter<T> it(data);
  T k; size_t y;
  while (it.next(k, y)) {
    ModelInput x = KeyTraits<T>::to_model_input(k);
    double c_pred = cubic.predict_to_float(x);
    double l_pred = linear.predict_to_float(x);
    our_error += std::fabs(c_pred - (double)y);
    lin_error += std::fabs(l_pred - (double)y);
  }
  if (lin_error < our_error) {
    Model m(K_CUBIC);
    m.fp = {0.0, 0.0, linear.fp[1], linear.fp[0]};
    return m;
  }
  return cubic;
}

// models/normal.rs:28-50 ncdf, :52-76 lncdf
template <class T> Model normal_new(const Data<T>& data, bool lognormal) {
  double scale = -std::numeric_limits<double>::infinity();
  double mean = 0.0, stdev = 0.0;
  double n = (double)data.len();
  T k; size_t y;
  {
    FixDupsIter<T> it(data);
    while (it.next(k, y)) {
      double x = KeyTraits<T>::as_float(k);
      if (lognormal) { double l = fit_ln(x); x = std::isfinite(l) ? l : 0.0; }
      mean += x / n;
      scale = rust_fmax(scale, (double)y);
    }
  }
  {
    FixDupsIter<T> it(data);
    while (it.next(k, y)) {
      double x = KeyTraits<T>::as_float(k);
      if (lognormal) { double l = fit_ln(x); x = std::isfinite(l) ? l : 0.0; }
      stdev += (x - mean) * (x - mean);
    }
  }
  stdev /= n;
  stdev = std::sqrt(stdev);
  Model m(lognormal ? K_LOGNORMAL : K_NORMAL);
  m.fp = {mean, stdev, scale};
  return m;
}

// models/utils.rs:13-21
inline uint8_t num_bits(uint64_t largest_target) {
  uint8_t nbits = 0;
  while (nbits + 1 < 64 && ((uint64_t)1 << (nbits + 1)) - 1 <= largest_target) nbits += 1;
  REF_ASSERT(nbits >= 1, "num_bits: assertion nbits >= 1 failed");
  return nbits;
}
// models/utils.rs:23-36
template <class T> uint8_t common_prefix_size(const Data<T>& data) {
  uint64_t any_ones = 0, no_ones = ~(uint64_t)0;
  FixDupsIter<T> it(data);
  T k; size_t y;
  while (it.next(k, y)) {
    uint64_t v = KeyTraits<T>::to_model_input(k).as_int();
    any_ones |= v;
    no_ones &= v;
  }
  uint64_t any_zeros = ~no_ones;
  uint64_t prefix_bits = any_zeros ^ any_ones;
  uint64_t inv = ~prefix_bits;
  return (uint8_t)(inv == 0 ? 64 : __builtin_clzll(inv));
}
template <class T> uint64_t max_scaled_y(const Data<T>& data) {
  uint64_t largest = 0;
  FixDupsIter<T> it(data);
  T k; size_t y;
  while (it.next(k, y)) largest = std::max<uint64_t>(largest, (uint64_t)y);
  return largest;
}

// models/radix.rs:18-40  RadixModel::new
template <class T> Model radix_new(const Data<T>& data) {
  Model m(K_RADIX);
  if (data.len() == 0) { m.ip = {0, 0}; return m; }
  uint64_t largest_value = max_scaled_y(data);
  uint8_t bits = num_bits(largest_value);
  uint8_t common_prefix = common_prefix_size(data);
  m.ip = {common_prefix, bits};
  return m;
}

// models/radix.rs:90-120  RadixTable::new
template <class T> Model radix_table_new(const Data<T>& data, uint8_t bits) {
  Model m(K_RADIX_TABLE);
  uint8_t prefix = common_prefix_size(data);
  m.table_bits = bits;
  m.ip = {prefix};
  m.t32.assign((size_t)1 << bits, 0);
  uint64_t last_radix = 0;
  FixDupsIter<T> it(data);
  T k; size_t y;
  while (it.next(k, y)) {
    uint64_t x = KeyTraits<T>::to_model_input(k).as_int();
    uint8_t nb = (prefix + bits > 64) ? 0 : (uint8_t)(64 - (prefix + bits));
    uint64_t current_radix = shr64(shr64(shl64(x, prefix), prefix), nb);
    if (current_radix == last_radix) continue;
    REF_ASSERT(current_radix < m.t32.size(), "radix table: current_radix out of range");
    m.t32[(size_t)current_radix] = (uint32_t)y;
    for (uint64_t i = last_radix + 1; i < current_radix; ++i) m.t32[(size_t)i] = (uint32_t)y;
    last_radix = current_radix;
  }
  for (size_t i = (size_t)last_radix + 1; i < m.t32.size(); ++i) m.t32[i] = (uint32_t)m.t32.size();
  return m;
}

// models/balanced_radix.rs:20-37  chi2 (counts are i32: `vec![0; n]` defaults to i32)
template <class T> double bradix_chi2(const Data<T>& data, uint64_t max_bin, const Model& model) {
  std::vector<int32_t> counts((size_t)max_bin, 0);
  FixDupsIter<T> it(data);
  T k; size_t y;
  while (it.next(k, y)) {
    uint64_t p = model.predict_to_int(KeyTraits<T>::to_model_input(k));
    REF_ASSERT(p < counts.size(), "bradix chi2: index out of bounds");
    counts[(size_t)p] = (int32_t)((uint32_t)counts[(size_t)p] + 1u);
  }
  double expected = (double)data.len() / (double)max_bin;
  double sum = 0.0;
  for (int32_t c : counts) {
    double dlt = (double)c - expected;
    sum += (dlt * dlt) / expected;
  }
  return sum;
}
// models/balanced_radix.rs:39-98  bradix / BalancedRadixModel::new
template <class T> Model bradix_new(const Data<T>& data) {
  Model none(K_BRADIX);
  if (data.len() == 0) { none.ip = {0, 0, 0}; none.high = true; return none; }
  uint64_t max_output = max_scaled_y(data);
  uint8_t bits = num_bits(max_output);
  uint8_t common_prefix = common_prefix_size(data);
  double best_score = std::numeric_limits<double>::infinity();
  bool have = false;
  Model best(K_BRADIX);
  for (unsigned tb = bits; tb < std::min<unsigned>(bits + 2u, 64u); ++tb) {
    uint8_t test_bits = (uint8_t)tb;
    uint64_t bits_max = shl64(1, (unsigned)(test_bits + 1)) - 1;
    Model hi(K_BRADIX);
    hi.ip = {common_prefix, test_bits, max_output - 1};
    hi.high = true;
    double hs = bradix_chi2(data, max_output, hi);
    if (hs < best_score) { best_score = hs; best = hi; have = true; }
    Model lo(K_BRADIX);
    lo.ip = {common_prefix, test_bits, max_output - bits_max};  // wraps in release
    lo.high = false;
    double ls = bradix_chi2(data, max_output, lo);
    if (ls < best_score) { best_score = ls; best = lo; have = true; }
  }
  REF_ASSERT(have, "bradix: best_result.unwrap() on None");
  return best;
}

// models/utils.rs:55-102 radix_index (the trailing self-check cannot fire on sorted pivots)
inline std::vector<uint64_t> radix_index(const std::vector<uint64_t>& points, uint8_t nbits) {
  std::vector<uint64_t> ri((size_t)1 << nbits, 0);
  uint64_t last_radix = 0;
  for (size_t idx = 0; idx < points.size(); ++idx) {
    uint64_t radix = points[idx] >> (64 - nbits);
    REF_ASSERT(radix < ri.size(), "radix_index: radix out of range");
    if (radix == last_radix) continue;
    for (uint64_t i = last_radix + 1; i < radix; ++i) ri[(size_t)i] = (uint64_t)idx;
    ri[(size_t)radix] = (uint64_t)idx;
    last_radix = radix;
  }
  for (uint64_t i = last_radix + 1; i < (uint64_t)ri.size(); ++i) ri[(size_t)i] = (uint64_t)points.size();
  ri.push_back((uint64_t)points.size());
  return ri;
}
// models/histogram.rs:20-54
template <class T> Model histogram_new(const Data<T>& data) {
  Model m(K_HISTOGRAM);
  if (data.len() == 0) { m.ip = {0}; return m; }
  size_t num_bins = data.get(data.len() - 1).second;
  REF_ASSERT(num_bins != 0, "histogram: attempt to divide by zero");
  size_t items_per_bin = data.len() / num_bins;
  REF_ASSERT(items_per_bin >= 1, "not enough items for equidepth histogram");
  m.a2.reserve(num_bins);
  for (size_t b = 0; b < num_bins; ++b) m.a2.push_back(KeyTraits<T>::as_uint(data.get_key(b * items_per_bin)));
  m.a1 = radix_index(m.a2, 20);
  m.ip = {(uint64_t)m.a2.size()};
  return m;
}

// train/mod.rs:35-57  train_model
template <class T> Model train_model(const std::string& model_type, const Data<T>& data) {
  if (model_type == "linear") return linear_new(data);
  if (model_type == "robust_linear") return robust_linear_new(data);
  if (model_type == "linear_spline") return linear_spline_new(data);
  if (model_type == "cubic") return cubic_new(data);
  if (model_type == "loglinear") return loglinear_new(data);
  if (model_type == "normal") return normal_new(data, false);
  if (model_type == "lognormal") return normal_new(data, true);
  if (model_type == "radix") return radix_new(data);
  if (model_type == "radix8") return radix_table_new(data, 8);
  if (model_type == "radix18") return radix_table_new(data, 18);
  if (model_type == "radix22") return radix_table_new(data, 22);
  if (model_type == "radix26") return radix_table_new(data, 26);
  if (model_type == "radix28") return radix_table_new(data, 28);
  if (model_type == "bradix") return bradix_new(data);
  if (model_type == "histogram") return histogram_new(data);
  throw Panic{"Unknown model type: " + model_type};
}

// train/mod.rs:59-85 validate.  (Constructing radix-table models on empty data only to read
// their restriction is elided: RadixTable's restriction is None, radix.rs:167.)
inline void validate(const std::vector<std::string>& spec) {
  Data<uint64_t> empty;
  size_t num_layers = spec.size();
  for (size_t idx = 0; idx < spec.size(); ++idx) {
    bool top_only;
    if (spec[idx].rfind("radix", 0) == 0 && spec[idx].size() > 5) {
      // radix8/18/22/26/28 — check the name is known, restriction None
      if (!(spec[idx] == "radix8" || spec[idx] == "radix18" || spec[idx] == "radix22" ||
            spec[idx] == "radix26" || spec[idx] == "radix28"))
        throw Panic{"Unknown model type: " + spec[idx]};
      top_only = false;
    } else {
      top_only = train_model(spec[idx], empty).must_be_top();
    }
    if (top_only) REF_ASSERT(idx == 0, "if used, model type " + spec[idx] + " must be the root model");
    (void)num_layers;
  }
}

// train/two_layer.rs:14-18
inline uint64_t error_between(uint64_t v1, uint64_t v2, uint64_t max_pred) {
  uint64_t p1 = std::min(v1, max_pred), p2 = std::min(v2, max_pred);
  return std::max(p1, p2) - std::min(p1, p2);
}

// train/two_layer.rs:20-99  build_models_from
template <class T>
std::vector<Model> build_models_from(const Data<T>& data, const Model& top_model, const std::string& model_type,
                                     size_t start_idx, size_t end_idx, size_t first_model_idx,
                                     size_t num_models) {
  REF_ASSERT(end_idx > start_idx, "start index was " + std::to_string(start_idx) + " but end index was " +
                                      std::to_string(end_idx));
  REF_ASSERT(end_idx <= data.len(), "end_idx <= data.len()");
  REF_ASSERT(start_idx <= data.len(), "start_idx <= data.len()");
  Data<T> dummy_md;
  std::vector<Model> leaf_models;
  leaf_models.reserve(num_models);
  std::vector<T> sk;         // second_layer_data keys
  std::vector<uint64_t> so;  // second_layer_data offsets
  size_t last_target = first_model_idx;

  auto train_on_vec = [&]() {
    Data<T> container;
    container.keys = sk.data();
    container.offs = so.data();
    container.n = sk.size();
    container.scale = 1.0;
    return train_model(model_type, container);
  };

  FixDupsIter<T> it(data);
  T x; size_t y;
  for (size_t j = 0; j < start_idx; ++j) if (!it.next(x, y)) break;  // .skip(start_idx)
  for (size_t cnt = 0; cnt < end_idx - start_idx; ++cnt) {          // .take(end - start)
    if (!it.next(x, y)) break;
    size_t model_pred = (size_t)top_model.predict_to_int(KeyTraits<T>::to_model_input(x));
    REF_ASSERT(top_model.needs_bounds_check() || model_pred < first_model_idx + num_models,
               "Top model gave an index of " + std::to_string(model_pred) + " which is out of bounds");
    size_t target = std::min(first_model_idx + num_models - 1, model_pred);
    REF_ASSERT(target >= last_target, "assertion failed: target >= last_target");
    if (target > last_target) {
      bool has_last_item = !sk.empty();
      T lk{}; uint64_t lo = 0;
      if (has_last_item) { lk = sk.back(); lo = so.back(); }
      sk.push_back(x); so.push_back((uint64_t)y);
      leaf_models.push_back(train_on_vec());
      for (size_t s = last_target + 1; s < target; ++s) leaf_models.push_back(train_model(model_type, dummy_md));
      REF_ASSERT(leaf_models.size() + first_model_idx == target, "leaf_models.len() + first_model_idx == target");
      sk.clear(); so.clear();
      if (has_last_item) { sk.push_back(lk); so.push_back(lo); }
    }
    sk.push_back(x); so.push_back((uint64_t)y);
    last_target = target;
  }
  REF_ASSERT(!sk.empty(), "assertion failed: !second_layer_data.is_empty()");
  leaf_models.push_back(train_on_vec());
  REF_ASSERT(leaf_models.size() <= num_models, "assertion failed: leaf_models.len() <= num_models");
  for (size_t s = last_target + 1; s < first_model_idx + num_models; ++s)
    leaf_models.push_back(train_model(model_type, dummy_md));
  REF_ASSERT(num_models == leaf_models.size(), "assertion failed: num_models == leaf_models.len()");
  return leaf_models;
}

// train/lower_bound_correction.rs:83-162
template <class T> struct LowerBoundCorrection {
  struct Opt { bool some = false; size_t idx = 0; T key{}; };
  std::vector<Opt> first, last;
  std::vector<std::pair<size_t, T>> next, prev;
  std::vector<uint64_t> run_lengths;

  template <class F> LowerBoundCorrection(F pred_func, uint64_t num_leaf_models, const Data<T>& data) {
    size_t N = (size_t)num_leaf_models;
    first.assign(N, Opt{});
    last.assign(N, Opt{});
    run_lengths.assign(N, 0);
    size_t last_target = 0;
    uint64_t current_run_length = 0;
    REF_ASSERT(data.len() > 0, "get_key(0) on empty data");
    T current_run_key = data.get_key(0);
    FixDupsIter<T> it(data);
    T x; size_t y;
    while (it.next(x, y)) {
      uint64_t leaf_idx = pred_func(x);
      size_t target = (size_t)std::min<uint64_t>(num_leaf_models - 1, leaf_idx);
      if (target == last_target && x == current_run_key) {
        current_run_length += 1;
      } else if (target != last_target || x != current_run_key) {
        run_lengths[last_target] = std::max(run_lengths[last_target], current_run_length);
        current_run_length = 1;
        current_run_key = x;
        last_target = target;
      }
      if (!first[target].some) { first[target].some = true; first[target].idx = y; first[target].key = x; }
      last[target].some = true; last[target].idx = y; last[target].key = x;
    }
    // :30-56 compute_next_for_leaf
    next.assign(N, {0, KeyTraits<T>::zero_value()});
    {
      size_t idx = 0;
      while (idx < N) {
        // find_first_above(:16-26)
        bool found = false; size_t nl = 0;
        if (idx != N - 1) {
          for (size_t i = idx + 1;; ++i) {
            if (first[i].some) { found = true; nl = i; break; }
            if (i == N - 1) break;
          }
        }
        if (found) {
          for (size_t i = idx; i < nl; ++i) next[i] = {first[nl].idx, first[nl].key};
          idx = nl;
        } else {
          for (size_t i = idx; i < N; ++i) next[i] = {data.len(), KeyTraits<T>::max_value()};
          break;
        }
      }
    }
    // :58-80 compute_prev_for_leaf
    prev.assign(N, {0, KeyTraits<T>::zero_value()});
    {
      size_t idx = N - 1;
      while (idx > 0) {
        bool found = false; size_t pl = 0;
        for (size_t i = idx - 1;; --i) {   // find_first_below(:4-14)
          if (last[i].some) { found = true; pl = i; break; }
          if (i == 0) break;
        }
        if (found) {
          for (size_t i = pl + 1; i < idx + 1; ++i) prev[i] = {last[pl].idx, last[pl].key};
          idx = pl;
        } else {
          break;
        }
      }
    }
  }
};

struct TrainedRMI {
  uint64_t num_rmi_rows = 0, num_data_rows = 0;
  double model_avg_error = 0, model_avg_l2_error = 0, model_avg_log2_error = 0, model_max_log2_error = 0;
  uint64_t model_max_error = 0, model_max_error_idx = 0;
  std::vector<uint64_t> last_layer_max_l1s;
  std::vector<uint64_t> leaf_counts;  // (n_j) of two_layer.rs:207-217, kept for parity checks
  std::unique_ptr<Model> top;
  std::vector<Model> leaves;
  uint64_t branching_factor = 0;
  std::string l1_name, l2_name;
  bool could_not_replace = false;
};

// Build a float-parameter top model directly from given parameters (test hook: lets the
// remaining pipeline be compared bit-for-bit when the top fit itself is tolerance-only).
inline Model model_from_params(const std::string& name, const double* p, int np) {
  Kind k;
  int need;
  if (name == "linear") { k = K_LINEAR; need = 2; }
  else if (name == "robust_linear") { k = K_ROBUST_LINEAR; need = 2; }
  else if (name == "linear_spline") { k = K_LINEAR_SPLINE; need = 2; }
  else if (name == "cubic") { k = K_CUBIC; need = 4; }
  else if (name == "loglinear") { k = K_LOGLINEAR; need = 2; }
  else if (name == "normal") { k = K_NORMAL; need = 3; }
  else if (name == "lognormal") { k = K_LOGNORMAL; need = 3; }
  else throw Panic{"l0 override unsupported for model " + name};
  REF_ASSERT(np == need, "l0 override: wrong parameter count");
  Model m(k);
  m.fp.assign(p, p + np);
  return m;
}

// train/two_layer.rs:101-306  train_two_layer
template <class T>
TrainedRMI train_two_layer(Data<T> md, const std::string& layer1_model, const std::string& layer2_model,
                           uint64_t num_leaf_models, const double* l0_override, int n_override, int threads) {
  validate({layer1_model, layer2_model});
  REF_ASSERT(num_leaf_models >= 1, "branching factor must be >= 1");
  size_t num_rows = md.len();
  md.scale = (double)num_leaf_models / (double)num_rows;             // :109
  Model top_model = l0_override ? model_from_params(layer1_model, l0_override, n_override)
                                : train_model(layer1_model, md);    // :110
  md.scale = 1.0;                                                    // :128

  auto top_pred = [&](T k) { return top_model.predict_to_int(KeyTraits<T>::to_model_input(k)); };

  // :131-136 + models/mod.rs:294-309 lower_bound_by
  uint64_t midpoint_model = num_leaf_models / 2;
  size_t split_idx;
  {
    auto less = [&](size_t i) {
      uint64_t model_idx = top_pred(md.get(i).first);
      uint64_t model_target = std::min<uint64_t>(num_leaf_models - 1, model_idx);
      return model_target < midpoint_model;
    };
    size_t size = md.len();
    if (size == 0) split_idx = 0;
    else {
      size_t base = 0;
      while (size > 1) {
        size_t half = size / 2, mid = base + half;
        base = less(mid) ? mid : base;
        size -= half;
      }
      split_idx = base + (less(base) ? 1 : 0);
    }
  }
  if (split_idx > 0 && split_idx < md.len()) {                        // :139-145
    uint64_t key_at = top_pred(md.get_key(split_idx));
    uint64_t key_pr = top_pred(md.get_key(split_idx - 1));
    REF_ASSERT(key_at > key_pr, "assertion failed: key_at > key_pr");
  }

  std::vector<Model> leaf_models;
  if (split_idx >= md.len()) {                                        // :147-150
    leaf_models = build_models_from(md, top_model, layer2_model, 0, md.len(), 0, (size_t)num_leaf_models);
  } else {                                                            // :151-175
    size_t split_idx_target = (size_t)std::min<uint64_t>(num_leaf_models - 1, top_pred(md.get_key(split_idx)));
    size_t first_half_models = split_idx_target;
    size_t second_half_models = (size_t)num_leaf_models - split_idx_target;
    std::vector<Model> hf1, hf2;
    if (threads >= 2) {   // rayon::join
      Panic p2{""}; bool failed2 = false;
      std::thread th([&]() {
        try {
          hf2 = build_models_from(md, top_model, layer2_model, split_idx + 1, md.len(), split_idx_target,
                                  second_half_models);
        } catch (Panic& p) { failed2 = true; p2 = p; }
      });
      Panic p1{""}; bool failed1 = false;
      try {
        hf1 = build_models_from(md, top_model, layer2_model, 0, split_idx, 0, first_half_models);
      } catch (Panic& p) { failed1 = true; p1 = p; }
      th.join();
      if (failed1) throw p1;
      if (failed2) throw p2;
    } else {
      hf1 = build_models_from(md, top_model, layer2_model, 0, split_idx, 0, first_half_models);
      hf2 = build_models_from(md, top_model, layer2_model, split_idx + 1, md.len(), split_idx_target,
                              second_half_models);
    }
    leaf_models = std::move(hf1);
    for (auto& m : hf2) leaf_models.push_back(std::move(m));
  }

  LowerBoundCorrection<T> lb(top_pred, num_leaf_models, md);         // :178-180

  bool could_not_replace = false;                                     // :185-197
  for (size_t idx = 0; idx + 1 < (size_t)num_leaf_models; ++idx) {
    REF_ASSERT(lb.first[idx].some == lb.last[idx].some, "first_key/last_key mismatch");
    if (!lb.last[idx].some) {
      size_t upper_bound = lb.next[idx].first;
      if (!leaf_models[idx].set_to_constant_model((uint64_t)upper_bound)) could_not_replace = true;
    }
  }

  std::vector<std::pair<uint64_t, uint64_t>> l1s((size_t)num_leaf_models, {0, 0});  // :207-217
  {
    FixDupsIter<T> it(md);
    T k; size_t y;
    while (it.next(k, y)) {
      ModelInput x = KeyTraits<T>::to_model_input(k);
      uint64_t leaf_idx = top_model.predict_to_int(x);
      size_t target = (size_t)std::min<uint64_t>(num_leaf_models - 1, leaf_idx);
      uint64_t pred = leaf_models[target].predict_to_int(x);
      uint64_t err = error_between(pred, (uint64_t)y, (uint64_t)md.len());
      l1s[target] = {l1s[target].first + 1, std::max(err, l1s[target].second)};
    }
  }

  for (size_t leaf_idx = 0; leaf_idx < (size_t)num_leaf_models; ++leaf_idx) {       // :227-259
    uint64_t curr_err = l1s[leaf_idx].second;
    uint64_t upper_error;
    {
      size_t idx_of_next = lb.next[leaf_idx].first;
      T key_of_next = lb.next[leaf_idx].second;
      uint64_t pred = leaf_models[leaf_idx].predict_to_int(
          KeyTraits<T>::to_model_input(KeyTraits<T>::minus_epsilon(key_of_next)));
      upper_error = error_between(pred, (uint64_t)idx_of_next + 1, (uint64_t)md.len());
    }
    uint64_t lower_error;
    {
      T first_key_before = lb.prev[leaf_idx].second;
      size_t prev_idx = leaf_idx == 0 ? 0 : leaf_idx - 1;
      size_t first_idx = lb.next[prev_idx].first;
      uint64_t pred = leaf_models[leaf_idx].predict_to_int(
          KeyTraits<T>::to_model_input(KeyTraits<T>::plus_epsilon(first_key_before)));
      lower_error = error_between(pred, (uint64_t)first_idx, (uint64_t)md.len());
    }
    uint64_t new_err = std::max(curr_err, std::max(upper_error, lower_error)) + lb.run_lengths[leaf_idx];
    l1s[leaf_idx] = {l1s[leaf_idx].first, new_err};
  }

  TrainedRMI r;
  // :267-269 max_by_key: the LAST of several equally-maximum elements is returned.
  {
    size_t m_idx = 0; uint64_t m_err = l1s[0].second;
    for (size_t i = 1; i < l1s.size(); ++i)
      if (l1s[i].second >= m_err) { m_err = l1s[i].second; m_idx = i; }
    r.model_max_error = m_err;
    r.model_max_error_idx = m_idx;
  }
  {
    uint64_t s = 0;  // :274-275 (u64 sum, wraps in release)
    for (auto& p : l1s) s += p.first * p.second;
    r.model_avg_error = (double)s / (double)num_rows;
  }
  {
    double s = 0.0;  // :277-279
    for (auto& p : l1s) { double v = (double)(p.first * p.second); s += (v * v) / (double)num_rows; }
    r.model_avg_l2_error = s;
  }
  {
    double s = 0.0;  // :281-282
    for (auto& p : l1s) s += (double)p.first * std::log2((double)(2 * p.second + 2));
    r.model_avg_log2_error = s / (double)num_rows;
  }
  r.model_max_log2_error = std::log2((double)r.model_max_error);     // :284
  r.last_layer_max_l1s.reserve(l1s.size());
  r.leaf_counts.reserve(l1s.size());
  for (auto& p : l1s) { r.leaf_counts.push_back(p.first); r.last_layer_max_l1s.push_back(p.second); }
  r.num_rmi_rows = r.num_data_rows = md.len();
  r.top.reset(new Model(std::move(top_model)));
  r.leaves = std::move(leaf_models);
  r.branching_factor = num_leaf_models;
  r.l1_name = layer1_model;
  r.l2_name = layer2_model;
  r.could_not_replace = could_not_replace;
  return r;
}

// train/mod.rs:100-126  train
template <class T>
TrainedRMI train(const Data<T>& data, const std::string& model_spec, uint64_t branch_factor,
                 const double* l0_override, int n_override, int threads) {
  std::vector<std::string> all_models;
  {
    size_t pos = 0;
    while (true) {
      size_t c = model_spec.find(',', pos);
      if (c == std::string::npos) { all_models.push_back(model_spec.substr(pos)); break; }
      all_models.push_back(model_spec.substr(pos, c - pos));
      pos = c + 1;
    }
  }
  validate(all_models);
  std::string last = all_models.back();
  all_models.pop_back();
  if (all_models.size() == 1) return train_two_layer(data, all_models[0], last, branch_factor, l0_override, n_override, threads);
  throw Panic{"only two-layer RMIs are supported (train/mod.rs:123-125 panic!())"};
}

thread_local std::string g_err;

struct Handle {
  TrainedRMI rmi;
};
struct ModelHandle {
  Model m;
  explicit ModelHandle(Model mm) : m(std::move(mm)) {}
};

template <class T>
Handle* do_train(const void* keys, uint64_t n, const char* spec, uint64_t bf, const double* l0, int nl0, int threads) {
  Data<T> d;
  d.keys = (const T*)keys;
  d.n = (size_t)n;
  auto h = std::make_unique<Handle>();
  h->rmi = train<T>(d, spec, bf, l0, nl0, threads);
  return h.release();
}

template <class T>
ModelHandle* do_model(const char* name, const void* keys, const uint64_t* offs, uint64_t n, double scale) {
  Data<T> d;
  d.keys = (const T*)keys;
  d.offs = offs;
  d.n = (size_t)n;
  d.scale = scale;
  return new ModelHandle(train_model<T>(name, d));
}

}  // namespace

extern "C" {

// key_type: 0 = u64, 1 = u32, 2 = f64 (same numbering as include/rmi_b200.h)
void* rmi_oracle_train(const void* keys, uint64_t n, int key_type, const char* model_spec, uint64_t branch_factor,
                       const double* l0_override, int n_override, int threads) {
  try {
    g_err.clear();
    switch (key_type) {
      case 0: return do_train<uint64_t>(keys, n, model_spec, branch_factor, l0_override, n_override, threads);
      case 1: return do_train<uint32_t>(keys, n, model_spec, branch_factor, l0_override, n_override, threads);
      case 2: return do_train<double>(keys, n, model_spec, branch_factor, l0_override, n_override, threads);
      default: g_err = "bad key type"; return nullptr;
    }
  } catch (Panic& p) {
    g_err = p.msg;
    return nullptr;
  } catch (std::exception& e) {
    g_err = e.what();
    return nullptr;
  }
}
const char* rmi_oracle_last_error() { return g_err.c_str(); }
void rmi_oracle_free(void* h) { delete (Handle*)h; }

// scalars[0..8): n, N, max_error, max_error_idx, l0_kind, l1_kind, l0_high, could_not_replace
// stats[0..4):   avg_error, avg_l2_error, avg_log2_error, max_log2_error
void rmi_oracle_summary(void* hh, uint64_t* scalars, double* stats) {
  auto& r = ((Handle*)hh)->rmi;
  scalars[0] = r.num_rmi_rows;
  scalars[1] = r.branching_factor;
  scalars[2] = r.model_max_error;
  scalars[3] = r.model_max_error_idx;
  scalars[4] = (uint64_t)r.top->kind;
  scalars[5] = (uint64_t)r.leaves[0].kind;
  scalars[6] = r.top->high ? 1 : 0;
  scalars[7] = r.could_not_replace ? 1 : 0;
  stats[0] = r.model_avg_error;
  stats[1] = r.model_avg_l2_error;
  stats[2] = r.model_avg_log2_error;
  stats[3] = r.model_max_log2_error;
}
// sizes[0..5): #float params, #int params, table32 len, a1 len, a2 len   of the top model
void rmi_oracle_l0_sizes(void* hh, uint64_t* sizes) {
  auto& m = *((Handle*)hh)->rmi.top;
  sizes[0] = m.fp.size(); sizes[1] = m.ip.size(); sizes[2] = m.t32.size(); sizes[3] = m.a1.size(); sizes[4] = m.a2.size();
}
void rmi_oracle_l0_get(void* hh, double* fp, uint64_t* ip, uint32_t* t32, uint64_t* a1, uint64_t* a2) {
  auto& m = *((Handle*)hh)->rmi.top;
  if (fp) std::copy(m.fp.begin(), m.fp.end(), fp);
  if (ip) std::copy(m.ip.begin(), m.ip.end(), ip);
  if (t32) std::copy(m.t32.begin(), m.t32.end(), t32);
  if (a1) std::copy(m.a1.begin(), m.a1.end(), a1);
  if (a2) std::copy(m.a2.begin(), m.a2.end(), a2);
}
uint32_t rmi_oracle_l1_params_per_model(void* hh) {
  return (uint32_t)((Handle*)hh)->rmi.leaves[0].fp.size();
}
// params: N x ppm doubles (leaf order), errors: N, counts: N
void rmi_oracle_l1_get(void* hh, double* params, uint64_t* errors, uint64_t* counts) {
  auto& r = ((Handle*)hh)->rmi;
  size_t ppm = r.leaves[0].fp.size();
  if (params)
    for (size_t j = 0; j < r.leaves.size(); ++j)
      for (size_t p = 0; p < ppm; ++p) params[j * ppm + p] = r.leaves[j].fp[p];
  if (errors) std::copy(r.last_layer_max_l1s.begin(), r.last_layer_max_l1s.end(), errors);
  if (counts) std::copy(r.leaf_counts.begin(), r.leaf_counts.end(), counts);
}
// RMI lookup as the generated code does it (codegen.rs:612-718): returns the position
// estimate and writes the leaf's error bound.
uint64_t rmi_oracle_lookup(void* hh, int key_is_float, uint64_t ikey, double fkey, uint64_t* err) {
  auto& r = ((Handle*)hh)->rmi;
  ModelInput in{key_is_float != 0, ikey, fkey};
  uint64_t N = r.branching_factor;
  uint64_t t = std::min<uint64_t>(N - 1, r.top->predict_to_int(in));
  uint64_t p = r.leaves[(size_t)t].predict_to_int(in);
  if (err) *err = r.last_layer_max_l1s[(size_t)t];
  return std::min<uint64_t>(p, r.num_rmi_rows - 1);
}

// Batch form of the lookup above over a key array (the reference's integration tests walk
// every key of the data set, tests/simple_model_wiki/main.cpp:26-42).
void rmi_oracle_lookup_batch(void* hh, const void* keys, uint64_t n, int key_type, uint64_t* pos, uint64_t* err) {
  for (uint64_t i = 0; i < n; ++i) {
    switch (key_type) {
      case 0: pos[i] = rmi_oracle_lookup(hh, 0, ((const uint64_t*)keys)[i], 0.0, &err[i]); break;
      case 1: pos[i] = rmi_oracle_lookup(hh, 0, ((const uint32_t*)keys)[i], 0.0, &err[i]); break;
      default: pos[i] = rmi_oracle_lookup(hh, 1, 0, ((const double*)keys)[i], &err[i]); break;
    }
  }
}

// --- single-model entry points (known-answer tests) -------------------------------------
void* rmi_oracle_model_train(const char* name, const void* keys, const uint64_t* offs, uint64_t n, int key_type,
                             double scale) {
  try {
    g_err.clear();
    switch (key_type) {
      case 0: return do_model<uint64_t>(name, keys, offs, n, scale);
      case 1: return do_model<uint32_t>(name, keys, offs, n, scale);
      case 2: return do_model<double>(name, keys, offs, n, scale);
      default: g_err = "bad key type"; return nullptr;
    }
  } catch (Panic& p) {
    g_err = p.msg;
    return nullptr;
  }
}
void rmi_oracle_model_free(void* m) { delete (ModelHandle*)m; }
uint64_t rmi_oracle_model_predict_int(void* m, int key_is_float, uint64_t ikey, double fkey) {
  return ((ModelHandle*)m)->m.predict_to_int(ModelInput{key_is_float != 0, ikey, fkey});
}
double rmi_oracle_model_predict_float(void* m, int key_is_float, uint64_t ikey, double fkey) {
  return ((ModelHandle*)m)->m.predict_to_float(ModelInput{key_is_float != 0, ikey, fkey});
}
void rmi_oracle_model_sizes(void* mm, uint64_t* sizes) {
  auto& m = ((ModelHandle*)mm)->m;
  sizes[0] = m.fp.size(); sizes[1] = m.ip.size(); sizes[2] = m.t32.size(); sizes[3] = m.a1.size(); sizes[4] = m.a2.size();
}
void rmi_oracle_model_get(void* mm, double* fp, uint64_t* ip, uint32_t* t32, uint64_t* a1, uint64_t* a2) {
  auto& m = ((ModelHandle*)mm)->m;
  if (fp) std::copy(m.fp.begin(), m.fp.end(), fp);
  if (ip) std::copy(m.ip.begin(), m.ip.end(), ip);
  if (t32) std::copy(m.t32.begin(), m.t32.end(), t32);
  if (a1) std::copy(m.a1.begin(), m.a1.end(), a1);
  if (a2) std::copy(m.a2.begin(), m.a2.end(), a2);
}
int rmi_oracle_model_high(void* mm) { return ((ModelHandle*)mm)->m.high ? 1 : 0; }

// models/mod.rs:238-250 map_scale!, exposed for the offset-scaling known-answer test.
uint64_t rmi_oracle_scale_offset(uint64_t off, double scale) {
  Data<uint64_t> d;
  d.scale = scale;
  return (uint64_t)d.map_scale((size_t)off);
}
void rmi_oracle_set_trailing_repeat(int on) { g_trailing_repeat = on != 0; }
uint8_t rmi_oracle_common_prefix_u64(const uint64_t* keys, uint64_t n) {
  Data<uint64_t> d;
  d.keys = keys;
  d.n = (size_t)n;
  return common_prefix_size(d);
}

}  // extern "C"
