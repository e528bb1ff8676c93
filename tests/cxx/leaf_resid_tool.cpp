// Test tool for rmi_b200/csrc/leaf_resid.cuh (no GPU): the chunk bounds a linear leaf's fit records, on adversarial
// leaves, against the true per-chunk maximum of the computed forward-pass error.
//   leaf_resid_tool
// Restates what k_leaf computes per item (t = RN(x - x0), r = RN(j - bt t), the float records) and per key of the
// forward pass (clamp(floor(RN(beta x + alpha)), 0, n) against the key's global offset), then checks, for every chunk,
// that resid_chunk_bound_f is not below the chunk's true maximum, and that the best-first evaluation of
// resid_max_error finds the leaf's maximum.  Prints one line per case family:
//   family=<name> leaves=<l> chunks=<c> evaluated=<e> tight=<t> fail=<f>
// (tight: chunks whose bound equals their true maximum) and exits 1 if any bound fails.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <map>
#include <string>
#include <vector>

#include "../../rmi_b200/csrc/leaf_resid.cuh"

using u64 = uint64_t;

namespace {

u64 rng_state = 0x9e3779b97f4a7c15ull;
u64 next_u64() {   // splitmix64
  u64 z = (rng_state += 0x9e3779b97f4a7c15ull);
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

// __double2ull_rd, then the clamp to n of leaf_predict_clamped (the 32-bit form saturates at 2^32 - 1 >= n first,
// which the clamp makes equivalent)
u64 predict_clamped(double alpha, double beta, double x, u64 n) {
  const double p = std::fma(beta, x, alpha);
  u64 v;
  if (!(p > 0.0)) v = 0;                        // negative, -0, NaN: the kernel's linear leaves never see NaN
  else if (p >= 0x1p64) v = ~0ull;
  else v = (u64)std::floor(p);
  return v < n ? v : n;
}

struct Stats { u64 leaves = 0, chunks = 0, evaluated = 0, tight = 0, fail = 0; };
std::map<std::string, Stats> stats;

// One leaf: sorted keys (the training vector, item j at global offset F0 + j), its 16-byte alignment offset `skip`
// (items before the vector in the first piece), keys per chunk `sw`, the provisional slope bt (the kernel takes the
// line through the first and last item; any slope must give valid bounds) and a fitted line (alpha, beta).
void check_leaf(const std::string& family, const std::vector<u64>& k, u64 F0, u64 n, int skip, int sw, double bt,
                double alpha, double beta) {
  Stats& s = stats[family];
  s.leaves++;
  const size_t L = k.size();
  const double x0 = (double)k[0];
  const size_t nch = (skip + L + sw - 1) / sw;
  std::vector<double> rmin(nch, INFINITY), rmax(nch, -INFINITY), tlast(nch, 0.0);
  std::vector<u64> truth(nch, 0);
  for (size_t j = 0; j < L; ++j) {
    const size_t c = (skip + j) / sw;
    const double x = (double)k[j];
    const double t = x - x0;
    const double r = std::fma(-bt, t, (double)j);
    rmin[c] = std::fmin(rmin[c], r);
    rmax[c] = std::fmax(rmax[c], r);
    tlast[c] = t;
    const u64 F = F0 + j, p = predict_clamped(alpha, beta, x, n);
    const u64 e = p > F ? p - F : F - p;
    if (e > truth[c]) truth[c] = e;
  }
  const rmi::ResidLeaf lf = rmi::resid_leaf(alpha, beta, x0, bt, (double)F0);
  std::vector<float> U(nch);
  float tl_prev = 0.0f;
  u64 leaf_max = 0;
  for (size_t c = 0; c < nch; ++c) {
    const float tl = rmi::resid_f32_down(tlast[c]);
    const double b = rmi::resid_chunk_bound_f(lf, tl_prev, tl, rmi::resid_f32_down(rmin[c]), rmi::resid_f32_up(rmax[c]));
    tl_prev = tl;
    U[c] = rmi::resid_f32_up(b);
    s.chunks++;
    if (!(b >= (double)truth[c])) {
      s.fail++;
      std::printf("FAIL family=%s chunk=%zu bound=%.17g true=%llu alpha=%a beta=%a bt=%a x0=%a F0=%llu\n", family.c_str(), c,
                  b, (unsigned long long)truth[c], alpha, beta, bt, x0, (unsigned long long)F0);
    }
    if (b == (double)truth[c]) s.tight++;
    if (truth[c] > leaf_max) leaf_max = truth[c];
  }
  // resid_max_error's selection: largest bound first, then only bounds above the running maximum
  u64 got = 0;
  for (;;) {
    float best = -1.0f;
    size_t bc = 0;
    for (size_t c = 0; c < nch; ++c)
      if (U[c] > best) { best = U[c]; bc = c; }
    if (!((double)best > (double)got)) break;
    U[bc] = -1.0f;
    s.evaluated++;
    if (truth[bc] > got) got = truth[bc];
  }
  if (got != leaf_max) {
    s.fail++;
    std::printf("FAIL family=%s best-first max=%llu true=%llu\n", family.c_str(), (unsigned long long)got,
                (unsigned long long)leaf_max);
  }
}

// least-squares line through (x_j, F0 + j), computed in long double and rounded: close to the leaf kernel's fit
void lsq(const std::vector<u64>& k, u64 F0, double& alpha, double& beta) {
  long double mx = 0, my = 0;
  const size_t L = k.size();
  for (size_t j = 0; j < L; ++j) { mx += (long double)(double)k[j]; my += (long double)(F0 + j); }
  mx /= L; my /= L;
  long double sxy = 0, sxx = 0;
  for (size_t j = 0; j < L; ++j) {
    const long double dx = (long double)(double)k[j] - mx;
    sxy += dx * ((long double)(F0 + j) - my);
    sxx += dx * dx;
  }
  beta = sxx > 0 ? (double)(sxy / sxx) : 0.0;
  alpha = sxx > 0 ? (double)(my - (long double)beta * mx) : (double)my;
}

double endpoint_slope(const std::vector<u64>& k) {
  const double x0 = (double)k.front(), xb = (double)k.back();
  return xb > x0 ? (double)(k.size() - 1) / (xb - x0) : 0.0;
}

// every family: the endpoint line and the kernel's fit stand-in, plus fits perturbed by a few ulps and lines far away
void check_all(const std::string& family, const std::vector<u64>& k, u64 F0, u64 n, int sw) {
  const int skip = (int)(next_u64() % (u64)(sw / 8));   // 0 .. KPP - 1 (KPP = sw / 8 keys per 16 bytes)
  double alpha, beta;
  lsq(k, F0, alpha, beta);
  const double bt = endpoint_slope(k);
  check_leaf(family, k, F0, n, skip, sw, bt, alpha, beta);
  for (int d = 1; d <= 4; ++d) {
    check_leaf(family, k, F0, n, skip, sw, bt, std::nextafter(alpha, d & 1 ? INFINITY : -INFINITY),
               std::nextafter(beta, d & 2 ? INFINITY : -INFINITY));
  }
  check_leaf(family + "/beta0", k, F0, n, skip, sw, bt, (double)(F0 + k.size() / 2), 0.0);
  check_leaf(family + "/far", k, F0, n, skip, sw, bt * 7.5 + 1e-9, alpha + 40.0, beta * 0.25);
  check_leaf(family + "/far", k, F0, n, skip, sw, -bt, alpha, beta);
  check_leaf(family + "/far", k, F0, n, skip, sw, 0.0, alpha, beta);
}

std::vector<u64> uniform_keys(u64 lo, u64 span, size_t L) {   // L distinct sorted keys in [lo, lo + span)
  std::vector<u64> k;
  std::map<u64, int> seen;
  while (k.size() < L) {
    const u64 v = lo + (span ? next_u64() % span : 0);
    if (seen.emplace(v, 0).second) k.push_back(v);
  }
  std::sort(k.begin(), k.end());
  return k;
}

}  // namespace

int main() {
  const int SW64 = 16, SW32 = 32;
  // uniform leaves as the headline build makes them (about 190 keys over 2^44), both key widths
  for (int i = 0; i < 400; ++i) {
    const size_t L = 150 + next_u64() % 90;
    const u64 F0 = next_u64() % (200000000ull);
    check_all("uniform64", uniform_keys(next_u64() >> 1, 1ull << 44, L), F0, 200000000ull, SW64);
    check_all("uniform32", uniform_keys(next_u64() % (1ull << 31), 1ull << 22, 2 * L), F0 % 100000000ull, 100001000ull, SW32);
  }
  // the maximum in the first or the last chunk: a gap right after the first key or right before the last
  for (int i = 0; i < 100; ++i) {
    const size_t L = 100 + next_u64() % 150;
    std::vector<u64> k = uniform_keys(1ull << 40, 1ull << 30, L);
    const u64 gap = 1ull << (30 + next_u64() % 6);
    if (i & 1) for (size_t j = 1; j < L; ++j) k[j] += gap;
    else k[L - 1] += gap;
    check_all(i & 1 ? "max_first" : "max_last", k, 1000 + i, 1ull << 33, SW64);
  }
  // ties: equally spaced keys with the same bump in every chunk, so every chunk holds the leaf's maximum
  for (int i = 0; i < 100; ++i) {
    const size_t L = 64 + 16 * (next_u64() % 12);
    const u64 step = 1 + next_u64() % 100000, bump = step * (1 + next_u64() % 5);
    std::vector<u64> k(L);
    for (size_t j = 0; j < L; ++j) k[j] = (1ull << 36) + j * step * 8 + ((j % 16) == 7 ? bump : 0);
    check_all("ties", k, next_u64() % (1ull << 32), 1ull << 33, SW64);
  }
  // keys near 2^64 whose doubles collide (2048 integers per double): runs of equal doubles, some leaves entirely one
  for (int i = 0; i < 200; ++i) {
    const size_t L = 2 + next_u64() % 250;
    const u64 hi = ~0ull - (next_u64() % 20000);
    std::vector<u64> k = uniform_keys(hi - 3 * L - next_u64() % 6000, 3 * L, L);
    check_all("collide64", k, (1ull << 32) + i, (1ull << 33), SW64);
    const double bt = 1.0 / 2048.0 * (1 + (i % 3));   // lines through colliding keys: the kernel never has one
    double a, b;
    lsq(k, 77, a, b);
    check_leaf("collide64/slope", k, 77, 1ull << 20, 0, SW64, bt, a, b);
  }
  // leaves that cross a power of two (where the spacing of doubles doubles, or integers stop being exact)
  const int pows[] = {32, 40, 52, 53, 54, 63};
  for (int p : pows) {
    for (int i = 0; i < 40; ++i) {
      const size_t L = 20 + next_u64() % 230;
      const u64 span = (p >= 52 ? (1ull << (p - 40)) : 1ull << 12) * L;
      std::vector<u64> k = uniform_keys((1ull << p) - span / 2, span, L);
      check_all("pow2_" + std::to_string(p), k, next_u64() % (1ull << 34), 1ull << 35, SW64);
    }
  }
  // one-key and two-key leaves, and a constant model over a long leaf
  for (int i = 0; i < 100; ++i) {
    const size_t L = 1 + (i % 2);
    std::vector<u64> k = uniform_keys(next_u64() >> 2, 1ull << 20, L);
    check_all("tiny", k, next_u64() % 1000000, 1000000 + 4, SW64);
    std::vector<u64> kl = uniform_keys(next_u64() >> 2, 1ull << 40, 200);
    check_leaf("beta0_long", kl, 5000, 1ull << 20, 1, SW64, endpoint_slope(kl), 5000.0 + i, 0.0);
  }
  // predictions clamped at 0 and at n: lines that put the leaf's keys far outside [0, n]
  for (int i = 0; i < 100; ++i) {
    std::vector<u64> k = uniform_keys(1ull << 50, 1ull << 38, 180);
    double a, b;
    lsq(k, 1000, a, b);
    check_leaf("clamped", k, 1000, 1000 + k.size(), 0, SW64, endpoint_slope(k), a - 5000.0 * (i % 3), b * (1 + (i % 5)));
  }
  u64 fails = 0;
  for (const auto& kv : stats) {
    const Stats& s = kv.second;
    std::printf("family=%s leaves=%llu chunks=%llu evaluated=%llu tight=%llu fail=%llu\n", kv.first.c_str(),
                (unsigned long long)s.leaves, (unsigned long long)s.chunks, (unsigned long long)s.evaluated,
                (unsigned long long)s.tight, (unsigned long long)s.fail);
    fails += s.fail;
  }
  return fails ? 1 : 0;
}
