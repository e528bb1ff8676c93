// libm's fma over arrays, for the tests' restatement of the bounded lookup (one rounding, f64::mul_add).
// Built with -ffp-contract=off and without -mfma, so every element goes through the C library's fma.
#include <cmath>
#include <cstddef>

extern "C" void fma_batch(const double* a, const double* b, const double* c, double* out, size_t n) {
  for (size_t i = 0; i < n; ++i) out[i] = std::fma(a[i], b[i], c[i]);
}
