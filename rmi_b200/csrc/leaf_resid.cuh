// leaf_resid.cuh — an upper bound on a linear leaf's forward-pass error over one key chunk, from residuals against a
// provisional line that k_leaf (kernels_leaf.cu) records while it fits the leaf.
//
// During the fit every item j of the training vector (key x_j = the key's double, vector offset j = 0, 1, ...) gets
//     t_j = RN(x_j - x0)                 x0: the vector's first item
//     r_j = RN(j - bt * t_j)             one fused multiply-add; bt: the slope of the provisional line
// and each chunk of the copy ring keeps, in float, a lower bound on its r_j (rounded down), an upper bound (rounded
// up) and its last t_j rounded down.  t_j is non-decreasing (x_j is, and rounding is monotone), so the chunk's t_j lie
// in [last t of the previous chunk, last t of this chunk].
//
// After the fit the forward pass needs, for the global offset F_j = F0 + j and the fitted alpha, beta,
//     e_j = | clamp(floor(p_j), 0, n) - F_j |,   p_j = RN(beta * x_j + alpha)   (leaf_predict_clamped)
// F_j lies in [0, n], so the clamp only brings floor(p_j) closer to it: e_j <= |floor(p_j) - F_j| = |floor(d_j)| with
// d_j = p_j - F_j (F_j is an integer).  With tau_j = x_j - x0 and rho_j = j - bt * t_j (both exact),
//     d_j = (p_j - (alpha + beta x_j)) + (alpha + beta x0 - F0) + (beta - bt) t_j + beta (tau_j - t_j) - rho_j,
// so d_j lies in [A + min(db tlo, db thi) - rmax, A + max(db tlo, db thi) - rmin] widened by every rounding, where
// A = alpha + beta x0 - F0 and db = beta - bt.  floor is monotone, so |floor(d_j)| <= max(floor(hi), -floor(lo)).
// The bound is rigorous for the computed prediction, not for real arithmetic; resid_chunk_bound derives its margin.
//
// __host__ __device__ and free of CUDA intrinsics outside __CUDA_ARCH__, so that g++ compiles it
// (tests/cxx/leaf_resid_tool.cpp checks the bound on adversarial leaves).
#pragma once
#include <cmath>

#ifdef __CUDACC__
#define RMI_RESID_HD __host__ __device__ __forceinline__
#else
#define RMI_RESID_HD inline
#endif

namespace rmi {

// float bounds of a double: rounded towards -inf / +inf
RMI_RESID_HD float resid_f32_down(double v) {
#ifdef __CUDA_ARCH__
  return __double2float_rd(v);
#else
  float f = (float)v;
  if ((double)f > v) f = std::nextafter(f, -INFINITY);
  return f;
#endif
}
RMI_RESID_HD float resid_f32_up(double v) {
#ifdef __CUDA_ARCH__
  return __double2float_ru(v);
#else
  float f = (float)v;
  if ((double)f < v) f = std::nextafter(f, INFINITY);
  return f;
#endif
}

// What the chunk bounds of one leaf share.
struct ResidLeaf {
  double A;      // RN(RN(beta * x0 + alpha) - F0)
  double db;     // RN(beta - bt)
  double s0;     // the leaf's part of the margin's sum S (below)
  double sthi;   // the coefficient of thi in S
};

RMI_RESID_HD ResidLeaf resid_leaf(double alpha, double beta, double x0, double bt, double F0) {
  ResidLeaf L;
  const double P = std::fma(beta, x0, alpha);
  L.A = P - F0;
  L.db = beta - bt;
  L.s0 = 2.0 * std::fabs(alpha) + 2.0 * std::fabs(beta) * x0 + std::fabs(P) + std::fabs(F0) + 2.0 * std::fabs(L.A);
  L.sthi = 4.0 * std::fabs(beta) + std::fabs(bt) + 3.0 * std::fabs(L.db);
  return L;
}

// Upper bound on max e_j over the items of a chunk whose computed t_j lie in [tlo, thi] (0 <= tlo <= thi) and whose
// computed r_j lie in [rmin, rmax].  Returns a whole number, or +inf when nothing can be said (non-finite inputs).
//
// The margin.  With u = 2^-53, every rounding is at most u times the magnitude of its exact result:
//   p_j                     u (1+u) (|alpha| + |beta| x_j),  x_j = x0 + tau_j <= x0 + 2 thi   (|tau - t| <= u tau)
//   t_j, times beta         u |beta| tau_j <= 2u |beta| thi
//   r_j                     u |rho_j| <= 2u R,   R = max(|rmin|, |rmax|)
//   P = RN(beta x0 + alpha) u (|alpha| + |beta| x0)
//   A = RN(P - F0)          u (|P| + |F0|)
//   db, times t_j <= thi    u (1+u) (|beta| + |bt|) thi
//   db * tlo, db * thi      u |db| thi
//   the two additions       2u (1+u)^2 (|A| + |db| thi + R)   (each side)
//   the margin's own subtraction / addition: u (|A| + |db| thi + R) (1 + 3u) + u m
// Their sum is at most 1.01 u S with
//   S = 2|alpha| + 2|beta| x0 + |P| + |F0| + 2|A| + thi (4|beta| + |bt| + 3|db|) + 4R,
// and m = 4u S (computed, so itself within 1 +- 16u of that) covers it with room to spare.
RMI_RESID_HD double resid_chunk_bound(const ResidLeaf& L, double tlo, double thi, double rmin, double rmax) {
  const double R = std::fmax(std::fabs(rmin), std::fabs(rmax));
  const double S = L.s0 + L.sthi * thi + 4.0 * R;
  const double m = 0x1p-51 * S;
  const double e1 = L.db * tlo, e2 = L.db * thi;
  const double lo = ((L.A + std::fmin(e1, e2)) - rmax) - m;
  const double hi = ((L.A + std::fmax(e1, e2)) - rmin) + m;
  const double U = std::fmax(std::floor(hi), -std::floor(lo));
  return U >= 0.0 ? U : INFINITY;   // NaN (and, impossibly, a negative bound) -> no bound
}

// The same from a chunk's float record: rmin / rmax rounded outwards, the last t of this chunk (tl) and of the chunk
// before (tl_prev; 0 for the first chunk) rounded down.  t_j is 0 or at least 1 (a difference of whole-number
// doubles) and below 2^65, so RD(t) <= t <= RD(t) (1 + 2^-23), and that product is exact in double.
RMI_RESID_HD double resid_chunk_bound_f(const ResidLeaf& L, float tl_prev, float tl, float rmin, float rmax) {
  return resid_chunk_bound(L, (double)tl_prev, (double)tl * (1.0 + 0x1p-23), (double)rmin, (double)rmax);
}

}  // namespace rmi
