// spline.cuh — closed-form part of the cubic spline model (reference
// rmi_lib/src/models/cubic_spline.rs:38-101), shared by the single-GPU top fit
// (kernels_top.cu: k_spline_prepare) and the range-partitioned one (kernels_shard.cu), which
// gathers the four defining points from different ranks.
#pragma once
#include "rust_math.cuh"

namespace rmi {

// scale(v, min, max) = (v - min) / (max - min)          cubic_spline.rs:14-16
__device__ __forceinline__ double scale3(double v, double mn, double mx) {
  return __ddiv_rn(__dadd_rn(v, -mn), __dadd_rn(mx, -mn));
}

// (a, b, c, d) of the monotone cubic Hermite segment through (xmin, ymin), (xmax, ymax) with
//   m1 = slope to (x_next, y_next): the first stream item whose scaled x is > 0   (:46-54)
//   m2 = slope from (x_prev, y_prev): the last raw item whose scaled x is < 1     (:56-65)
// rescaled when m1^2 + m2^2 > 9 (:67-72), expanded into monomial coefficients (:74-101).
// Every operation rounds once, in the reference's order; x^3 goes through a double-double
// cube (rust_math.cuh) in place of libm's powf(3.0).
__device__ __forceinline__ void cubic_from_points(double xmin, double ymin, double xmax, double ymax, double x_next,
                                                  double y_next, double x_prev, double y_prev, double& a, double& b,
                                                  double& c, double& d) {
  double sxn = scale3(x_next, xmin, xmax);
  double syn = scale3(y_next, ymin, ymax);
  double m1 = __ddiv_rn(__dadd_rn(syn, -0.0), __dadd_rn(sxn, -0.0));
  double sxp = scale3(x_prev, xmin, xmax);
  double syp = scale3(y_prev, ymin, ymax);
  double m2 = __ddiv_rn(__dadd_rn(1.0, -syp), __dadd_rn(1.0, -sxp));
  double ss = __dadd_rn(__dmul_rn(m1, m1), __dmul_rn(m2, m2));
  if (ss > 9.0) {
    double tau = __ddiv_rn(3.0, __dsqrt_rn(ss));
    m1 = __dmul_rn(m1, tau);
    m2 = __dmul_rn(m2, tau);
  }
  double d3 = cube_dd(__dadd_rn(xmax, -xmin));
  // (m1 + m2 - 2) / d3
  a = __ddiv_rn(__dadd_rn(__dadd_rn(m1, m2), -2.0), d3);
  // -(xmax*(2*m1 + m2 - 3) + xmin*(m1 + 2*m2 - 3)) / d3
  double t1 = __dmul_rn(xmax, __dadd_rn(__dadd_rn(__dmul_rn(2.0, m1), m2), -3.0));
  double t2 = __dmul_rn(xmin, __dadd_rn(__dadd_rn(m1, __dmul_rn(2.0, m2)), -3.0));
  b = __ddiv_rn(-__dadd_rn(t1, t2), d3);
  // (m1*xmax^2 + m2*xmin^2 + xmax*xmin*(2*m1 + 2*m2 - 6)) / d3
  double xmax2 = __dmul_rn(xmax, xmax), xmin2 = __dmul_rn(xmin, xmin);
  double u1 = __dmul_rn(m1, xmax2), u2 = __dmul_rn(m2, xmin2);
  double u3 = __dmul_rn(__dmul_rn(xmax, xmin), __dadd_rn(__dadd_rn(__dmul_rn(2.0, m1), __dmul_rn(2.0, m2)), -6.0));
  c = __ddiv_rn(__dadd_rn(__dadd_rn(u1, u2), u3), d3);
  // -xmin*(m1*xmax^2 + xmax*xmin*(m2 - 3) + xmin^2) / d3
  double v2 = __dmul_rn(__dmul_rn(xmax, xmin), __dadd_rn(m2, -3.0));
  double inner = __dadd_rn(__dadd_rn(u1, v2), xmin2);
  d = __ddiv_rn(__dmul_rn(-xmin, inner), d3);
  double dy = __dadd_rn(ymax, -ymin);
  a = __dmul_rn(a, dy); b = __dmul_rn(b, dy); c = __dmul_rn(c, dy); d = __dmul_rn(d, dy);
  d = __dadd_rn(d, ymin);
}

// The cache-fix spline's interpolation between (x0, y0) and (x1, y1) at x (cache_fix.rs:36-43, and the generated
// spline lookup, codegen.rs:410-437): t = (x - x0) / (x1 - x0) with wrapping u64 subtractions,
// fma(1 - t, y0, t * y1), then Rust's saturating `as u64` (NaN -> 0).  Shared by the bounded lookup
// (kernels_lookup.cu) and the device cache-fix scan (kernels_cachefix.cu), which must agree with the host bit for bit.
__device__ __forceinline__ u64 cache_fix_interp(u64 x, u64 x0, u64 y0, u64 x1, u64 y1) {
  const double t = __ddiv_rn(__ull2double_rn(x - x0), __ull2double_rn(x1 - x0));
  return f64_to_u64_sat(__fma_rn(__dsub_rn(1.0, t), __ull2double_rn(y0), __dmul_rn(t, __ull2double_rn(y1))));
}

}  // namespace rmi
