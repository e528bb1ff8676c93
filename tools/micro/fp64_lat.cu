// Microbenchmark (developer tool): FP64 dependent-op latency and the cost of one Welford step
// for a single resident warp on sm_90a.  nvcc -arch=sm_90a -fmad=false -O3 fp64_lat.cu
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k_lat(double* out, long long* cyc, int iters, double a, double b) {
  double v = a;
  long long t0 = clock64();
  for (int i = 0; i < iters; ++i) { v = __dadd_rn(v, b); v = __dadd_rn(v, b); v = __dadd_rn(v, b); v = __dadd_rn(v, b); }
  long long t1 = clock64();
  double w = a;
  for (int i = 0; i < iters; ++i) { w = __fma_rn(w, b, a); w = __fma_rn(w, b, a); w = __fma_rn(w, b, a); w = __fma_rn(w, b, a); }
  long long t2 = clock64();
  double u = a;
  for (int i = 0; i < iters; ++i) { u = __dmul_rn(u, b); u = __dmul_rn(u, b); u = __dmul_rn(u, b); u = __dmul_rn(u, b); }
  long long t3 = clock64();
  // independent: 4 chains of dadd
  double p0 = a, p1 = a + 1, p2 = a + 2, p3 = a + 3;
  for (int i = 0; i < iters; ++i) { p0 = __dadd_rn(p0, b); p1 = __dadd_rn(p1, b); p2 = __dadd_rn(p2, b); p3 = __dadd_rn(p3, b); }
  long long t4 = clock64();
  if (threadIdx.x == 0) { cyc[0] = t1 - t0; cyc[1] = t2 - t1; cyc[2] = t3 - t2; cyc[3] = t4 - t3; }
  out[threadIdx.x] = v + w + u + p0 + p1 + p2 + p3;
}
struct W {
  double mean_x, mean_y, c, m2, nf;
  __device__ __forceinline__ double dv(double a, double rc) const {
    double q0 = __dmul_rn(a, rc); double rem = __fma_rn(-nf, q0, a); return __fma_rn(rem, rc, q0); }
  __device__ __forceinline__ void push(double x, double y, double rc) {
    nf = __dadd_rn(nf, 1.0);
    double dx = __dadd_rn(x, -mean_x);
    mean_x = __dadd_rn(mean_x, dv(dx, rc));
    mean_y = __dadd_rn(mean_y, dv(__dadd_rn(y, -mean_y), rc));
    c = __dadd_rn(c, __dmul_rn(dx, __dadd_rn(y, -mean_y)));
    double dx2 = __dadd_rn(x, -mean_x);
    m2 = __dadd_rn(m2, __dmul_rn(dx, dx2));
  }
};
// the solo loop of kernels_leaf.cu: x / rc per lane, replayed from shuffles
template <int UNROLL>
__global__ void k_solo(const unsigned long long* keys, int n, double* out, long long* cyc) {
  const unsigned FULL = 0xffffffffu;
  int lane = threadIdx.x & 31;
  W w; w.mean_x = w.mean_y = w.c = w.m2 = w.nf = 0.0;
  double idxd = 0.0;
  long long t0 = clock64();
  unsigned long long cur = keys[lane];
  for (int base = 0; base < n; base += 32) {
    unsigned long long nxt = base + 32 + lane < n ? keys[base + 32 + lane] : 0ull;
    double xl = (double)cur;
    double rcl = __drcp_rn(__dadd_rn(w.nf, (double)(lane + 1)));
#pragma unroll UNROLL
    for (int q = 0; q < 32; ++q) {
      double xq = __shfl_sync(FULL, xl, q), rq = __shfl_sync(FULL, rcl, q);
      double yd = idxd;
      idxd = __dadd_rn(idxd, 1.0);
      w.push(xq, yd, rq);
    }
    cur = nxt;
  }
  long long t1 = clock64();
  if (threadIdx.x == 0) cyc[0] = t1 - t0;
  out[threadIdx.x] = w.mean_x + w.mean_y + w.c + w.m2;
}
// variant: x / rc / y staged through shared memory (LDS broadcast instead of 4 SHFL per step)
__global__ void k_solo_smem(const unsigned long long* keys, int n, double* out, long long* cyc) {
  __shared__ double sx[2][32], sr[2][32];
  int lane = threadIdx.x & 31;
  W w; w.mean_x = w.mean_y = w.c = w.m2 = w.nf = 0.0;
  double idxd = 0.0;
  long long t0 = clock64();
  unsigned long long cur = keys[lane];
  int buf = 0;
  for (int base = 0; base < n; base += 32, buf ^= 1) {
    unsigned long long nxt = base + 32 + lane < n ? keys[base + 32 + lane] : 0ull;
    sx[buf][lane] = (double)cur;
    sr[buf][lane] = __drcp_rn(__dadd_rn(w.nf, (double)(lane + 1)));
    __syncwarp();
#pragma unroll 8
    for (int q = 0; q < 32; ++q) {
      double xq = sx[buf][q], rq = sr[buf][q];
      double yd = idxd;
      idxd = __dadd_rn(idxd, 1.0);
      w.push(xq, yd, rq);
    }
    cur = nxt;
  }
  long long t1 = clock64();
  if (threadIdx.x == 0) cyc[0] = t1 - t0;
  out[threadIdx.x] = w.mean_x + w.mean_y + w.c + w.m2;
}

// V1: the x and y chains interleaved in source order; V2: also software-pipelined (the c / m2
// updates of step k are issued inside step k+1's dependency stalls).  Same values, same order.
struct W2 {
  double mean_x, mean_y, c, m2, nf;
  double pdx, px, py; bool have;
  __device__ __forceinline__ void push_v1(double x, double y, double rc) {
    nf = __dadd_rn(nf, 1.0);
    double dx = __dadd_rn(x, -mean_x), dy = __dadd_rn(y, -mean_y);
    double qx = __dmul_rn(dx, rc), qy = __dmul_rn(dy, rc);
    double rx = __fma_rn(-nf, qx, dx), ry = __fma_rn(-nf, qy, dy);
    qx = __fma_rn(rx, rc, qx); qy = __fma_rn(ry, rc, qy);
    mean_x = __dadd_rn(mean_x, qx); mean_y = __dadd_rn(mean_y, qy);
    double dy2 = __dadd_rn(y, -mean_y), dx2 = __dadd_rn(x, -mean_x);
    c = __dadd_rn(c, __dmul_rn(dx, dy2));
    m2 = __dadd_rn(m2, __dmul_rn(dx, dx2));
  }
  // pipelined: call with the previous step's (pdx, px, py) pending
  __device__ __forceinline__ void push_v2(double x, double y, double rc) {
    nf = __dadd_rn(nf, 1.0);
    double dx = __dadd_rn(x, -mean_x), dy = __dadd_rn(y, -mean_y);
    double dy2 = __dadd_rn(py, -mean_y), dx2 = __dadd_rn(px, -mean_x);       // previous step's tail
    double qx = __dmul_rn(dx, rc), qy = __dmul_rn(dy, rc);
    double t1 = __dmul_rn(pdx, dy2), t2 = __dmul_rn(pdx, dx2);
    double rx = __fma_rn(-nf, qx, dx), ry = __fma_rn(-nf, qy, dy);
    c = __dadd_rn(c, t1); m2 = __dadd_rn(m2, t2);
    qx = __fma_rn(rx, rc, qx); qy = __fma_rn(ry, rc, qy);
    mean_x = __dadd_rn(mean_x, qx); mean_y = __dadd_rn(mean_y, qy);
    pdx = dx; px = x; py = y;
  }
  __device__ __forceinline__ void flush() {
    double dy2 = __dadd_rn(py, -mean_y), dx2 = __dadd_rn(px, -mean_x);
    c = __dadd_rn(c, __dmul_rn(pdx, dy2)); m2 = __dadd_rn(m2, __dmul_rn(pdx, dx2));
  }
};
template <int V, int UNROLL>
__global__ void k_solo2(const unsigned long long* keys, int n, double* out, long long* cyc, const double* init) {
  __shared__ double sx[2][32], sr[2][32];
  int lane = threadIdx.x & 31;
  W2 w; w.mean_x = init[lane]; w.mean_y = init[32 + lane]; w.c = init[64 + lane]; w.m2 = init[96 + lane]; w.nf = init[128 + lane];
  // pending "previous step" that contributes exactly zero: pdx = 0
  w.pdx = 0.0; w.px = 0.0; w.py = 0.0;
  double idxd = init[160 + lane];
  long long t0 = clock64();
  unsigned long long cur = keys[lane];
  int buf = 0;
  for (int base = 0; base < n; base += 32, buf ^= 1) {
    unsigned long long nxt = base + 32 + lane < n ? keys[base + 32 + lane] : 0ull;
    sx[buf][lane] = (double)cur;
    sr[buf][lane] = __drcp_rn(__dadd_rn(w.nf, (double)(lane + 1)));
    __syncwarp();
#pragma unroll UNROLL
    for (int q = 0; q < 32; ++q) {
      double xq = sx[buf][q], rq = sr[buf][q];
      double yd = idxd;
      idxd = __dadd_rn(idxd, 1.0);
      if (V == 1) w.push_v1(xq, yd, rq); else w.push_v2(xq, yd, rq);
    }
    cur = nxt;
  }
  if (V == 2) w.flush();
  long long t1 = clock64();
  if (threadIdx.x == 0) cyc[0] = t1 - t0;
  out[threadIdx.x] = w.mean_x + w.mean_y + w.c + w.m2;
}

// V3: lane-pair formulation.  Even lanes run the mean_x chain and odd lanes the mean_y chain in
// the SAME instruction stream (m += RN((v - m) / n)); dx and the new means go to shared memory;
// after 32 steps lane q forms step q's two products, and the serial c / m2 accumulations of one
// batch ride along the next batch's chain loop (even lanes: c, odd lanes: m2).
template <int UNROLL>
__global__ void k_solo3(const unsigned long long* keys, int n, double* out, long long* cyc, const double* init) {
  __shared__ double2 sV[32][2];   // {v, tprev} per (step, half)
  __shared__ double2 sR[32];      // {rc, nf} per step
  __shared__ double sD[32];       // dx per step
  __shared__ double sM[32][2];    // means after the step
  const int lane = threadIdx.x & 31, h = lane & 1;
  double m = init[h], acc = init[64 + h];
  double nf0 = init[128], idxd0 = init[160];
  sV[lane][0].y = 0.0; sV[lane][1].y = 0.0;
  long long t0 = clock64();
  unsigned long long cur = keys[lane];
  for (int base = 0; base < n; base += 32) {
    unsigned long long nxt = base + 32 + lane < n ? keys[base + 32 + lane] : 0ull;
    const double xl = (double)cur, yl = __dadd_rn(idxd0, (double)lane);
    const double nfl = __dadd_rn(nf0, (double)(lane + 1));
    sV[lane][0].x = xl; sV[lane][1].x = yl;
    sR[lane] = make_double2(__drcp_rn(nfl), nfl);
    __syncwarp();
    double2 vt1 = sV[0][h], rn1 = sR[0], vt2 = sV[1][h], rn2 = sR[1];
#pragma unroll UNROLL
    for (int q = 0; q < 32; ++q) {
      const double2 vt = vt1, rn = rn1;
      vt1 = vt2; rn1 = rn2;
      vt2 = sV[(q + 2) & 31][h]; rn2 = sR[(q + 2) & 31];    // two steps ahead of the stores below
      const double d = __dadd_rn(vt.x, -m);
      const double q0 = __dmul_rn(d, rn.x);
      const double r = __fma_rn(-rn.y, q0, d);
      m = __dadd_rn(m, __fma_rn(r, rn.x, q0));
      acc = __dadd_rn(acc, vt.y);
      if (h == 0) sD[q] = d;
      sM[q][h] = m;
    }
    __syncwarp();
    {
      const double dx = sD[lane];
      sV[lane][0].y = __dmul_rn(dx, __dadd_rn(yl, -sM[lane][1]));
      sV[lane][1].y = __dmul_rn(dx, __dadd_rn(xl, -sM[lane][0]));
    }
    nf0 = __dadd_rn(nf0, 32.0); idxd0 = __dadd_rn(idxd0, 32.0);
    cur = nxt;
  }
  __syncwarp();
  for (int q = 0; q < 32; ++q) acc = __dadd_rn(acc, sV[q][h].y);
  long long t1 = clock64();
  if (threadIdx.x == 0) cyc[0] = t1 - t0;
  const double mx = __shfl_sync(0xffffffffu, m, 0), my = __shfl_sync(0xffffffffu, m, 1);
  const double c = __shfl_sync(0xffffffffu, acc, 0), m2 = __shfl_sync(0xffffffffu, acc, 1);
  out[threadIdx.x] = mx + my + c + m2;
}

// dissect the lane-pair loop: F&1 = stores, F&2 = acc chain, F&4 = operands from shared memory
template <int F>
__global__ void k_chain(double* out, long long* cyc, const double* init, int n) {
  __shared__ double2 sV[32][2];
  __shared__ double2 sR[32];
  __shared__ double sD[32];
  __shared__ double sM[32][2];
  const int lane = threadIdx.x & 31, h = lane & 1;
  double m = init[h], acc = init[64 + h];
  sV[lane][0] = make_double2(1.0 + lane, 0.0); sV[lane][1] = make_double2(2.0 + lane, 0.0);
  sR[lane] = make_double2(1.0 / (lane + 1), lane + 1.0);
  __syncwarp();
  double2 cv = sV[lane][h], cr = sR[lane];
  long long t0 = clock64();
  for (int base = 0; base < n; base += 32) {
    double2 vt1 = sV[0][h], rn1 = sR[0], vt2 = sV[1][h], rn2 = sR[1];
    double pd = 0, pm = 0, keepA = 0, keepB = 0;
#pragma unroll (F & 16 ? 32 : 4)
    for (int q = 0; q < 32; ++q) {
      double2 vt = vt1, rn = rn1;
      if (q == 0) { pd = 0; pm = 0; }
      if (F & 4) { vt1 = vt2; rn1 = rn2; vt2 = sV[(q + 2) & 31][h]; rn2 = sR[(q + 2) & 31]; }
      else { vt = cv; rn = cr; }
      const double d = __dadd_rn(vt.x, -m);
      const double q0 = __dmul_rn(d, rn.x);
      const double r = __fma_rn(-rn.y, q0, d);
      m = __dadd_rn(m, __fma_rn(r, rn.x, q0));
      if (F & 2) acc = __dadd_rn(acc, vt.y);
      if ((F & 1) && !(F & 8)) { if (h == 0) sD[q] = d; sM[q][h] = m; }
      if ((F & 1) && (F & 8)) { if (q > 0) { if (h == 0) sD[q - 1] = pd; sM[q - 1][h] = pm; } }
      pd = d; pm = m;
      if (F & 16) { if ((q & 15) == (lane >> 1)) { if (q < 16) keepA = m; else keepB = m; } }
    }
    if (F & 16) { cv.y += __shfl_sync(0xffffffffu, keepA, (lane * 2) & 31) + __shfl_sync(0xffffffffu, keepB, (lane * 2 + 1) & 31); }
    if ((F & 1) && (F & 8)) { if (h == 0) sD[31] = pd; sM[31][h] = pm; }
    if (F & 1) { __syncwarp(); cv.y += sD[lane] + sM[lane][1]; }
  }
  long long t1 = clock64();
  if (threadIdx.x == 0) cyc[0] = t1 - t0;
  out[threadIdx.x] = m + acc + cv.y;
}
int main() {
  double* out; long long* cyc; unsigned long long* keys;
  int n = 1 << 14;
  cudaMalloc(&out, 1024); cudaMallocManaged(&cyc, 64); cudaMallocManaged(&keys, n * 8);
  for (int i = 0; i < n; ++i) keys[i] = 1000ull * i + (i * 7919ull) % 997;
  int iters = 10000;
  for (int rep = 0; rep < 2; ++rep) {
    k_lat<<<1, 32>>>(out, cyc, iters, 1.5, 1.0000001); cudaDeviceSynchronize();
    if (rep) printf("dadd %.2f  dfma %.2f  dmul %.2f  4-indep-dadd(per op) %.2f cycles\n", cyc[0] / (4.0 * iters), cyc[1] / (4.0 * iters),
                    cyc[2] / (4.0 * iters), cyc[3] / (4.0 * iters));
    k_solo<1><<<1, 32>>>(keys, n, out, cyc); cudaDeviceSynchronize();
    if (rep) printf("solo shfl unroll1: %.1f cycles/step\n", (double)cyc[0] / n);
    k_solo<8><<<1, 32>>>(keys, n, out, cyc); cudaDeviceSynchronize();
    if (rep) printf("solo shfl unroll8: %.1f cycles/step\n", (double)cyc[0] / n);
    k_solo<32><<<1, 32>>>(keys, n, out, cyc); cudaDeviceSynchronize();
    if (rep) printf("solo shfl unroll32: %.1f cycles/step\n", (double)cyc[0] / n);
    k_solo_smem<<<1, 32>>>(keys, n, out, cyc); cudaDeviceSynchronize();
    if (rep) printf("solo smem unroll8: %.1f cycles/step\n", (double)cyc[0] / n);
  }
  double* init; cudaMallocManaged(&init, 192 * 8); for (int i = 0; i < 192; ++i) init[i] = 0.0;
  double* o2; cudaMallocManaged(&o2, 1024);
  k_solo_smem<<<1, 32>>>(keys, n, o2, cyc); cudaDeviceSynchronize(); double ref = o2[0];
  k_solo2<1, 8><<<1, 32>>>(keys, n, o2, cyc, init); cudaDeviceSynchronize();
  printf("v1 interleaved unroll8: %.1f cycles/step  same=%d\n", (double)cyc[0] / n, o2[0] == ref);
  k_solo2<2, 8><<<1, 32>>>(keys, n, o2, cyc, init); cudaDeviceSynchronize();
  printf("v2 pipelined unroll8: %.1f cycles/step  same=%d\n", (double)cyc[0] / n, o2[0] == ref);
  k_solo2<2, 32><<<1, 32>>>(keys, n, o2, cyc, init); cudaDeviceSynchronize();
  printf("v2 pipelined unroll32: %.1f cycles/step  same=%d\n", (double)cyc[0] / n, o2[0] == ref);
  k_solo2<2, 4><<<1, 32>>>(keys, n, o2, cyc, init); cudaDeviceSynchronize();
  printf("v2 pipelined unroll4: %.1f cycles/step  same=%d\n", (double)cyc[0] / n, o2[0] == ref);
  k_solo3<4><<<1, 32>>>(keys, n, o2, cyc, init); cudaDeviceSynchronize();
  printf("v3 lane-pair unroll4: %.1f cycles/step  same=%d\n", (double)cyc[0] / n, o2[0] == ref);
  k_solo3<8><<<1, 32>>>(keys, n, o2, cyc, init); cudaDeviceSynchronize();
  printf("v3 lane-pair unroll8: %.1f cycles/step  same=%d\n", (double)cyc[0] / n, o2[0] == ref);
  k_solo3<32><<<1, 32>>>(keys, n, o2, cyc, init); cudaDeviceSynchronize();
  printf("v3 lane-pair unroll32: %.1f cycles/step  same=%d\n", (double)cyc[0] / n, o2[0] == ref);
  k_chain<0><<<1, 32>>>(o2, cyc, init, n); cudaDeviceSynchronize(); printf("chain only (regs): %.1f\n", (double)cyc[0] / n);
  k_chain<2><<<1, 32>>>(o2, cyc, init, n); cudaDeviceSynchronize(); printf("chain + acc: %.1f\n", (double)cyc[0] / n);
  k_chain<4><<<1, 32>>>(o2, cyc, init, n); cudaDeviceSynchronize(); printf("chain + lds: %.1f\n", (double)cyc[0] / n);
  k_chain<6><<<1, 32>>>(o2, cyc, init, n); cudaDeviceSynchronize(); printf("chain + lds + acc: %.1f\n", (double)cyc[0] / n);
  k_chain<5><<<1, 32>>>(o2, cyc, init, n); cudaDeviceSynchronize(); printf("chain + lds + sts: %.1f\n", (double)cyc[0] / n);
  k_chain<15><<<1, 32>>>(o2, cyc, init, n); cudaDeviceSynchronize(); printf("chain + lds + acc + delayed sts: %.1f\n", (double)cyc[0] / n);
  k_chain<22><<<1, 32>>>(o2, cyc, init, n); cudaDeviceSynchronize(); printf("chain + lds + acc + keep-in-reg: %.1f\n", (double)cyc[0] / n);
  k_chain<7><<<1, 32>>>(o2, cyc, init, n); cudaDeviceSynchronize(); printf("chain + lds + acc + sts: %.1f\n", (double)cyc[0] / n);
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
