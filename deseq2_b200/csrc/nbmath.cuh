// nbmath.cuh -- fp64 device math for the NB-GLM kernels (sm_90a).
//
// Own implementations of the special functions the reference pulls from R's nmath
// (Rf_lgammafn / Rf_digamma / Rf_trigamma, call sites /root/reference/src/DESeq2.cpp:50-58,90-96,139-145)
// and of log() for strictly positive normal arguments.  Written for the GPU's FP64 pipe:
//   * one log + one reciprocal per fused lgamma/digamma pair, the rest FMAs;
//   * every polynomial coefficient lives in a __constant__ table so it reaches the DFMA as a uniform-register
//     operand (two coefficients per instruction) instead of issue slots spent on UMOV/IMAD.MOV pairs
//     materialising 64-bit immediates;
//   * no special-case branches (callers guarantee positive, finite, normal inputs).
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace nb {

constexpr double kHalfLog2Pi = 0.918938533204672741780329736406;  // log(sqrt(2*pi))
constexpr double kShift = 10.0;  // arguments below this are shifted up before the asymptotic series

// coefficient tables (constant bank)
//  kLogC[k-1]  = 1 / ((2k+1) 4^k), k = 1..9 : log((1+s)/(1-s)) = t + t^3/12 + t^5/80 + ...,  t = 2s
//  kStirC[k-1] = B_2k / (2k (2k-1)), k = 1..7
//  kDigC[k-1]  = B_2k / (2k),        k = 1..7
//  kTriC[k-1]  = B_2k,               k = 1..7
__constant__ double kLogC[10] = {1.0 / 12.0,        1.0 / 80.0,         1.0 / 448.0,        1.0 / 2304.0,
                                 1.0 / 11264.0,     1.0 / 53248.0,      1.0 / 245760.0,     1.0 / 1114112.0,
                                 1.0 / 4980736.0,   0.0};
__constant__ double kStirC[8] = {1.0 / 12.0,  -1.0 / 360.0, 1.0 / 1260.0, -1.0 / 1680.0,
                                 1.0 / 1188.0, -691.0 / 360360.0, 1.0 / 156.0, 0.0};
__constant__ double kDigC[8] = {1.0 / 12.0, -1.0 / 120.0, 1.0 / 252.0, -1.0 / 240.0,
                                1.0 / 132.0, -691.0 / 32760.0, 1.0 / 12.0, 0.0};
__constant__ double kTriC[8] = {1.0 / 6.0, -1.0 / 30.0, 1.0 / 42.0, -1.0 / 30.0,
                                5.0 / 66.0, -691.0 / 2730.0, 7.0 / 6.0, 0.0};
// log1p series for the table-driven log: -1/2, 1/3, -1/4, 1/5, -1/6, 1/7
__constant__ double kLogT[6] = {-1.0 / 2.0, 1.0 / 3.0, -1.0 / 4.0, 1.0 / 5.0, -1.0 / 6.0, 1.0 / 7.0};
// ln2 split: hi has 32 trailing zero bits cleared so e*hi is exact for |e| < 2^11
__constant__ double kLn2[2] = {6.93147180369123816490e-01, 1.90821492927058770002e-10};

// fast fp64 reciprocal: MUFU.RCP64H seed (~20 bits) + 2 Newton steps (<= 1 ulp for normal inputs).
// Callers use it only where the operand is known positive, finite and normal.
__device__ __forceinline__ double rcp_fast(double x) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  double e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  return r;
}

// ---------------------------------------------------------------- table-driven log
// log(x) for positive, finite, normal x (no zero / denormal / inf / nan handling), Tang-style:
//   x = 2^e m, m in [1, 2);  c = 1 + k/128 the grid point nearest to m (k = 0..128);  r = (m - c) / c, |r| <= 2^-8
//   log x = e ln2 + log c + (r - r^2/2 + ... + r^7/7)
// {1/c, hi(log c), lo(log c)} come from a 129-entry table (gen_logtab.py) that every kernel using log_pos copies
// into shared memory once per CTA (init_log_table): 3 integer ops for the index, one reciprocal-free reduction,
// a degree-6 polynomial -- ~27 instructions against ~45 for the division-based fdlibm scheme (kept below as
// log_pos_poly).  c = 1 and c = 2 are grid points, so results near x = 1 keep full relative accuracy.
// Max error 1.06 ulp (host emulation over 3e7 points, see DESIGN.md).
__device__ const double4 g_logtab[129] = {
#include "logtab.inc"
};
// The grid point c is rebuilt from k with two integer instructions instead of being loaded, and the table is split into
// {1/c, hi(log c)} (one LDS.128) and lo(log c) (one LDS.64): 24 instead of 32 bytes of shared-memory traffic per call.
// The random-index fetch is the kernels' top short-scoreboard stall and bank-conflict source.
__shared__ double2 s_logA[129];
__shared__ double s_logL[129];

// every thread of the CTA must call this before the first log_pos (contains a __syncthreads)
__device__ __forceinline__ void init_log_table() {
  for (int i = threadIdx.x + threadIdx.y * blockDim.x; i < 129; i += blockDim.x * blockDim.y) {
    const double4 t = g_logtab[i];
    s_logA[i] = make_double2(t.x, t.y);
    s_logL[i] = t.z;
  }
  __syncthreads();
}

__device__ __forceinline__ double log_pos(double x) {
  const int hi = __double2hiint(x);
  const int lo = __double2loint(x);
  const int e = (hi >> 20) - 1023;
  const int k = ((hi >> 13) & 0x7f) + ((hi >> 12) & 1);
  const double m = __hiloint2double((hi & 0x000fffff) | 0x3ff00000, lo);
  const double2 ta = s_logA[k];
  const double4 t = make_double4(ta.x, ta.y, s_logL[k], __hiloint2double(0x3ff00000 + (k << 13), 0));
  const double r = (m - t.w) * t.x;
  double p = kLogT[5];
  p = fma(p, r, kLogT[4]);
  p = fma(p, r, kLogT[3]);
  p = fma(p, r, kLogT[2]);
  p = fma(p, r, kLogT[1]);
  p = fma(p, r, kLogT[0]);
  const double de = __hiloint2double(0x43300000, e ^ 0x80000000) - 4503601774854144.0;
  const double h = fma(de, kLn2[0], t.y);
  const double l = fma(de, kLn2[1], t.z);
  return h + (r + fma(r * r, p, l));
}

// division-based fdlibm-style log (no table): used where no shared-memory table is set up
__device__ __forceinline__ double log_pos_poly(double x) {
  int hi = __double2hiint(x);
  const int lo = __double2loint(x);
  int e = (hi >> 20) - 1023;
  hi = (hi & 0x000fffff) | 0x3ff00000;
  if (hi >= 0x3ff6a09f) {  // m >= ~sqrt(2): halve
    hi -= 0x00100000;
    e += 1;
  }
  const double m = __hiloint2double(hi, lo);
  const double f = m - 1.0;
  const double r = rcp_fast(m + 1.0);
  double t = f * r;
  t = fma(f, r, t);                                  // t ~= 2 f / (2 + f)
  const double z = t * t;
  const double c = r * fma(f, -t, 2.0 * (f - t));    // exact_t - t
  const double z2 = z * z;
  const double a0 = fma(kLogC[1], z, kLogC[0]);
  const double a1 = fma(kLogC[3], z, kLogC[2]);
  const double a2 = fma(kLogC[5], z, kLogC[4]);
  const double a3 = fma(kLogC[7], z, kLogC[6]);
  const double z4 = z2 * z2;
  const double b0 = fma(a1, z2, a0);
  const double b1 = fma(a3, z2, a2);
  const double p = fma(fma(kLogC[8], z4, b1), z4, b0);
  const double res_lo = fma(t * z, p, c);
  const double de = __hiloint2double(0x43300000, e ^ 0x80000000) - 4503601774854144.0;
  const double q = fma(de, kLn2[0], t);
  const double rem = fma(de, -kLn2[0], q) - t;       // rounding error of q
  return q + fma(de, kLn2[1], res_lo - rem);
}

// 1/k!, k = 2..13 (exp_fast)
__constant__ double kExpC[12] = {1.0 / 2.0,          1.0 / 6.0,           1.0 / 24.0,           1.0 / 120.0,
                                 1.0 / 720.0,        1.0 / 5040.0,        1.0 / 40320.0,        1.0 / 362880.0,
                                 1.0 / 3628800.0,    1.0 / 39916800.0,    1.0 / 479001600.0,    1.0 / 6227020800.0};

// exp(x) for |x| < 700 (no overflow / underflow / nan handling): x = k ln2 + r, |r| <= ln2/2, Taylor to r^13,
// scaled by 2^k through the exponent field.  < 1 ulp-ish (checked on the device against mpmath in tests).
__device__ __forceinline__ double exp_fast(double x) {
  const double kf = rint(x * 1.4426950408889634);
  const double r = fma(kf, -kLn2[1], fma(kf, -kLn2[0], x));
  // Estrin: 12 coefficients (1/2! .. 1/13!) in r
  const double r2 = r * r;
  const double e0 = fma(kExpC[1], r, kExpC[0]);
  const double e1 = fma(kExpC[3], r, kExpC[2]);
  const double e2 = fma(kExpC[5], r, kExpC[4]);
  const double e3 = fma(kExpC[7], r, kExpC[6]);
  const double e4 = fma(kExpC[9], r, kExpC[8]);
  const double e5 = fma(kExpC[11], r, kExpC[10]);
  const double r4 = r2 * r2;
  const double f0 = fma(e1, r2, e0);
  const double f1 = fma(e3, r2, e2);
  const double f2 = fma(e5, r2, e4);
  double p = fma(fma(f2, r4, f1), r4, f0);
  p = fma(p * r, r, r);          // r + r^2 * poly
  const double e = 1.0 + p;
  const int k = (int)kf;
  return __hiloint2double(__double2hiint(e) + (k << 20), __double2loint(e));
}

// log1p(x) for x >= 0 (finite): log(u) + (x - (u - 1)) / u with u = 1 + x recovers the bits 1 + x rounds away
__device__ __forceinline__ double log1p_pos(double x) {
  const double u = 1.0 + x;
  return log_pos(u) + (x - (u - 1.0)) * rcp_fast(u);
}

// Stirling tail  sum_{k>=1} B_2k / (2k (2k-1) x^(2k-1))  evaluated as xi * poly(xi^2), x >= kShift
__device__ __forceinline__ double stirling_tail(double xi, double xi2) {
  double p = kStirC[6];
  p = fma(p, xi2, kStirC[5]);
  p = fma(p, xi2, kStirC[4]);
  p = fma(p, xi2, kStirC[3]);
  p = fma(p, xi2, kStirC[2]);
  p = fma(p, xi2, kStirC[1]);
  p = fma(p, xi2, kStirC[0]);
  return p * xi;
}

// sum_{k>=1} B_2k / (2k x^2k), x >= kShift
__device__ __forceinline__ double digamma_tail(double xi2) {
  double p = kDigC[6];
  p = fma(p, xi2, kDigC[5]);
  p = fma(p, xi2, kDigC[4]);
  p = fma(p, xi2, kDigC[3]);
  p = fma(p, xi2, kDigC[2]);
  p = fma(p, xi2, kDigC[1]);
  p = fma(p, xi2, kDigC[0]);
  return p * xi2;
}

// lgamma(x) for x > 0.
__device__ __forceinline__ double lgamma_pos(double x) {
  double prod = 1.0;
  const bool shifted = x < kShift;
  while (x < kShift) {
    prod *= x;
    x += 1.0;
  }
  const double xi = rcp_fast(x);
  const double lx = log_pos(x);
  double r = fma(x - 0.5, lx, -x) + kHalfLog2Pi + stirling_tail(xi, xi * xi);
  if (shifted) r -= log_pos(prod);
  return r;
}

// fused lgamma(x), digamma(x) for x > 0: shares log(x) and 1/x.
__device__ __forceinline__ void lgamma_digamma_pos(double x, double& lg, double& dg) {
  // shift: prod = x (x+1) ... (x+n-1), dprod = d prod / dx
  double prod = 1.0, dprod = 0.0;
  const bool shifted = x < kShift;
  while (x < kShift) {
    dprod = fma(dprod, x, prod);
    prod *= x;
    x += 1.0;
  }
  const double xi = rcp_fast(x);
  const double xi2 = xi * xi;
  const double lx = log_pos(x);
  lg = fma(x - 0.5, lx, -x) + kHalfLog2Pi + stirling_tail(xi, xi2);
  dg = lx - 0.5 * xi - digamma_tail(xi2);
  if (shifted) {
    lg -= log_pos(prod);
    dg -= dprod * rcp_fast(prod);
  }
}

// no-shift variant for x >= kShift (caller guarantees)
__device__ __forceinline__ void lgamma_digamma_big(double x, double& lg, double& dg) {
  const double xi = rcp_fast(x);
  const double xi2 = xi * xi;
  const double lx = log_pos(x);
  lg = fma(x - 0.5, lx, -x) + kHalfLog2Pi + stirling_tail(xi, xi2);
  dg = lx - 0.5 * xi - digamma_tail(xi2);
}

__device__ __forceinline__ double digamma_pos(double x) {
  double lg, dg;
  lgamma_digamma_pos(x, lg, dg);
  return dg;
}

// trigamma(x), x > 0.  Used once per gene (d2lp), so the shift loop may divide.
__device__ __forceinline__ double trigamma_pos(double x) {
  double s = 0.0;
  while (x < kShift) {
    const double xi = 1.0 / x;
    s = fma(xi, xi, s);
    x += 1.0;
  }
  const double xi = 1.0 / x, xi2 = xi * xi;
  double p = kTriC[6];
  p = fma(p, xi2, kTriC[5]);
  p = fma(p, xi2, kTriC[4]);
  p = fma(p, xi2, kTriC[3]);
  p = fma(p, xi2, kTriC[2]);
  p = fma(p, xi2, kTriC[1]);
  p = fma(p, xi2, kTriC[0]);
  return s + xi + 0.5 * xi2 + p * xi2 * xi;
}

// ---------------------------------------------------------------- warp helpers
// xor-butterfly all-reduces inside aligned groups of GL lanes (GL = 32: the whole warp); every lane of a group ends
// with the same bits
template <int GL>
__device__ __forceinline__ double group_allreduce_sum(double v) {
#pragma unroll
  for (int o = GL / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <int GL>
__device__ __forceinline__ double group_allreduce_max(double v) {
#pragma unroll
  for (int o = GL / 2; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <int N, int GL>
__device__ __forceinline__ void group_allreduce_sum_n(double (&v)[N]) {
#pragma unroll
  for (int o = GL / 2; o > 0; o >>= 1) {
#pragma unroll
    for (int i = 0; i < N; i++) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
  }
}

__device__ __forceinline__ double warp_allreduce_sum(double v) { return group_allreduce_sum<32>(v); }
__device__ __forceinline__ double warp_allreduce_max(double v) { return group_allreduce_max<32>(v); }
template <int N>
__device__ __forceinline__ void warp_allreduce_sum_n(double (&v)[N]) { group_allreduce_sum_n<N, 32>(v); }

// All-reduce of N per-lane partial sums, N a power of two <= 32, as a butterfly reduce-scatter followed by
// an all-gather: log2(N) halving exchange rounds (N/2 + N/4 + ... + 1 values shuffled), plain butterflies for
// the remaining rounds, then N indexed shuffles.  ~2.4x fewer SHFL than N independent butterflies for N = 8.
// The result is bitwise identical in every lane (each value is reduced along one fixed tree).
template <int N>
__device__ __forceinline__ void warp_allreduce_sum_rs(double (&v)[N], int lane) {
  static_assert(N >= 1 && N <= 32 && (N & (N - 1)) == 0, "N must be a power of two <= 32");
  int width = N;  // number of live values in v[0 .. width)
  int o = 16;
#pragma unroll
  for (; o > 0 && width > 1; o >>= 1) {
    const bool upper = (lane & o) != 0;
    const int half = width / 2;
#pragma unroll
    for (int i = 0; i < N / 2; i++) {
      if (i < half) {
        // lower lanes keep v[i], send v[i+half]; upper lanes keep v[i+half], send v[i]
        const double keep = upper ? v[i + half] : v[i];
        const double send = upper ? v[i] : v[i + half];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
      }
    }
    width = half;
  }
#pragma unroll
  for (; o > 0; o >>= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
  // value index i (original) now sits in v[0] of the lanes whose upper bits spell i: gather
  const double mine = v[0];
  constexpr int LOGN = (N == 1) ? 0 : (N == 2) ? 1 : (N == 4) ? 2 : (N == 8) ? 3 : (N == 16) ? 4 : 5;
#pragma unroll
  for (int i = 0; i < N; i++) {
    // lane holding original index i: bit (16 >> s) set iff bit (LOGN-1-s) of i ... built below
    int src = 0;
#pragma unroll
    for (int s = 0; s < LOGN; s++) {
      // round s (offset 16>>s) split the live range in halves: upper lanes kept the upper half
      if ((i >> (LOGN - 1 - s)) & 1) src |= (16 >> s);
    }
    v[i] = __shfl_sync(0xffffffffu, mine, src);
  }
}

// The same reduce-scatter + all-gather inside lane groups of GL lanes (GL = 16 or 8; lg = lane index inside the group,
// N <= GL): used by the several-genes-per-warp experiment kernels, never instantiated by the product kernels.
template <int N, int GL>
__device__ __forceinline__ void group_allreduce_sum_rs(double (&v)[N], int lg) {
  static_assert(N >= 1 && N <= GL && (N & (N - 1)) == 0 && (GL == 16 || GL == 8), "N must be a power of two <= GL");
  int width = N;
  int o = GL / 2;
#pragma unroll
  for (; o > 0 && width > 1; o >>= 1) {
    const bool upper = (lg & o) != 0;
    const int half = width / 2;
#pragma unroll
    for (int i = 0; i < N / 2; i++) {
      if (i < half) {
        const double keep = upper ? v[i + half] : v[i];
        const double send = upper ? v[i] : v[i + half];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
      }
    }
    width = half;
  }
#pragma unroll
  for (; o > 0; o >>= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
  const double mine = v[0];
  constexpr int LOGN = (N == 1) ? 0 : (N == 2) ? 1 : (N == 4) ? 2 : (N == 8) ? 3 : 4;
#pragma unroll
  for (int i = 0; i < N; i++) {
    int src = 0;
#pragma unroll
    for (int s = 0; s < LOGN; s++)
      if ((i >> (LOGN - 1 - s)) & 1) src |= ((GL / 2) >> s);
    v[i] = __shfl_sync(0xffffffffu, mine, src, GL);   // width GL: the source lane is taken inside the caller's group
  }
}

}  // namespace nb
