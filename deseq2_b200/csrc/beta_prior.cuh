// beta_prior.cuh -- estimateBetaPriorVar's weighted upper quantile on the device (betaPriorMethod "weighted").
// Reference: estimateBetaPriorVar R/core.R:1601-1689, matchWeightedUpperQuantileForVariance
// :2416-2419, Hmisc.wtd.quantile / Hmisc.wtd.table :2762-2900 (type "quantile", normwt = TRUE), addAllContrasts
// R/expanded.R:76-98.  For every requested column c (one CTA each):
//   x_i  = |beta[a_c, i] - (b_c < 0 ? 0 : beta[b_c, i])|     a column of the MLE log2 fold changes, or a contrast
//   w_i  = 1 / (1 / baseMean_i + dispFit_i)
//   kept: |x_i| < 10 (NaN is not kept) and w_i neither NaN nor 0;  N kept entries, S = sum of their weights
//   w'_i = w_i N / S                                           (normwt); ties in x share one cumulative weight
//   order = 1 + (N - 1) prob, low = max(floor(order), 1), high = min(low + 1, N), frac = order mod 1
//   x_(v) = the smallest x whose cumulative weight reaches v - 1e-12 max(1, v), the largest x if none does (rule = 2)
//   q_c  = (1 - frac) x_(low) + frac x_(high);  NaN when nothing is kept.
// No sort and no scratch in global memory: after one pass for N and S, 16 passes refine BOTH order statistics
// together, 4 bits per pass, most significant first, over the 64-bit pattern of x (non-negative doubles order like
// their bit patterns).  A pass histograms the weight of the entries that share the prefix found so far; every thread
// owns one column of the shared histogram and the columns are summed in a fixed order, so two calls give the same
// bits (no floating-point atomics anywhere).  The histogram (2 x 16 x 128 doubles = 32 KB) is static shared memory.
// Included by size_factors.cu, whose column-select launch helper starts it (one CTA per column, like the size-factor
// medians).
#pragma once
#include "engine.h"
#include "nbmath.cuh"

#include <math.h>

namespace nb {
namespace {

constexpr int kBpThreads = 128;
constexpr int kBpDigits = 16;                                  // 4-bit digits, 16 passes over 64 bits

// ---- the steps of the refinement, shared with rlog's prior variance (rlog.cuh), which runs them over many CTAs
// Hmisc's order statistics for N kept entries: frac and the cumulative-weight targets of x_(low) and x_(high), in the
// host restatement's arithmetic, unfused (nvcc would contract these into FMAs)
__device__ __forceinline__ void bp_targets(double dN, double prob, double& frac, double& t_low, double& t_high) {
  const double order = __dadd_rn(1.0, __dmul_rn(dN - 1.0, prob));
  const double low = fmax(floor(order), 1.0);
  const double high = fmin(low + 1.0, dN);
  frac = order - floor(order);
  t_low = __dadd_rn(low, -__dmul_rn(1e-12, fmax(1.0, low)));
  t_high = __dadd_rn(high, -__dmul_rn(1e-12, fmax(1.0, high)));
}

// one entry into the calling thread's histogram column hl (row stride kBpThreads): digit `shift` of its bit pattern,
// for each target whose prefix it shares
__device__ __forceinline__ void bp_hist_add(double* hl, unsigned long long bits, double wn, int shift,
                                            unsigned long long mask, unsigned long long p0, unsigned long long p1,
                                            int& md0, int& md1) {
  const int d = (int)(bits >> shift) & (kBpDigits - 1);
  const unsigned long long hi = bits & mask;
  if (hi == p0) { hl[d * kBpThreads] += wn; md0 = max(md0, d); }
  if (hi == p1) { hl[(kBpDigits + d) * kBpThreads] += wn; md1 = max(md1, d); }
}

// bucket totals of the 2 x kBpDigits x kBpThreads histogram: warp w sums the rows w, w + 4, ...; each lane 4
// consecutive columns, then a fixed tree
__device__ __forceinline__ void bp_bucket_totals(const double* s_hist, double (*bucket)[kBpDigits], int warp,
                                                 int lane) {
  for (int row = warp; row < 2 * kBpDigits; row += kBpThreads / 32) {
    const double* col = s_hist + row * kBpThreads + lane * (kBpThreads / 32);
    double v = 0.0;
    for (int k = 0; k < kBpThreads / 32; k++) v += col[k];
    v = warp_allreduce_sum(v);
    if (lane == 0) bucket[row / kBpDigits][row % kBpDigits] = v;
  }
}

// the digit of one target: the first whose cumulative weight reaches it; none (rounding, or the target lies beyond the
// total weight: rule = 2) -> the largest digit present under the prefix (maxd).  Advances below and prefix.
__device__ __forceinline__ void bp_pick_digit(const double* bucket, const int& maxd, double target, int shift,
                                              double& below, unsigned long long& prefix) {
  double b = below;
  int pick = -1;
  for (int d = 0; d < kBpDigits; d++) {
    if (b + bucket[d] >= target) { pick = d; break; }
    b += bucket[d];
  }
  if (pick < 0) {
    pick = max(maxd, 0);
    b = below;
    for (int d = 0; d < pick; d++) b += bucket[d];
  }
  below = b;
  prefix |= (unsigned long long)pick << shift;
}

// one entry of column (a, b): its |x| bit pattern and weight; false if the entry does not take part
__device__ __forceinline__ bool bp_entry(const BetaPriorQArgs& A, int a, int b, int i, unsigned long long& bits,
                                         double& w) {
  double x = A.beta[(size_t)a * A.n + i];
  if (b >= 0) x -= A.beta[(size_t)b * A.n + i];
  x = fabs(x);
  w = 1.0 / (1.0 / A.base_mean[i] + A.disp_fit[i]);
  bits = (unsigned long long)__double_as_longlong(x);
  return x < 10.0 && !isnan(w) && w != 0.0;
}

__global__ void __launch_bounds__(kBpThreads) beta_prior_quantile_kernel(const BetaPriorQArgs A) {
  __shared__ double s_hist[2 * kBpDigits * kBpThreads];        // [target 2][digit 16][thread]
  __shared__ double s_red[kBpThreads / 32];
  __shared__ double s_bucket[2][kBpDigits];
  __shared__ double s_below[2];
  __shared__ unsigned long long s_prefix[2];
  __shared__ int s_cnt, s_maxd[2];
  const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int a = A.col_a[c], b = A.col_b[c];
  unsigned long long bits;
  double w;

  // ---- pass 1: kept count and weight sum (per-thread sums in element order, then a fixed tree)
  int cnt = 0;
  double sw = 0.0;
  for (int i = tid; i < A.n; i += kBpThreads)
    if (bp_entry(A, a, b, i, bits, w)) { cnt++; sw += w; }
  if (tid == 0) { s_cnt = 0; s_prefix[0] = s_prefix[1] = 0ull; s_below[0] = s_below[1] = 0.0; }
  __syncthreads();
  sw = warp_allreduce_sum(sw);
  if (lane == 0) s_red[warp] = sw;
  if (cnt) atomicAdd(&s_cnt, cnt);
  __syncthreads();
  const int N = s_cnt;
  if (N == 0) {
    if (tid == 0) A.out_q[c] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  double S = 0.0;
  for (int k = 0; k < kBpThreads / 32; k++) S += s_red[k];
  const double dN = (double)N;
  double frac, t_low, t_high;
  bp_targets(dN, A.prob, frac, t_low, t_high);

  // ---- 16 refinement passes, both order statistics at once
  double* hl = s_hist + tid;
  for (int r = 0; r < kBpDigits; r++) {
    const int shift = 60 - 4 * r;
    const unsigned long long mask = r == 0 ? 0ull : (~0ull << (shift + 4));
    for (int k = 0; k < 2 * kBpDigits; k++) hl[k * kBpThreads] = 0.0;
    if (tid < 2) s_maxd[tid] = -1;
    __syncthreads();
    const unsigned long long p0 = s_prefix[0], p1 = s_prefix[1];
    int md0 = -1, md1 = -1;
    for (int i = tid; i < A.n; i += kBpThreads) {
      if (!bp_entry(A, a, b, i, bits, w)) continue;
      bp_hist_add(hl, bits, (w * dN) / S, shift, mask, p0, p1, md0, md1);   // normwt, as w * length(x) / sum(w)
    }
    if (md0 >= 0) atomicMax(&s_maxd[0], md0);
    if (md1 >= 0) atomicMax(&s_maxd[1], md1);
    __syncthreads();
    bp_bucket_totals(s_hist, s_bucket, warp, lane);
    __syncthreads();
    if (tid < 2) bp_pick_digit(s_bucket[tid], s_maxd[tid], tid ? t_high : t_low, shift, s_below[tid], s_prefix[tid]);
    __syncthreads();
  }
  if (tid == 0) {
    const double xl = __longlong_as_double((long long)s_prefix[0]);
    const double xh = __longlong_as_double((long long)s_prefix[1]);
    A.out_q[c] = __dadd_rn(__dmul_rn(1.0 - frac, xl), __dmul_rn(frac, xh));
  }
}

}  // namespace
}  // namespace nb
