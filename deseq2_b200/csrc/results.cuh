// results.cuh -- results() and pvalueAdjustment() (R/results.R:298-740) on the device (included by size_factors.cu,
// launched through its launch_per_column).
//
// results_gene_kernel: one warp per gene (the count-row reads are coalesced along the sample axis).  From the
// selected column (log2FoldChange, lfcSE, stat, pvalue) it applies, in R's order:
//   1. the swapped reference level (LFC and, for the Wald test, stat negated, :910-925) and contrastAllZero
//      (:1237-1270: the original counts of the contrast's samples are all zero -> LFC 0; for the Wald test stat 0
//      and p 1, the LRT keeps its own stat and p, :1032-1037);
//   2. lfcThreshold / altHypothesis (:464-518), with pnorm(q, sd = se) = pnorm(q / se) and the upper tail
//      pnorm(q, lower.tail = FALSE) = erfc(q / sqrt 2) / 2;
//   3. the Cook's cutoff (:520-565): maxCooks > cutoff (NaN never flags) and not kept by the two-group heuristic
//      -> p NA;
//   4. replaced rows that are now all zero (:567-575) -> LFC, SE, stat 0 and p 1.
// results_heuristic_kernel: one warp per gene the cutoff flags: outCount = the count at which.max of the gene's Cook's
// row (the first maximum, NaN skipped); the gene is kept when at least 3 of its counts are > outCount.
//
// filter_cutoff_kernel: one CTA per theta: quantile(filter, theta, type = 7) by size_factors.cu's MSB-first radix
// select (select_key / next_key), no sort of the filter:
//   index = 1 + (n - 1) theta, lo = floor(index); x[lo], replaced by (1 - h) x[lo] + h x[lo + 1] (h = index - lo,
//   no contraction) when index > lo and x[lo + 1] != x[lo].
// filter_numrej_kernel: one CTA per theta: the number of rejections, sum(p.adjust(p[filter >= cutoff]) < alpha),
// without the adjusted column.  The p-values come sorted ascending (NaN last) with their filter values; a block-wide
// scan gives every member its rank r among the n_theta members, and R's expressions (n = n_theta: the lazy default
// length(p) is forced after the NAs are dropped) give the count directly, because pmin(1, v) < alpha <=> v < alpha:
//   BH / BY / hochberg  padj_(r) = min_{s >= r} term_s: the count is the largest r with term_r < alpha,
//                       term = n / r * p, ((q * n) / r) * p with q = sum(1 / (1:n)), (n + 1 - r) * p;
//   holm                padj_(r) = max_{s <= r} (n - s + 1) p_(s): the length of the prefix with term < alpha;
//   bonferroni / none   the plain count of n p < alpha, p < alpha.
// padj_kernel: one CTA: the adjusted column of one subset (filter >= cutoff, or every non-NA p), a suffix-min
// (BH / BY / hochberg) or prefix-max (holm) scan in sorted order, pmin(1, .), scattered to the genes' positions;
// the other genes get NA.
// Tied p-values cannot change an adjusted value, whatever order the sort leaves them in: within a run of ties the
// cummin (cummax) reaches the term of the run's last (first) rank from every member of the run, so all of them get
// that value.  The sort therefore needs no stability.  No floating-point atomics: the counts are integer reductions,
// BY's q is summed in a fixed tree order, so two calls give the same bits.
#pragma once
#include "../../include/b200nb.h"
#include "engine.h"
#include "nbmath.cuh"

namespace nb {
namespace {

constexpr int kRsThreads = 128;                    // per-gene kernels: one warp per gene
constexpr int kRsScanThreads = 512;                // one-CTA-per-subset kernels
constexpr int kRsWarps = kRsScanThreads / 32;

__device__ __forceinline__ double rs_nan() { return __longlong_as_double(0x7ff8000000000000ll); }

template <class T>
__device__ __forceinline__ double rs_count(const void* y, size_t k) {
  return (double)__ldg(static_cast<const T*>(y) + k);
}

// pnorm(q, lower.tail = FALSE)
__device__ __forceinline__ double rs_upper(double q) { return 0.5 * erfc(q * 0.70710678118654752440); }
// pnorm(q)
__device__ __forceinline__ double rs_lower(double q) { return 0.5 * erfc(-q * 0.70710678118654752440); }
// R's pmax / pmin: NA when either argument is
__device__ __forceinline__ double rs_pmax(double a, double b) { return (isnan(a) || isnan(b)) ? rs_nan() : fmax(a, b); }
__device__ __forceinline__ double rs_pmin(double a, double b) { return (isnan(a) || isnan(b)) ? rs_nan() : fmin(a, b); }
__device__ __forceinline__ double rs_sign(double v) { return isnan(v) ? v : (v > 0.0 ? 1.0 : (v < 0.0 ? -1.0 : 0.0)); }
__device__ __forceinline__ double rs_sub(double a, double b) { return __dadd_rn(a, -b); }

template <class T>
__global__ void __launch_bounds__(kRsThreads) results_gene_kernel(const ResultsGeneArgs A) {
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * (kRsThreads / 32) + (threadIdx.x >> 5);
  if (g >= A.n) return;                                      // whole warps leave together
  double lfc = A.lfc[g], se = A.se[g], stat = A.stat[g], p = A.pvalue[g];
  if (A.negate) {
    lfc = -lfc;
    if (!A.lrt) stat = -stat;
  }
  if (A.zero_mask != nullptr) {
    const size_t off = (size_t)g * A.ld;
    double s = 0.0;
    for (int j = lane; j < A.m; j += 32)
      if (A.zero_mask[j]) s += rs_count<T>(A.y, off + j);
    s = warp_allreduce_sum(s);                               // counts are >= 0: the sum is 0 iff all are
    if (s == 0.0) {
      lfc = 0.0;
      if (!A.lrt) {
        stat = 0.0;
        p = 1.0;
      }
    }
  }
  const double T_ = A.lfc_threshold;
  switch (A.alt) {
    case B200NB_ALT_GREATER_ABS:
      stat = lfc / se;
      p = rs_lower(__dadd_rn(-fabs(lfc), T_) / se) + rs_lower(rs_sub(-fabs(lfc), T_) / se);
      break;
    case B200NB_ALT_GREATER_ABS_2014: {
      const double q = rs_sub(fabs(lfc), T_) / se;
      stat = rs_sign(lfc) * rs_pmax(q, 0.0);
      p = rs_pmin(1.0, 2.0 * rs_upper(q));
      break;
    }
    case B200NB_ALT_LESS_ABS: {
      const double qa = rs_sub(T_, lfc) / se, qb = __dadd_rn(lfc, T_) / se;
      stat = rs_pmin(rs_pmax(qa, 0.0), rs_pmax(qb, 0.0));
      p = rs_pmax(rs_upper(qa), rs_upper(qb));
      break;
    }
    case B200NB_ALT_GREATER: {
      const double q = rs_sub(lfc, T_) / se;
      stat = rs_pmax(q, 0.0);
      p = rs_upper(q);
      break;
    }
    case B200NB_ALT_LESS:
      stat = rs_pmin(__dadd_rn(lfc, T_) / se, 0.0);
      p = rs_upper(rs_sub(-T_, lfc) / se);
      break;
    default: break;                                          // B200NB_ALT_NONE: T = 0 and greaterAbs
  }
  if (A.max_cooks != nullptr && A.max_cooks[g] > A.cooks_cutoff && !(A.keep != nullptr && A.keep[g] != 0))
    p = rs_nan();
  if (A.replace != nullptr && A.replace[g] != 0 && A.base_mean[g] == 0.0) {
    lfc = se = stat = 0.0;
    p = 1.0;
  }
  if (lane == 0) {
    A.out_lfc[g] = lfc;
    A.out_se[g] = se;
    A.out_stat[g] = stat;
    A.out_pvalue[g] = p;
  }
}

template <class T>
__global__ void __launch_bounds__(kRsThreads) results_heuristic_kernel(const ResultsHeuristicArgs A) {
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * (kRsThreads / 32) + (threadIdx.x >> 5);
  if (k >= A.k) return;
  const long long row = A.rows[k];
  const double* c = A.cooks + (size_t)k * A.ld_cooks;
  // which.max: the first index of the largest non-NaN value (m if there is none)
  double best = 0.0;
  int bi = A.m;
  for (int j = lane; j < A.m; j += 32) {
    const double v = c[j];
    if (!isnan(v) && (bi == A.m || v > best)) {
      best = v;
      bi = j;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (oi != A.m && (bi == A.m || ob > best || (ob == best && oi < bi))) {
      best = ob;
      bi = oi;
    }
  }
  int above = 0;
  if (bi < A.m) {
    const size_t off = (size_t)row * A.ld;
    const double out_count = rs_count<T>(A.y, off + bi);
    for (int j = lane; j < A.m; j += 32) above += rs_count<T>(A.y, off + j) > out_count;
  }
  above = (int)warp_allreduce_sum((double)above);
  if (lane == 0) A.keep[row] = above >= 3;
}

// block-wide inclusive scan of one value per thread (kRsScanThreads threads) under an associative, exact op;
// `total` is the op over the whole block.  s_warp: kRsWarps shared slots.
template <class V, class Op>
__device__ __forceinline__ V rs_block_scan(V v, Op op, V* s_warp, V& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const V u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v = op(u, v);
  }
  if (lane == 31) s_warp[warp] = v;
  __syncthreads();
  if (warp == 0) {
    V w = s_warp[lane < kRsWarps ? lane : kRsWarps - 1];
    for (int o = 1; o < 32; o <<= 1) {
      const V u = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w = op(u, w);
    }
    if (lane < kRsWarps) s_warp[lane] = w;
  }
  __syncthreads();
  if (warp > 0) v = op(s_warp[warp - 1], v);
  total = s_warp[kRsWarps - 1];
  __syncthreads();                                           // s_warp is reused by the next call
  return v;
}

struct RsAdd { __device__ int operator()(int a, int b) const { return a + b; } };
struct RsMax { __device__ int operator()(int a, int b) const { return a > b ? a : b; } };
struct RsMin { __device__ int operator()(int a, int b) const { return a < b ? a : b; } };
struct RsDMin { __device__ double operator()(double a, double b) const { return fmin(a, b); } };
struct RsDMax { __device__ double operator()(double a, double b) const { return fmax(a, b); } };

__global__ void __launch_bounds__(kRsScanThreads) filter_cutoff_kernel(const FilterCutoffArgs A) {
  __shared__ unsigned int hist[256];
  __shared__ unsigned long long s_prefix, s_next;
  __shared__ unsigned int s_k, s_le;
  const int n = A.n, tid = threadIdx.x;
  const double index = __dadd_rn(1.0, __dmul_rn((double)(n - 1), A.theta[blockIdx.x]));
  const double lo = floor(index);
  const unsigned int rank = (unsigned int)lo - 1u;           // 0-based rank of x[lo]
  if (tid == 0) s_prefix = 0;
  const unsigned long long k1 = select_key(A.filter, n, rank, hist, s_prefix, s_k);
  const double xlo = value_of(k1);
  double qs = xlo;
  if (index > lo) {
    const double xhi = value_of(next_key(A.filter, n, rank, k1, s_le, s_next));
    if (xhi != xlo) {
      const double h = rs_sub(index, lo);
      qs = __dadd_rn(__dmul_rn(1.0 - h, xlo), __dmul_rn(h, xhi));
    }
  }
  if (tid == 0) A.out[blockIdx.x] = qs;
}

// membership of sorted position i in the subset of cutoff `cut`
__device__ __forceinline__ int rs_member(const PadjArgs& A, int i, double cut) {
  return i < A.n && !isnan(A.p_sorted[i]) && A.filter_sorted[i] >= cut;
}

// the number of members, and BY's q = sum(1 / (1:n)) in a fixed tree order
__device__ __forceinline__ int rs_subset_size(const PadjArgs& A, double cut, int* s_int, double* s_dbl, double& q) {
  const int tid = threadIdx.x;
  int c = 0;
  for (int i = tid; i < A.n; i += kRsScanThreads) c += rs_member(A, i, cut);
  int nt;
  rs_block_scan(c, RsAdd(), s_int, nt);
  q = 1.0;
  if (A.method == B200NB_PADJ_BY) {
    double s = 0.0;
    for (int k = nt - tid; k >= 1; k -= kRsScanThreads) s += 1.0 / (double)k;
    s_dbl[tid] = s;
    __syncthreads();
    for (int w = kRsScanThreads >> 1; w > 0; w >>= 1) {
      if (tid < w) s_dbl[tid] += s_dbl[tid + w];
      __syncthreads();
    }
    q = s_dbl[0];
    __syncthreads();
  }
  return nt;
}

// R's term of the member of rank r (1-based, ascending p) among nt
__device__ __forceinline__ double rs_term(int method, double p, int r, int nt, double q) {
  const double n = (double)nt;
  switch (method) {
    case B200NB_PADJ_BH: return (n / (double)r) * p;
    case B200NB_PADJ_BY: return (__dmul_rn(q, n) / (double)r) * p;
    case B200NB_PADJ_HOLM: return (double)(nt - r + 1) * p;
    case B200NB_PADJ_HOCHBERG: return (double)(nt + 1 - r) * p;
    case B200NB_PADJ_BONFERRONI: return n * p;
    default: return p;
  }
}

__global__ void __launch_bounds__(kRsScanThreads) filter_numrej_kernel(const PadjArgs A) {
  __shared__ int s_int[kRsWarps];
  __shared__ double s_dbl[kRsScanThreads];
  const int tid = threadIdx.x;
  const double cut = A.cutoffs[blockIdx.x];
  double q;
  const int nt = rs_subset_size(A, cut, s_int, s_dbl, q);
  const int method = A.method;
  const bool suffix = method == B200NB_PADJ_BH || method == B200NB_PADJ_BY || method == B200NB_PADJ_HOCHBERG;
  int best = 0, first_bad = nt + 1, cnt = 0;
  int base = 0;
  for (int c0 = 0; c0 < A.n; c0 += kRsScanThreads) {
    const int i = c0 + tid;
    const int mem = rs_member(A, i, cut);
    int tot;
    const int r = base + rs_block_scan(mem, RsAdd(), s_int, tot);
    if (mem) {
      const bool below = rs_term(method, A.p_sorted[i], r, nt, q) < A.alpha;
      if (suffix) {
        if (below) best = max(best, r);
      } else if (method == B200NB_PADJ_HOLM) {
        if (!below) first_bad = min(first_bad, r);
      } else {
        cnt += below;
      }
    }
    base += tot;
  }
  int v = suffix ? best : (method == B200NB_PADJ_HOLM ? first_bad : cnt);
  int all;
  if (suffix) rs_block_scan(v, RsMax(), s_int, all);
  else if (method == B200NB_PADJ_HOLM) rs_block_scan(v, RsMin(), s_int, all);
  else rs_block_scan(v, RsAdd(), s_int, all);
  if (tid == 0) A.out_numrej[blockIdx.x] = method == B200NB_PADJ_HOLM ? all - 1 : all;
}

__global__ void __launch_bounds__(kRsScanThreads) padj_kernel(const PadjArgs A) {
  __shared__ int s_int[kRsWarps];
  __shared__ double s_dbl[kRsScanThreads];
  __shared__ double s_warp_d[kRsWarps];
  const int tid = threadIdx.x;
  const double cut = A.cutoffs != nullptr ? A.cutoffs[A.j] : -INFINITY;
  double q;
  const int nt = rs_subset_size(A, cut, s_int, s_dbl, q);
  const int method = A.method;
  const double nan = rs_nan();
  if (method == B200NB_PADJ_HOLM) {                          // prefix max, forward
    int base = 0;
    double carry = -INFINITY;
    for (int c0 = 0; c0 < A.n; c0 += kRsScanThreads) {
      const int i = c0 + tid;
      const int mem = rs_member(A, i, cut);
      int tot;
      const int r = base + rs_block_scan(mem, RsAdd(), s_int, tot);
      const double t = mem ? rs_term(method, A.p_sorted[i], r, nt, q) : -INFINITY;
      double ctot;
      const double v = fmax(carry, rs_block_scan(t, RsDMax(), s_warp_d, ctot));
      if (i < A.n) A.out[A.order[i]] = mem ? fmin(1.0, v) : nan;
      carry = fmax(carry, ctot);
      base += tot;
    }
    return;
  }
  const bool suffix = method == B200NB_PADJ_BH || method == B200NB_PADJ_BY || method == B200NB_PADJ_HOCHBERG;
  if (!suffix) {                                             // bonferroni / none: elementwise
    for (int i = tid; i < A.n; i += kRsScanThreads) {
      const int mem = rs_member(A, i, cut);
      const double t = mem ? rs_term(method, A.p_sorted[i], 0, nt, q) : nan;
      A.out[A.order[i]] = (mem && method == B200NB_PADJ_BONFERRONI) ? fmin(1.0, t) : t;
    }
    return;
  }
  // suffix min, backward: thread tid of a chunk takes position hi - 1 - tid
  int after = 0;                                             // members at positions past the chunk
  double carry = INFINITY;
  const int chunks = (A.n + kRsScanThreads - 1) / kRsScanThreads;
  for (int ch = chunks - 1; ch >= 0; ch--) {
    const int hi = min(A.n, (ch + 1) * kRsScanThreads);
    const int i = hi - 1 - tid;
    const int mem = i >= ch * kRsScanThreads && rs_member(A, i, cut);
    int tot;
    const int r = nt - (after + rs_block_scan(mem, RsAdd(), s_int, tot)) + 1;
    const double t = mem ? rs_term(method, A.p_sorted[i], r, nt, q) : INFINITY;
    double ctot;
    const double v = fmin(carry, rs_block_scan(t, RsDMin(), s_warp_d, ctot));
    if (i >= ch * kRsScanThreads) A.out[A.order[i]] = mem ? fmin(1.0, v) : nan;
    carry = fmin(carry, ctot);
    after += tot;
  }
}

}  // namespace
}  // namespace nb
