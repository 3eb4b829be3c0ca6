// size_factors.cu -- median-of-ratios size factors on the device (SURVEY.md section 8f row 4).
// Reference: estimateSizeFactorsForMatrix, /root/reference/R/core.R:535-578 (locfunc = median, no geoMeans /
// controlGenes):
//   type "ratio":     loggeomean_i = mean_j log K_ij                 (-Inf as soon as one count of the gene is 0)
//   type "poscounts": loggeomean_i = mean_j [K_ij > 0] log K_ij      (-Inf only for all-zero genes)
//   s_j = exp(median_i { log K_ij - loggeomean_i : loggeomean_i finite and K_ij > 0 })
// Three launches, no host round trip:
//   sf_ratio_kernel   one warp per gene: log ratios into a gene-major n x ld matrix, +Inf where the entry does not
//                     take part; counts the genes with a finite log geometric mean (R stops if there are none)
//   to_col_major      (layout.cu) makes the ratios of one sample contiguous
//   sf_median_kernel  one CTA per sample: exact median by a most-significant-byte-first radix select on the
//                     order-preserving 64-bit image of the doubles (8 histogram passes + one pass for the upper
//                     middle element when the count is even) -- no sort, no scratch beyond 256 shared counters.
// The same one-CTA-per-column radix refinement computes estimateBetaPriorVar's weighted upper quantiles
// (beta_prior_quantile_kernel, beta_prior.cuh) and the trimmed sums of estimateSizeFactorsIterate's objective
// (iterate_trim_sum_kernel, sf_iterate.cuh, whose per-gene kernel starts the same way); all start through
// launch_per_column, as does the transform of the normalized counts (transform_kernel, transform.cuh: VST and
// normTransform), one CTA per block of rows, rlog's fit and prior variance (rlog.cuh: one CTA per block of genes;
// a fixed grid of histogram CTAs and one picking CTA per refinement pass), and results()' per-gene steps, filter
// cutoffs, rejection counts and adjusted p-values (results.cuh: one warp per gene, one CTA per theta).
#include "engine.h"
#include "beta_prior.cuh"
#include "nbmath.cuh"

#include <math.h>

namespace nb {
namespace {

__device__ __forceinline__ unsigned long long key_of(double v) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(v);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);      // ascending doubles <-> ascending unsigned keys
}
__device__ __forceinline__ double value_of(unsigned long long k) {
  const unsigned long long b = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
  return __longlong_as_double((long long)b);
}

// Column order statistics for the one-CTA-per-column kernels (every thread of the CTA calls these; the shared
// variables are the caller's; s_prefix must be 0 on entry).  select_key: the key of 0-based rank `rank` among key_of(col[0..n)), by an MSB-first
// 8-bit radix select (8 histogram passes, 256 shared counters).  next_key: the key of rank rank + 1 given that of rank
// `rank`: k1 again if more than rank + 1 keys are <= k1, otherwise the smallest key above k1.
__device__ __forceinline__ unsigned long long select_key(const double* col, int n, unsigned int rank,
                                                         unsigned int* hist, unsigned long long& s_prefix,
                                                         unsigned int& s_k) {
  const int tid = threadIdx.x;
  if (tid == 0) s_k = rank;
  for (int pass = 7; pass >= 0; pass--) {
    for (int b = tid; b < 256; b += blockDim.x) hist[b] = 0;
    __syncthreads();
    const unsigned long long prefix = s_prefix;
    const unsigned long long mask = (pass == 7) ? 0ull : (~0ull << (8 * (pass + 1)));
    for (int i = tid; i < n; i += blockDim.x) {
      const unsigned long long k = key_of(col[i]);
      if ((k & mask) == prefix) atomicAdd(&hist[(unsigned int)(k >> (8 * pass)) & 255u], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      unsigned int k = s_k, b = 0;
      while (b < 255u && k >= hist[b]) { k -= hist[b]; b++; }   // k < number of keys under this prefix; b is bounded anyway
      s_k = k;
      s_prefix = prefix | ((unsigned long long)b << (8 * pass));
    }
    __syncthreads();
  }
  return s_prefix;
}
__device__ __forceinline__ unsigned long long next_key(const double* col, int n, unsigned int rank,
                                                       unsigned long long k1, unsigned int& s_le,
                                                       unsigned long long& s_next) {
  const int tid = threadIdx.x;
  if (tid == 0) { s_le = 0; s_next = ~0ull; }
  __syncthreads();
  unsigned int le = 0;
  unsigned long long nxt = ~0ull;
  for (int i = tid; i < n; i += blockDim.x) {
    const unsigned long long k = key_of(col[i]);
    le += k <= k1;
    if (k > k1 && k < nxt) nxt = k;
  }
  if (le) atomicAdd(&s_le, le);
  atomicMin(&s_next, nxt);
  __syncthreads();
  return (s_le > rank + 1u) ? k1 : s_next;
}

// DIV: the ratios of K / divisor (estimateNormFactors, R/core.R:2160): log(K/d) - loggeomean, where loggeomean is the
// mean of log(K/d) for "ratio" and log(geoMeanNZ(K)) = log(exp(sum log K[K > 0] / m)) of the raw counts for
// "poscounts" (the geoMeans estimateSizeFactors passes, R/methods.R:377-390)
template <bool DIV>
__global__ void __launch_bounds__(256) sf_ratio_kernel(const SizeFactorArgs A) {
  init_log_table();
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (g >= A.n) return;                                      // whole warps leave together
  const size_t off = (size_t)g * A.ld;
  const double inf = __longlong_as_double(0x7ff0000000000000ll);
  double s = 0.0;
  int zeros = 0, pos = 0;
  for (int j = lane; j < A.m; j += 32) {
    const double y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + j]
                                : (double)static_cast<const int32_t*>(A.y)[off + j];
    if (y > 0.0) {
      if constexpr (DIV) {
        const double l = log(y / A.divisor[off + j]);
        A.ratios[off + j] = l;
        s += A.poscounts ? log_pos(y) : l;
      } else {
        const double l = log_pos(y);
        A.ratios[off + j] = l;                               // log K_ij for now; the mean is subtracted below
        s += l;
      }
      pos++;
    } else {
      zeros++;
    }
  }
  s = warp_allreduce_sum(s);
  zeros = (int)warp_allreduce_sum((double)zeros);
  pos = (int)warp_allreduce_sum((double)pos);
  const bool finite = A.poscounts ? (pos > 0) : (zeros == 0);
  double lg = finite ? s / (double)A.m : -inf;
  if constexpr (DIV)
    if (finite && A.poscounts) lg = log(exp(lg));
  __syncwarp();
  for (int j = lane; j < A.m; j += 32) {
    const double y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + j]
                                : (double)static_cast<const int32_t*>(A.y)[off + j];
    A.ratios[off + j] = (finite && y > 0.0) ? A.ratios[off + j] - lg : inf;
  }
  if (lane == 0) {
    A.loggeomeans[g] = lg;
    if (finite) atomicAdd(A.n_finite, 1);
  }
}

// col: the n ratios of one sample (contiguous); +Inf marks entries that do not take part.
__global__ void __launch_bounds__(512) sf_median_kernel(const double* __restrict__ ratios_colmajor, int n,
                                                        double* __restrict__ size_factors) {
  __shared__ unsigned int hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ unsigned int s_k, s_nv, s_le;
  __shared__ unsigned long long s_next;
  const double* col = ratios_colmajor + (size_t)blockIdx.x * n;
  const int tid = threadIdx.x;
  const unsigned long long kinf = key_of(__longlong_as_double(0x7ff0000000000000ll));
  if (tid == 0) { s_nv = 0; s_prefix = 0; }
  __syncthreads();
  unsigned int mine = 0;
  for (int i = tid; i < n; i += blockDim.x) mine += key_of(col[i]) < kinf;
  if (mine) atomicAdd(&s_nv, mine);
  __syncthreads();
  const unsigned int nv = s_nv;
  if (nv == 0) {                                             // median of nothing: NA in R
    if (tid == 0) size_factors[blockIdx.x] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  const unsigned int rank = (nv - 1) / 2;                    // lower middle element (0-based rank)
  const unsigned long long k1 = select_key(col, n, rank, hist, s_prefix, s_k);
  double med = value_of(k1);
  if ((nv & 1u) == 0) med = 0.5 * (med + value_of(next_key(col, n, rank, k1, s_le, s_next)));   // upper middle
  if (tid == 0) size_factors[blockIdx.x] = exp(med);
}

}  // namespace
}  // namespace nb

#include "sf_iterate.cuh"
#include "transform.cuh"
#include "rlog.cuh"
#include "results.cuh"

namespace nb {
namespace {

// One CTA per column (or per block of rows) with static shared memory only: the launch site of the kernels of this
// file and its headers.
template <class... P, class... A>
cudaError_t launch_per_column(void (*kern)(P...), int columns, int threads, cudaStream_t stream, A... args) {
  kern<<<columns, threads, 0, stream>>>(args...);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_size_factors(const SizeFactorArgs& a, cudaStream_t stream) {
  if (a.n == 0 || a.m == 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(a.n_finite, 0, sizeof(int), stream);
  if (e != cudaSuccess) return e;
  const auto ratio = a.divisor != nullptr ? sf_ratio_kernel<true> : sf_ratio_kernel<false>;
  ratio<<<(a.n + 7) / 8, 256, 0, stream>>>(a);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  e = launch_to_col_major(a.ratios, a.ratios_colmajor, a.n, a.m, a.ld, stream);
  if (e != cudaSuccess) return e;
  return launch_per_column(sf_median_kernel, a.m, 512, stream, a.ratios_colmajor, a.n, a.size_factors);
}

cudaError_t launch_beta_prior_quantile(const BetaPriorQArgs& a, cudaStream_t stream) {
  if (a.k == 0) return cudaSuccess;
  return launch_per_column(beta_prior_quantile_kernel, a.k, kBpThreads, stream, a);
}

cudaError_t launch_sf_iterate_objective(const SfIterateArgs& a, cudaStream_t stream) {
  const int cols = 2 * a.m + 1;
  for (int c0 = 0; c0 < cols; c0 += a.tile) {
    const int t = cols - c0 < a.tile ? cols - c0 : a.tile;
    cudaError_t e = launch_per_column(iterate_loglik_kernel, (a.n + 7) / 8, kItLlThreads, stream, a, c0, t);
    if (e != cudaSuccess) return e;
    e = launch_per_column(iterate_trim_sum_kernel, t, kItSumThreads, stream, a, c0);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t launch_transform(const TransformArgs& a, cudaStream_t stream) {
  if (a.n == 0 || a.m == 0) return cudaSuccess;
  const int rows = transform_rows_per_cta(a.m);
  return launch_per_column(transform_kernel_for(a), (int)(((long long)a.n + rows - 1) / rows), kTfThreads, stream, a,
                           rows);
}

cudaError_t launch_rlog_fit(const RlogFitArgs& a, cudaStream_t stream) {
  if (a.n == 0 || a.m == 0) return cudaSuccess;
  const int genes = rlog_genes_per_cta(a.m);
  return launch_per_column(rlog_fit_kernel_for(a), (int)(((long long)a.n + genes - 1) / genes), kRlThreads, stream, a);
}

size_t rlog_prior_scratch_bytes(int n, int m) {
  int rows = 0, ctas = 0;
  rlog_prior_grid(n, m, rows, ctas);
  return sizeof(RlogPriorState) + (size_t)ctas * kRpPart * sizeof(double);
}

// the scratch (rlog_prior_scratch_bytes) starts at a.st; the partials follow the state
cudaError_t launch_rlog_prior_var(const RlogPriorArgs& a, cudaStream_t stream) {
  RlogPriorArgs b = a;
  rlog_prior_grid(a.n, a.m, b.rows_per_block, b.ctas);
  b.part = reinterpret_cast<double*>(b.st + 1);
  const auto hist = rlog_prior_hist_for(b);
  for (int pass = -1; pass < kBpDigits; pass++) {
    cudaError_t e = launch_per_column(hist, b.ctas, kBpThreads, stream, b, pass);
    if (e != cudaSuccess) return e;
    e = launch_per_column(rlog_prior_pick_kernel, 1, kBpThreads, stream, b, pass);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t launch_results_gene(const ResultsGeneArgs& a, cudaStream_t stream) {
  if (a.n == 0) return cudaSuccess;
  constexpr int genes = kRsThreads / 32;
  return launch_per_column(a.y_is_f64 ? results_gene_kernel<double> : results_gene_kernel<int32_t>,
                           (int)(((long long)a.n + genes - 1) / genes), kRsThreads, stream, a);
}

cudaError_t launch_results_heuristic(const ResultsHeuristicArgs& a, cudaStream_t stream) {
  if (a.k == 0) return cudaSuccess;
  constexpr int genes = kRsThreads / 32;
  return launch_per_column(a.y_is_f64 ? results_heuristic_kernel<double> : results_heuristic_kernel<int32_t>,
                           (a.k + genes - 1) / genes, kRsThreads, stream, a);
}

cudaError_t launch_filter_cutoffs(const FilterCutoffArgs& a, int n_theta, cudaStream_t stream) {
  return launch_per_column(filter_cutoff_kernel, n_theta, kRsScanThreads, stream, a);
}

cudaError_t launch_filter_numrej(const PadjArgs& a, int n_theta, cudaStream_t stream) {
  return launch_per_column(filter_numrej_kernel, n_theta, kRsScanThreads, stream, a);
}

cudaError_t launch_padj(const PadjArgs& a, cudaStream_t stream) {
  return launch_per_column(padj_kernel, 1, kRsScanThreads, stream, a);
}

}  // namespace nb
