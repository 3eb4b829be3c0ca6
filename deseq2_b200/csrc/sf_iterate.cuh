// sf_iterate.cuh -- the objective of estimateSizeFactorsIterate (R/core.R:2589-2622) and its central differences, for
// all perturbations in one call (included by size_factors.cu, launched through its launch_per_column).
//   fn(p) = sum(gene.ll[gene.ll > quantile(gene.ll, Q)]),  gene.ll_i = sum_j log dnbinom(K_ij; q_ij s_j, 1/alpha_i),
//   s = exp(p - mean(p)).
// optim's gradient (fmingr, no gradient given) needs fn at par + h e_k and par - h e_k for every k; column c of the
// output is fn at: c = 0: par; c = 1 + k: par + h e_k; c = 1 + m + k: par - h e_k.
// Perturbing par_k by +-h scales every s_j by e^{-+h/m} and s_k by a further e^{+-h}, so a gene's log-likelihood at
// column 1 + k is B_i + (t(s_k e^{h - h/m}) - t(s_k e^{-h/m})) with B_i the row sum at the uniform scale e^{-h/m} and
// t the entry's log density (C_i and e^{+h/m} for the minus columns): three row sums per gene (A at scale 1, B, C)
// plus two log densities per perturbation, instead of 2m + 1 row sums.
//   iterate_loglik_kernel   one warp per gene: the gene log-likelihoods of a tile of perturbation columns,
//                           column-major n x tile; the first tile also computes and keeps A / B / C
//   iterate_trim_sum_kernel one CTA per column: R's quantile(type = 7) at Q by an MSB-first radix select of the order
//                           statistics floor(h) and floor(h) + 1 (h = (n - 1) Q, 1-based index 1 + h), then the sum of
//                           the values strictly above it, reduced in a fixed order (two calls give the same bits).
#pragma once
#include "engine.h"
#include "nb_logdens.cuh"

namespace nb {
namespace {

constexpr int kItLlThreads = 256;   // 8 genes per CTA
constexpr int kItSumThreads = 512;

// the entry's log density at mu = mu0 * scale, lmu = lmu0 + lscale; dnbinom_mu's point mass at mu = 0
__device__ __forceinline__ double it_term(double y, double cst, double mu, double lmu, double alpha, double log_alpha,
                                          double r) {
  if (mu == 0.0) return (y == 0.0) ? 0.0 : -INFINITY;
  return cst + nb_logdens_mu(y, mu, lmu, alpha, log_alpha, r);
}

__global__ void __launch_bounds__(kItLlThreads) iterate_loglik_kernel(const SfIterateArgs A, int c0, int tile) {
  init_log_table();
  init_lfact_table();
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (g >= A.n) return;                                      // whole warps leave together
  const size_t off = (size_t)g * A.ld;
  const int m = A.m;
  const double alpha = A.alpha[g];
  const double r = 1.0 / alpha, log_alpha = log(alpha), lg_r = lgamma_pos(r);
  double ps = 0.0;
  for (int j = lane; j < m; j += 32) ps += A.par[j];
  const double pbar = warp_allreduce_sum(ps) / (double)m;
  const double dm = A.h / (double)m;
  const double eB = exp(-dm), eC = exp(dm);                  // uniform scales of the plus / minus columns
  double abc[3];
  if (c0 == 0) {
    abc[0] = abc[1] = abc[2] = 0.0;
    for (int j = lane; j < m; j += 32) {
      const double y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + j]
                                  : (double)static_cast<const int32_t*>(A.y)[off + j];
      const double q = A.q[off + j], ls = A.par[j] - pbar;
      const double cst = lgamma_diff(y, r, lg_r) - log_factorial(y);
      const double mu = q * exp(ls), lmu = log(q) + ls;
      abc[0] += it_term(y, cst, mu, lmu, alpha, log_alpha, r);
      abc[1] += it_term(y, cst, mu * eB, lmu - dm, alpha, log_alpha, r);
      abc[2] += it_term(y, cst, mu * eC, lmu + dm, alpha, log_alpha, r);
    }
    warp_allreduce_sum_n(abc);
    if (lane == 0) {
      A.abc[g] = abc[0];
      A.abc[(size_t)A.n + g] = abc[1];
      A.abc[2 * (size_t)A.n + g] = abc[2];
    }
  } else {
    abc[0] = A.abc[g];
    abc[1] = A.abc[(size_t)A.n + g];
    abc[2] = A.abc[2 * (size_t)A.n + g];
  }
  // columns c0 .. c0 + tile - 1 of [par | par + h e_k | par - h e_k]; entry k serves columns 1 + k and 1 + m + k, so
  // its mu-independent part and log(q) are formed once for both
  const int c1 = c0 + tile;
  if (lane == 0 && c0 == 0) A.ll[g] = abc[0];
  for (int k = lane; k < m; k += 32) {
    const int cp = 1 + k, cm = 1 + m + k;
    const bool wp = cp >= c0 && cp < c1, wm = cm >= c0 && cm < c1;
    if (!wp && !wm) continue;
    const double y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + k]
                                : (double)static_cast<const int32_t*>(A.y)[off + k];
    const double q = A.q[off + k], ls = A.par[k] - pbar;
    const double cst = lgamma_diff(y, r, lg_r) - log_factorial(y);
    const double mu = q * exp(ls), lmu = log(q) + ls;
    if (wp) {                                                // s_k e^{h - h/m}, every other s_j e^{-h/m}
      const double tb = it_term(y, cst, mu * eB, lmu - dm, alpha, log_alpha, r);
      const double tp = it_term(y, cst, mu * exp(A.h - dm), lmu + (A.h - dm), alpha, log_alpha, r);
      A.ll[(size_t)(cp - c0) * A.n + g] = abc[1] + (tp - tb);
    }
    if (wm) {                                                // s_k e^{h/m - h}, every other s_j e^{+h/m}
      const double tb = it_term(y, cst, mu * eC, lmu + dm, alpha, log_alpha, r);
      const double tp = it_term(y, cst, mu * exp(dm - A.h), lmu + (dm - A.h), alpha, log_alpha, r);
      A.ll[(size_t)(cm - c0) * A.n + g] = abc[2] + (tp - tb);
    }
  }
}

// column t of the tile: the n gene log-likelihoods of objective column c0 + t
__global__ void __launch_bounds__(kItSumThreads) iterate_trim_sum_kernel(const SfIterateArgs A, int c0) {
  __shared__ unsigned int hist[256];
  __shared__ unsigned long long s_prefix, s_next;
  __shared__ unsigned int s_k, s_le;
  __shared__ double s_part[kItSumThreads];
  const int n = A.n, tid = threadIdx.x;
  const double* col = A.ll + (size_t)blockIdx.x * n;
  // quantile.default, type 7: index = 1 + (n - 1) Q, lo = floor(index), hi = ceiling(index),
  // qs = x[lo], replaced by (1 - h) x[lo] + h x[hi] when index > lo and x[hi] != x[lo]
  const double index = 1.0 + (double)(n - 1) * A.Q;
  const double lo = floor(index);
  const unsigned int rank = (unsigned int)lo - 1u;           // 0-based rank of x[lo]
  if (tid == 0) s_prefix = 0;
  const unsigned long long k1 = select_key(col, n, rank, hist, s_prefix, s_k);
  const double xlo = value_of(k1);
  double qs = xlo;
  if (index > lo) {
    const double xhi = value_of(next_key(col, n, rank, k1, s_le, s_next));   // x[hi] = x[lo + 1]
    if (xhi != xlo) {
      const double h = index - lo;
      qs = __dadd_rn(__dmul_rn(1.0 - h, xlo), __dmul_rn(h, xhi));   // no contraction: R's rounding
    }
  }
  double s = 0.0;
  for (int i = tid; i < n; i += blockDim.x) {
    const double v = col[i];
    if (v > qs) s += v;
  }
  s_part[tid] = s;
  __syncthreads();
  for (int w = blockDim.x >> 1; w > 0; w >>= 1) {            // fixed-order tree: the same bits on every call
    if (tid < w) s_part[tid] += s_part[tid + w];
    __syncthreads();
  }
  if (tid == 0) A.out[c0 + blockIdx.x] = s_part[0];
}

}  // namespace
}  // namespace nb
