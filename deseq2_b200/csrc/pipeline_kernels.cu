// pipeline_kernels.cu -- the per-gene pre-steps that feed the hot path, and the global dispersion-trend fit,
// as device kernels (SURVEY.md section 8f row 2: "host pre-steps on device").  In the reference these are R:
//   getBaseMeansAndVariances  R/core.R:2138-2157      baseMean, baseVar, allZero
//   linearModelMu             R/core.R:2454-2459      (y Q)(x R^-1)'  ==  X (X'X)^-1 X' y
//   roughDispEstimate         R/core.R:2422-2437
//   momentsDispEstimate       R/core.R:2439-2448
//   alpha_hat bounds          R/core.R:716,727-728    min(rough, moments) clamped to [minDisp, max(10, m)]
//   linearModelMuNormalized   R/core.R:2461-2467      mu = linear-model fit * size factor, clamped at minmu
//   beta start values         R/fitNbinomGLMs.R:139-155  QR least squares of log(K/s + 0.1) on X
//   parametricDispersionFit   R/core.R:2166-2189      Gamma GLM (identity link) disp ~ a0 + a1/mean, iterated trimming
// prep_kernel: one warp per gene; the projection P = (X'X)^-1 X' (p x m) is computed once on the host.
// trend_fit_kernel: ONE CTA runs the whole iteratively re-trimmed IRLS on the device (no host round trips).
// With observation weights (template flag W, b200nb_prep_weighted_dev) the same read of the count row also reads the
// raw weight row and adds, from getAndCheckWeights (R/core.R:2697-2752) and the weighted getBaseMeansAndVariances:
//   baseMean / baseVar of w * K/s with the RAW weights (R/core.R:2140-2145); moments dispersion from this pair,
//   rough dispersion and the start values unweighted as in the reference;
//   weights / rowmax(weights) written to an n x ld matrix; rows with a negative / NaN / infinite weight or no positive
//   weight counted into a status word (the reference stops on them: stopifnot, then qr() on NaN);
//   weightsFail = !(rank(w * X) == p && rank(X[w > threshold, nonzero columns]) == ncol), R's qr() rank (LINPACK
//   dqrdc2, tol 1e-7) decided from the two p x p Gram matrices (gram_full_rank).
#include <mutex>

#include "engine.h"
#include "nbmath.cuh"

namespace nb {
namespace {

// Whether R's qr(Z)$rank equals the number of active columns of Z, decided from the Gram matrix A = Z'Z alone (p x p
// row-major in this warp's shared memory, p <= 32; overwritten).  `active`: bit k = column k of Z takes part (the
// rest are left out, as R drops all-zero columns before its second test); nrows: the number of rows of Z.
// dqrdc2 walks the columns in order and moves a column to the end when its norm after the Householder steps so far is
// below tol = 1e-7 times its original norm (1 for a zero column); the rank is then (columns - moved), at most nrows.
// So the rank is full exactly when nrows >= columns and no column is moved.  The squared norm of column c left after
// the steps for the columns before it is the Schur-complement diagonal of A, so an unpivoted elimination that compares
// each diagonal with tol^2 times the original one makes the same decision in exact arithmetic.  In floating point it
// can differ from dqrdc2 only at knife edges: a squared norm ratio within a few dozen ulps of tol^2 (dqrdc2 also
// downdates its column norms instead of recomputing them).
__device__ bool gram_full_rank(double* A, int p, int nrows, unsigned active, int lane) {
  if (nrows < __popc(active)) return false;
  const double tol = 1e-7;
  const double orig = (lane < p) ? A[lane * p + lane] : 0.0;
  for (int c = 0; c < p; c++) {
    if (!((active >> c) & 1u)) continue;
    const double d = A[c * p + c];
    const double oc = __shfl_sync(0xffffffffu, orig, c);
    if (!(d >= tol * tol * (oc == 0.0 ? 1.0 : oc))) return false;   // moved to the end: rank < columns (NaN too)
    if (lane > c && lane < p && ((active >> lane) & 1u)) {
      const double f = A[lane * p + c] / d;
      for (int k = c + 1; k < p; k++)
        if ((active >> k) & 1u) A[lane * p + k] = fma(-f, A[c * p + k], A[lane * p + k]);
    }
    __syncwarp();
  }
  return true;
}

// the columns of a Gram matrix with a non-zero diagonal (R: mm.sub[, colSums(abs(mm.sub)) > 0])
__device__ __forceinline__ unsigned gram_nonzero_columns(const double* A, int p, int lane) {
  return __ballot_sync(0xffffffffu, lane < p && A[lane * p + lane] > 0.0);
}

// per-warp shared-memory doubles the weighted kernels add after the unweighted layout (0 for W = false)
template <bool W>
__host__ __device__ __forceinline__ size_t prep_weighted_extra(int mpad, int p, bool grouped) {
  if constexpr (W) return grouped ? (size_t)p * p + 64 : (size_t)mpad + 2 * (size_t)p * p;
  else return 0;
}

// the divisor of sample j of the gene at row offset off: its normalization factor (NF) or its size factor
template <bool NF>
__device__ __forceinline__ double norm_factor(const double* __restrict__ nf, const double* sf, size_t off, int j) {
  if constexpr (NF) return __ldg(nf + off + j);
  else return sf[j];
}

// the per-gene outputs of the weighted variant (lane 0)
__device__ __forceinline__ void store_weight_flags(const PrepArgs& A, int g, bool invalid, bool ok) {
  A.weights_fail[g] = ok ? 0 : 1;
  if (invalid) atomicAdd(A.status, 1);
}

template <bool W, bool NF>
__global__ void __launch_bounds__(256) prep_kernel(const PrepArgs A) {
  static_assert(!(W && NF), "observation weights together with normalization factors are not supported");
  extern __shared__ __align__(16) double smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int mpad = (A.m + 3) & ~3;
  double* sf = smem;                                   // mpad
  double* wrow = smem + mpad + (size_t)warp * (2 * mpad + 64 + prep_weighted_extra<W>(mpad, A.p, false));
  double* vn = wrow;                                   // normalised counts
  double* vl = wrow + mpad;                            // log(norm + 0.1)
  double* coef = wrow + 2 * mpad;                      // 32: P * norm
  double* coefl = coef + 32;                           // 32: P * log(norm + .1)
  double* wn = coefl + 32;                             // W: mpad, the weights (raw, then normalised)
  double* gram = wn + mpad;                            // W: 2 p x p Gram matrices
  if constexpr (!NF)
    for (int j = threadIdx.x; j < A.m; j += blockDim.x) sf[j] = A.size_factors[j];
  __syncthreads();
  const int g = blockIdx.x * (blockDim.x >> 5) + warp;
  if (g >= A.n) return;
  const size_t off = (size_t)g * A.ld;
  double s = 0.0, s2 = 0.0, raw = 0.0;
  double wmax = 0.0;
  bool bad = false;
  for (int j = lane; j < A.m; j += 32) {
    const double y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + j] : (double)static_cast<const int32_t*>(A.y)[off + j];
    const double v = y / norm_factor<NF>(A.nf, sf, off, j);   // NF: the gene's row, read again for mu_lin
    vn[j] = v;
    vl[j] = log(v + 0.1);
    if constexpr (W) {
      const double w = A.weights[off + j];
      wn[j] = w;
      s += w * v;
      wmax = fmax(wmax, w);
      bad = bad || !(w >= 0.0);
    } else {
      s += v;
    }
    raw += y;
  }
  s = warp_allreduce_sum(s);
  raw = warp_allreduce_sum(raw);
  const double bm = s / (double)A.m;
  for (int j = lane; j < A.m; j += 32) {
    double d;
    if constexpr (W) d = wn[j] * vn[j] - bm;
    else d = vn[j] - bm;
    s2 = fma(d, d, s2);
  }
  s2 = warp_allreduce_sum(s2);
  const double bv = s2 / (double)(A.m - 1);
  __syncwarp();
  // coef = P v: lanes stride over samples (coalesced reads of P), one warp reduction per coefficient
  for (int k = 0; k < A.p; k++) {
    const double* Pk = A.proj + (size_t)k * A.m;
    double c = 0.0, cl = 0.0;
    for (int j = lane; j < A.m; j += 32) {
      const double pk = __ldg(Pk + j);
      c = fma(pk, vn[j], c);
      cl = fma(pk, vl[j], cl);
    }
    c = warp_allreduce_sum(c);
    cl = warp_allreduce_sum(cl);
    if (lane == 0) {
      coef[k] = c;
      coefl[k] = cl;
      if (A.beta0 != nullptr) A.beta0[(size_t)g + (size_t)A.n * k] = cl;
    }
  }
  __syncwarp();
  // fitted = X coef; rough dispersion; linear mu
  double rs = 0.0;
  for (int j = lane; j < A.m; j += 32) {
    double f = 0.0;
    for (int k = 0; k < A.p; k++) f = fma(__ldg(A.x + (size_t)k * A.m + j), coef[k], f);
    const double mu1 = fmax(1.0, f);
    const double d = vn[j] - mu1;
    rs += (d * d - mu1) / (mu1 * mu1);
    if (A.mu_lin != nullptr) A.mu_lin[off + j] = fmax(f * norm_factor<NF>(A.nf, sf, off, j), A.minmu);
  }
  rs = warp_allreduce_sum(rs);
  bool invalid = false, ok = true;
  if constexpr (W) {
    // normalise by the row maximum, then the Gram matrices of w * X and of X on the samples with w > threshold
    wmax = warp_allreduce_max(wmax);
    invalid = __any_sync(0xffffffffu, bad) || !(wmax > 0.0) || !(wmax < INFINITY);
    double kept = 0.0;
    for (int j = lane; j < A.m; j += 32) {
      const double w = wn[j] / wmax;
      wn[j] = w;
      A.weights_norm[off + j] = w;
      kept += (w > A.weight_threshold) ? 1.0 : 0.0;
    }
    for (int j = A.m + lane; j < A.ld; j += 32) A.weights_norm[off + j] = 0.0;
    kept = warp_allreduce_sum(kept);
    __syncwarp();
    const int p = A.p;
    double* g1 = gram;
    double* g2 = gram + p * p;
    for (int a = 0; a < p; a++) {
      for (int b = a; b < p; b++) {
        double t1 = 0.0, t2 = 0.0;
        for (int j = lane; j < A.m; j += 32) {
          const double xx = __ldg(A.x + (size_t)a * A.m + j) * __ldg(A.x + (size_t)b * A.m + j);
          const double w = wn[j];
          t1 = fma(w * w, xx, t1);
          if (w > A.weight_threshold) t2 += xx;
        }
        t1 = warp_allreduce_sum(t1);
        t2 = warp_allreduce_sum(t2);
        if (lane == 0) {
          g1[a * p + b] = g1[b * p + a] = t1;
          g2[a * p + b] = g2[b * p + a] = t2;
        }
      }
    }
    __syncwarp();
    const unsigned act2 = gram_nonzero_columns(g2, p, lane);
    ok = gram_full_rank(g1, p, A.m, (p == 32) ? 0xffffffffu : ((1u << p) - 1u), lane);
    ok = gram_full_rank(g2, p, (int)kept, act2, lane) && ok;
  }
  if (lane == 0) {
    const double rough = fmax(rs / (double)(A.m - A.p), 0.0);
    const double moments = (bv - A.xim * bm) / (bm * bm);
    double a0 = fmin(rough, moments);
    a0 = fmin(fmax(A.min_disp, a0), A.max_disp);   // pmin(pmax(minDisp, alpha_hat), maxDisp): NaN -> minDisp like pmax
    A.base_mean[g] = bm;
    A.base_var[g] = bv;
    A.alpha0[g] = a0;
    A.all_zero[g] = (raw == 0.0) ? 1 : 0;
    if constexpr (W) store_weight_flags(A, g, invalid, ok);
  }
}

// The same pre-steps for a design with G <= 32 distinct rows (factor designs: config 4 has m = 1000, p = 10, G = 10).
// prep_kernel streams the p x m projection and the m x p design through every gene (2 p m loads and FMAs per gene,
// L2 latency bound at 8 warps per SM); here a sample only adds its value and its log to its
// group's lane-private slot, the projection is applied to the G group sums and the fitted value is read per group.
template <bool W, bool NF>
__global__ void __launch_bounds__(256) prep_grouped_kernel(const PrepArgs A, int mpad, int ps) {
  static_assert(!(W && NF), "observation weights together with normalization factors are not supported");
  extern __shared__ __align__(16) double smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int G = A.G, p = A.p;
  double* sf = smem;                                   // mpad
  double* Pg = sf + mpad;                              // p x G: the projection's column of each group
  double* xg = Pg + (size_t)p * G;                     // G x ps
  int* rep = reinterpret_cast<int*>(xg + (size_t)G * ps);          // 32: one sample of each group
  unsigned char* gidb = reinterpret_cast<unsigned char*>(rep + 32);   // mpad
  double* wrow = reinterpret_cast<double*>(gidb + mpad) +
                 (size_t)warp * (mpad + 2 * (size_t)G * 32 + 3 * 32 + 2 * 32 + prep_weighted_extra<W>(mpad, p, true) +
                                 (NF ? mpad : 0));
  double* vn = wrow;                                   // normalised counts
  double* accN = wrow + mpad;                          // G x 32 lane-private sums of the normalised counts
  double* accL = accN + (size_t)G * 32;                // G x 32: of log(norm + 0.1)
  double* gsN = accL + (size_t)G * 32;                 // 32: group sums
  double* gsL = gsN + 32;
  double* fit = gsL + 32;                              // 32: fitted value of each group
  double* coef = fit + 32;                             // 32: P * norm
  double* coefl = coef + 32;                           // 32: P * log(norm + .1)
  double* gsW = coefl + 32;                            // W, 32: group sums of the squared normalised weights
  double* gsC = gsW + 32;                              // W, 32: group counts of normalised weights > threshold
  double* gram = gsC + 32;                             // W: p x p Gram matrix
  double* nfw = coefl + 32;                            // NF: mpad, the gene's normalization factors
  for (int j = threadIdx.x; j < A.m; j += blockDim.x) {
    if constexpr (!NF) sf[j] = A.size_factors[j];
    const int g = A.gid[j];
    gidb[j] = (unsigned char)g;
    rep[g] = j;                                        // any sample of the group (racing writers, all valid)
  }
  for (int i = threadIdx.x; i < G * ps; i += blockDim.x) xg[i] = A.xg[i];
  __syncthreads();
  for (int i = threadIdx.x; i < p * G; i += blockDim.x) Pg[i] = A.proj[(size_t)(i / G) * A.m + rep[i % G]];
  __syncthreads();
  const int g = blockIdx.x * (blockDim.x >> 5) + warp;
  if (g >= A.n) return;
  const size_t off = (size_t)g * A.ld;
  for (int t = 0; t < G; t++) {
    accN[t * 32 + lane] = 0.0;
    accL[t * 32 + lane] = 0.0;
  }
  double s = 0.0, s2 = 0.0, raw = 0.0;
  double wmax = 0.0;
  bool bad = false;
  // NF: the gene's factors go to a per-warp shared row first (each lane its own entries), so that the loops below
  // keep no more live state than with size factors (a second read of the global row spilled)
  if constexpr (NF)
    for (int j = lane; j < A.m; j += 32) nfw[j] = A.nf[off + j];
  const double* nfr = NF ? nfw : sf;
  for (int j = lane; j < A.m; j += 32) {
    const double y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + j] : (double)static_cast<const int32_t*>(A.y)[off + j];
    const double v = y / nfr[j];                       // NF: group sums of K/nf, fits scaled by nf_ij
    vn[j] = v;
    const int slot = gidb[j] * 32 + lane;
    accN[slot] += v;
    accL[slot] += log(v + 0.1);
    if constexpr (W) {
      const double w = A.weights[off + j];
      s += w * v;
      wmax = fmax(wmax, w);
      bad = bad || !(w >= 0.0);
    } else {
      s += v;
    }
    raw += y;
  }
  s = warp_allreduce_sum(s);
  raw = warp_allreduce_sum(raw);
  const double bm = s / (double)A.m;
  for (int j = lane; j < A.m; j += 32) {
    double d;
    if constexpr (W) d = A.weights[off + j] * vn[j] - bm;     // the row is in L1 from the pass above
    else d = vn[j] - bm;
    s2 = fma(d, d, s2);
  }
  s2 = warp_allreduce_sum(s2);
  const double bv = s2 / (double)(A.m - 1);
  __syncwarp();
  if (lane < G) {
    double a = 0.0, b = 0.0;
    for (int l = 0; l < 32; l++) {
      a += accN[lane * 32 + ((l + lane) & 31)];
      b += accL[lane * 32 + ((l + lane) & 31)];
    }
    gsN[lane] = a;
    gsL[lane] = b;
  }
  __syncwarp();
  if (lane < p) {
    double c = 0.0, cl = 0.0;
    for (int t = 0; t < G; t++) {
      c = fma(Pg[lane * G + t], gsN[t], c);
      cl = fma(Pg[lane * G + t], gsL[t], cl);
    }
    coef[lane] = c;
    coefl[lane] = cl;
    if (A.beta0 != nullptr) A.beta0[(size_t)g + (size_t)A.n * lane] = cl;
  }
  __syncwarp();
  if (lane < G) {
    double f = 0.0;
    for (int k = 0; k < p; k++) f = fma(xg[lane * ps + k], coef[k], f);
    fit[lane] = f;
  }
  __syncwarp();
  double rs = 0.0;
  for (int j = lane; j < A.m; j += 32) {
    const double f = fit[gidb[j]];
    const double mu1 = fmax(1.0, f);
    const double d = vn[j] - mu1;
    rs += (d * d - mu1) / (mu1 * mu1);
    if (A.mu_lin != nullptr) A.mu_lin[off + j] = fmax(f * nfr[j], A.minmu);
  }
  rs = warp_allreduce_sum(rs);
  bool invalid = false, ok = true;
  if constexpr (W) {
    // normalise by the row maximum; the Gram matrices need only each group's sum of w^2 and count of w > threshold
    // (the lane-private slots are free again: their group sums were taken above)
    wmax = warp_allreduce_max(wmax);
    invalid = __any_sync(0xffffffffu, bad) || !(wmax > 0.0) || !(wmax < INFINITY);
    for (int t = 0; t < G; t++) {
      accN[t * 32 + lane] = 0.0;
      accL[t * 32 + lane] = 0.0;
    }
    for (int j = lane; j < A.m; j += 32) {
      const double w = A.weights[off + j] / wmax;
      A.weights_norm[off + j] = w;
      const int slot = gidb[j] * 32 + lane;
      accN[slot] = fma(w, w, accN[slot]);
      accL[slot] += (w > A.weight_threshold) ? 1.0 : 0.0;
    }
    for (int j = A.m + lane; j < A.ld; j += 32) A.weights_norm[off + j] = 0.0;
    __syncwarp();
    if (lane < G) {
      double a = 0.0, b = 0.0;
      for (int l = 0; l < 32; l++) {
        a += accN[lane * 32 + ((l + lane) & 31)];
        b += accL[lane * 32 + ((l + lane) & 31)];
      }
      gsW[lane] = a;
      gsC[lane] = b;
    }
    __syncwarp();
    double kept = 0.0;
    for (int t = 0; t < G; t++) kept += gsC[t];
    // lane b builds column b of sum_t c_t x_t x_t' (x_t: the distinct design rows), first c = w^2, then c = count
    for (int pass = 0; pass < 2; pass++) {
      const double* c = pass == 0 ? gsW : gsC;
      if (lane < p)
        for (int a = 0; a < p; a++) {
          double t1 = 0.0;
          for (int t = 0; t < G; t++) t1 = fma(c[t] * xg[t * ps + a], xg[t * ps + lane], t1);
          gram[a * p + lane] = t1;
        }
      __syncwarp();
      const bool full = pass == 0 ? gram_full_rank(gram, p, A.m, (p == 32) ? 0xffffffffu : ((1u << p) - 1u), lane)
                                  : gram_full_rank(gram, p, (int)kept, gram_nonzero_columns(gram, p, lane), lane);
      ok = ok && full;
      __syncwarp();
    }
  }
  if (lane == 0) {
    const double rough = fmax(rs / (double)(A.m - A.p), 0.0);
    const double moments = (bv - A.xim * bm) / (bm * bm);
    double a0 = fmin(rough, moments);
    a0 = fmin(fmax(A.min_disp, a0), A.max_disp);   // pmin(pmax(minDisp, alpha_hat), maxDisp): NaN -> minDisp like pmax
    A.base_mean[g] = bm;
    A.base_var[g] = bv;
    A.alpha0[g] = a0;
    A.all_zero[g] = (raw == 0.0) ? 1 : 0;
    if constexpr (W) store_weight_flags(A, g, invalid, ok);
  }
}

// ---------------------------------------------------------------- dispersion trend (one CTA per SM, grid barrier)
// The fit is a sequence of full passes over all genes (five weighted sums, then the deviance), dozens of them, each
// needing the previous one's result: a single CTA spends ~0.25 ms per pass at a million genes (config 5 on 8 GPUs: the
// global step is on ALL genes, 15 ms).  Here every CTA reduces a slice, writes its partial sums to a double-buffered
// global slot, the grid meets at a counter barrier, and every CTA then adds the partials in the same fixed order, so
// all CTAs carry bit-identical coefficients and take the same branches.  The launch is cooperative (co-residency is
// guaranteed or the launch fails; no spinning on CTAs that were never scheduled).
constexpr int kTrendVals = 5;
struct TrendGrid {
  double* part;          // [2][gridDim.x][kTrendVals]
  unsigned int* bar;     // arrival counter, zeroed before the launch
  double* red;           // shared: 32 * kTrendVals + kTrendVals
  unsigned int phase;
};

// v[0..K) summed over the whole grid; every thread of every CTA returns with the same totals in v
template <int K>
__device__ __forceinline__ void grid_sum(TrendGrid& G, double (&v)[K]) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int ncta = gridDim.x;
#pragma unroll
  for (int k = 0; k < K; k++) v[k] = warp_allreduce_sum(v[k]);
  __syncthreads();   // the previous call's totals in red[] have been read by everybody
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < K; k++) G.red[warp * kTrendVals + k] = v[k];
  __syncthreads();
  double* slot = G.part + ((size_t)(G.phase & 1u) * ncta + blockIdx.x) * kTrendVals;
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < K; k++) {
      double t = (lane < nw) ? G.red[lane * kTrendVals + k] : 0.0;
      t = warp_allreduce_sum(t);
      if (lane == 0) slot[k] = t;
    }
    if (ncta > 1) {
      if (lane == 0) {
        __threadfence();
        atomicAdd(G.bar, 1u);
        const unsigned int want = (G.phase + 1u) * (unsigned int)ncta;
        while (*reinterpret_cast<volatile unsigned int*>(G.bar) < want) {}
        __threadfence();
      }
      __syncwarp();
    }
    const double* base = G.part + (size_t)(G.phase & 1u) * ncta * kTrendVals;
#pragma unroll
    for (int k = 0; k < K; k++) {
      double t = 0.0;
      for (int c = lane; c < ncta; c += 32) t += __ldcg(base + (size_t)c * kTrendVals + k);
      t = warp_allreduce_sum(t);
      if (lane == 0) G.red[32 * kTrendVals + k] = t;
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; k++) v[k] = G.red[32 * kTrendVals + k];
  G.phase++;
}

// out[0..1] = coefficients (asymptDisp, extraPois); out[2] = status (0 ok, 1 not converged, 2 non-positive
// coefficients, 3 no usable genes); out[3] = outer iterations used.
__global__ void __launch_bounds__(512) trend_fit_kernel(const double* __restrict__ means,
                                                         const double* __restrict__ disps, int n, double min_disp,
                                                         double* __restrict__ out, double* part, unsigned int* bar) {
  __shared__ double red[33 * kTrendVals];
  TrendGrid G{part, bar, red, 0u};
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gnt = gridDim.x * blockDim.x;
  double c0 = 0.1, c1 = 1.0;
  int status = 1, outer = 0;
  for (; outer <= 10; outer++) {   // R: iter > 10 => "dispersion fit did not converge"
    // glm(disps[good] ~ I(1/means[good]), Gamma(identity), start = coefs): IRLS, weights 1/mu^2, response y
    const double t0 = c0, t1 = c1;   // trimming uses the coefficients at loop entry
    double b0 = c0, b1 = c1;
    double dev_old;
    {
      double a[2] = {0.0, 0.0};   // deviance, count
      for (int i = gtid; i < n; i += gnt) {
        const double d = disps[i], mn = means[i];
        if (!(d > 100.0 * min_disp)) continue;
        const double resid = d / (t0 + t1 / mn);
        if (!(resid > 1e-4 && resid < 15.0)) continue;
        const double mu = b0 + b1 / mn;
        a[0] += -log(d / mu) + (d - mu) / mu;
        a[1] += 1.0;
      }
      grid_sum(G, a);
      dev_old = 2.0 * a[0];
      if (a[1] < 2.0) { status = 3; break; }
    }
    bool converged = false, bad = false;
    for (int it = 0; it < 25; it++) {
      double sv[5] = {0.0, 0.0, 0.0, 0.0, 0.0};   // sw, swx, swxx, swy, swxy
      for (int i = gtid; i < n; i += gnt) {
        const double d = disps[i], mn = means[i];
        if (!(d > 100.0 * min_disp)) continue;
        const double resid = d / (t0 + t1 / mn);
        if (!(resid > 1e-4 && resid < 15.0)) continue;
        const double xi = 1.0 / mn;
        const double mu = b0 + b1 * xi;
        const double w = 1.0 / (mu * mu);
        sv[0] += w; sv[1] += w * xi; sv[2] += w * xi * xi; sv[3] += w * d; sv[4] += w * xi * d;
      }
      grid_sum(G, sv);
      const double sw = sv[0], swx = sv[1], swxx = sv[2], swy = sv[3], swxy = sv[4];
      const double det = sw * swxx - swx * swx;
      b0 = (swxx * swy - swx * swxy) / det;
      b1 = (sw * swxy - swx * swy) / det;
      double a[2] = {0.0, 0.0};   // deviance, number of non-positive means
      for (int i = gtid; i < n; i += gnt) {
        const double d = disps[i], mn = means[i];
        if (!(d > 100.0 * min_disp)) continue;
        const double resid = d / (t0 + t1 / mn);
        if (!(resid > 1e-4 && resid < 15.0)) continue;
        const double mu = b0 + b1 / mn;
        if (!(mu > 0.0)) a[1] += 1.0;
        a[0] += -log(d / mu) + (d - mu) / mu;
      }
      grid_sum(G, a);
      const double dev = 2.0 * a[0];
      if (a[1] > 0.0) { bad = true; break; }
      if (fabs(dev - dev_old) / (fabs(dev) + 0.1) < 1e-8) { converged = true; break; }
      dev_old = dev;
    }
    if (bad || !(b0 > 0.0) || !(b1 > 0.0)) { status = 2; c0 = b0; c1 = b1; break; }
    const double l0 = log(b0 / c0), l1 = log(b1 / c1);
    c0 = b0;
    c1 = b1;
    if ((l0 * l0 + l1 * l1 < 1e-6) && converged) { status = 0; break; }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    out[0] = c0;
    out[1] = c1;
    out[2] = (double)status;
    out[3] = (double)outer;
  }
}

}  // namespace

// a.weights != nullptr selects the weighted instantiations (their larger per-warp scratch may run fewer warps per
// CTA), a.nf != nullptr the normalization-factor ones (the grouped one adds an mpad row per warp; the shared
// size-factor row goes unused)
cudaError_t launch_prep(const PrepArgs& a, cudaStream_t stream) {
  if (a.n == 0) return cudaSuccess;
  const bool weighted = a.weights != nullptr;
  const bool nf = a.nf != nullptr;
  if (a.G > 0 && a.G <= 32) {
    const int mpad = (a.m + 7) & ~7, ps = a.p | 1;
    int warps = 8;
    const size_t fixed = ((size_t)mpad + (size_t)a.p * a.G + (size_t)a.G * ps) * sizeof(double) + 32 * sizeof(int) + mpad;
    const size_t per_warp = ((size_t)mpad + 2 * (size_t)a.G * 32 + 5 * 32 +
                             (weighted ? prep_weighted_extra<true>(mpad, a.p, true) : 0) + (nf ? mpad : 0)) *
                            sizeof(double);
    size_t smem = fixed + warps * per_warp;
    while ((weighted || nf) && warps > 1 && smem > 200 * 1024) {
      warps >>= 1;
      smem = fixed + warps * per_warp;
    }
    if (smem <= 200 * 1024) {
      const auto kern = weighted ? prep_grouped_kernel<true, false>
                                 : (nf ? prep_grouped_kernel<false, true> : prep_grouped_kernel<false, false>);
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
      kern<<<(a.n + warps - 1) / warps, warps * 32, smem, stream>>>(a, mpad, ps);
      return cudaGetLastError();
    }
  }
  const int mpad = (a.m + 3) & ~3;
  const size_t per_warp = 2 * (size_t)mpad + 64 + (weighted ? prep_weighted_extra<true>(mpad, a.p, false) : 0);
  int warps = 8;
  size_t smem = ((size_t)mpad + (size_t)warps * per_warp) * sizeof(double);
  while (warps > 1 && smem > 200 * 1024) {
    warps >>= 1;
    smem = ((size_t)mpad + (size_t)warps * per_warp) * sizeof(double);
  }
  const auto kern = weighted ? prep_kernel<true, false> : (nf ? prep_kernel<false, true> : prep_kernel<false, false>);
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<(a.n + warps - 1) / warps, warps * 32, smem, stream>>>(a);
  return cudaGetLastError();
}

// scratch of the grid reduction: partial sums of every CTA (double-buffered) + the barrier counter.  One buffer per
// process (the device pipeline runs on one stream); trend fits on two streams at once are serialised by the mutex only
// up to the launch, so callers must not overlap them.
cudaError_t launch_trend_fit(const double* means, const double* disps, int n, double min_disp, double* out,
                             cudaStream_t stream) {
  static std::mutex mu;
  static void* scratch = nullptr;
  constexpr int kMaxCtas = 256;
  constexpr size_t kPartBytes = 2 * (size_t)kMaxCtas * kTrendVals * sizeof(double);
  std::lock_guard<std::mutex> lk(mu);
  if (scratch == nullptr) {
    cudaError_t e = cudaMalloc(&scratch, kPartBytes + 256);
    if (e != cudaSuccess) return e;
  }
  double* part = static_cast<double*>(scratch);
  unsigned int* bar = reinterpret_cast<unsigned int*>(static_cast<char*>(scratch) + kPartBytes);
  cudaError_t e = cudaMemsetAsync(bar, 0, sizeof(unsigned int), stream);
  if (e != cudaSuccess) return e;
#ifdef SIMT_EMU
  // the emulator runs the CTAs of a grid one after the other: a grid barrier needs the one-CTA grid
  trend_fit_kernel<<<1, 512, 0, stream>>>(means, disps, n, min_disp, out, part, bar);
  return cudaGetLastError();
#else
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, trend_fit_kernel, 512, 0);
  if (e != cudaSuccess) return e;
  if (per_sm < 1) return cudaErrorLaunchOutOfResources;
  int grid = (n + 2047) / 2048;                 // at least four genes per thread before another CTA pays its barrier
  const int cap = device_sm_count() < kMaxCtas ? device_sm_count() : kMaxCtas;
  if (grid > cap) grid = cap;
  if (grid < 1) grid = 1;
  void* args[] = {(void*)&means, (void*)&disps, (void*)&n, (void*)&min_disp, (void*)&out, (void*)&part, (void*)&bar};
  return cudaLaunchCooperativeKernel((const void*)trend_fit_kernel, dim3(grid), dim3(512), args, 0, stream);
#endif
}

}  // namespace nb

// ================================================================ Cook's distances (SURVEY.md section 8f row 1)
// R/core.R:2277-2359: robustMethodOfMomentsDisp (per-cell trimmed mean, trimmed mean of squared errors, max over
// cells), Cook's distance from the hat diagonal, and the per-gene maximum over samples with >= 3 replicates in
// their cell.  One warp per gene.  The trimmed means need the floor(n*trim) smallest and largest values of a cell:
// they are extracted one at a time with a warp arg-min / arg-max over the lanes' unmarked candidates (cells have
// tens to hundreds of samples, floor(n/8) extractions), which avoids a full sort.
namespace nb {
namespace {

// mean of vals[list[0..n)] after removing its k smallest and k largest entries (k = floor(n * trim), trim < 0.5).
// Each round removes the current minimum AND the current maximum among the unmarked candidates (one scan, two
// interleaved warp arg-reductions; ties: lowest index for the minimum, highest for the maximum, so the two are
// distinct while at least two candidates remain).  `taken`: n-byte scratch in shared memory.
__device__ __forceinline__ double trimmed_mean_list(const double* vals, const int* list, int n, int k,
                                                    unsigned char* taken, int lane) {
  double tot = 0.0;
  for (int i = lane; i < n; i += 32) {
    tot += vals[list[i]];
    taken[i] = 0;
  }
  tot = warp_allreduce_sum(tot);
  __syncwarp();
  double removed = 0.0;
  for (int round = 0; round < k; round++) {
    double lo = 1e308, hi = -1e308;
    int ilo = 0x7fffffff, ihi = -1;
    for (int i = lane; i < n; i += 32) {
      if (taken[i]) continue;
      const double v = vals[list[i]];
      if (v < lo) { lo = v; ilo = i; }
      if (v >= hi) { hi = v; ihi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double olo = __shfl_xor_sync(0xffffffffu, lo, o);
      const int oilo = __shfl_xor_sync(0xffffffffu, ilo, o);
      const double ohi = __shfl_xor_sync(0xffffffffu, hi, o);
      const int oihi = __shfl_xor_sync(0xffffffffu, ihi, o);
      if (olo < lo || (olo == lo && oilo < ilo)) { lo = olo; ilo = oilo; }
      if (ohi > hi || (ohi == hi && oihi > ihi)) { hi = ohi; ihi = oihi; }
    }
    removed += lo + hi;
    if (lane == (ilo & 31)) taken[ilo] = 1;   // candidate i is owned by lane i % 32
    if (lane == (ihi & 31)) taken[ihi] = 1;
    __syncwarp();
  }
  return (tot - removed) / (double)(n - 2 * k);
}

// The same trimmed mean for a COMPACT list cv[0..n), n <= 32 NQ <= 256, by rank counting: every lane owns NQ entries
// and counts, for each, the entries that precede it in the total order (value, index) -- one broadcast load and NQ
// integer compares per visited entry, all independent, no warp reduction per removed value (the extraction above is a
// serial chain of k five-level shuffle reductions: ncu on the config-4 shape, 100 samples per cell, showed the
// Cook's kernel bound by that latency).  Values are non-negative doubles, so their bit patterns order like the
// values; "v_j precedes v_i" is bits_j < bits_i + [j < i], and [j < i] depends only on the 32-entry blocks of j and i
// and, inside the same block, on the lanes.  Entries of rank in [k, n - k) are kept and summed.
template <int NQ>
__device__ __forceinline__ double trimmed_mean_rank(const double* cv, int n, int k, int lane) {
  unsigned long long thr0[NQ], thr1[NQ];
  double own[NQ];
  int rank[NQ];
#pragma unroll
  for (int q = 0; q < NQ; q++) {
    const int i = lane + 32 * q;
    own[q] = (i < n) ? cv[i] : 0.0;
    thr0[q] = (unsigned long long)__double_as_longlong(own[q]);
    thr1[q] = thr0[q] + 1ull;
    rank[q] = 0;
  }
#pragma unroll
  for (int b = 0; b < NQ; b++) {
    const int jn = (n - 32 * b < 32) ? n - 32 * b : 32;   // warp-uniform
    for (int jl = 0; jl < jn; jl++) {
      const unsigned long long vb = (unsigned long long)__double_as_longlong(cv[32 * b + jl]);
#pragma unroll
      for (int q = 0; q < NQ; q++) {
        const unsigned long long thr = (q > b) ? thr1[q] : ((q < b) ? thr0[q] : ((jl < lane) ? thr1[q] : thr0[q]));
        rank[q] += (vb < thr) ? 1 : 0;
      }
    }
  }
  double s = 0.0;
#pragma unroll
  for (int q = 0; q < NQ; q++)
    if (lane + 32 * q < n && rank[q] >= k && rank[q] < n - k) s += own[q];
  return warp_allreduce_sum(s) / (double)(n - 2 * k);
}
__device__ __forceinline__ double trimmed_mean_compact(const double* cv, int n, int k, int lane) {
  if (n <= 32) return trimmed_mean_rank<1>(cv, n, k, lane);
  if (n <= 64) return trimmed_mean_rank<2>(cv, n, k, lane);
  if (n <= 128) return trimmed_mean_rank<4>(cv, n, k, lane);
  return trimmed_mean_rank<8>(cv, n, k, lane);
}

__device__ __forceinline__ int trim_bin(int n) { return n <= 3 ? 0 : (n <= 23 ? 1 : 2); }

// per-warp scratch: the row of normalised counts, `sqlen` doubles for the values / squared errors of one cell (the whole
// row when a cell has more than 256 samples or the cell sizes are unknown: extraction path), `taken` flags likewise
__host__ __device__ inline int cooks_sqlen(int m, int mpad, int max_cell) {
  // max_cell < 3: no cell has three replicates and the whole row is trimmed at once (needs the full scratch)
  return (max_cell >= 3 && max_cell <= 256 && m > 256) ? 256 : mpad;
}
__host__ __device__ inline size_t cooks_warp_doubles(int m, int mpad, int max_cell) {
  const int sqlen = cooks_sqlen(m, mpad, max_cell);
  return (size_t)mpad + sqlen + (sqlen == mpad ? (mpad + 7) / 8 : 0);
}

// NF: the robust dispersion and the trimmed means are of K/nf (gene-major nf); otherwise of K/s (shared s)
template <bool NF>
__global__ void __launch_bounds__(256) cooks_kernel(const CooksArgs A) {
  extern __shared__ __align__(16) double smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int mpad = (A.m + 3) & ~3;
  const int sqlen = cooks_sqlen(A.m, mpad, A.max_cell);
  int* cell_ptr = reinterpret_cast<int*>(smem);                 // ncell + 1
  int* cell_samples = cell_ptr + A.ncell + 1;                   // m
  double* sf = smem + ((A.ncell + 1 + A.m + 1) / 2 + 1);        // mpad
  double* wbase = sf + mpad + (size_t)warp * cooks_warp_doubles(A.m, mpad, A.max_cell);
  double* vn = wbase;                                           // normalised counts
  double* sq = wbase + mpad;                                    // one cell's values, then its squared errors
  unsigned char* taken = reinterpret_cast<unsigned char*>(wbase + mpad + sqlen);   // extraction path only
  for (int i = threadIdx.x; i <= A.ncell; i += blockDim.x) cell_ptr[i] = A.cell_ptr[i];
  for (int i = threadIdx.x; i < A.m; i += blockDim.x) {
    cell_samples[i] = A.cell_samples[i];
    if constexpr (!NF) sf[i] = A.size_factors[i];
  }
  __syncthreads();
  const double trimratio[3] = {1.0 / 3.0, 1.0 / 4.0, 1.0 / 8.0};
  const double scale_c[3] = {2.04, 1.86, 1.51};
  const int g = blockIdx.x * (blockDim.x >> 5) + warp;
  if (g >= A.n) return;
  const size_t off = (size_t)g * A.ld;
  double s = 0.0;
  if constexpr (NF)                                             // staged in vn and divided in place (as in prep)
    for (int j = lane; j < A.m; j += 32) vn[j] = A.nf[off + j];
  for (int j = lane; j < A.m; j += 32) {
    const double y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + j] : (double)static_cast<const int32_t*>(A.y)[off + j];
    const double v = y / (NF ? vn[j] : sf[j]);
    vn[j] = v;
    s += v;
  }
  const double mean = warp_allreduce_sum(s) / (double)A.m;
  __syncwarp();
  double vmax = -1e308;
  bool any3 = false;
  for (int c = 0; c < A.ncell; c++) {
    const int lo = cell_ptr[c], nc = cell_ptr[c + 1] - lo;
    if (nc < 3) continue;
    any3 = true;
    const int tb = trim_bin(nc);
    const int k = (int)floor((double)nc * trimratio[tb]);
    double ve;
    if (nc <= 256) {
      // the cell's values, compact, in the `sq` row; squared errors in place for the second trimmed mean
      __syncwarp();
      for (int i = lane; i < nc; i += 32) sq[i] = vn[cell_samples[lo + i]];
      __syncwarp();
      const double cm = trimmed_mean_compact(sq, nc, k, lane);
      for (int i = lane; i < nc; i += 32) {
        const double d = sq[i] - cm;
        sq[i] = d * d;
      }
      __syncwarp();
      ve = scale_c[tb] * trimmed_mean_compact(sq, nc, k, lane);
    } else {
      const double cm = trimmed_mean_list(vn, cell_samples + lo, nc, k, taken, lane);
      for (int i = lane; i < nc; i += 32) {
        const int j = cell_samples[lo + i];
        const double d = vn[j] - cm;
        sq[j] = d * d;
      }
      __syncwarp();
      ve = scale_c[tb] * trimmed_mean_list(sq, cell_samples + lo, nc, k, taken, lane);
    }
    vmax = fmax(vmax, ve);
  }
  if (!any3) {
    // trimmedVariance over all samples (R/core.R:2327-2332); cell_samples is a permutation of 0..m-1
    const int k = (int)floor((double)A.m / 8.0);
    const bool small = A.m <= 256;   // vn[0..m) is the compact list itself
    const double rm = small ? trimmed_mean_compact(vn, A.m, k, lane) : trimmed_mean_list(vn, cell_samples, A.m, k, taken, lane);
    for (int j = lane; j < A.m; j += 32) {
      const double d = vn[j] - rm;
      sq[j] = d * d;
    }
    __syncwarp();
    vmax = 1.51 * (small ? trimmed_mean_compact(sq, A.m, k, lane) : trimmed_mean_list(sq, cell_samples, A.m, k, taken, lane));
  }
  const double alpha_r = fmax((vmax - mean) / (mean * mean), 0.04);
  // Cook's distance and its maximum over samples in cells with >= 3 replicates
  double mx = -1e308;
  for (int c = 0; c < A.ncell; c++) {
    const int lo = cell_ptr[c], nc = cell_ptr[c + 1] - lo;
    for (int i = lane; i < nc; i += 32) {
      const int j = cell_samples[lo + i];
      const double y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + j] : (double)static_cast<const int32_t*>(A.y)[off + j];
      const double mu = A.mu[off + j], h = A.hat[off + j];
      const double V = mu + alpha_r * mu * mu;
      const double d = y - mu;
      const double ck = d * d / V / (double)A.p * h / ((1.0 - h) * (1.0 - h));
      if (A.cooks != nullptr) A.cooks[off + j] = ck;
      if (nc >= 3) mx = fmax(mx, ck);
    }
  }
  mx = warp_allreduce_max(mx);
  if (lane == 0) {
    A.robust_disp[g] = alpha_r;
    A.max_cooks[g] = (any3 && A.m > A.p) ? mx : nan("");
  }
}

}  // namespace

cudaError_t launch_cooks(const CooksArgs& a, cudaStream_t stream) {
  if (a.n == 0) return cudaSuccess;
  const int mpad = (a.m + 3) & ~3;
  auto bytes = [&](int w) {
    return (((size_t)(a.ncell + 1 + a.m + 1) / 2 + 1) + mpad + (size_t)w * cooks_warp_doubles(a.m, mpad, a.max_cell)) *
           sizeof(double);
  };
  // several CTAs per SM: 4 warps each, 8 when the per-warp scratch is small enough for two such CTAs
  int warps = (2 * bytes(8) <= 220 * 1024) ? 8 : 4;
  while (warps > 1 && bytes(warps) > 200 * 1024) warps >>= 1;
  const size_t smem = bytes(warps);
  const auto kern = a.nf != nullptr ? cooks_kernel<true> : cooks_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<(a.n + warps - 1) / warps, warps * 32, smem, stream>>>(a);
  return cudaGetLastError();
}

}  // namespace nb
