// rlog.cuh -- rlogData (R/rlog.R:172-272) on the device: its one fitNbinomGLMs call and its prior variance (included
// by size_factors.cu, launched through its launch_per_column).
//
// rlog_fit_kernel: fitBeta's IRLS (src/DESeq2.cpp:283-465, betaTol, useQR = TRUE, useOptim = FALSE) for the design
// X = [1 | I_m] with the ridge Lambda = diag(lambda0, lambda, ..., lambda), or X = I_m when the intercept is frozen.
// X'WX + Lambda is an arrow matrix (a dense first row and column over a diagonal); eliminating the sample rows solves
// it exactly in O(m), with w_j = mu_j / (1 + alpha mu_j) and z_j the working response:
//   c_j   = w_j lambda / (w_j + lambda)
//   beta0 = sum_j c_j z_j / (lambda0 + sum_j c_j)          (sum w - sum w^2 / (w + lambda) formed as sum c: no cancellation)
//   beta_j = w_j (z_j - beta0) / (w_j + lambda)
// and with a frozen intercept (X = I_m, nf' = nf 2^intercept) beta_j = w_j z_j / (w_j + lambda).  Start values as
// fitNbinomGLMs (R/fitNbinomGLMs.R:139-155): [1 | I_m] has rank m < p, so beta0 = log(rowMeans(K / nf)), beta_j = 0; for
// I_m the QR start log(K / nf' + 0.1).  The divergence test (|beta_k| > kBetaLarge over all coefficients, intercept
// included) and the deviance stop are deseq_rules.cuh's; the deviance is the direct form of nb_logdens.cuh with its
// mu-independent part formed once per gene.  No hat diagonals and no sandwich variances: rlogData discards them.
// Outputs: (beta0 + beta_j) / log 2 (log2 scale, R's modelMatrix %*% betaMatrix), or beta_j / log 2 + intercept; the
// log2 intercept; iter.  Rows that R leaves out (all-zero counts; a non-finite frozen intercept) get 0, intercept -Inf
// and iter 0.  The output row holds the sample coefficients between iterations, so nothing is sized by m: each pass
// re-forms w and z of the previous coefficients (one exp) before it takes the next ones (a second exp).
// GL lanes per gene (8 / 16 / 32 from m), consecutive lanes on consecutive samples (coalesced along the sample axis);
// the groups of a warp run their passes together until the last one stops.  Static shared memory only (the log table;
// log(y!) is lgamma_pos(y + 1), the value of nb_logdens.cuh's table, formed once per entry).
//
// rlog_prior_hist_kernel / rlog_prior_pick_kernel: rlogData's betaPriorVar (R/rlog.R:233-240),
//   x_ij = log2(K_ij / s_ij + 0.5) - log2(baseMean_i + 0.5),  w_i = 1 / (1 / baseMean_i + dispFit_i)
//   betaPriorVar = (Hmisc.wtd.quantile(|x|, w, 0.95, normwt = TRUE) / qnorm(0.975))^2   (R/core.R:2416-2419)
// over all n m entries: beta_prior.cuh's MSB-first refinement of both order statistics (bp_targets, bp_hist_add,
// bp_bucket_totals, bp_pick_digit) without its |x| < 10 cut, spread over many CTAs.  Each pass, every CTA of a fixed
// grid histograms its row blocks into its own partials; one CTA then sums the partials in CTA order and picks the digit.
// x is recomputed from the counts in every pass (no n x m scratch) and no floating-point atomic is used, so two calls
// give the same bits.
#pragma once
#include "beta_prior.cuh"
#include "deseq_rules.cuh"
#include "engine.h"
#include "nb_logdens.cuh"

namespace nb {
namespace {

constexpr int kRlThreads = 128;
// per-CTA partials of the quantile: 2 x kBpDigits bucket sums, 2 largest digits, kept count and weight sum
constexpr int kRpMaxd = 2 * kBpDigits, kRpCnt = kRpMaxd + 2, kRpSum = kRpCnt + 1, kRpPart = kRpSum + 1;
constexpr int kRpMaxCtas = 528;                   // 4 per SM of an H100 SXM; fixed so the sum order does not depend on the card
constexpr int kRpEntriesPerBlock = kBpThreads * 8;

// lanes per gene: 8 up to 40 samples, 16 up to 160, a warp above (at most ~10 samples per lane and pass)
inline int rlog_group_lanes(int m) { return m <= 40 ? 8 : (m <= 160 ? 16 : 32); }

template <class T>
__device__ __forceinline__ double rl_count(const void* y, size_t k) {
  return (double)__ldg(static_cast<const T*>(y) + k);
}

// mu = max(nf' exp(eta), minmu) (src/DESeq2.cpp:361-364), w and the working response z = log(mu / nf') + (y - mu) / mu
// (:340, :349; log(mu / nf') = eta unless the clamp bites); returns mu
__device__ __forceinline__ double rl_working(double y, double nfp, double eta, double alpha, const RlogFitArgs& A,
                                             double& w, double& z) {
  const double mu = fmax(nfp * exp(eta), A.minmu);
  const double lmn = (mu == A.minmu) ? log(A.minmu * rcp_fast(nfp)) : eta;
  const double imu = rcp_fast(mu);
  w = mu * rcp_fast(fma(alpha, mu, 1.0));
  z = lmn + fma(y, imu, -1.0);
  return mu;
}

template <int GL, bool NF, bool FROZEN, class T>
__global__ void __launch_bounds__(kRlThreads) rlog_fit_kernel(const RlogFitArgs A) {
  init_log_table();
  const int lg = threadIdx.x % GL;
  const int g = (int)((blockIdx.x * (unsigned)kRlThreads + threadIdx.x) / GL);
  const bool valid = g < A.n;
  if (__all_sync(0xffffffffu, !valid)) return;               // whole warps leave together
  const int m = A.m;
  const size_t off = (size_t)(valid ? g : 0) * A.ld;
  double* out = A.out + (size_t)(valid ? g : 0) * A.ld_out;
  const double lam = A.lambda;

  // nf'_j: the factor (and with a frozen intercept 2^intercept) of sample j
  double scale = 1.0, icpt = 0.0;
  bool active = valid;
  if (FROZEN && valid) {
    icpt = A.intercept[g];
    active = isfinite(icpt);
    scale = exp2(icpt);
  }
  const auto nfp_of = [&](int j) {
    const double f = NF ? __ldg(A.nf + off + j) : __ldg(A.size_factors + j);
    return FROZEN ? f * scale : f;
  };
  // a dispersion that is not finite and > 0 gives the row NaN (the C ABI does not read device data; lgamma_pos needs
  // r > 0)
  double alpha = active ? A.disp_fit[g] : 1.0;
  const bool alpha_ok = alpha > 0.0 && alpha < HUGE_VAL;
  if (!alpha_ok) alpha = 1.0;
  const double r = 1.0 / alpha, log_alpha = log(alpha), lg_r = lgamma_pos(r);

  // ---- row sum of K / nf' (the start intercept) and the mu-independent part of the deviance
  double s2[2] = {0.0, 0.0};
  if (active)
    for (int j = lg; j < m; j += GL) {
      const double y = rl_count<T>(A.y, off + j);
      s2[0] = fma(y, rcp_fast(nfp_of(j)), s2[0]);
      s2[1] += lgamma_diff(y, r, lg_r) - lgamma_pos(y + 1.0);   // once per gene: no log-factorial table
    }
  group_allreduce_sum_n<2, GL>(s2);
  if (!FROZEN && s2[0] == 0.0) active = false;               // an all-zero row: R leaves it out
  const bool fitted = active;
  if (!alpha_ok) active = false;
  const double devc = s2[1];
  double b0 = FROZEN ? 0.0 : log(s2[0] / (double)m);

  // ---- the pass at the start values: store them; the sums of the first solve
  s2[0] = s2[1] = 0.0;
  if (active)
    for (int j = lg; j < m; j += GL) {
      const double y = rl_count<T>(A.y, off + j);
      const double nfp = nfp_of(j);
      const double bj = FROZEN ? log(fma(y, rcp_fast(nfp), 0.1)) : 0.0;
      out[j] = bj;
      if (!FROZEN) {
        double w, z;
        rl_working(y, nfp, b0 + bj, alpha, A, w, z);
        const double c = w * lam * rcp_fast(w + lam);
        s2[0] = fma(c, z, s2[0]);
        s2[1] += c;
      }
    }
  if (!FROZEN) group_allreduce_sum_n<2, GL>(s2);

  // ---- IRLS: solve, then one pass that re-forms w, z of the previous coefficients, takes the new ones, and forms
  // the deviance and the sums of the next solve at them
  IrlsProgress ir;
  for (int t = 0; t < A.maxit; t++) {
    double b0n = 0.0;
    if (active) {
      ir.start_iteration();
      if (!FROZEN) b0n = s2[0] * rcp_fast(A.lambda0 + s2[1]);
    }
    double acc[4] = {0.0, 0.0, 0.0, 0.0};                    // S1, S2, deviance (mu-dependent), diverged
    if (active)
      for (int j = lg; j < m; j += GL) {
        const double y = rl_count<T>(A.y, off + j);
        const double nfp = nfp_of(j);
        double w, z;
        rl_working(y, nfp, b0 + out[j], alpha, A, w, z);
        const double bj = w * (z - b0n) * rcp_fast(w + lam);
        out[j] = bj;
        if (fabs(bj) > kBetaLarge) acc[3] = 1.0;
        const double mu = rl_working(y, nfp, b0n + bj, alpha, A, w, z);
        acc[2] += nb_logdens_mu(y, mu, log(mu), alpha, log_alpha, r);
        if (!FROZEN) {
          const double c = w * lam * rcp_fast(w + lam);
          acc[0] = fma(c, z, acc[0]);
          acc[1] += c;
        }
      }
    group_allreduce_sum_n<4, GL>(acc);
    s2[0] = acc[0];
    s2[1] = acc[1];
    if (active) {
      b0 = b0n;
      if (acc[3] != 0.0 || fabs(b0n) > kBetaLarge) {
        ir.diverged(A.maxit);
        active = false;
      } else if (ir.stop_after_pass(acc[2], devc, A)) {
        active = false;
      }
    }
    if (!__any_sync(0xffffffffu, active)) break;
  }

  // ---- the values on the log2 scale
  if (!valid) return;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  for (int j = lg; j < m; j += GL) {
    double v = 0.0;
    if (fitted) v = FROZEN ? __dadd_rn(out[j] / A.ln2, icpt) : __dadd_rn(b0 / A.ln2, out[j] / A.ln2);
    out[j] = (fitted && !alpha_ok) ? nan : v;
  }
  if (lg == 0) {
    if (!FROZEN && A.out_intercept != nullptr) A.out_intercept[g] = !fitted ? -INFINITY : (alpha_ok ? b0 / A.ln2 : nan);
    A.iter[g] = !fitted ? 0.0 : (alpha_ok ? ir.it : nan);
  }
}

inline int rlog_genes_per_cta(int m) { return kRlThreads / rlog_group_lanes(m); }

template <int GL, bool NF, bool FROZEN>
void (*rlog_fit_kernel_for_type(const RlogFitArgs& a))(RlogFitArgs) {
  return a.y_is_f64 ? rlog_fit_kernel<GL, NF, FROZEN, double> : rlog_fit_kernel<GL, NF, FROZEN, int32_t>;
}

template <int GL, bool NF>
void (*rlog_fit_kernel_for_mode(const RlogFitArgs& a))(RlogFitArgs) {
  return a.intercept != nullptr ? rlog_fit_kernel_for_type<GL, NF, true>(a) : rlog_fit_kernel_for_type<GL, NF, false>(a);
}

template <int GL>
void (*rlog_fit_kernel_for_factors(const RlogFitArgs& a))(RlogFitArgs) {
  return a.nf != nullptr ? rlog_fit_kernel_for_mode<GL, true>(a) : rlog_fit_kernel_for_mode<GL, false>(a);
}

// the instantiation for a's sample count, factors, frozen intercept and count type
void (*rlog_fit_kernel_for(const RlogFitArgs& a))(RlogFitArgs) {
  switch (rlog_group_lanes(a.m)) {
    case 8: return rlog_fit_kernel_for_factors<8>(a);
    case 16: return rlog_fit_kernel_for_factors<16>(a);
    default: return rlog_fit_kernel_for_factors<32>(a);
  }
}

// ---------------------------------------------------------------- prior variance

// one entry (i, j): false if it does not take part (its weight is NaN or 0, as Hmisc drops them)
template <bool NF, class T>
__device__ __forceinline__ bool rp_entry(const RlogPriorArgs& A, size_t i, int j, unsigned long long& bits,
                                         double& w) {
  const double bm = __ldg(A.base_mean + i);
  w = 1.0 / (1.0 / bm + __ldg(A.disp_fit + i));
  if (isnan(w) || w == 0.0) return false;
  const double s = NF ? __ldg(A.nf + i * A.ld + j) : __ldg(A.size_factors + j);
  const double x = log2(__dadd_rn(rl_count<T>(A.y, i * A.ld + j) / s, 0.5)) - log2(__dadd_rn(bm, 0.5));
  bits = (unsigned long long)__double_as_longlong(fabs(x));
  return true;
}

// f(bits, w) for every entry that takes part among the calling CTA's row blocks (blocks blockIdx.x, + ctas, ...), in a
// fixed order per thread; consecutive threads on consecutive samples
template <bool NF, class T, class F>
__device__ __forceinline__ void rp_for_entries(const RlogPriorArgs& A, F&& f) {
  const unsigned m = (unsigned)A.m;
  const int blocks = (A.n + A.rows_per_block - 1) / A.rows_per_block;
  for (int rb = blockIdx.x; rb < blocks; rb += A.ctas) {
    const int r0 = rb * A.rows_per_block;
    const unsigned total = (unsigned)min(A.rows_per_block, A.n - r0) * m;
    for (unsigned k = threadIdx.x; k < total; k += kBpThreads) {
      const unsigned di = k / m;
      unsigned long long bits;
      double w;
      if (rp_entry<NF, T>(A, (size_t)r0 + di, (int)(k - di * m), bits, w)) f(bits, w);
    }
  }
}

// pass < 0: kept count and weight sum of the CTA's entries; pass r >= 0: the histograms of digit r of both targets
template <bool NF, class T>
__global__ void __launch_bounds__(kBpThreads) rlog_prior_hist_kernel(const RlogPriorArgs A, int pass) {
  __shared__ double s_hist[2 * kBpDigits * kBpThreads];        // [target 2][digit 16][thread]
  __shared__ double s_bucket[2][kBpDigits];
  __shared__ double s_red[kBpThreads / 32];
  __shared__ int s_maxd[2];
  __shared__ unsigned int s_cnt;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double* part = A.part + (size_t)blockIdx.x * kRpPart;
  if (pass < 0) {
    unsigned int cnt = 0;
    double sw = 0.0;
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    rp_for_entries<NF, T>(A, [&](unsigned long long, double w) { cnt++; sw += w; });
    sw = warp_allreduce_sum(sw);
    if (lane == 0) s_red[warp] = sw;
    if (cnt) atomicAdd(&s_cnt, cnt);
    __syncthreads();
    if (tid == 0) {
      double S = 0.0;
      for (int k = 0; k < kBpThreads / 32; k++) S += s_red[k];
      part[kRpCnt] = (double)s_cnt;
      part[kRpSum] = S;
    }
    return;
  }
  const double dN = A.st->dN, S = A.st->S;
  if (dN == 0.0) return;
  const int shift = 60 - 4 * pass;
  const unsigned long long mask = pass == 0 ? 0ull : (~0ull << (shift + 4));
  const unsigned long long p0 = A.st->prefix[0], p1 = A.st->prefix[1];
  double* hl = s_hist + tid;
  for (int k = 0; k < 2 * kBpDigits; k++) hl[k * kBpThreads] = 0.0;
  if (tid < 2) s_maxd[tid] = -1;
  __syncthreads();
  int md0 = -1, md1 = -1;
  rp_for_entries<NF, T>(A, [&](unsigned long long bits, double w) {
    bp_hist_add(hl, bits, (w * dN) / S, shift, mask, p0, p1, md0, md1);   // normwt, as w * length(x) / sum(w)
  });
  if (md0 >= 0) atomicMax(&s_maxd[0], md0);
  if (md1 >= 0) atomicMax(&s_maxd[1], md1);
  __syncthreads();
  bp_bucket_totals(s_hist, s_bucket, warp, lane);
  __syncthreads();
  if (tid < 2 * kBpDigits) part[tid] = s_bucket[tid / kBpDigits][tid % kBpDigits];
  if (tid < 2) part[kRpMaxd + tid] = (double)s_maxd[tid];
}

// one CTA: the partials of the pass summed in CTA order; pass < 0 sets up the targets, pass r picks digit r and the
// last pass writes betaPriorVar (NaN when no entry takes part)
__global__ void __launch_bounds__(kBpThreads) rlog_prior_pick_kernel(const RlogPriorArgs A, int pass) {
  __shared__ double s_bucket[2][kBpDigits];
  __shared__ int s_maxd[2];
  const int tid = threadIdx.x;
  RlogPriorState* st = A.st;
  if (pass < 0) {
    if (tid == 0) {
      double cnt = 0.0, S = 0.0;
      for (int c = 0; c < A.ctas; c++) {
        cnt += A.part[(size_t)c * kRpPart + kRpCnt];
        S += A.part[(size_t)c * kRpPart + kRpSum];
      }
      RlogPriorState s{};
      s.dN = cnt;
      s.S = S;
      if (cnt > 0.0) bp_targets(cnt, A.prob, s.frac, s.t_low, s.t_high);
      *st = s;
      if (cnt == 0.0) *A.out_var = __longlong_as_double(0x7ff8000000000000ll);
    }
    return;
  }
  if (st->dN == 0.0) return;
  if (tid < 2 * kBpDigits) {
    double v = 0.0;
    for (int c = 0; c < A.ctas; c++) v += A.part[(size_t)c * kRpPart + tid];
    s_bucket[tid / kBpDigits][tid % kBpDigits] = v;
  } else if (tid < 2 * kBpDigits + 2) {
    int md = -1;
    for (int c = 0; c < A.ctas; c++) md = max(md, (int)A.part[(size_t)c * kRpPart + kRpMaxd + tid - 2 * kBpDigits]);
    s_maxd[tid - 2 * kBpDigits] = md;
  }
  __syncthreads();
  if (tid < 2)
    bp_pick_digit(s_bucket[tid], s_maxd[tid], tid ? st->t_high : st->t_low, 60 - 4 * pass, st->below[tid],
                  st->prefix[tid]);
  if (pass < kBpDigits - 1) return;
  __syncthreads();
  if (tid == 0) {
    const double xl = __longlong_as_double((long long)st->prefix[0]);
    const double xh = __longlong_as_double((long long)st->prefix[1]);
    const double q = __dadd_rn(__dmul_rn(1.0 - st->frac, xl), __dmul_rn(st->frac, xh));
    const double sd = q / A.sd_scale;
    *A.out_var = sd * sd;
  }
}

// rows per histogram block and CTAs of the histogram grid for n x m entries
inline void rlog_prior_grid(int n, int m, int& rows_per_block, int& ctas) {
  rows_per_block = m >= kRpEntriesPerBlock ? 1 : kRpEntriesPerBlock / m;
  const long long blocks = ((long long)n + rows_per_block - 1) / rows_per_block;
  ctas = (int)(blocks < kRpMaxCtas ? blocks : kRpMaxCtas);
}

template <bool NF>
void (*rlog_prior_hist_for_type(const RlogPriorArgs& a))(RlogPriorArgs, int) {
  return a.y_is_f64 ? rlog_prior_hist_kernel<NF, double> : rlog_prior_hist_kernel<NF, int32_t>;
}

void (*rlog_prior_hist_for(const RlogPriorArgs& a))(RlogPriorArgs, int) {
  return a.nf != nullptr ? rlog_prior_hist_for_type<true>(a) : rlog_prior_hist_for_type<false>(a);
}

}  // namespace
}  // namespace nb
