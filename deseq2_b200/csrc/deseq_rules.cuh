// deseq_rules.cuh -- the reference's per-gene decision rules, written once for every fit kernel family
// (fit_disp.cu / fit_disp_grp.cuh, fit_beta.cu / fit_beta_grp.cuh, fit_generic.cu / fit_generic_seg.cuh).
//
// Each kernel keeps its own gene -> lane mapping, loop structure and evaluation code and drives these rules from its
// loop.  The parity tests compare `iter` / `iter_accept` per gene, so every decision here is the reference's, and
// every floating-point expression is kept textually as it is: nvcc contracts them into FMAs, and a re-associated or
// split expression changes bits.
#pragma once
#include "engine.h"

namespace nb {

// ---------------------------------------------------------------- fitDisp (src/DESeq2.cpp:201-265)
// Armijo back-tracking ascent on log alpha.  Per gene:
//   a = propose();  evaluate lp, dlp at a;  if (take(lp, dlp, A)) stop;
// The first proposal is the starting point (:205-206); take() then records the initial values.  Every later proposal
// is a + kappa dlp with kappa shrunk so that the step stays inside [-30, 10]; take() applies the acceptance test and
// the kappa schedule and reports whether the gene stopped (converged, or fell below min_log_alpha).  The caller
// bounds the number of proposals by maxit (the reference's `for (t = 0; t < maxit; t++)`); `it` counts them.
struct DispLineSearch {
  double a, a_new;
  double lp = 0.0, dlp = 0.0, initial_lp = 0.0, initial_dlp = 0.0;
  double kappa;
  double change = -1.0;
  int it = 0, acc_n = 0;
  bool first = true;

  __device__ __forceinline__ DispLineSearch(double a0, double kappa_0) : a(a0), a_new(a0), kappa(kappa_0) {}

  __device__ __forceinline__ double propose() {
    a_new = a;
    if (!first) {
      it++;
      const double a_propose = a + kappa * dlp;
      if (a_propose < -30.0) kappa = (-30.0 - a) / dlp;
      if (a_propose > 10.0) kappa = (10.0 - a) / dlp;
      a_new = a + kappa * dlp;
    }
    return a_new;
  }

  __device__ __forceinline__ bool take(double lp_new, double dlp_new, const DispArgs& A) {
    const double epsilon = 1.0e-4;
    if (first) {
      lp = initial_lp = lp_new;
      dlp = initial_dlp = dlp_new;
      first = false;
      return false;
    }
    const double theta_kappa = -1.0 * lp_new;
    const double theta_hat_kappa = -1.0 * lp - kappa * epsilon * dlp * dlp;
    if (theta_kappa <= theta_hat_kappa) {
      acc_n++;
      a = a_new;
      change = lp_new - lp;
      if (change < A.tol) {
        lp = lp_new;
        return true;
      }
      if (a < A.min_log_alpha) return true;
      lp = lp_new;
      dlp = dlp_new;
      kappa = fmin(kappa * 1.1, A.kappa_0);
      if (acc_n % 5 == 0) kappa = kappa / 2.0;
    } else {
      kappa = kappa / 2.0;
    }
    return false;
  }

  // the nine per-gene outputs; d2 = second derivative of the log posterior at the final a
  __device__ __forceinline__ void store(const DispArgs& A, unsigned int g, double d2) const {
    A.log_alpha[g] = a;
    A.iter[g] = it;
    A.iter_accept[g] = acc_n;
    A.last_change[g] = change;
    A.initial_lp[g] = initial_lp;
    A.initial_dlp[g] = initial_dlp;
    A.last_lp[g] = lp;
    A.last_dlp[g] = dlp;
    A.last_d2lp[g] = d2;
  }
};

// ---------------------------------------------------------------- fitDispGrid (src/DESeq2.cpp:492-510)
// The coarse grid A.grid[0 .. n), then n points over [a_hat - delta, a_hat + delta] around its argmax (delta = one
// coarse grid step).  Per gene: for (t = 0; t < evaluations(); t++) { a = point(t); evaluate lp at a; take(t, a, lp); }
// and the result is a_best.  Ties keep the first point.
struct DispGridSearch {
  const double* grid;
  int n;
  double delta;
  double best = 0.0, a_hat = 0.0, a_best = 0.0, start = 0.0, end = 0.0, step = 0.0;

  __device__ __forceinline__ explicit DispGridSearch(const DispArgs& A)
      : grid(A.grid), n(A.grid_n), delta(A.grid[1] - A.grid[0]) {}

  __device__ __forceinline__ int evaluations() const { return 2 * n; }

  __device__ __forceinline__ double point(int t) {
    const int tt = (t < n) ? t : t - n;
    if (t == n) {
      start = a_hat - delta;
      end = a_hat + delta;
      step = (end - start) / (double)(n - 1);
    }
    return (t < n) ? grid[tt] : ((tt == n - 1) ? end : start + tt * step);
  }

  __device__ __forceinline__ void take(int t, double a, double lp) {
    const int tt = (t < n) ? t : t - n;
    if (tt == 0 || lp > best) {
      best = lp;
      if (t < n) a_hat = a; else a_best = a;
    }
  }
};

// ---------------------------------------------------------------- fitBeta (src/DESeq2.cpp:344-383)
// |beta_k| > kBetaLarge after a solve: the gene diverged.  Its iteration count becomes maxit and the diverged beta is
// kept without a further pass (:357-360).  Where beta lives (a register array, or one coefficient per lane) decides
// how the test is written, so each kernel writes it against this constant.
constexpr double kBetaLarge = 30.0;

// IRLS iteration count and deviance stop rule.  Per iteration: start_iteration(); solve; on divergence diverged() and
// stop; pass; if (stop_after_pass(dv, devc, A)) stop.  The pass at the starting values comes before the first
// iteration and is not scored.  NaN in the relative change stops with it = maxit; convergence is tested from the
// second iteration on.
struct IrlsProgress {
  double dev = 0.0, dev_old = 0.0;
  double it = 0.0;   // a double, as in the reference's NumericVector

  __device__ __forceinline__ void start_iteration() { it += 1.0; }
  __device__ __forceinline__ void diverged(int maxit) { it = (double)maxit; }

  // dv + devc: the log-likelihood sum of the pass (mu-dependent and mu-independent parts); Args: BetaArgs, or any
  // argument block with the same tol and maxit (RlogFitArgs)
  template <class Args>
  __device__ __forceinline__ bool stop_after_pass(double dv, double devc, const Args& A) {
    dev = -2.0 * (dv + devc);
    const double conv_test = fabs(dev - dev_old) / (fabs(dev) + 0.1);
    if (isnan(conv_test)) {
      it = (double)A.maxit;
      return true;
    }
    if ((it > 1.0) && (conv_test < A.tol)) return true;
    dev_old = dev;
    return false;
  }
};

}  // namespace nb
