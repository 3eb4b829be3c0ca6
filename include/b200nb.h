/*
 * b200nb.h -- C ABI of the H100-native batched negative-binomial GLM engine (libb200nb.so, sm_90a).
 *
 * This is the drop-in boundary for the ONE hot path of thelovelab/DESeq2: the three native routines the R
 * package reaches through .Call (registration table /root/reference/src/RcppExports.cpp:84-94):
 *
 *   b200nb_fit_disp       replaces  _DESeq2_fitDisp      src/RcppExports.cpp:16-38, body src/DESeq2.cpp:164-277
 *   b200nb_fit_disp_grid  replaces  _DESeq2_fitDispGrid  src/RcppExports.cpp:64-82, body src/DESeq2.cpp:469-513
 *   b200nb_fit_beta       replaces  _DESeq2_fitBeta      src/RcppExports.cpp:41-61, body src/DESeq2.cpp:283-465
 *
 * Argument order follows the reference signatures (SEXP list -> plain pointers + explicit dimensions,
 * named-list members -> caller-allocated output buffers with the reference's member names).  The R-side
 * .Call shim that re-creates the SEXP interface on top of these symbols is in INTEGRATION.md.
 *
 * Conventions
 *   - matrices are R layout: column-major, genes = rows: y[i + n*j] is gene i, sample j; x is m x p.
 *   - host entry points take HOST pointers, copy to the current CUDA device, run the kernels, copy the
 *     results back; they are synchronous.  Inputs are never modified.
 *   - *_dev entry points take DEVICE pointers in the engine's gene-major layout (one gene per row, sample
 *     axis contiguous, row stride ld >= m elements) and enqueue on `stream` (a cudaStream_t passed as void*;
 *     NULL = legacy default stream) without synchronising.  The GLM, prep, Cook's, size-factor and
 *     sf_iterate_objective entry points read rows with 16-byte loads: there ld % 4 == 0 and every matrix base is
 *     16-byte aligned.  The layout helpers, transform, rlog_* and results_* entry points accept any ld >= m.
 *   - arguments are checked before anything is enqueued: y_type is B200NB_Y_INT32 or B200NB_Y_F64, every ld
 *     (ld_out, ld_cooks) is >= m, and no pointer an entry point reads or writes is NULL when it has work
 *     (n > 0); the pointers documented as optional may be NULL.  A call with n == 0 that passes its checks
 *     does nothing and succeeds, unless its entry point states that it needs n >= 1.
 *   - every function returns 0 on success, non-zero on failure; b200nb_last_error() then returns a
 *     message (thread-local).  Per-gene numerical failure is in-band exactly as in the reference
 *     (iter == maxit sentinel, NaN coefficients), never an error (src/DESeq2.cpp:357-360,375-378).
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails.
 *   - p (design columns) is limited to B200NB_MAX_P.
 */
#ifndef B200NB_H
#define B200NB_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200NB_MAX_P 32
#define B200NB_Y_INT32 0
#define B200NB_Y_F64 1
#define B200NB_TRANSFORM_VST_PARAMETRIC 0
#define B200NB_TRANSFORM_VST_MEAN 1
#define B200NB_TRANSFORM_LOG2 2
/* results(): altHypothesis (B200NB_ALT_NONE: lfcThreshold = 0 with "greaterAbs", the columns pass unchanged) */
#define B200NB_ALT_NONE 0
#define B200NB_ALT_GREATER_ABS 1
#define B200NB_ALT_GREATER_ABS_2014 2
#define B200NB_ALT_LESS_ABS 3
#define B200NB_ALT_GREATER 4
#define B200NB_ALT_LESS 5
/* p.adjust methods ("fdr" is BH) */
#define B200NB_PADJ_BH 0
#define B200NB_PADJ_BY 1
#define B200NB_PADJ_HOLM 2
#define B200NB_PADJ_HOCHBERG 3
#define B200NB_PADJ_BONFERRONI 4
#define B200NB_PADJ_NONE 5

/* ---- fitDisp: src/DESeq2.cpp:164.  Outputs = list members at :268-276 (length n each). */
int b200nb_fit_disp(const void* y, int y_type, const double* x, const double* mu_hat, const double* log_alpha,
                    const double* log_alpha_prior_mean, double log_alpha_prior_sigmasq, double min_log_alpha,
                    double kappa_0, double tol, int maxit, int use_prior, const double* weights, int use_weights,
                    double weight_threshold, int use_cr, int n, int m, int p,
                    double* out_log_alpha, int32_t* out_iter, int32_t* out_iter_accept, double* out_last_change,
                    double* out_initial_lp, double* out_initial_dlp, double* out_last_lp, double* out_last_dlp,
                    double* out_last_d2lp);

/* ---- fitDispGrid: src/DESeq2.cpp:469.  Output = list member log_alpha (:512). */
int b200nb_fit_disp_grid(const void* y, int y_type, const double* x, const double* mu_hat, const double* disp_grid,
                         int disp_grid_n, const double* log_alpha_prior_mean, double log_alpha_prior_sigmasq,
                         int use_prior, const double* weights, int use_weights, double weight_threshold, int use_cr,
                         int n, int m, int p, double* out_log_alpha);

/* ---- fitBeta: src/DESeq2.cpp:283.  beta_mat (n x p) is the starting value; outputs = list members at
 * :458-464: out_beta_mat n x p, out_beta_var_mat n x p, out_iter n (double, NumericVector in the reference),
 * out_hat_diagonals n x m, out_contrast_num n, out_contrast_denom n, out_deviance n.
 * nf is the n x m normalisation-factor matrix the reference receives (R/core.R:2221-2228).
 * out_mu (n x m, may be NULL) is an extension: the fitted mean nf*exp(x beta) clamped at minmu, which the
 * reference recomputes in R right after the call (R/fitNbinomGLMs.R:180). */
int b200nb_fit_beta(const void* y, int y_type, const double* x, const double* nf, const double* alpha_hat,
                    const double* contrast, const double* beta_mat, const double* lambda, const double* weights,
                    int use_weights, double tol, int maxit, int use_qr, double minmu, int n, int m, int p,
                    double* out_beta_mat, double* out_beta_var_mat, double* out_iter, double* out_hat_diagonals,
                    double* out_contrast_num, double* out_contrast_denom, double* out_deviance, double* out_mu);

/* ---- device-resident variants (gene-major n x ld matrices, see header comment) */
int b200nb_fit_disp_dev(const void* y, int y_type, const double* x, const double* mu_hat, const double* log_alpha,
                        const double* log_alpha_prior_mean, double log_alpha_prior_sigmasq, double min_log_alpha,
                        double kappa_0, double tol, int maxit, int use_prior, const double* weights,
                        int use_weights, double weight_threshold, int use_cr, int n, int m, int p, long long ld,
                        double* out_log_alpha, int32_t* out_iter, int32_t* out_iter_accept,
                        double* out_last_change, double* out_initial_lp, double* out_initial_dlp,
                        double* out_last_lp, double* out_last_dlp, double* out_last_d2lp, void* stream);

int b200nb_fit_disp_grid_dev(const void* y, int y_type, const double* x, const double* mu_hat,
                             const double* disp_grid, int disp_grid_n, const double* log_alpha_prior_mean,
                             double log_alpha_prior_sigmasq, int use_prior, const double* weights, int use_weights,
                             double weight_threshold, int use_cr, int n, int m, int p, long long ld,
                             double* out_log_alpha, void* stream);

/* nf_is_vector != 0: nf is the length-m size-factor vector instead of the n x ld matrix.
 * beta_mat / out_beta_mat / out_beta_var_mat stay column-major n x p.  out_hat_diagonals / out_mu are
 * gene-major n x ld and may be NULL. */
int b200nb_fit_beta_dev(const void* y, int y_type, const double* x, const double* nf, int nf_is_vector,
                        const double* alpha_hat, const double* contrast, const double* beta_mat,
                        const double* lambda, const double* weights, int use_weights, double tol, int maxit,
                        int use_qr, double minmu, int n, int m, int p, long long ld, double* out_beta_mat,
                        double* out_beta_var_mat, double* out_iter, double* out_hat_diagonals,
                        double* out_contrast_num, double* out_contrast_denom, double* out_deviance, double* out_mu,
                        void* stream);

/* b200nb_nb_loglik_dev: what R recomputes right after fitBeta (R/fitNbinomGLMs.R:180-182): the fitted mean
 * mu = nf * exp(x beta) WITHOUT the minmu clamp (out_mu, gene-major n x ld, may be NULL) and
 * logLike = rowSums([w *] dnbinom(y, mu, size = 1/alpha, log = TRUE)) (nbinomLogLike, R/core.R:2208-2217; out_loglik[n]).
 * nbinomLRT's statistic (R/core.R:1877) and Cook's distances (R/core.R:1457) are built from these, not from the
 * clamped quantities inside the IRLS.  beta_mat: n x p column-major, natural-log scale (fitBeta's out_beta_mat).
 * minmu > 0 evaluates the log-likelihood (not out_mu) at max(mu, minmu): what fitNbinomGLMsOptim stores for the rows
 * it refits (R/fitNbinomGLMs.R:386-398); 0 = no clamp. */
int b200nb_nb_loglik_dev(const void* y, int y_type, const double* x, const double* nf, int nf_is_vector,
                         const double* alpha_hat, const double* beta_mat, const double* weights, int use_weights,
                         double minmu, int n, int m, int p, long long ld, double* out_loglik, double* out_mu,
                         void* stream);

/* b200nb_beta_optim_dev: fitNbinomGLMsOptim (R/fitNbinomGLMs.R:340-407) for the rows whose IRLS did not converge /
 * diverged / gave NA: box-constrained maximisation of logLike + log prior (ridge lambda, natural-log scale here:
 * lambda_log2 / ln(2)^2; box |beta| <= 30 ln 2 = |beta_log2| <= 30).  The objective is strictly concave, so the unique
 * maximiser is what optim(method = "L-BFGS-B") converges to; a projected Newton iteration finds it (maxit iterations
 * at most; out_converged = 1 plays optim's convergence == 0).  Pass ONLY the rows to refit (gathered gene-major rows).
 * beta_start / out_beta_mat: n x p column-major, natural-log scale.  Standard errors, fitted means and the
 * log-likelihood at the optimum come from b200nb_fit_beta_dev(maxit = 0) and b200nb_nb_loglik_dev. */
int b200nb_beta_optim_dev(const void* y, int y_type, const double* x, const double* nf, int nf_is_vector,
                          const double* alpha_hat, const double* lambda, const double* beta_start,
                          const double* weights, int use_weights, int maxit, int n, int m, int p, long long ld,
                          double* out_beta_mat, int32_t* out_converged, int32_t* out_iter, void* stream);

/* layout helpers on device buffers: R column-major n x m <-> gene-major n x ld.  elem_size 4 (int32) or 8. */
int b200nb_to_gene_major_dev(const void* src_colmajor, void* dst, int n, int m, long long ld, int elem_size,
                             void* stream);
int b200nb_to_col_major_dev(const double* src, double* dst_colmajor, int n, int m, long long ld, void* stream);

/* ---- pre-steps of the hot path on device buffers (the R glue around the native calls, SURVEY.md 8f row 2)
 * b200nb_prep_dev: per gene, from the counts (gene-major n x ld) and size factors:
 *   base_mean, base_var, all_zero      getBaseMeansAndVariances   R/core.R:2138-2157
 *   alpha0 = clamp(min(roughDispEstimate, momentsDispEstimate), min_disp, max_disp)   R/core.R:2422-2448, 716, 727
 *   mu_lin (optional) = linearModelMuNormalized clamped at minmu                      R/core.R:2454-2467, 764
 *   beta0 (optional, n x p column-major) = QR least squares of log(K/s + 0.1) on X    R/fitNbinomGLMs.R:139-145
 * x is m x p column-major; proj is (X'X)^-1 X' as p x m row-major; xim = mean(1/size_factor).
 * b200nb_trend_fit_dev: parametricDispersionFit (R/core.R:2166-2189) over genes with disps > 100*min_disp;
 *   out4 = {asymptDisp, extraPois, status (0 ok, 1 not converged, 2 non-positive, 3 no usable genes), rounds}. */
int b200nb_prep_dev(const void* y, int y_type, const double* x, const double* proj, const double* size_factors,
                    double xim, double min_disp, double max_disp, double minmu, int n, int m, int p, long long ld,
                    double* base_mean, double* base_var, int32_t* all_zero, double* alpha0, double* mu_lin,
                    double* beta0, void* stream);
int b200nb_trend_fit_dev(const double* means, const double* disps, int n, double min_disp, double* out4,
                         void* stream);
/* b200nb_prep_weighted_dev: b200nb_prep_dev with observation weights (gene-major n x ld, raw assay weights), p <= 32:
 *   base_mean, base_var of w * K/s with the raw weights (R/core.R:2140-2145); alpha0 from the weighted moments and
 *   the unweighted rough dispersion; mu_lin and beta0 unweighted (pass mu_lin = NULL: with weights the reference
 *   fits mu by IRLS);
 *   out_weights_norm (gene-major n x ld) = weights / row maximum, padding columns 0       R/core.R:2700-2702
 *   out_weights_fail[n] = 1 where rank(w * X) < p or X on the samples with normalised w > weight_threshold (all-zero
 *     columns dropped) is rank deficient, R's qr() rank with tol 1e-7                     R/core.R:2706-2722
 *   out_status (one device int, zeroed by the call) = number of rows with a negative, NaN or infinite weight or no
 *     positive weight; the reference stops on them, so the caller must raise when it is not 0. */
int b200nb_prep_weighted_dev(const void* y, int y_type, const double* x, const double* proj,
                             const double* size_factors, double xim, double min_disp, double max_disp, double minmu,
                             int n, int m, int p, long long ld, double* base_mean, double* base_var,
                             int32_t* all_zero, double* alpha0, double* mu_lin, double* beta0, const double* weights,
                             double weight_threshold, double* out_weights_norm, int32_t* out_weights_fail,
                             int32_t* out_status, void* stream);
/* b200nb_prep_nf_dev: b200nb_prep_dev with gene-specific normalization factors nf (gene-major n x ld, positive) in
 * place of the size-factor vector: base_mean / base_var of K/nf, the rough dispersion and beta0 from K/nf,
 * mu_lin = linearModelMu(K/nf) * nf clamped at minmu (linearModelMuNormalized, R/core.R:2465-2471).  xim is
 * mean(1 / colMeans(nf)) over the rows the moments estimate is for (R/core.R:2439-2448), computed by the caller. */
int b200nb_prep_nf_dev(const void* y, int y_type, const double* x, const double* proj, const double* nf, double xim,
                       double min_disp, double max_disp, double minmu, int n, int m, int p, long long ld,
                       double* base_mean, double* base_var, int32_t* all_zero, double* alpha0, double* mu_lin,
                       double* beta0, void* stream);

/* b200nb_cooks_dev: calculateCooksDistance + recordMaxCooks + robustMethodOfMomentsDisp (R/core.R:2277-2359).
 * cells = distinct design rows: cell_ptr (ncell+1) / cell_samples (m, sample indices grouped by cell), device ints.
 * cooks (gene-major n x ld) may be NULL; max_cooks[n] is NaN when no cell has >= 3 replicates or m <= p. */
int b200nb_cooks_dev(const void* y, int y_type, const double* mu, const double* hat, const double* size_factors,
                     const int32_t* cell_ptr, const int32_t* cell_samples, int ncell, int n, int m, int p,
                     long long ld, double* cooks, double* max_cooks, double* robust_disp, void* stream);
/* b200nb_cooks_nf_dev: b200nb_cooks_dev with normalization factors nf (gene-major n x ld) in place of the size
 * factors: the robust dispersion and the trimmed cell means work on K/nf; mu already carries nf. */
int b200nb_cooks_nf_dev(const void* y, int y_type, const double* mu, const double* hat, const double* nf,
                        const int32_t* cell_ptr, const int32_t* cell_samples, int ncell, int n, int m, int p,
                        long long ld, double* cooks, double* max_cooks, double* robust_disp, void* stream);

/* b200nb_size_factors_dev: estimateSizeFactorsForMatrix (R/core.R:535-578; locfunc = median, no geoMeans /
 * controlGenes).  poscounts = 0 is type "ratio", 1 is type "poscounts".  y gene-major (n x ld); loggeomeans[n] and
 * size_factors[m] are outputs; scratch_gm (n x ld doubles) and scratch_cm (n x m doubles) are caller-provided device
 * scratch; n_finite (device int) receives the number of genes with a finite log geometric mean -- R stops with
 * "every gene contains at least one zero" when it is 0, the caller must do the same.  A sample with no usable
 * ratio gets NaN (median of an empty set is NA in R).  scratch_cm is also an output: on return it holds the log
 * ratios log K_ij - loggeomean_i the median is taken over, column-major (sample j at scratch_cm + j n), +Inf where an
 * entry does not take part; the gene-sharded estimator takes the median over every rank's ratios from it.  The same
 * holds for b200nb_size_factors_norm_dev below. */
int b200nb_size_factors_dev(const void* y, int y_type, int poscounts, int n, int m, long long ld,
                            double* loggeomeans, double* scratch_gm, double* scratch_cm, double* size_factors,
                            int32_t* n_finite, void* stream);
/* b200nb_size_factors_norm_dev: the size factors of K / d for a positive divisor matrix d (gene-major n x ld), the
 * first step of estimateNormFactors (R/core.R:2159-2163).  Ratios log(K/d) - loggeomean over the entries with K > 0;
 * poscounts = 0: loggeomean = mean log(K/d) (type "ratio"); 1: loggeomean = log(geoMeanNZ(K)) of the RAW counts, the
 * geoMeans that estimateSizeFactors passes for type "poscounts" (R/methods.R:377-390).  The caller applies the
 * incoming-geoMeans rescaling sf / exp(mean(log sf)) (R/core.R:573-576) for poscounts.  Other arguments as above. */
int b200nb_size_factors_norm_dev(const void* y, int y_type, const double* divisor, int poscounts, int n, int m,
                                 long long ld, double* loggeomeans, double* scratch_gm, double* scratch_cm,
                                 double* size_factors, int32_t* n_finite, void* stream);

/* b200nb_beta_prior_quantile_dev: the weighted upper quantile of estimateBetaPriorVar (betaPriorMethod "weighted",
 * R/core.R:1601-1689, 2416-2419; Hmisc.wtd.quantile with normwt = TRUE, :2762-2900).  For each of the k columns
 * x_c = beta[:, a] - (b < 0 ? 0 : beta[:, b]) (col_a / col_b are device ints; b >= 0 gives addAllContrasts'
 * differences, R/expanded.R:76-98) out_q[c] = wtd.quantile(|x_c|, w, prob) over the entries with |x_c| < 10 and a
 * weight w = 1/(1/base_mean + disp_fit) that is neither NaN nor 0; NaN when no entry is kept.  beta_log2 is n x p
 * column-major (log2 scale).  Deterministic: two calls on the same input give the same bits.  Needs n >= 1, p >= 1,
 * k >= 0, 0 <= a < p, -1 <= b < p, 0 < prob < 1 (the indices are fetched to the host once to check them). */
int b200nb_beta_prior_quantile_dev(const double* beta_log2, int n, int p, const double* base_mean,
                                   const double* disp_fit, const int32_t* col_a, const int32_t* col_b, int k,
                                   double prob, double* out_q, void* stream);

/* b200nb_sf_iterate_objective_dev: the objective of estimateSizeFactorsIterate (R/core.R:2589-2622) at the log size
 * factors par[m] and at the 2m points optim's finite-difference gradient needs (ndeps = h):
 *   fn(p) = sum(gene.ll[gene.ll > quantile(gene.ll, Q)]),  gene.ll_i = sum_j log dnbinom(K_ij; q_ij s_j, 1/alpha_i),
 *   s = exp(p - mean(p)),  quantile type 7.
 * out[0] = fn(par), out[1 + k] = fn(par + h e_k), out[1 + m + k] = fn(par - h e_k), k < m.  y: counts, gene-major
 * (n x ld, int32 or f64); q: gene-major n x ld, mu / s of the dispersion fit; alpha: n dispersions.  Needs n, m >= 1,
 * finite h > 0, 0 <= Q < 1 and no NULL pointer.  The gene log-likelihoods are formed for tiles of at most
 * max_tile_cols objective columns (0: as many as 128 MB of workspace hold) in a workspace the library keeps per
 * process, shared with the host entry points (calls on different streams must not overlap).  Enqueue only;
 * deterministic: two calls on the same input give the same bits. */
int b200nb_sf_iterate_objective_dev(const void* y, int y_type, const double* q, const double* alpha,
                                    const double* par, double h, double Q, int n, int m, long long ld,
                                    int max_tile_cols, double* out, void* stream);

/* b200nb_transform_dev: a transform of the normalized counts q = K / s_j (size_factors[m]) or K / nf_ij (nf, gene-major
 * n x ld): exactly one of the two is non-NULL.  y: counts, gene-major (n x ld, int32 or f64); out: gene-major n x ld_out
 * float64, columns >= m untouched.  mode and its constants c0, c1:
 *   B200NB_TRANSFORM_VST_PARAMETRIC  getVarianceStabilizedData for fitType "parametric" (R/vst.R:153-155),
 *     c0 = asymptDisp, c1 = extraPois (both finite and > 0):
 *     log((1 + c1 + 2 c0 q + 2 sqrt(c0 q (1 + c1 + c0 q))) / (4 c0)) / log(2)
 *   B200NB_TRANSFORM_VST_MEAN  fitType "mean" (R/vst.R:185-189), c0 = alpha (finite and > 0), c1 unused:
 *     (2 asinh(sqrt(c0 q)) - log(c0) - log(4)) / log(2)
 *   B200NB_TRANSFORM_LOG2  normTransform(f = log2, pc = c0) (R/helper.R:421-435), c0 finite and >= 0, c1 unused:
 *     log2(q + c0)
 * q is an IEEE division and the formulas are evaluated in R's operand order without contraction.  Needs n, m >= 0,
 * ld >= m, ld_out >= m and no NULL pointer.  Enqueue only. */
int b200nb_transform_dev(const void* y, int y_type, const double* size_factors, const double* nf, int n, int m,
                         long long ld, int mode, double c0, double c1, double* out, long long ld_out, void* stream);

/* b200nb_rlog_fit_dev: rlogData's fitNbinomGLMs call (R/rlog.R:249-253: betaTol = tol, useQR, no optim) for every row
 * of y (gene-major n x ld, int32 or f64 counts), with exactly one of size_factors[m] and nf (gene-major n x ld):
 *   intercept == NULL: the design [1 | I_m], ridge 1e-6 on the intercept and 1 / beta_prior_var on the samples (log2
 *     scale); start beta0 = log(rowMeans(K / nf)), beta_j = 0.  out_ij = (beta0 + beta_j) / log(2) and
 *     out_intercept_i = beta0 / log(2); an all-zero row gets out = 0 and out_intercept = -Inf.
 *   intercept != NULL (n log2 intercepts, the frozen rlog): the design I_m on nf' = nf 2^intercept, start
 *     log(K / nf' + 0.1); out_ij = beta_j / log(2) + intercept_i; a row with a non-finite intercept gets out = 0.
 *     out_intercept is not written (may be NULL).
 * disp_fit: n dispersions (R's dispFit); a fitted row whose dispersion is not finite and > 0 gets NaN in out,
 * out_intercept and out_iter.  out: gene-major n x ld_out, columns >= m untouched; out_iter: n IRLS iterations (maxit
 * for a diverged row, |beta| > 30; 0 for a row left out).  Needs n >= 0, m >= 1, ld >= m, ld_out >= m, finite
 * beta_prior_var > 0, tol > 0 and minmu > 0, maxit >= 1 and no NULL pointer among y, disp_fit, out, out_iter (and
 * out_intercept without an intercept).  Enqueue only. */
int b200nb_rlog_fit_dev(const void* y, int y_type, const double* size_factors, const double* nf,
                        const double* intercept, const double* disp_fit, int n, int m, long long ld,
                        double beta_prior_var, double tol, int maxit, double minmu, double* out, long long ld_out,
                        double* out_intercept, double* out_iter, void* stream);

/* b200nb_rlog_prior_var_dev: rlogData's betaPriorVar (R/rlog.R:233-240) over the n x m entries of y (gene-major n x
 * ld) with exactly one of size_factors[m] and nf (gene-major n x ld):
 *   x_ij = log2(K_ij / s_ij + 0.5) - log2(base_mean_i + 0.5), weight 1 / (1 / base_mean_i + disp_fit_i)
 *   *out_var = (Hmisc weighted quantile of |x| at 0.95, normwt = TRUE, / qnorm(0.975))^2
 * Entries whose weight is NaN or 0 (an all-zero row: base_mean 0) do not take part; NaN when none does.  Two calls
 * give the same bits.  Needs n, m >= 1, ld >= m and no NULL pointer.  Enqueue only. */
int b200nb_rlog_prior_var_dev(const void* y, int y_type, const double* size_factors, const double* nf,
                              const double* base_mean, const double* disp_fit, int n, int m, long long ld,
                              double* out_var, void* stream);

/* b200nb_results_gene_dev: results()' per-gene steps (R/results.R:298-575) for n genes, in R's order, from the selected
 * column lfc, se, stat, pvalue (n each):
 *   negate != 0 (the numerator is the reference level): LFC negated, and stat too unless lrt != 0;
 *   zero_mask (m int32 flags, or NULL): contrastAllZero -- when the counts of y (gene-major n x ld, int32 or f64: the
 *     original counts) at the flagged samples are all zero, LFC = 0 and, unless lrt != 0, stat = 0 and p = 1;
 *   alt (B200NB_ALT_*) with lfc_threshold T >= 0: the thresholded stat and p (pnorm);
 *   max_cooks (n, or NULL: no Cook's cutoff): p = NaN where max_cooks > cooks_cutoff, unless keep (n int32, or NULL)
 *     is non-zero there;
 *   replace (n int32, or NULL) with base_mean (n): where replace != 0 and base_mean == 0, LFC, SE, stat = 0, p = 1.
 * Writes out_lfc, out_se, out_stat, out_pvalue (n each; may alias the inputs).  Needs n >= 0, m >= 1, ld >= m, a known
 * alt, finite T >= 0, and no NULL pointer among the column inputs and outputs (y with zero_mask, base_mean with
 * replace).  Enqueue only. */
int b200nb_results_gene_dev(const void* y, int y_type, int n, int m, long long ld, const double* lfc, const double* se,
                            const double* stat, const double* pvalue, int negate, const int32_t* zero_mask, int lrt,
                            int alt, double lfc_threshold, const double* max_cooks, double cooks_cutoff,
                            const int32_t* keep, const int32_t* replace, const double* base_mean, double* out_lfc,
                            double* out_se, double* out_stat, double* out_pvalue, void* stream);

/* b200nb_results_heuristic_dev: results()' two-group Cook's heuristic (R/results.R:538-556) for k flagged genes:
 * rows (k gene indices into y, gene-major n x ld counts), cooks (gene-major k x ld_cooks: row r holds the Cook's
 * distances of gene rows[r]).  outCount = y[rows[r], which.max(cooks row)] (first maximum, NaN skipped);
 * keep[rows[r]] = (at least 3 counts of the gene are > outCount).  Other entries of keep are not written.  Needs
 * k >= 0, m >= 1, ld >= m, ld_cooks >= m and no NULL pointer.  Enqueue only. */
int b200nb_results_heuristic_dev(const void* y, int y_type, const int64_t* rows, int k, int m, long long ld,
                                 const double* cooks, long long ld_cooks, int32_t* keep, void* stream);

/* b200nb_filter_cutoffs_dev: quantile(filter, theta, type = 7) (R/results.R:725) of the n filter values (none NaN) at
 * n_theta probabilities in [0, 1], one CTA per probability by radix select.  Needs n >= 1, 1 <= n_theta <= 65535 and
 * no NULL pointer.  Enqueue only. */
int b200nb_filter_cutoffs_dev(const double* filter, int n, const double* theta, int n_theta, double* out,
                              void* stream);

/* b200nb_filter_numrej_dev: numRej of pvalueAdjustment (R/results.R:652): for every cutoff c_t (n_theta of them) the
 * number of genes with filter >= c_t whose p.adjust(method) over that subset is < alpha.  p_sorted: the n p-values in
 * ascending order, NaN last (NaN never belongs to a subset); filter_sorted: their filter values.  out_numrej: n_theta
 * int32.  Needs n >= 1, 1 <= n_theta <= 65535, a known method, 0 < alpha < 1 and no NULL pointer.  Enqueue only. */
int b200nb_filter_numrej_dev(const double* p_sorted, const double* filter_sorted, int n, const double* cutoffs,
                             int n_theta, int method, double alpha, int32_t* out_numrej, void* stream);

/* b200nb_padj_dev: the adjusted p-values of one subset: p.adjust(method) over the genes with filter >= cutoffs[j]
 * (cutoffs == NULL: every gene with a p-value), written to out[order[i]] for the gene at sorted position i; the
 * others get NaN.  p_sorted, filter_sorted as for b200nb_filter_numrej_dev; order: the n gene positions (0 <= order[i]
 * < n_out, each once).  Needs n >= 1, j >= 0, a known method and no NULL pointer among p_sorted, filter_sorted,
 * order, out.  Enqueue only. */
int b200nb_padj_dev(const double* p_sorted, const double* filter_sorted, const int64_t* order, int n,
                    const double* cutoffs, int j, int method, double* out, void* stream);

/* ---- housekeeping */
const char* b200nb_last_error(void);
int b200nb_device_count(void);            /* number of visible CUDA devices (0 if none / no driver) */
long long b200nb_kernel_launches(void);   /* kernels this library has launched in this process */
void b200nb_release_workspace(void);      /* frees cached device / pinned buffers of the host entry points */
/* The host entry points keep the gene-major device copies of the large input matrices of recent calls, addressed by
 * CONTENT (dimensions + a 128-bit hash of every byte, recomputed from the caller's buffer on each call), so the count
 * matrix and the fitted means that one DESeq() run passes to fitDisp, fitDisp and fitBeta cross PCIe once.
 * b200nb_cache_clear() forgets them (the memory stays allocated for reuse); B200NB_CACHE_MB=0 disables the cache. */
void b200nb_cache_clear(void);
/* Page-locked memory for RESULT matrices (pooled).  A result buffer obtained here receives its data by one DMA; any
 * other buffer is filled through the library's pinned staging ring by host threads and pays first-touch page faults
 * when it is fresh (~3 ms for a 50 000 x 100 hat-diagonal matrix).  Returns NULL when page-locked memory cannot be had
 * (use ordinary memory then).  In R: allocVector3(REALSXP, n, &allocator) with these two as mem_alloc / mem_free
 * (deseq2_b200/r_shim/deseq2_b200_shim.c). */
void* b200nb_host_alloc(size_t bytes);
void b200nb_host_free(void* p);
/* cumulative counters of the host entry points: out[0] bytes copied host->device, [1] device->host, [2] cache hits,
 * [3] cache misses, [4] bytes served from the cache instead of being uploaded, [5] bytes hashed / scanned on the host.
 * Writes min(n, 6) values, returns 6. */
int b200nb_host_stats(long long* out, int n);
const char* b200nb_version(void);

/* test hook: lgamma / digamma / trigamma of the device math on host arrays x[0..n) (x > 0) */
int b200nb_test_special(const double* x, int n, double* out_lgamma, double* out_digamma, double* out_trigamma);
/* test hook: the host content hash of `count` elements of `elem` (4 | 8) bytes at p, canonical indices first_index...,
 * by every instruction-set variant this CPU can run (scalar, AVX2, AVX-512): out[0..1] receive the scalar value;
 * returns the number of variants compared, or -1 if two of them disagree. */
int b200nb_test_hash(const void* p, long long count, int elem, long long first_index, unsigned long long* out2);

#ifdef __cplusplus
}
#endif
#endif /* B200NB_H */
