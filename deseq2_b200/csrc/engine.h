// engine.h -- internal launcher interface between the C ABI (capi.cu) and the sm_90a kernels.
// Device layout ("gene-major"): every n x m matrix is stored one gene per row with the sample axis
// contiguous, row stride `ld` elements (ld % 4 == 0 so rows start 32-byte aligned for 128-bit loads).
// The design matrix x stays in R's column-major m x p form (it is tiny and staged into shared memory).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nb {

constexpr int kMaxSmallP = 4;    // register-resident normal equations
constexpr int kMaxP = 32;        // shared-memory path upper bound

// Sample layout of the segmented general-p kernels (fit_generic_seg.cuh; grouped designs, m <= 65535).  The samples are
// sorted by design group and dealt to the 32 lanes as contiguous chunks of the sorted sequence (lane l gets sorted
// samples [l q + min(l, rem), ...), q = m / 32, rem = m % 32); the sample that lane l visits in trip i of the loop
// `for (j = lane; j < m; j += 32)` sits at position i * 32 + l.  A lane therefore sees a short run of consecutive
// groups ("segments"), accumulates the per-group sums of a pass in registers and stores one value per segment.
// All arrays are device pointers prepared by the C-ABI layer together with xg / gid; `pos == nullptr`: no layout.
struct SegLayout {
  const unsigned short* pos;      // m: position of sample j
  const unsigned short* inv;      // m: sample at position q
  const unsigned short* seg_end;  // kmax x 32: trip count after which segment r of lane l ends (0xffff: no such segment)
  const unsigned char* gfirst;    // 32: group of lane l's first segment
  const unsigned char* glo;       // G: first lane holding samples of group g
  const unsigned char* ghi;       // G: last lane holding samples of group g
  int kmax;                       // most segments any lane has
};

struct DispArgs {
  // inputs (device pointers)
  const void* y;        // gene-major counts, int32 or f64
  int y_is_f64;
  const double* mu;     // gene-major
  const double* w;      // gene-major observation weights or nullptr
  const double* x;      // m x p column-major
  const double* log_alpha_in;  // n
  const double* prior_mean;    // n
  double prior_sigmasq, min_log_alpha, kappa_0, tol;
  int maxit, use_prior, use_weights, use_cr;
  double weight_threshold;
  int n, m, p;
  long long ld;
  // outputs (device pointers, length n)
  double* log_alpha;
  int32_t* iter;
  int32_t* iter_accept;
  double* last_change;
  double* initial_lp;
  double* initial_dlp;
  double* last_lp;
  double* last_dlp;
  double* last_d2lp;
  // grid mode (fitDispGrid): when grid != nullptr the line search is replaced by the two-level grid
  const double* grid;
  int grid_n;
  // general-p path (fit_generic.cu): distinct design rows and per-sample row ids, prepared by the C-ABI layer
  const double* xg;   // G x (p|1) (grouped) or m x (p|1) (samplewise)
  const int* gid;     // m
  int G, grouped;
  double* row_scratch;   // general-p path, long rows: per-warp global scratch for the sample rows (set by the launcher)
  // saturated design (G == p, distinct rows X_g invertible): X'WX = X_g' diag(W_g) X_g, so
  // log det = 2 log|det X_g| + sum_g log W_g and tr(B^-1 dB) = sum_g dW_g / W_g -- no p x p algebra at all
  int saturated;
  double sat_logdet;  // 2 log|det X_g|
  SegLayout seg;
  // device scratch supplied by the caller: (4 + 3 n) 32-bit words
  // [work-queue counter | 3 per-mode gene counts | 3 per-mode gene lists]; the launcher zeroes the header
  unsigned int* scratch;
  // filled by the launcher from `scratch`
  unsigned int* counter;
  const unsigned int* mode_counts;
  const int* mode_lists;
};

// experiment: [queue counter | 3 mode counters | 2 more queue counters | pad to 8 | 8 bucket counts | 8 bucket fills | pad],
// then the three gene lists, one bucket code per gene and a scratch list for the bucket sort
constexpr int kDispScratchHead = 32;
constexpr int kDispScratchLists = 5;
inline size_t disp_scratch_bytes(int n) {
  return (kDispScratchHead + kDispScratchLists * (size_t)n) * sizeof(unsigned int);
}

struct BetaArgs {
  const void* y;
  int y_is_f64;
  const double* nf;      // gene-major n x m normalisation factors, or length-m size-factor vector
  int nf_is_vector;
  const double* w;       // gene-major weights or nullptr
  const double* x;       // m x p column-major
  const double* alpha_hat;   // n
  const double* contrast;    // p
  const double* beta_in;     // n x p column-major (R layout), starting values
  const double* lambda;      // p
  int use_weights;
  double tol;
  int maxit;
  int use_qr;                // accepted for interface parity; both settings use the equilibrated Cholesky
  double minmu;
  int n, m, p;
  long long ld;
  // outputs
  double* beta_out;          // n x p column-major
  double* beta_var;          // n x p column-major
  double* iter;              // n (double, as in the reference's NumericVector)
  double* hat_diag;          // gene-major n x m (ld), may be nullptr
  double* mu_out;            // gene-major n x m (ld), may be nullptr (fused mu = nf * exp(x beta))
  double* contrast_num;      // n
  double* contrast_denom;    // n
  double* deviance;          // n
  unsigned int* counter;
  // general-p path (fit_generic.cu)
  const double* xg;
  const int* gid;
  int G, grouped;
  double* row_scratch;   // long rows: per-warp global scratch for the sample rows (set by the launcher)
  SegLayout seg;
};

// nbinomLogLike at the unclamped fitted mean (fit_beta.cu::nb_loglik_kernel)
struct LogLikArgs {
  const void* y;
  int y_is_f64;
  const double* x;        // m x p column-major
  const double* nf;       // gene-major n x ld, or length-m size-factor vector
  int nf_is_vector;
  const double* alpha;    // n
  const double* beta;     // n x p column-major, natural log scale
  const double* w;        // gene-major weights or nullptr
  int n, m, p;
  long long ld;
  double minmu;           // > 0: the log-likelihood (not mu_out) is evaluated at max(mu, minmu) -- what
                          // fitNbinomGLMsOptim stores for the rows it refits (R/fitNbinomGLMs.R:386-398); 0: no clamp
  double* loglik;         // n
  double* mu_out;         // gene-major n x ld or nullptr: nf * exp(x beta), not clamped
};
cudaError_t launch_nb_loglik(const LogLikArgs& a, cudaStream_t stream);

// box-constrained maximisation of the penalised NB log-likelihood for rows the IRLS left unfitted (fit_optim.cu)
struct OptimArgs {
  const void* y;
  int y_is_f64;
  const double* x;        // m x p column-major
  const double* nf;       // gene-major n x ld, or length-m size-factor vector
  int nf_is_vector;
  const double* alpha;    // n
  const double* lambda;   // p, natural-log scale (lambda_log2 / ln(2)^2)
  const double* beta_in;  // n x p column-major start values, natural-log scale (NaN -> 0, clipped into the box)
  const double* w;        // gene-major weights or nullptr
  double bound;           // box half-width on the natural-log scale (30 ln 2)
  int maxit;
  int n, m, p;
  long long ld;
  double* beta_out;       // n x p column-major
  int32_t* converged;     // n: 1 = stationary point reached (optim's convergence == 0)
  int32_t* iter;          // n: Newton iterations used
};
cudaError_t launch_beta_optim(const OptimArgs& a, cudaStream_t stream);

// per-gene pre-steps (pipeline_kernels.cu)
struct PrepArgs {
  const void* y;
  int y_is_f64;
  const double* x;             // m x p column-major
  const double* proj;          // p x m row-major: (X'X)^-1 X'
  const double* size_factors;  // m
  double xim;                  // mean(1 / size factor)
  double min_disp, max_disp, minmu;
  int n, m, p;
  long long ld;
  double* base_mean;           // n
  double* base_var;            // n
  int32_t* all_zero;           // n
  double* alpha0;              // n: min(rough, moments) dispersion, clamped
  double* mu_lin;              // gene-major n x ld or nullptr: linear-model mu * size factor, clamped at minmu
  double* beta0;               // n x p column-major or nullptr: least-squares start values on log(K/s + 0.1)
  // grouped designs (G <= 32 distinct rows; G == 0: not used): P = (X'X)^-1 X' has one distinct column per design
  // group, so P v = sum_g P_g (sum_{j in g} v_j) and the fitted value of a sample is its group's
  const int* gid;              // m: design group of sample j
  const double* xg;            // G x (p|1): the distinct design rows
  int G;
  // observation weights (b200nb_prep_weighted_dev; the unweighted kernels never read these).  base_mean / base_var
  // are then of w * K/s with the RAW weights; rough dispersion, mu_lin and beta0 stay unweighted.
  const double* weights;       // gene-major n x ld, raw assay weights
  double weight_threshold;     // rank test 2 keeps the samples with normalised weight > this
  double* weights_norm;        // gene-major n x ld: weights / row maximum (padding columns written as 0)
  int32_t* weights_fail;       // n: 1 = a rank test of getAndCheckWeights fails
  int32_t* status;             // 1 int, incremented once per row with a negative / NaN / infinite weight or no
                               // positive weight (the reference stops on each of these)
  // gene-specific normalization factors (b200nb_prep_nf_dev; nullptr: size_factors): gene-major n x ld, read in place
  // of size_factors; xim is then mean(1 / colMeans(nf)) over the non-all-zero rows
  const double* nf;
};
cudaError_t launch_prep(const PrepArgs& a, cudaStream_t stream);

// median-of-ratios size factors (size_factors.cu)
struct SizeFactorArgs {
  const void* y;
  int y_is_f64;
  int poscounts;               // 0: type "ratio", 1: type "poscounts" (R/core.R:541-549)
  int n, m;
  long long ld;
  double* loggeomeans;         // n (out)
  double* ratios;              // gene-major n x ld scratch
  double* ratios_colmajor;     // n x m column-major scratch
  double* size_factors;        // m (out)
  int* n_finite;               // out: genes with a finite log geometric mean
  const double* divisor;       // gene-major n x ld or nullptr: the size factors of K / divisor (estimateNormFactors)
};
cudaError_t launch_size_factors(const SizeFactorArgs& a, cudaStream_t stream);

// estimateBetaPriorVar's weighted upper quantile (beta_prior.cuh, launched from size_factors.cu)
struct BetaPriorQArgs {
  const double* beta;          // n x p column-major, log2 scale
  int n;
  const double* base_mean;     // n
  const double* disp_fit;      // n
  const int32_t* col_a;        // k: column c = beta[:, a] - (b < 0 ? 0 : beta[:, b])
  const int32_t* col_b;        // k
  int k;
  double prob;
  double* out_q;               // k (out)
};
cudaError_t launch_beta_prior_quantile(const BetaPriorQArgs& a, cudaStream_t stream);

// estimateSizeFactorsIterate's objective at par and its 2m central-difference points (sf_iterate.cuh, launched from
// size_factors.cu)
struct SfIterateArgs {
  const void* y;
  int y_is_f64;
  const double* q;             // gene-major n x ld: mu / s
  const double* alpha;         // n
  const double* par;           // m: log size factors
  double h, Q;                 // optim's ndeps, the trimmed quantile
  int n, m;
  long long ld;
  int tile;                    // objective columns per tile (>= 1)
  double* abc;                 // 3n scratch: the row sums at the scales 1, e^{-h/m}, e^{+h/m}
  double* ll;                  // n x tile column-major scratch
  double* out;                 // 2m + 1 (out)
};
cudaError_t launch_sf_iterate_objective(const SfIterateArgs& a, cudaStream_t stream);

// The transforms of the normalized counts (transform.cuh, launched from size_factors.cu): VST for fitType "parametric" / "mean", log2(q + pc)
enum TransformMode { kTfVstParametric = 0, kTfVstMean = 1, kTfLog2 = 2 };
struct TransformArgs {
  const void* y;
  int y_is_f64;
  const double* size_factors;  // m, or nullptr when nf is given
  const double* nf;            // gene-major n x ld normalization factors, or nullptr
  int n, m;
  long long ld, ld_out;
  int mode;                    // TransformMode
  double c0, c1, c2, c3, ln2;  // per-mode constants, see transform.cuh
  double* out;                 // gene-major n x ld_out (out)
};
cudaError_t launch_transform(const TransformArgs& a, cudaStream_t stream);

// rlog (rlog.cuh, launched from size_factors.cu): the IRLS fit of rlogData's design [1 | I_m] (or I_m with a frozen
// intercept) and the prior variance of its sample coefficients
struct RlogFitArgs {
  const void* y;
  int y_is_f64;
  const double* size_factors;  // m, or nullptr when nf is given
  const double* nf;            // gene-major n x ld normalization factors, or nullptr
  const double* intercept;     // n frozen log2 intercepts, or nullptr (fit [1 | I_m])
  const double* disp_fit;      // n
  double lambda, lambda0;      // natural-log-scale ridge of the sample columns and of the intercept
  double tol, minmu, log_minmu, ln2;
  int maxit;
  int n, m;
  long long ld, ld_out;
  double* out;                 // gene-major n x ld_out: the rlog values (the sample coefficients while fitting)
  double* out_intercept;       // n fitted log2 intercepts, or nullptr (not written with a frozen intercept)
  double* iter;                // n
};
cudaError_t launch_rlog_fit(const RlogFitArgs& a, cudaStream_t stream);

// Per-CTA partials and running state of the multi-CTA weighted quantile (rlog.cuh)
struct RlogPriorState {
  unsigned long long prefix[2];
  double below[2];
  double dN, S, frac, t_low, t_high;
};
struct RlogPriorArgs {
  const void* y;
  int y_is_f64;
  const double* size_factors;  // m, or nullptr when nf is given
  const double* nf;            // gene-major n x ld, or nullptr
  const double* base_mean;     // n
  const double* disp_fit;      // n
  int n, m;
  long long ld;
  double prob, sd_scale;       // quantile probability; the normal quantile the upper quantile is matched to
  RlogPriorState* st;          // rlog_prior_scratch_bytes(n, m) of device scratch (the state, then per-CTA partials)
  double* out_var;             // 1
  // set by the launcher: the histogram grid (fixed by n and m, so the partials are summed in the same order)
  int ctas, rows_per_block;
  double* part;
};
cudaError_t launch_rlog_prior_var(const RlogPriorArgs& a, cudaStream_t stream);
size_t rlog_prior_scratch_bytes(int n, int m);

// results() and pvalueAdjustment() (results.cuh, launched from size_factors.cu)
struct ResultsGeneArgs {
  const void* y;               // gene-major n x ld original counts (read only with zero_mask)
  int y_is_f64;
  int n, m;
  long long ld;
  const double *lfc, *se, *stat, *pvalue;   // the selected column, n each
  int negate, lrt, alt;        // alt: B200NB_ALT_*
  const int32_t* zero_mask;    // m flags of contrastAllZero's samples, or nullptr
  double lfc_threshold, cooks_cutoff;
  const double* max_cooks;     // n, or nullptr: no Cook's cutoff
  const int32_t* keep;         // n, or nullptr: the two-group heuristic's kept genes
  const int32_t* replace;      // n, or nullptr
  const double* base_mean;     // n (with replace)
  double *out_lfc, *out_se, *out_stat, *out_pvalue;
};
cudaError_t launch_results_gene(const ResultsGeneArgs& a, cudaStream_t stream);

struct ResultsHeuristicArgs {
  const void* y;
  int y_is_f64;
  const int64_t* rows;         // k gene rows of y
  int k, m;
  long long ld, ld_cooks;
  const double* cooks;         // gene-major k x ld_cooks
  int32_t* keep;               // indexed by gene row
};
cudaError_t launch_results_heuristic(const ResultsHeuristicArgs& a, cudaStream_t stream);

struct FilterCutoffArgs {
  const double* filter;        // n
  int n;
  const double* theta;         // one CTA per probability
  double* out;
};
cudaError_t launch_filter_cutoffs(const FilterCutoffArgs& a, int n_theta, cudaStream_t stream);

// the p-values in ascending order (NaN last) and their filter values; a subset is {i : p not NaN, filter >= cutoff}
struct PadjArgs {
  const double* p_sorted;
  const double* filter_sorted;
  const int64_t* order;        // padj: gene position of sorted position i
  int n;
  const double* cutoffs;       // numrej: one per CTA; padj: cutoffs[j], or nullptr for every non-NaN p
  int j, method;               // method: B200NB_PADJ_*
  double alpha;
  int32_t* out_numrej;
  double* out;
};
cudaError_t launch_filter_numrej(const PadjArgs& a, int n_theta, cudaStream_t stream);
cudaError_t launch_padj(const PadjArgs& a, cudaStream_t stream);

// Cook's distances (pipeline_kernels.cu)
struct CooksArgs {
  const void* y;
  int y_is_f64;
  const double* mu;            // gene-major fitted means
  const double* hat;           // gene-major hat diagonals
  const double* size_factors;  // m
  const int* cell_ptr;         // ncell + 1: samples of cell c are cell_samples[cell_ptr[c] .. cell_ptr[c+1])
  const int* cell_samples;     // m: a permutation of 0..m-1 grouped by cell
  int ncell, n, m, p;
  int max_cell;                // samples in the largest cell (the launcher sizes the per-warp scratch by it); 0: unknown
  long long ld;
  double* cooks;               // gene-major n x ld or nullptr
  double* max_cooks;           // n
  double* robust_disp;         // n
  const double* nf;            // gene-major n x ld normalization factors, read in place of size_factors; or nullptr
};
cudaError_t launch_cooks(const CooksArgs& a, cudaStream_t stream);
cudaError_t launch_trend_fit(const double* means, const double* disps, int n, double min_disp, double* out4,
                             cudaStream_t stream);

// returns cudaSuccess or the launch error; kernels are enqueued on `stream`
cudaError_t launch_fit_disp(const DispArgs& a, cudaStream_t stream);
cudaError_t launch_fit_beta(const BetaArgs& a, cudaStream_t stream);
// any p <= kMaxP (shared-memory normal equations, grouped design); used for p > kMaxSmallP
cudaError_t launch_fit_disp_generic(const DispArgs& a, cudaStream_t stream);
cudaError_t launch_fit_beta_generic(const BetaArgs& a, cudaStream_t stream);

// layout helpers (layout.cu)
// column-major n x m (R) -> gene-major n x ld.  elem_size 4 or 8.
cudaError_t launch_to_gene_major(const void* src_colmajor, void* dst, int n, int m, long long ld, int elem_size,
                                 cudaStream_t stream);
// gene-major n x ld -> column-major n x m (f64)
cudaError_t launch_to_col_major(const double* src, double* dst_colmajor, int n, int m, long long ld,
                                cudaStream_t stream);
// 128-bit content hash of a gene-major matrix into out2[0..1] (device); see hostrt.h::hash_elems
cudaError_t launch_hash_gene_major(const void* src, int n, int m, long long ld, int elem_size,
                                   unsigned long long* out2, cudaStream_t stream);
cudaError_t launch_special_test(const double* x, int n, double* lg, double* dg, double* tg, cudaStream_t stream);

int device_sm_count();

// Grid of a persistent-queue kernel: one resident wave (SMs x the CTAs per SM the occupancy calculator allows for
// `threads` and `smem` bytes of dynamic shared memory), and no more CTAs than ceil(n / genes_per_cta) can keep busy;
// at least 1.  Raises the kernel's dynamic shared-memory limit to `smem` first.  The occupancy answer is cached per
// (kernel address, threads, smem).
cudaError_t persistent_grid(const void* kernel, int threads, size_t smem, int genes_per_cta, int n, unsigned* grid);

}  // namespace nb
