// fit_beta_grp.cuh -- several genes per warp for the IRLS kernel (the default for m <= ~330 samples: two genes per
// warp at C2's 100 samples, four at 12).  See fit_disp_grp.cuh for the idea;
// included by fit_beta.cu inside namespace nb::{anonymous}.
//
// A warp holds NG = 32 / GL genes, GL lanes each.  Control flow is warp-uniform: a round loads one gene per group, all
// groups run IRLS passes together, a group whose gene has converged / diverged (or that got no gene) keeps executing the
// pass at the coefficients of its last valid pass -- an idempotent recomputation, shared memory and X'WX end up with
// the same values -- until the slowest group of the warp is done.  Arithmetic per gene: the product kernel's
// (stage_beta_row, beta_pass, beta_finish with GL lanes); decisions: deseq_rules.cuh::IrlsProgress.
#pragma once

// CTA shape per group width: 16 lanes (2 genes per warp): 256 threads, 2 CTAs per SM; 8 lanes (4 genes per warp): 128
// threads, 3 CTAs per SM, so that 12 warps x 4 gene slices still fit in shared memory.
#ifndef NB_GRP_SHAPE_DEFINED
#define NB_GRP_SHAPE_DEFINED
#ifndef NB_GRP16_CTAS
#define NB_GRP16_CTAS 2   // resident CTAs per SM the register allocation is bounded for (A/B knobs of the build)
#endif
#ifndef NB_GRP8_CTAS
#define NB_GRP8_CTAS 3
#endif
template <int GL>
struct GrpShape {
  static_assert(GL == 16 || GL == 8, "group width must be 16 or 8 lanes");
  static constexpr int threads = (GL == 8) ? 128 : 256;
  static constexpr int ctas = (GL == 8) ? NB_GRP8_CTAS : NB_GRP16_CTAS;
};
#endif

// Which width this kernel uses for m samples: B200NB_GROUP_LANES_BETA, else B200NB_GROUP_LANES, = 8 | 16 | 32 forces one
// (32 = the product kernel); otherwise 8 lanes up to 40 samples, 16 above (the launcher falls back to the product
// kernel when the slices do not fit in shared memory).
inline int group_lanes_beta(int m) {
  static const int forced = [] {
    const char* e = getenv("B200NB_GROUP_LANES_BETA");
    if (!e) e = getenv("B200NB_GROUP_LANES");
    const int v = e ? atoi(e) : 0;
    return (v == 8 || v == 16 || v == 32) ? v : 0;
  }();
  if (forced) return forced;
  return m <= 40 ? 8 : 16;
}

// IND: the variant for indicator designs (smallp.cuh); both variants are launched, and the one that does not fit the
// design returns at once.
template <int P, bool USE_W, int GL, bool IND>
__global__ void __launch_bounds__(GrpShape<GL>::threads, GrpShape<GL>::ctas) fit_beta_grp_kernel(const BetaArgs A, int mpad) {
  extern __shared__ __align__(16) double smem[];
  if (indicator_design<P>(A.x, A.m) != IND) return;
  init_log_table();
  init_lfact_table();
  constexpr int NG = 32 / GL;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int grp = lane / GL, lg = lane % GL;
  const int nrow = 2 + (A.nf_is_vector ? 0 : 1) + (USE_W ? 1 : 0);
  double* xs = smem;                                 // P * mpad
  double* lnf_shared = xs + (size_t)P * mpad;        // mpad (used when nf is a vector)
  double* rowbase = lnf_shared + mpad + ((size_t)warp * NG + grp) * nrow * mpad;
  double* ys = rowbase;
  double* mus = rowbase + mpad;
  double* lnfs = A.nf_is_vector ? lnf_shared : rowbase + 2 * mpad;
  double* wsm = USE_W ? rowbase + (size_t)(A.nf_is_vector ? 2 : 3) * mpad : nullptr;

  for (int idx = threadIdx.x; idx < P * A.m; idx += blockDim.x) {
    const int k = idx / A.m, j = idx - k * A.m;
    xs[k * mpad + j] = A.x[idx];
  }
  if (A.nf_is_vector)
    for (int j = threadIdx.x; j < A.m; j += blockDim.x) lnf_shared[j] = log(A.nf[j]);
  // slices are evaluated even before a group holds a gene: give them finite contents (y = 1, log nf = 0, w = 1)
  {
    double* rows = lnf_shared + mpad;
    const size_t total = (size_t)(blockDim.x >> 5) * NG * nrow * mpad;
    for (size_t i = threadIdx.x; i < total; i += blockDim.x) {
      const int rowkind = (int)((i / mpad) % nrow);
      rows[i] = (!A.nf_is_vector && rowkind == 2) ? 0.0 : 1.0;
    }
  }
  __syncthreads();

  BetaRow rv{ys, lnfs, mus, wsm, xs, A.m, mpad};
  double lam[P], contrast[P];
#pragma unroll
  for (int k = 0; k < P; k++) {
    lam[k] = A.lambda[k];
    contrast[k] = A.contrast[k];
  }
  const double minmu = A.minmu, log_minmu = log(A.minmu);

  for (;;) {
    unsigned int g = 0;
    if (lg == 0) g = atomicAdd(A.counter, 1u);
    g = __shfl_sync(0xffffffffu, g, grp * GL);
    const bool valid = g < (unsigned int)A.n;
    if (!__any_sync(0xffffffffu, valid)) break;
    if (!valid) g = 0;
    stage_beta_row<USE_W, GL>(A, (size_t)g * A.ld, valid, mpad, lg, ys, lnfs, wsm);

    double beta[P], beta_eval[P];
#pragma unroll
    for (int k = 0; k < P; k++) beta_eval[k] = beta[k] = valid ? A.beta_in[(size_t)g + (size_t)A.n * k] : 0.0;
    const double alpha = valid ? A.alpha_hat[g] : 1.0;
    const double r = 1.0 / alpha;
    const double log_alpha = log(alpha);

    const double devc = deviance_const<USE_W, GL>(A, rv, r, lg);

    SymP<P> XtWX;
    double XtWz[P];
#pragma unroll
    for (int i = 0; i < SymP<P>::N; i++) XtWX.v[i] = 0.0;
#pragma unroll
    for (int k = 0; k < P; k++) XtWz[k] = 0.0;
    IrlsProgress ir;
    bool first = true;       // the pass at the starting values is still to come
    bool active = valid;
    while (__any_sync(0xffffffffu, active)) {
      if (active && !first) {
        ir.start_iteration();
        SymP<P> M = XtWX;
#pragma unroll
        for (int k = 0; k < P; k++) {
          M.at(k, k) += lam[k];
          beta[k] = XtWz[k];
        }
        spd_solve_equilibrated<P>(M, beta);
        bool big = false;
#pragma unroll
        for (int k = 0; k < P; k++) big = big || (fabs(beta[k]) > kBetaLarge);
        if (big) {             // diverged: keep the diverged beta, do not re-evaluate
          ir.diverged(A.maxit);
          active = false;
        }
      }
      // a stopped group re-evaluates at the coefficients of its last valid pass: same mu, same X'WX
      double bev[P];
#pragma unroll
      for (int k = 0; k < P; k++) bev[k] = active ? beta[k] : beta_eval[k];
      SymP<P> XtWX_new;
      double XtWz_new[P];
      double dv;
      beta_pass<P, USE_W, GL, IND>(rv, bev, alpha, r, log_alpha, minmu, log_minmu, lg, dv, XtWX_new, XtWz_new);
      if (active) {
        XtWX = XtWX_new;
#pragma unroll
        for (int k = 0; k < P; k++) {
          XtWz[k] = XtWz_new[k];
          beta_eval[k] = beta[k];
        }
        if (first) first = false;
        else if (ir.stop_after_pass(dv, devc, A)) active = false;
        if (ir.it >= (double)A.maxit) active = false;   // the reference's `for (t = 0; t < maxit; t++)`
      }
    }

    beta_finish<P, USE_W, GL, IND>(A, g, valid, lg, rv, XtWX, lam, contrast, beta, alpha, ir);
    __syncwarp();
  }
}
