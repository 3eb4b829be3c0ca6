// fit_disp_grp.cuh -- several genes per warp (the default for m <= ~330 samples: two genes per warp at C2's 100
// samples, four with table-length ordering at 12).
//
// Included by fit_disp.cu inside namespace nb::{anonymous}.  The product kernel gives a gene the whole warp: at
// m = 100 the sample loop is 4 sweeps of 32 lanes (22 % of the last sweep idle) and everything that happens once per
// evaluation -- exp / reciprocal of alpha, the reduction of the 8 partial sums, the Cox-Reid determinant and trace,
// the prior, the Armijo bookkeeping -- is paid per gene; the work model in DESIGN.md section 4.1 puts that fixed part
// at roughly 40 % of the ~1000 warp-instructions of an evaluation.  Here a warp holds NG = 32 / GL genes, GL lanes
// each (GL = 16: 7 sweeps of 16 lanes for m = 100), and every instruction of the fixed part serves NG genes at once.
//
// Control flow stays warp-uniform (every lane reaches every shuffle): a ROUND loads one gene per group, then all groups
// iterate the line search together; a group whose gene has stopped (or that got no gene) keeps executing with its
// state frozen until the slowest group of the warp is done.  Iteration counts of the C2 workload are 11 +/- 1.5, so
// the expected loss is E[max of 2] / mean ~ 8 %.  The arithmetic per gene is the product kernel's (same
// disp_eval_mode / disp_d2 templates with GL lanes), the decisions are the reference's (src/DESeq2.cpp:201-265).
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

// Which width this kernel uses for m samples: B200NB_GROUP_LANES_DISP, else B200NB_GROUP_LANES, = 8 | 16 | 32 forces one
// (32 = the product kernel); otherwise 8 lanes up to 40 samples, 16 above (the launcher falls back to the product
// kernel when the slices do not fit in shared memory).
inline int group_lanes_disp(int m) {
  static const int forced = [] {
    const char* e = getenv("B200NB_GROUP_LANES_DISP");
    if (!e) e = getenv("B200NB_GROUP_LANES");
    const int v = e ? atoi(e) : 0;
    return (v == 8 || v == 16 || v == 32) ? v : 0;
  }();
  if (forced) return forced;
  return m <= 40 ? 8 : 16;
}

// One round of the line search for the NG genes a warp holds (deseq_rules.cuh::DispLineSearch), warp-uniform control
// flow: a group whose gene has stopped, or that got no gene, evaluates at its frozen a until every group is done.
template <int P, bool USE_W, int MODE, int GL, bool IND>
__device__ __forceinline__ void line_search_round(const DispArgs& A, const DispRow& rv, const DispScal& sc,
                                                  unsigned int g, bool valid, double sum_wy, int lg) {
  const double pm = valid ? A.prior_mean[g] : 0.0;
  DispLineSearch ls(valid ? A.log_alpha_in[g] : 0.0, A.kappa_0);
  bool active = valid;               // false once this group's gene has stopped
  while (__any_sync(0xffffffffu, active)) {
    const double a_new = active ? ls.propose() : ls.a;
    double lp_new, dlp_new;
    disp_eval_mode<P, USE_W, true, MODE, GL, IND>(rv, sc, a_new, pm, sum_wy, lg, lp_new, dlp_new);
    // the reference's `for (t = 0; t < maxit; t++)` bounds the proposals
    if (active) active = !ls.take(lp_new, dlp_new, A) && ls.it < A.maxit;
  }
  const double d2 = disp_d2<P, USE_W, GL, IND>(rv, sc, MODE, ls.a, lg);
  if (valid && lg == 0) ls.store(A, g, d2);
}

// One kernel for the three evaluation-mode families, one family after the other, each with its own queue counter
// (scratch[0], [4], [5]) so that all groups of a warp always run the same MODE code.  IND: the variant for indicator
// designs (smallp.cuh); both variants are launched, and the one that does not fit the design returns at once.
template <int P, bool USE_W, int GL, bool IND>
__global__ void __launch_bounds__(GrpShape<GL>::threads, GrpShape<GL>::ctas) fit_disp_grp_kernel(const DispArgs A, int mpad) {
  extern __shared__ __align__(16) double smem[];
  if (indicator_design<P>(A.x, A.m) != IND) return;
  init_log_table();
  constexpr int NG = 32 / GL;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int grp = lane / GL, lg = lane % GL;
  constexpr int NROW = USE_W ? 3 : 2;
  double* xs = smem;                                   // P * mpad
  const size_t slice = (size_t)NROW * mpad + kTabMax;
  double* rowbase = smem + (size_t)P * mpad + ((size_t)warp * NG + grp) * slice;
  DispWarpSmem S{rowbase, rowbase + mpad, USE_W ? rowbase + 2 * mpad : nullptr, rowbase + (size_t)NROW * mpad};
  for (int idx = threadIdx.x; idx < P * A.m; idx += blockDim.x) {
    const int k = idx / A.m, j = idx - k * A.m;
    xs[k * mpad + j] = A.x[idx];
  }
  // the slices are evaluated even when a group holds no gene yet: give them finite contents
  for (size_t i = threadIdx.x; i < (size_t)(blockDim.x >> 5) * NG * slice; i += blockDim.x)
    smem[(size_t)P * mpad + i] = 1.0;
  __syncthreads();

  DispRow rv{S.ys, S.mus, S.wsm, xs, S.tab, A.m, mpad, 0};
  const DispScal sc{A.prior_sigmasq, 1.0 / A.prior_sigmasq, A.weight_threshold, A.use_prior, A.use_cr};
  const unsigned int n0 = A.mode_counts[MODE_TAB], n1 = A.mode_counts[MODE_BIG];
  const unsigned int n2 = (unsigned int)A.n - n0 - n1;

#pragma unroll 1
  for (int mode = 0; mode < 3; mode++) {
    const unsigned int limit = (mode == MODE_TAB) ? n0 : (mode == MODE_BIG) ? n1 : n2;
    unsigned int* counter = (mode == MODE_TAB) ? A.counter : A.counter + 3 + mode;   // scratch[0], [4], [5]
    const int* list = A.mode_lists + (size_t)mode * A.n;
    for (;;) {
      unsigned int q = 0;
      if (lg == 0) q = atomicAdd(counter, 1u);
      q = __shfl_sync(0xffffffffu, q, grp * GL);
      const bool valid = q < limit;
      if (!__any_sync(0xffffffffu, valid)) break;
      const unsigned int g = valid ? (unsigned int)list[q] : 0u;
      double sum_wy, ymax;
      stage_row<USE_W, GL>(A, g, valid, mpad, lg, S, sum_wy, ymax);
      if (mode == MODE_TAB) {
        build_table<USE_W, GL>(S, A.m, lg);
        rv.ntab = valid ? (int)ymax : 0;
        line_search_round<P, USE_W, MODE_TAB, GL, IND>(A, rv, sc, g, valid, sum_wy, lg);
      } else if (mode == MODE_BIG) {
        line_search_round<P, USE_W, MODE_BIG, GL, IND>(A, rv, sc, g, valid, sum_wy, lg);
      } else {
        line_search_round<P, USE_W, MODE_GEN, GL, IND>(A, rv, sc, g, valid, sum_wy, lg);
      }
      __syncwarp();
    }
  }
}
