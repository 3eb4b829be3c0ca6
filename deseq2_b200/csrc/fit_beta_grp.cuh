// fit_beta_grp.cuh -- several genes per warp for the IRLS kernel (the default for m <= ~330 samples: two genes per
// warp at C2's 100 samples, four at 12).  See fit_disp_grp.cuh for the idea;
// included by fit_beta.cu inside namespace nb::{anonymous}.
//
// A warp holds NG = 32 / GL genes, GL lanes each.  Control flow is warp-uniform: a round loads one gene per group, all
// groups run IRLS passes together, a group whose gene has converged / diverged (or that got no gene) keeps executing the
// pass at the coefficients of its last valid pass -- an idempotent recomputation, shared memory and X'WX end up with
// the same values -- until the slowest group of the warp is done.  Arithmetic per gene: the product kernel's
// (beta_pass with GL lanes); decisions: the reference's (src/DESeq2.cpp:334-383 / :388-425, post-loop :429-455).
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

template <int P, bool USE_W, int GL>
__global__ void __launch_bounds__(GrpShape<GL>::threads, GrpShape<GL>::ctas) fit_beta_grp_kernel(const BetaArgs A, int mpad) {
  extern __shared__ __align__(16) double smem[];
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
  const double large = 30.0;

  for (;;) {
    unsigned int g = 0;
    if (lg == 0) g = atomicAdd(A.counter, 1u);
    g = __shfl_sync(0xffffffffu, g, grp * GL);
    const bool valid = g < (unsigned int)A.n;
    if (!__any_sync(0xffffffffu, valid)) break;
    if (!valid) g = 0;
    const size_t off = (size_t)g * A.ld;

    // ---- stage the row (128-bit loads), GL lanes
    if (valid) {
      for (int j4 = lg * 4; j4 < mpad; j4 += 4 * GL) {
        double yv[4];
        if (A.y_is_f64) {
          const double2* p2 = reinterpret_cast<const double2*>(static_cast<const double*>(A.y) + off + j4);
          const double2 a0 = __ldg(p2), a1 = __ldg(p2 + 1);
          yv[0] = a0.x; yv[1] = a0.y; yv[2] = a1.x; yv[3] = a1.y;
        } else {
          const int4 v = __ldg(reinterpret_cast<const int4*>(static_cast<const int32_t*>(A.y) + off + j4));
          yv[0] = v.x; yv[1] = v.y; yv[2] = v.z; yv[3] = v.w;
        }
#pragma unroll
        for (int q = 0; q < 4; q++) ys[j4 + q] = yv[q];
        if (!A.nf_is_vector) {
          const double2* n2 = reinterpret_cast<const double2*>(A.nf + off + j4);
          const double2 n0 = __ldg(n2), n1 = __ldg(n2 + 1);
          lnfs[j4 + 0] = log(n0.x); lnfs[j4 + 1] = log(n0.y); lnfs[j4 + 2] = log(n1.x); lnfs[j4 + 3] = log(n1.y);
        }
        if (USE_W) {
          const double2* w2 = reinterpret_cast<const double2*>(A.w + off + j4);
          const double2 w0 = __ldg(w2), w1 = __ldg(w2 + 1);
          wsm[j4 + 0] = w0.x; wsm[j4 + 1] = w0.y; wsm[j4 + 2] = w1.x; wsm[j4 + 3] = w1.y;
        }
      }
    }
    __syncwarp();

    double beta[P], beta_eval[P];
#pragma unroll
    for (int k = 0; k < P; k++) beta_eval[k] = beta[k] = valid ? A.beta_in[(size_t)g + (size_t)A.n * k] : 0.0;
    const double alpha = valid ? A.alpha_hat[g] : 1.0;
    const double r = 1.0 / alpha;
    const double log_alpha = log(alpha);

    // mu-independent part of the deviance
    double devc = 0.0;
    if (A.maxit > 0) {
      const double lg_r = lgamma_pos(r);
      double c = 0.0;
      for (int j = lg; j < A.m; j += GL) {
        const double y = ys[j];
        double t = lgamma_diff(y, r, lg_r) - log_factorial(y);
        if (USE_W) t *= wsm[j];
        c += t;
      }
#pragma unroll
      for (int o = GL / 2; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
      devc = c;
    }

    SymP<P> XtWX;
    double XtWz[P];
#pragma unroll
    for (int i = 0; i < SymP<P>::N; i++) XtWX.v[i] = 0.0;
#pragma unroll
    for (int k = 0; k < P; k++) XtWz[k] = 0.0;
    double dev = 0.0, dev_old = 0.0;
    double it = 0.0;
    bool first = true;       // the pass at the starting values is still to come
    bool active = valid;
    while (__any_sync(0xffffffffu, active)) {
      if (active && !first) {
        it += 1.0;
        SymP<P> M = XtWX;
#pragma unroll
        for (int k = 0; k < P; k++) {
          M.at(k, k) += lam[k];
          beta[k] = XtWz[k];
        }
        spd_solve_equilibrated<P>(M, beta);
        bool big = false;
#pragma unroll
        for (int k = 0; k < P; k++) big = big || (fabs(beta[k]) > large);
        if (big) {             // diverged: keep the diverged beta, do not re-evaluate (src/DESeq2.cpp:357-360)
          it = (double)A.maxit;
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
      beta_pass<P, USE_W, GL>(rv, bev, alpha, r, log_alpha, minmu, log_minmu, lg, dv, XtWX_new, XtWz_new);
      if (active) {
        XtWX = XtWX_new;
#pragma unroll
        for (int k = 0; k < P; k++) {
          XtWz[k] = XtWz_new[k];
          beta_eval[k] = beta[k];
        }
        if (first) {
          first = false;
        } else {
          dev = -2.0 * (dv + devc);
          const double conv_test = fabs(dev - dev_old) / (fabs(dev) + 0.1);
          if (isnan(conv_test)) {
            it = (double)A.maxit;
            active = false;
          } else if ((it > 1.0) && (conv_test < A.tol)) {
            active = false;
          } else {
            dev_old = dev;
          }
        }
        if (it >= (double)A.maxit) active = false;
      }
    }

    // ---- post-loop block (src/DESeq2.cpp:429-455); XtWX belongs to the mu currently in shared memory
    SymP<P> M = XtWX, Ainv;
    double s[P];
#pragma unroll
    for (int k = 0; k < P; k++) M.at(k, k) += lam[k];
#pragma unroll
    for (int k = 0; k < P; k++) s[k] = rsqrt(M.get(k, k));
#pragma unroll
    for (int a = 0; a < P; a++)
#pragma unroll
      for (int b = 0; b <= a; b++) M.at(a, b) *= s[a] * s[b];
    chol_factor<P>(M);
    chol_inverse<P>(M, Ainv);
#pragma unroll
    for (int a = 0; a < P; a++)
#pragma unroll
      for (int b = 0; b <= a; b++) Ainv.at(a, b) *= s[a] * s[b];

    __syncwarp();
    if (valid && (A.hat_diag != nullptr || A.mu_out != nullptr)) {
      for (int j = lg; j < A.m; j += GL) {
        const double mu = mus[j];
        if (A.mu_out != nullptr) A.mu_out[off + j] = mu;
        if (A.hat_diag != nullptr) {
          double w = mu * rcp_fast(fma(alpha, mu, 1.0));
          if (USE_W) w *= wsm[j];
          double xv[P];
#pragma unroll
          for (int k = 0; k < P; k++) xv[k] = xs[k * mpad + j];
          double q = 0.0;
#pragma unroll
          for (int a = 0; a < P; a++) {
            q = fma(xv[a] * xv[a], Ainv.get(a, a), q);
#pragma unroll
            for (int b = 0; b < a; b++) q = fma(2.0 * xv[a] * xv[b], Ainv.get(a, b), q);
          }
          A.hat_diag[off + j] = w * q;
        }
      }
    }
    // sigma = Ainv * XtWX * Ainv
    double T[P][P];
    sym_mul_full<P>(Ainv, XtWX, T);
    double cn = 0.0, cd = 0.0;
    double var[P];
    double sc_[P];   // sigma * contrast
#pragma unroll
    for (int a = 0; a < P; a++) sc_[a] = 0.0;
#pragma unroll
    for (int a = 0; a < P; a++) {
#pragma unroll
      for (int b = 0; b < P; b++) {
        double sab = 0.0;
#pragma unroll
        for (int k = 0; k < P; k++) sab = fma(T[a][k], Ainv.get(k, b), sab);
        if (a == b) var[a] = sab;
        sc_[a] = fma(sab, contrast[b], sc_[a]);
      }
      cn = fma(contrast[a], beta[a], cn);
    }
#pragma unroll
    for (int a = 0; a < P; a++) cd = fma(contrast[a], sc_[a], cd);
    if (valid && lg == 0) {
#pragma unroll
      for (int k = 0; k < P; k++) {
        A.beta_out[(size_t)g + (size_t)A.n * k] = beta[k];
        A.beta_var[(size_t)g + (size_t)A.n * k] = var[k];
      }
      A.iter[g] = it;
      A.contrast_num[g] = cn;
      A.contrast_denom[g] = sqrt(cd);
      A.deviance[g] = dev;
    }
    __syncwarp();
  }
}
