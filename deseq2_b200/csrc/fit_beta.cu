// fit_beta.cu -- per-gene ridge-penalised NB IRLS on sm_90a, one warp per gene.
//
// Behavioural contract (WHAT): /root/reference/src/DESeq2.cpp:283-465 (fitBeta): mu = max(nf*exp(X b), minmu),
// w = [wt*]mu/(1+alpha*mu), z = log(mu/nf) + (y-mu)/mu, b = argmin ridge WLS, |b|>30 => iter=maxit (diverged b
// kept), deviance = -2 sum [wt*] log NB(y; mu, 1/alpha), stop when t>0 and |dev-dev_old|/(|dev|+0.1) < tol, NaN =>
// iter=maxit (the stop and divergence rules are deseq_rules.cuh's); post-loop hat diagonal, sandwich covariance,
// contrast numerator/denominator (:429-455).
// HOW is new:
//   * one fused pass per iteration updates mu, the deviance, AND accumulates X'WX / X'Wz for the next solve,
//     so a gene costs (iterations + 1) passes over its row (held in shared memory) and one warp all-reduce
//     per pass; the post-loop block reuses the last pass's X'WX (the reference recomputes it three times);
//   * both reference branches (QR :344-356, normal equations :398) map to one Jacobi-equilibrated Cholesky of
//     X'WX + Lambda in registers (smallp.cuh) -- algebraically identical, agrees with the QR branch far inside
//     the 1e-6 contract (tests/test_parity_gpu.py, incl. the badly scaled covariate of test_optim.R);
//   * log NB is evaluated in the direct form with the mu-independent part
//     sum [wt*](lgamma(y+r)-lgamma(r)-lgamma(y+1)) hoisted out of the loop and the mu-dependent part written as
//     y (log mu + log alpha) - (y + r) log1p(mu alpha), r = 1/alpha: one exp and one log1p per sample per
//     iteration, accurate for every alpha in [1e-8, m];
//   * log(mu/nf) is never formed: mu = exp(eta + log nf) so log(mu/nf) = eta unless the minmu clamp bites.
#include "deseq_rules.cuh"
#include "engine.h"
#include "nb_logdens.cuh"
#include "smallp.cuh"

namespace nb {
namespace {

struct BetaRow {
  const double* y;
  const double* lnf;   // log normalisation factor per sample (CTA-shared when nf is a size-factor vector)
  double* mu;
  const double* w;
  const double* x;     // shared, column-major stride mpad
  int m, mpad;
};

constexpr int pow2_ceil_b(int n) { int p = 1; while (p < n) p <<= 1; return p; }

// One fused IRLS pass: mu (stored to shared memory), mu-dependent part of the deviance, X'WX and X'Wz.
// Four samples per lane per trip (clamped index + validity factor) for instruction-level parallelism.
// GL = lanes per gene: 32 (one warp per gene) or 16 / 8 (fit_beta_grp.cuh; `lane` is then the lane index
// inside the group and the reduction stays inside the group).
template <int P, bool USE_W, int GL = 32>
__device__ __forceinline__ void beta_pass(const BetaRow& rv, const double (&beta)[P], double alpha, double r,
                                          double log_alpha, double minmu, double log_minmu, int lane, double& dev_var,
                                          SymP<P>& XtWX, double (&XtWz)[P]) {
  constexpr int NS = SymP<P>::N;
  constexpr int NA = pow2_ceil_b(1 + NS + P);
  double acc[NA];
#pragma unroll
  for (int i = 0; i < NA; i++) acc[i] = 0.0;
  const int mlast = rv.m - 1;
  for (int j0 = lane; j0 < rv.m; j0 += 4 * GL) {
#pragma unroll
    for (int u = 0; u < 4; u++) {
      if (GL != 32 && (j0 - lane) + GL * u >= rv.m) break;   // narrow groups: skip sweeps with no sample at all
      const int jr = j0 + GL * u;
      const int j = min(jr, mlast);
      double vw = (jr < rv.m) ? 1.0 : 0.0;
      double xv[P];
      double eta = 0.0;
#pragma unroll
      for (int k = 0; k < P; k++) {
        xv[k] = rv.x[k * rv.mpad + j];
        eta = fma(xv[k], beta[k], eta);
      }
      const double lnf = rv.lnf[j];
      const double le = eta + lnf;
      // fmax(NaN, minmu) = minmu, as in the reference (:326); huge |eta| takes libm's exp for inf / 0
      double mu = fmax((fabs(le) < 700.0) ? exp_fast(le) : exp(le), minmu);
      const double lmu = (mu == minmu) ? log_minmu : le;
      if (jr < rv.m) rv.mu[j] = mu;
      const double y = rv.y[j];
      const double am = mu * alpha;
      const double u1 = 1.0 + am;
      const double iu1 = rcp_fast(u1);
      double w = mu * iu1 * vw;
      if (USE_W) {
        const double wt = rv.w[j];
        w *= wt;
        vw *= wt;
      }
      const double z = (lmu - lnf) + fma(y, rcp_fast(mu), -1.0);
      // log1p(am) = log(u1) + (am - (u1 - 1)) / u1
      const double l1p = log_pos(u1) + (am - (u1 - 1.0)) * iu1;
      acc[0] = fma(vw, fma(y, lmu + log_alpha, -(y + r) * l1p), acc[0]);
      const double wz = w * z;
#pragma unroll
      for (int a = 0; a < P; a++) {
        acc[1 + NS + a] = fma(wz, xv[a], acc[1 + NS + a]);
        const double wx = w * xv[a];
#pragma unroll
        for (int b = 0; b <= a; b++) acc[1 + a * (a + 1) / 2 + b] = fma(wx, xv[b], acc[1 + a * (a + 1) / 2 + b]);
      }
    }
  }
  if constexpr (GL == 32) {
    warp_allreduce_sum_rs<NA>(acc, lane);
  } else if constexpr (NA <= GL) {
    group_allreduce_sum_rs<NA, GL>(acc, lane);
  } else {
    group_allreduce_sum_n<NA, GL>(acc);
  }
  dev_var = acc[0];
#pragma unroll
  for (int i = 0; i < NS; i++) XtWX.v[i] = acc[1 + i];
#pragma unroll
  for (int a = 0; a < P; a++) XtWz[a] = acc[1 + NS + a];
}

// stage the row of gene g (128-bit loads) into the group's shared-memory rows: y, log nf (nf matrix only), w (USE_W);
// lg = lane inside the group of GL lanes.  `valid` false: the group has no gene this round and nothing is loaded.
template <bool USE_W, int GL>
__device__ __forceinline__ void stage_beta_row(const BetaArgs& A, size_t off, bool valid, int mpad, int lg, double* ys,
                                               double* lnfs, double* wsm) {
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
}

// mu-independent part of the deviance: sum_j [w_j] (lgamma(y_j + r) - lgamma(r) - lgamma(y_j + 1)), 0 when maxit = 0
template <bool USE_W, int GL>
__device__ __forceinline__ double deviance_const(const BetaArgs& A, const BetaRow& rv, double r, int lg) {
  if (A.maxit <= 0) return 0.0;
  const double lg_r = lgamma_pos(r);
  double c = 0.0;
  for (int j = lg; j < A.m; j += GL) {
    const double y = rv.y[j];
    double t = lgamma_diff(y, r, lg_r) - log_factorial(y);
    if (USE_W) t *= rv.w[j];
    c += t;
  }
  return group_allreduce_sum<GL>(c);
}

// post-loop block (src/DESeq2.cpp:429-455): hat diagonal, sandwich variance, contrast and the stores of gene g.  XtWX
// belongs to the mu currently in shared memory.  Every lane of the group computes; `valid` false stores nothing.
template <int P, bool USE_W, int GL>
__device__ __forceinline__ void beta_finish(const BetaArgs& A, unsigned int g, bool valid, int lg, const BetaRow& rv,
                                            const SymP<P>& XtWX, const double (&lam)[P], const double (&contrast)[P],
                                            const double (&beta)[P], double alpha, const IrlsProgress& ir) {
  const size_t off = (size_t)g * A.ld;
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
      const double mu = rv.mu[j];
      if (A.mu_out != nullptr) A.mu_out[off + j] = mu;
      if (A.hat_diag != nullptr) {
        double w = mu * rcp_fast(fma(alpha, mu, 1.0));
        if (USE_W) w *= rv.w[j];
        double xv[P];
#pragma unroll
        for (int k = 0; k < P; k++) xv[k] = rv.x[k * rv.mpad + j];
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
    A.iter[g] = ir.it;
    A.contrast_num[g] = cn;
    A.contrast_denom[g] = sqrt(cd);
    A.deviance[g] = ir.dev;
  }
}

#ifndef NB_LB_THREADS
#define NB_LB_THREADS 256
#define NB_LB_CTAS 2
#endif
template <int P, bool USE_W>
__global__ void __launch_bounds__(NB_LB_THREADS, NB_LB_CTAS) fit_beta_kernel(const BetaArgs A, int warps_per_cta, int mpad) {
  extern __shared__ __align__(16) double smem[];
  init_log_table();
  init_lfact_table();
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  // per-warp rows: y, mu, [lnf if nf is a matrix], [w]
  const int nrow = 2 + (A.nf_is_vector ? 0 : 1) + (USE_W ? 1 : 0);
  double* xs = smem;                                 // P * mpad
  double* lnf_shared = xs + (size_t)P * mpad;        // mpad (used when nf is a vector)
  double* rowbase = lnf_shared + mpad + (size_t)warp * nrow * mpad;
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
    if (lane == 0) g = atomicAdd(A.counter, 1u);
    g = __shfl_sync(0xffffffffu, g, 0);
    if (g >= (unsigned int)A.n) break;
    stage_beta_row<USE_W, 32>(A, (size_t)g * A.ld, true, mpad, lane, ys, lnfs, wsm);

    double beta[P];
#pragma unroll
    for (int k = 0; k < P; k++) beta[k] = A.beta_in[(size_t)g + (size_t)A.n * k];
    const double alpha = A.alpha_hat[g];
    const double r = 1.0 / alpha;
    const double log_alpha = log(alpha);
    const double devc = deviance_const<USE_W, 32>(A, rv, r, lane);

    SymP<P> XtWX;
    double XtWz[P];
    double dv;
    IrlsProgress ir;
    // t = -1: the pass at the starting values (mu, weights for the first solve); t >= 0: IRLS iterations
    for (int t = -1; t < A.maxit; t++) {
      if (t >= 0) {
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
        if (big) { ir.diverged(A.maxit); break; }
      }
      beta_pass<P, USE_W>(rv, beta, alpha, r, log_alpha, minmu, log_minmu, lane, dv, XtWX, XtWz);
      if (t >= 0 && ir.stop_after_pass(dv, devc, A)) break;
    }
    beta_finish<P, USE_W, 32>(A, g, true, lane, rv, XtWX, lam, contrast, beta, alpha, ir);
    __syncwarp();
  }
}

#include "fit_beta_grp.cuh"

template <int P, bool USE_W, int GL>
cudaError_t launch_beta_grp(const BetaArgs& a, int mpad, size_t fixed, size_t rowbytes, cudaStream_t stream,
                            bool& launched) {
  constexpr int NG = 32 / GL, GW = GrpShape<GL>::threads / 32;
  const size_t gsmem = fixed + (size_t)GW * NG * rowbytes;
  launched = false;
  if (gsmem > (size_t)227 * 1024 / GrpShape<GL>::ctas) return cudaSuccess;
  auto kg = fit_beta_grp_kernel<P, USE_W, GL>;
  unsigned grid = 0;
  const cudaError_t e = persistent_grid(reinterpret_cast<const void*>(kg), GrpShape<GL>::threads, gsmem, GW * NG, a.n, &grid);
  if (e != cudaSuccess) return e;
  kg<<<grid, GrpShape<GL>::threads, gsmem, stream>>>(a, mpad);
  launched = true;
  return cudaGetLastError();
}

// shared memory of the small-p IRLS kernels: the staged design and the log size-factor row (P + 1 rows of mpad) once
// per CTA, and per warp (or lane group) the y and mu rows, the log nf row of an nf matrix and the weights
struct BetaSmem {
  int mpad;
  size_t fixed, rowbytes;
};
BetaSmem beta_smem(int m, int p, bool use_w, bool nf_is_vector) {
  const int mpad = (m + 3) & ~3;
  const int nrow = 2 + (nf_is_vector ? 0 : 1) + (use_w ? 1 : 0);
  return {mpad, (size_t)(p + 1) * mpad * sizeof(double), (size_t)nrow * mpad * sizeof(double)};
}
constexpr size_t kBetaSmemCap = 227 * 1024;
// a one-warp plan must also leave room for the kernels' static shared memory, which counts against the same 227 KB per
// block: the log and log y! tables, 5152 bytes (ptxas -v)
constexpr size_t kBetaSmemCapOneWarp = kBetaSmemCap - 5152;

template <int P, bool USE_W>
cudaError_t launch_beta_t(const BetaArgs& a, cudaStream_t stream) {
  const BetaSmem S = beta_smem(a.m, P, USE_W, a.nf_is_vector != 0);
  const int mpad = S.mpad;
  const size_t fixed = S.fixed, rowbytes = S.rowbytes;
  const size_t smem_cap = kBetaSmemCap;
  int warps = NB_LB_THREADS / 32;
  while (warps > 1 && fixed + warps * rowbytes > smem_cap / 2) warps >>= 1;
  if (fixed + warps * rowbytes > kBetaSmemCapOneWarp) return cudaErrorInvalidValue;   // callers check fit_beta_smallp_fits
  const size_t smem = fixed + warps * rowbytes;
  auto kern = fit_beta_kernel<P, USE_W>;
  cudaError_t e = cudaMemsetAsync(a.counter, 0, sizeof(unsigned int), stream);
  if (e != cudaSuccess) return e;
  {
    const int gl = group_lanes_beta(a.m);
    bool launched = false;
    if (gl == 8) e = launch_beta_grp<P, USE_W, 8>(a, mpad, fixed, rowbytes, stream, launched);
    else if (gl == 16) e = launch_beta_grp<P, USE_W, 16>(a, mpad, fixed, rowbytes, stream, launched);
    if (e != cudaSuccess || launched) return e;
  }
  unsigned grid = 0;
  e = persistent_grid(reinterpret_cast<const void*>(kern), warps * 32, smem, warps, a.n, &grid);
  if (e != cudaSuccess) return e;
  kern<<<grid, warps * 32, smem, stream>>>(a, warps, mpad);
  return cudaGetLastError();
}

template <bool USE_W>
cudaError_t launch_beta_p(const BetaArgs& a, cudaStream_t stream) {
  switch (a.p) {
    case 1: return launch_beta_t<1, USE_W>(a, stream);
    case 2: return launch_beta_t<2, USE_W>(a, stream);
    case 3: return launch_beta_t<3, USE_W>(a, stream);
    case 4: return launch_beta_t<4, USE_W>(a, stream);
    default: return cudaErrorInvalidValue;
  }
}

// ---------------------------------------------------------------- nbinomLogLike at the UNCLAMPED fitted mean
// What R recomputes right after the native call (R/fitNbinomGLMs.R:180-182): mu = nf * exp(x beta) -- no minmu clamp --
// and logLike = rowSums([w *] dnbinom(y, mu = mu, size = 1/alpha, log = TRUE)) (nbinomLogLike, R/core.R:2208-2217).
// nbinomLRT's statistic is 2 (logLike_full - logLike_reduced) (R/core.R:1877) and Cook's distances use this mean
// (R/core.R:1457): both differ from the IRLS kernel's clamped deviance / mean whenever a fitted mean sits below minmu
// (a design cell of zeros).  One warp per gene, any p <= kMaxP, same direct-form log NB as beta_pass.
__global__ void __launch_bounds__(256) nb_loglik_kernel(const LogLikArgs A) {
  init_log_table();
  init_lfact_table();
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (g >= A.n) return;
  const size_t off = (size_t)g * A.ld;
  const double alpha = A.alpha[g];
  const double r = 1.0 / alpha, log_alpha = log(alpha), lg_r = lgamma_pos(r);
  double acc = 0.0;
  for (int j = lane; j < A.m; j += 32) {
    double eta = 0.0;
    for (int k = 0; k < A.p; k++) eta = fma(__ldg(A.x + (size_t)k * A.m + j), A.beta[(size_t)g + (size_t)A.n * k], eta);
    const double nf = A.nf_is_vector ? __ldg(A.nf + j) : A.nf[off + j];
    const double le = eta + log(nf);
    double mu = (fabs(le) < 700.0) ? exp_fast(le) : exp(le);
    if (A.mu_out != nullptr) A.mu_out[off + j] = mu;
    double lmu = le;
    if (A.minmu > 0.0 && !(mu >= A.minmu)) {
      mu = A.minmu;
      lmu = log(A.minmu);
    }
    const double y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + j]
                                : (double)static_cast<const int32_t*>(A.y)[off + j];
    double t;
    if (mu == 0.0) {
      t = (y == 0.0) ? 0.0 : -INFINITY;            // dnbinom_mu: point mass at zero
    } else {
      const double am = mu * alpha, u1 = 1.0 + am;
      const double l1p = log_pos(u1) + (am - (u1 - 1.0)) * rcp_fast(u1);
      t = lgamma_diff(y, r, lg_r) - log_factorial(y) + fma(y, lmu + log_alpha, -(y + r) * l1p);
    }
    if (A.w != nullptr) t *= A.w[off + j];
    acc += t;
  }
  acc = warp_allreduce_sum(acc);
  if (lane == 0) A.loglik[g] = acc;
}

}  // namespace

cudaError_t launch_nb_loglik(const LogLikArgs& a, cudaStream_t stream) {
  if (a.n == 0) return cudaSuccess;
  nb_loglik_kernel<<<(a.n + 7) / 8, 256, 0, stream>>>(a);
  return cudaGetLastError();
}

bool fit_beta_smallp_fits(int m, int p, int use_weights, int nf_is_vector) {
  const BetaSmem S = beta_smem(m, p, use_weights != 0, nf_is_vector != 0);
  return S.fixed + S.rowbytes <= kBetaSmemCapOneWarp;
}

cudaError_t launch_fit_beta(const BetaArgs& a, cudaStream_t stream) {
  if (a.n == 0) return cudaSuccess;
  return a.use_weights ? launch_beta_p<true>(a, stream) : launch_beta_p<false>(a, stream);
}

}  // namespace nb
