// fit_generic.cu -- fitDisp / fitDispGrid / fitBeta for any design width p <= 32 (configs with p > 4, e.g. the
// 10-level factor of BASELINE.json config 4 and its 11-column expanded matrix), one warp per gene.
//
// Same behavioural contract as fit_disp.cu / fit_beta.cu (src/DESeq2.cpp:31-158, 164-277, 283-465, 469-513).
// What changes is how the p x p normal equations are formed, because p(p+1)/2 accumulators per lane no longer
// fit in registers:
//   * the design matrix is reduced on the host to its G distinct rows ("groups", exactly what the reference's
//     modelMatrixGroups() computes, R/core.R:2450) plus a group id per sample.  X'WX = sum_g W_g x_g x_g' with
//     W_g = sum_{j in g} w_j, so a sample pass only accumulates per-group scalars (lane-private shared-memory
//     slots, no conflicts), and the p x p matrices are assembled from G terms instead of m;
//     tr(B^-1 dB) = sum_g dW_g x_g' B^-1 x_g needs no dB at all.  Factor designs have G ~ p (config 4: G = 10);
//   * designs with more than 32 distinct rows (continuous covariates) take the same code with "group" = sample
//     (SAMPLEWISE): per-sample weights are kept in a shared-memory row and the matrices are summed over m terms;
//   * matrices live in the warp's shared-memory slice (row stride p|1, conflict-free); Cholesky, inverse and
//     triangular solves are cooperative with lanes = rows.
// The per-sample arithmetic (fused lp/dlp pass, integer-count factor table, fused IRLS pass) is the same as in the
// register-resident small-p kernels.
#include <stdlib.h>

#include <mutex>

#include "deseq_rules.cuh"
#include "engine.h"
#include "nbmath.cuh"

// Unroll factors of the two per-sample loops.  These kernels are instruction-cache bound, not latency bound (large
// bodies, few warps per SM at the config-4 shape), so the loops are not unrolled by default.
#ifndef NB_EXP_GEN_UNROLL_DISP
#define NB_EXP_GEN_UNROLL_DISP 1
#endif
#ifndef NB_EXP_GEN_UNROLL_BETA
#define NB_EXP_GEN_UNROLL_BETA 1
#endif

namespace nb {
namespace {

constexpr int kTabMaxG = 256;
constexpr int kUnrollDisp = NB_EXP_GEN_UNROLL_DISP, kUnrollBeta = NB_EXP_GEN_UNROLL_BETA;

// ---------------------------------------------------------------- cooperative dense helpers (lanes = rows)

// in-place lower Cholesky of the p x p matrix A (row stride ps); upper triangle is left untouched
__device__ __forceinline__ void chol_smem(double* A, int p, int ps, int lane) {
  for (int c = 0; c < p; c++) {
    __syncwarp();
    const double l = sqrt(A[c * ps + c]);
    const double il = 1.0 / l;
    __syncwarp();
    if (lane == c) A[c * ps + c] = l;
    if (lane > c && lane < p) A[lane * ps + c] *= il;
    __syncwarp();
    if (lane > c && lane < p) {
      const double arc = A[lane * ps + c];
      for (int k = c + 1; k <= lane; k++) A[lane * ps + k] -= arc * A[k * ps + c];
    }
  }
  __syncwarp();
}

// inv = (L L')^-1, full symmetric storage; lane c computes column c
__device__ __forceinline__ void chol_inverse_smem(const double* L, double* inv, int p, int ps, int lane) {
  if (lane < p) {
    const int c = lane;
    for (int k = 0; k < c; k++) inv[k * ps + c] = 0.0;
    for (int k = c; k < p; k++) {
      double s = (k == c) ? 1.0 : 0.0;
      for (int i = c; i < k; i++) s -= L[k * ps + i] * inv[i * ps + c];
      inv[k * ps + c] = s / L[k * ps + k];
    }
    for (int k = p - 1; k >= 0; k--) {
      double s = inv[k * ps + c];
      for (int i = k + 1; i < p; i++) s -= L[i * ps + k] * inv[i * ps + c];
      inv[k * ps + c] = s / L[k * ps + k];
    }
  }
  __syncwarp();
}

struct Design {
  const double* xg;   // Gx x ps: distinct design rows (GROUPED) or all m rows (SAMPLEWISE)
  const int* gid;     // m: row of xg used by sample j
  int p, ps, G, grouped, m;
  // number of summation terms and the xg row of term t
  __device__ __forceinline__ int terms() const { return grouped ? G : m; }
  __device__ __forceinline__ const double* row(int t) const { return xg + (size_t)(grouped ? t : gid[t]) * ps; }
};

// M = sum_t W[t] x_t x_t'  (full symmetric storage); lane a builds row a
__device__ __forceinline__ void build_xtwx(const Design& D, const double* W, double* M, int lane) {
  const int T = D.terms();
  if (lane < D.p) {
    const int a = lane;
    for (int b = 0; b <= a; b++) M[a * D.ps + b] = 0.0;
    for (int t = 0; t < T; t++) {
      const double* xr = D.row(t);
      const double wa = W[t] * xr[a];
      for (int b = 0; b <= a; b++) M[a * D.ps + b] = fma(wa, xr[b], M[a * D.ps + b]);
    }
  }
  __syncwarp();
  if (lane < D.p)
    for (int b = 0; b < lane; b++) M[b * D.ps + lane] = M[lane * D.ps + b];
  __syncwarp();
}

// q[t] = x_t' Ainv x_t for every term; lanes over terms
__device__ __forceinline__ void quad_forms(const Design& D, const double* Ainv, double* q, int lane) {
  const int T = D.terms();
  for (int t = lane; t < T; t += 32) {
    const double* xr = D.row(t);
    double s = 0.0;
    for (int a = 0; a < D.p; a++) {
      double r = 0.0;
      for (int b = 0; b < D.p; b++) r = fma(Ainv[a * D.ps + b], xr[b], r);
      s = fma(xr[a], r, s);
    }
    q[t] = s;
  }
  __syncwarp();
}

// reduce lane-private accumulators acc[g*32 + lane] into out[g] (GROUPED mode)
__device__ __forceinline__ void reduce_group_acc(const double* acc, double* out, int G, int lane) {
  for (int g = lane; g < G; g += 32) {
    double s = 0.0;
    for (int l = 0; l < 32; l++) s += acc[g * 32 + ((l + lane) & 31)];
    out[g] = s;
  }
  __syncwarp();
}

struct GenWarp {
  double *ys, *r1, *r2, *wsm, *tab;   // rows: y, (mu | lnf), (imu | mu), weights, factor table
  double *accA, *accB, *accC;         // GROUPED: G*32 lane-private slots; SAMPLEWISE: rows of mpad
  double *WA, *WB, *WC, *q;           // per-term sums (GROUPED) / aliases of the rows (SAMPLEWISE), quad forms
  double *M0, *M1, *M2, *M3;          // p x ps matrices
  double *v0, *v1, *v2, *v3;          // length-32 vectors
};

// per-warp shared-memory layout.  Rows of length mpad: y, r1 (optional), r2 (optional), weights (optional);
// factor table (optional); `nacc` accumulator sets (3 for the dispersion kernel, 2 for IRLS).
struct GenShape {
  int has_r1, has_r2, use_w, has_tab, nacc;
  // 0: everything in shared memory.  1: the sample rows live in a per-warp slice of a GLOBAL scratch buffer
  // (L2-resident).  2: so do the samplewise accumulators and quad forms, and the kernel reads the design rows and the
  // row ids from global memory: no array of length m is left in shared memory, so any m fits.
  int rows_global;
};
__host__ __device__ inline int gen_rows(GenShape sh) { return 1 + sh.has_r1 + sh.has_r2 + sh.use_w; }
// the samplewise per-sample sums and quad forms are global (rows_global == 2)
__host__ __device__ inline bool gen_acc_global(int grouped, GenShape sh) { return sh.rows_global == 2 && !grouped; }
__host__ __device__ inline size_t gen_warp_doubles(int mpad, int p, int ps, int G, int grouped, GenShape sh) {
  const size_t terms = grouped ? (size_t)G : (size_t)mpad;
  const size_t acc = grouped ? (size_t)G * 32 : (size_t)mpad;
  const size_t rows = sh.rows_global ? 0 : (size_t)gen_rows(sh);
  const size_t sums = gen_acc_global(grouped, sh) ? 0 : sh.nacc * acc + (grouped ? sh.nacc * terms : 0) + terms;
  return rows * mpad + (sh.has_tab ? kTabMaxG : 0) + sums + 4 * (size_t)p * ps + 4 * 32;
}
// a warp's slice of the global scratch: its sample rows, then (rows_global == 2, samplewise) the nacc sums and q
__host__ __device__ inline size_t gen_global_doubles(int mpad, int grouped, GenShape sh) {
  if (!sh.rows_global) return 0;
  return ((size_t)gen_rows(sh) + (gen_acc_global(grouped, sh) ? sh.nacc + 1 : 0)) * mpad;
}

// `rowbase`: the warp's slice of the global row scratch when sh.rows_global, else ignored (rows come first in `base`)
__device__ __forceinline__ GenWarp carve(double* base, double* rowbase, int mpad, int p, int ps, int G, int grouped,
                                         GenShape sh) {
  GenWarp S;
  const size_t terms = grouped ? (size_t)G : (size_t)mpad;
  const size_t acc = grouped ? (size_t)G * 32 : (size_t)mpad;
  double* q = base;
  double* rq = sh.rows_global ? rowbase : base;
  S.ys = rq; rq += mpad;
  S.r1 = sh.has_r1 ? rq : nullptr; rq += sh.has_r1 ? mpad : 0;
  S.r2 = sh.has_r2 ? rq : nullptr; rq += sh.has_r2 ? mpad : 0;
  S.wsm = sh.use_w ? rq : nullptr; rq += sh.use_w ? mpad : 0;
  if (!sh.rows_global) q = rq;
  S.tab = sh.has_tab ? q : nullptr; q += sh.has_tab ? kTabMaxG : 0;
  const bool acc_global = gen_acc_global(grouped, sh);
  double* t = acc_global ? rq : q;   // the sums and quad forms: in shared memory after the table, or after the rows
  S.accA = t; t += acc;
  S.accB = t; t += acc;
  S.accC = (sh.nacc > 2) ? t : nullptr; t += (sh.nacc > 2) ? acc : 0;
  if (grouped) {
    S.WA = t; t += terms;
    S.WB = t; t += terms;
    S.WC = (sh.nacc > 2) ? t : nullptr; t += (sh.nacc > 2) ? terms : 0;
  } else {
    S.WA = S.accA; S.WB = S.accB; S.WC = S.accC;
  }
  S.q = t; t += terms;
  if (!acc_global) q = t;
  S.M0 = q; q += (size_t)p * ps;
  S.M1 = q; q += (size_t)p * ps;
  S.M2 = q; q += (size_t)p * ps;
  S.M3 = q; q += (size_t)p * ps;
  S.v0 = q; q += 32;
  S.v1 = q; q += 32;
  S.v2 = q; q += 32;
  S.v3 = q;
  return S;
}

__device__ __forceinline__ void zero_acc(double* acc, int G, int lane) {
  for (int g = 0; g < G; g++) acc[g * 32 + lane] = 0.0;
}

// ================================================================ dispersion

struct GDispCtx {
  Design D;
  GenWarp S;
  double prior_sigmasq, inv_sigmasq, weight_threshold;
  int use_prior, use_cr, use_w;
  int tab_mode, ntab;
  int saturated;
  double sat_logdet;
  double sum_wy;
};

// lp, dlp (and, when want2, the second derivative) at log-alpha a.  src/DESeq2.cpp:31-158.
__device__ __forceinline__ void gdisp_eval(const GDispCtx& C, double a, double pm, int lane, bool want_d, bool want2,
                                           double& lp, double& dlp, double& d2lp) {
  const Design& D = C.D;
  const GenWarp& S = C.S;
  const double alpha = exp_fast(a);   // a is confined to [-30, 10] by the line search / grid
  const double r = rcp_fast(alpha);
  const double r2 = r * r;
  double lg_r = 0.0, dg_r = 0.0, tg_r = 0.0;
  if (!C.tab_mode) {
    lgamma_digamma_pos(r, lg_r, dg_r);
    if (want2) tg_r = trigamma_pos(r);
  }
  double s_ll = 0.0, s_dl = 0.0, s_d2 = 0.0;
  if (C.tab_mode) {
    for (int k = lane; k < C.ntab; k += 32) {
      const double ck = S.tab[k];
      const double xk = r + (double)k;
      const double ik = rcp_fast(xk);
      s_ll = fma(ck, log_pos(xk), s_ll);
      s_dl = fma(-ck, ik, s_dl);
      if (want2) s_d2 = fma(-ck * r2, ik * ik, s_d2);
    }
  }
  if (C.use_cr && D.grouped) {
    zero_acc(S.accA, D.G, lane);
    if (want_d) zero_acc(S.accB, D.G, lane);
    if (want2) zero_acc(S.accC, D.G, lane);
  }
  const double* ys = S.ys;
  const double* mus = S.r1;
#pragma unroll kUnrollDisp
  for (int j = lane; j < D.m; j += 32) {
    const double y = ys[j], mu = mus[j];
    // wd = 1/(1/mu + alpha) = mu/(1 + mu alpha); 1/mu never needed: y/mu - 1 = (y - mu)/mu cancels against wd
    const double onema = fma(mu, alpha, 1.0);
    const double wi = rcp_fast(onema);
    const double wd = mu * wi;
    const double l2 = log_pos(onema);
    const double xr = y + r;
    double t = -xr * l2;
    double d = l2 + alpha * (y - mu) * wi;
    double d2 = wd * wd * alpha + y * wi * wi;
    if (!C.tab_mode) {
      double lg, dg;
      lgamma_digamma_pos(xr, lg, dg);
      t += lg - lg_r;
      d += dg_r - dg;
      if (want2) d2 += r2 * (trigamma_pos(xr) - tg_r);
    }
    double wt = 1.0;
    if (C.use_w) wt = S.wsm[j];
    s_ll = fma(wt, t, s_ll);
    s_dl = fma(wt, d, s_dl);
    if (want2) s_d2 = fma(wt, d2, s_d2);
    if (C.use_cr) {
      double wdm = wd;
      if (C.use_w && !(wt > C.weight_threshold)) wdm = 0.0;
      const double dwd = -wdm * wd;
      if (D.grouped) {
        const int slot = D.gid[j] * 32 + lane;
        S.accA[slot] += wdm;
        if (want_d) S.accB[slot] += dwd;
        if (want2) S.accC[slot] += 2.0 * wdm * wd * wd;
      } else {
        S.accA[j] = wdm;
        if (want_d) S.accB[j] = dwd;
        if (want2) S.accC[j] = 2.0 * wdm * wd * wd;
      }
    }
  }
  __syncwarp();
  double red[3] = {s_ll, s_dl, s_d2};
  warp_allreduce_sum_n(red);
  double cr = 0.0, dcr = 0.0, cr2 = 0.0;
  if (C.use_cr && C.saturated) {
    // saturated design: lane g owns group g.  log det B = 2 log|det X_g| + sum log W_g,
    // tr(B^-1 dB) = sum dW/W, tr(B^-1 dB B^-1 dB) = sum (dW/W)^2, tr(B^-1 d2B) = sum d2W/W
    double lw = 0.0, t1 = 0.0, t2 = 0.0, t3 = 0.0;
    for (int g = lane; g < D.G; g += 32) {
      double W = 0.0, dW = 0.0, d2W = 0.0;
      for (int l = 0; l < 32; l++) {
        const int sl = g * 32 + ((l + lane) & 31);
        W += S.accA[sl];
        if (want_d) dW += S.accB[sl];
        if (want2) d2W += S.accC[sl];
      }
      lw += log_pos(W);
      if (want_d) {
        const double iw = rcp_fast(W);
        const double q = dW * iw;
        t1 += q;
        t2 = fma(q, q, t2);
        if (want2) t3 = fma(d2W, iw, t3);
      }
    }
    double rr[4] = {lw, t1, t2, t3};
    warp_allreduce_sum_n(rr);
    cr = -0.5 * (rr[0] + C.sat_logdet);
    dcr = -0.5 * rr[1];
    if (want2) cr2 = 0.5 * rr[1] * rr[1] - 0.5 * (rr[1] * rr[1] - rr[2] + rr[3]);
  } else if (C.use_cr) {
    if (D.grouped) {
      reduce_group_acc(S.accA, S.WA, D.G, lane);
      if (want_d) reduce_group_acc(S.accB, S.WB, D.G, lane);
      if (want2) reduce_group_acc(S.accC, S.WC, D.G, lane);
    }
    double* B = S.M0;
    build_xtwx(D, S.WA, B, lane);
    if (C.use_w) {
      // a column that is all zero on the kept rows is dropped by the reference (:42): make it inert
      if (lane < D.p && B[lane * D.ps + lane] == 0.0) B[lane * D.ps + lane] = 1.0;
      __syncwarp();
    }
    chol_smem(B, D.p, D.ps, lane);
    double ld = (lane < D.p) ? log(B[lane * D.ps + lane]) : 0.0;
    ld = warp_allreduce_sum(ld);
    cr = -0.5 * (2.0 * ld);
    if (want_d) {
      double* Bi = S.M1;
      chol_inverse_smem(B, Bi, D.p, D.ps, lane);
      quad_forms(D, Bi, S.q, lane);
      const int T = D.terms();
      double tr1 = 0.0, tr3 = 0.0;
      for (int t = lane; t < T; t += 32) {
        tr1 = fma(S.WB[t], S.q[t], tr1);
        if (want2) tr3 = fma(S.WC[t], S.q[t], tr3);
      }
      tr1 = warp_allreduce_sum(tr1);
      dcr = -0.5 * tr1;
      if (want2) {
        tr3 = warp_allreduce_sum(tr3);
        double* dB = S.M2;
        double* Mm = S.M3;
        build_xtwx(D, S.WB, dB, lane);
        if (lane < D.p)
          for (int c = 0; c < D.p; c++) {
            double s = 0.0;
            for (int k = 0; k < D.p; k++) s = fma(Bi[lane * D.ps + k], dB[k * D.ps + c], s);
            Mm[lane * D.ps + c] = s;
          }
        __syncwarp();
        double tr2 = 0.0;
        if (lane < D.p)
          for (int k = 0; k < D.p; k++) tr2 = fma(Mm[lane * D.ps + k], Mm[k * D.ps + lane], tr2);
        tr2 = warp_allreduce_sum(tr2);
        cr2 = 0.5 * tr1 * tr1 - 0.5 * (tr1 * tr1 - tr2 + tr3);
      }
    }
  }
  double prior = 0.0, dprior = 0.0;
  if (C.use_prior) {
    const double dd = a - pm;
    prior = -0.5 * dd * dd * C.inv_sigmasq;
    dprior = -dd * C.inv_sigmasq;
  }
  lp = (red[0] + a * C.sum_wy) + prior + cr;
  const double dlp_noprior = (r2 * red[1] + dcr) * alpha;
  dlp = dlp_noprior + dprior;
  if (want2) {
    const double ll2 = -2.0 * r2 * r * red[1] + r2 * red[2];
    d2lp = ((ll2 + cr2) * alpha * alpha + dlp_noprior) + (C.use_prior ? -C.inv_sigmasq : 0.0);
  }
}

// stage y, mu, 1/mu, [w]; returns sum w y, max y, integrality
__device__ __forceinline__ void gstage_disp(const DispArgs& A, unsigned int g, int mpad, int lane, const GenWarp& S,
                                            double& sum_wy, double& ymax, bool& integral) {
  const size_t off = (size_t)g * A.ld;
  double swy = 0.0, ym = 0.0, ymin = 0.0;
  bool integ = true;
  for (int j = lane; j < mpad; j += 32) {
    double y = 0.0, mu = 1.0, w = 1.0;
    if (j < A.m) {
      y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + j] : (double)static_cast<const int32_t*>(A.y)[off + j];
      mu = A.mu[off + j];
      if (A.use_weights) w = A.w[off + j];
      swy += w * y;
      ym = fmax(ym, y);
      ymin = fmin(ymin, y);
      integ = integ && (y == floor(y));
    }
    S.ys[j] = y;
    S.r1[j] = mu;
    if (A.use_weights) S.wsm[j] = w;
  }
  sum_wy = warp_allreduce_sum(swy);
  ymax = warp_allreduce_max(ym);
  ymin = -warp_allreduce_max(-ymin);
  integral = __all_sync(0xffffffffu, integ) && (ymin >= 0.0);
  __syncwarp();
}

// histogram tab[v] = #{y == v + 1} (weighted) -> tab[k] = c_k = sum_j w_j [y_j > k], in place
__device__ __forceinline__ void tab_suffix_sums(double* tab, int lane) {
  constexpr int PER = kTabMaxG / 32;
  double loc[PER];
  double run = 0.0;
#pragma unroll
  for (int q = PER - 1; q >= 0; q--) {
    run += tab[lane * PER + q];
    loc[q] = run;
  }
  double above = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double t = __shfl_down_sync(0xffffffffu, above, o);
    if (lane + o < 32) above += t;
  }
  above -= run;
  __syncwarp();
#pragma unroll
  for (int q = 0; q < PER; q++) tab[lane * PER + q] = loc[q] + above;
  __syncwarp();
}

__device__ __forceinline__ void gbuild_table(const GenWarp& S, int m, bool use_w, int lane) {
  for (int k = lane; k < kTabMaxG; k += 32) S.tab[k] = 0.0;
  __syncwarp();
  if (use_w) {
    // weighted histogram in a fixed order (bin k belongs to lane k % 32): see fit_disp.cu::build_table
    for (int j = 0; j < m; j++) {
      const int v = (int)S.ys[j];
      if (v >= 1 && ((v - 1) & 31) == lane) S.tab[v - 1] += S.wsm[j];
    }
  } else {
    for (int j = lane; j < m; j += 32) {
      const int v = (int)S.ys[j];
      if (v >= 1) atomicAdd(&S.tab[v - 1], 1.0);
    }
  }
  __syncwarp();
  tab_suffix_sums(S.tab, lane);
}

__global__ void __launch_bounds__(256, 1) fit_disp_generic_kernel(const DispArgs A, int mpad, int ps, size_t warp_doubles) {
  extern __shared__ __align__(16) double smem[];
  init_log_table();
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  // rows_global == 2: the samplewise design and the row ids stay in global memory
  const bool all_global = A.rows_global == 2;
  const int xrows = A.grouped ? A.G : (all_global ? 0 : A.m);
  const int gids = all_global ? 0 : A.m;
  double* xg = smem;                                         // xrows * ps
  int* gid = reinterpret_cast<int*>(xg + (size_t)xrows * ps);  // gids ints (padded to doubles)
  double* wbase = xg + (size_t)xrows * ps + (gids + 1) / 2 + (size_t)warp * warp_doubles;
  for (int i = threadIdx.x; i < xrows * ps; i += blockDim.x) xg[i] = A.xg[i];
  for (int i = threadIdx.x; i < gids; i += blockDim.x) gid[i] = A.gid[i];
  __syncthreads();
  GDispCtx C;
  C.D = Design{xrows ? xg : A.xg, gids ? gid : A.gid, A.p, ps, A.G, A.grouped, A.m};
  const GenShape shp{1, 0, A.use_weights != 0, 1, 3, A.rows_global};
  const size_t gwarp = (size_t)blockIdx.x * (blockDim.x >> 5) + warp;
  C.S = carve(wbase, A.row_scratch ? A.row_scratch + gwarp * gen_global_doubles(mpad, A.grouped, shp) : nullptr, mpad, A.p,
              ps, A.G, A.grouped, shp);
  C.prior_sigmasq = A.prior_sigmasq;
  C.inv_sigmasq = 1.0 / A.prior_sigmasq;
  C.weight_threshold = A.weight_threshold;
  C.use_prior = A.use_prior;
  C.use_cr = A.use_cr;
  C.use_w = A.use_weights;
  C.saturated = A.saturated && A.grouped && A.G == A.p && !A.use_weights;
  C.sat_logdet = A.sat_logdet;

  for (;;) {
    unsigned int g = 0;
    if (lane == 0) g = atomicAdd(A.counter, 1u);
    g = __shfl_sync(0xffffffffu, g, 0);
    if (g >= (unsigned int)A.n) break;
    double ymax;
    bool integral;
    gstage_disp(A, g, mpad, lane, C.S, C.sum_wy, ymax, integral);
    C.tab_mode = integral && (ymax < (double)kTabMaxG);
    C.ntab = 0;
    if (C.tab_mode) {
      gbuild_table(C.S, A.m, A.use_weights != 0, lane);
      C.ntab = (int)ymax;
    }
    const double pm = A.prior_mean[g];
    double lp_new, dlp_new, d2;

    if (A.grid != nullptr) {
      DispGridSearch gs(A);
      for (int t = 0; t < gs.evaluations(); t++) {
        const double a = gs.point(t);
        gdisp_eval(C, a, pm, lane, false, false, lp_new, dlp_new, d2);
        gs.take(t, a, lp_new);
      }
      if (lane == 0) A.log_alpha[g] = gs.a_best;
      __syncwarp();
      continue;
    }

    DispLineSearch ls(A.log_alpha_in[g], A.kappa_0);
    for (int t = -1; t < A.maxit; t++) {   // t = -1: the evaluation at the starting point
      const double a_new = ls.propose();
      gdisp_eval(C, a_new, pm, lane, true, false, lp_new, dlp_new, d2);
      if (ls.take(lp_new, dlp_new, A)) break;
    }
    gdisp_eval(C, ls.a, pm, lane, true, true, lp_new, dlp_new, d2);
    if (lane == 0) ls.store(A, g, d2);
    __syncwarp();
  }
}

// ================================================================ beta (IRLS)

struct GBetaCtx {
  Design D;
  GenWarp S;
  const double* lnf;   // shared (vector nf) or the warp's row
  int use_w;
  double minmu, log_minmu;
};

// one fused pass: eta per term -> mu (stored), deviance part, per-term sums W = sum w, WZ = sum w z
__device__ __forceinline__ double gbeta_pass(const GBetaCtx& C, const double* beta, double alpha, double r,
                                             double log_alpha, bool want_dev, int lane) {
  const Design& D = C.D;
  const GenWarp& S = C.S;
  const int T = D.terms();
  // eta per term into q[]
  for (int t = lane; t < T; t += 32) {
    const double* xr = D.row(t);
    double e = 0.0;
    for (int k = 0; k < D.p; k++) e = fma(xr[k], beta[k], e);
    S.q[t] = e;
  }
  if (D.grouped) {
    zero_acc(S.accA, D.G, lane);
    zero_acc(S.accB, D.G, lane);
  }
  __syncwarp();
  double dev = 0.0;
  double* mus = S.r2;
#pragma unroll kUnrollBeta
  for (int j = lane; j < D.m; j += 32) {
    const int t = D.grouped ? D.gid[j] : j;
    const double lnf = C.lnf[j];
    const double le = S.q[t] + lnf;
    const double mu = fmax((fabs(le) < 700.0) ? exp_fast(le) : exp(le), C.minmu);
    const double lmu = (mu == C.minmu) ? C.log_minmu : le;
    mus[j] = mu;
    const double y = S.ys[j];
    const double am = mu * alpha;
    const double u1 = 1.0 + am;
    const double iu1 = rcp_fast(u1);
    double w = mu * iu1;
    double wt = 1.0;
    if (C.use_w) {
      wt = S.wsm[j];
      w *= wt;
    }
    const double z = (lmu - lnf) + fma(y, rcp_fast(mu), -1.0);
    if (want_dev) {
      const double l1p = log_pos(u1) + (am - (u1 - 1.0)) * iu1;   // log1p(am)
      dev = fma(wt, fma(y, lmu + log_alpha, -(y + r) * l1p), dev);
    }
    if (D.grouped) {
      const int slot = t * 32 + lane;
      S.accA[slot] += w;
      S.accB[slot] = fma(w, z, S.accB[slot]);
    } else {
      S.accA[j] = w;
      S.accB[j] = w * z;
    }
  }
  __syncwarp();
  if (D.grouped) {
    reduce_group_acc(S.accA, S.WA, D.G, lane);
    reduce_group_acc(S.accB, S.WB, D.G, lane);
  }
  return want_dev ? warp_allreduce_sum(dev) : 0.0;
}

__device__ __forceinline__ double lgamma_diff_g(double y, double r, double lg_r) {
  if (r >= kShift) {
    const double xr = y + r;
    const double ixr = rcp_fast(xr), ir = rcp_fast(r);
    const double tail = stirling_tail(ixr, ixr * ixr) - stirling_tail(ir, ir * ir);
    return fma(y, log_pos(xr), fma(r - 0.5, log1p_pos(y * ir), -y)) + tail;
  }
  return lgamma_pos(y + r) - lg_r;
}

__global__ void __launch_bounds__(256, 1) fit_beta_generic_kernel(const BetaArgs A, int mpad, int ps, size_t warp_doubles) {
  extern __shared__ __align__(16) double smem[];
  init_log_table();
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int p = A.p;
  // rows_global == 2: the samplewise design and the row ids stay in global memory, and each warp keeps the log size
  // factors in its own global row, as it does for an nf matrix
  const bool all_global = A.rows_global == 2;
  const int xrows = A.grouped ? A.G : (all_global ? 0 : A.m);
  const int gids = all_global ? 0 : A.m;
  const bool lnf_in_smem = A.nf_is_vector && !all_global;
  double* xg = smem;
  int* gid = reinterpret_cast<int*>(xg + (size_t)xrows * ps);
  double* lnf_shared = xg + (size_t)xrows * ps + (gids + 1) / 2;    // mpad (unused when the log nf are per warp)
  double* lam = lnf_shared + (all_global ? 0 : mpad);               // 32
  double* contrast = lam + 32;                                      // 32
  double* wbase = contrast + 32 + (size_t)warp * warp_doubles;
  for (int i = threadIdx.x; i < xrows * ps; i += blockDim.x) xg[i] = A.xg[i];
  for (int i = threadIdx.x; i < gids; i += blockDim.x) gid[i] = A.gid[i];
  if (lnf_in_smem)
    for (int j = threadIdx.x; j < A.m; j += blockDim.x) lnf_shared[j] = log(A.nf[j]);
  for (int k = threadIdx.x; k < p; k += blockDim.x) {
    lam[k] = A.lambda[k];
    contrast[k] = A.contrast[k];
  }
  __syncthreads();
  GBetaCtx C;
  C.D = Design{xrows ? xg : A.xg, gids ? gid : A.gid, p, ps, A.G, A.grouped, A.m};
  const GenShape shp{lnf_in_smem ? 0 : 1, 1, A.use_weights != 0, 0, 2, A.rows_global};
  const size_t gwarp = (size_t)blockIdx.x * (blockDim.x >> 5) + warp;
  C.S = carve(wbase, A.row_scratch ? A.row_scratch + gwarp * gen_global_doubles(mpad, A.grouped, shp) : nullptr, mpad, p,
              ps, A.G, A.grouped, shp);
  C.use_w = A.use_weights;
  C.minmu = A.minmu;
  C.log_minmu = log(A.minmu);
  C.lnf = lnf_in_smem ? lnf_shared : C.S.r1;
  const GenWarp& S = C.S;
  double* B = S.M0;      // X'WX
  double* L = S.M1;      // equilibrated, factored X'WX + Lambda
  double* Ainv = S.M2;
  double* Tm = S.M3;
  double* beta = S.v0;
  double* rhs = S.v1;
  double* sc = S.v2;     // equilibration scales
  double* tmp = S.v3;

  for (;;) {
    unsigned int g = 0;
    if (lane == 0) g = atomicAdd(A.counter, 1u);
    g = __shfl_sync(0xffffffffu, g, 0);
    if (g >= (unsigned int)A.n) break;
    const size_t off = (size_t)g * A.ld;
    for (int j = lane; j < mpad; j += 32) {
      double y = 0.0;
      if (j < A.m)
        y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + j] : (double)static_cast<const int32_t*>(A.y)[off + j];
      S.ys[j] = y;
      if (!lnf_in_smem) S.r1[j] = (j < A.m) ? log(A.nf_is_vector ? A.nf[j] : A.nf[off + j]) : 0.0;
      if (A.use_weights) S.wsm[j] = (j < A.m) ? A.w[off + j] : 0.0;
    }
    if (lane < p) beta[lane] = A.beta_in[(size_t)g + (size_t)A.n * lane];
    __syncwarp();
    const double alpha = A.alpha_hat[g];
    const double r = 1.0 / alpha;
    const double log_alpha = log(alpha);
    double devc = 0.0;
    if (A.maxit > 0) {
      const double lg_r = lgamma_pos(r);
      double c = 0.0;
      for (int j = lane; j < A.m; j += 32) {
        const double y = S.ys[j];
        double t = lgamma_diff_g(y, r, lg_r) - lgamma_pos(y + 1.0);
        if (A.use_weights) t *= S.wsm[j];
        c += t;
      }
      devc = warp_allreduce_sum(c);
    }
    gbeta_pass(C, beta, alpha, r, log_alpha, false, lane);
    IrlsProgress ir;
    for (int t = 0; t < A.maxit; t++) {
      ir.start_iteration();
      // normal equations (X'WX + Lambda) b = X'Wz, Jacobi-equilibrated Cholesky
      build_xtwx(C.D, S.WA, B, lane);
      if (lane < p) {
        double s = 0.0;
        const int T = C.D.terms();
        for (int q = 0; q < T; q++) s = fma(S.WB[q], C.D.row(q)[lane], s);
        rhs[lane] = s;
        sc[lane] = rsqrt(B[lane * ps + lane] + lam[lane]);
      }
      __syncwarp();
      if (lane < p) {
        for (int b = 0; b < p; b++) {
          const double v = B[lane * ps + b] + ((b == lane) ? lam[lane] : 0.0);
          L[lane * ps + b] = v * sc[lane] * sc[b];
        }
        rhs[lane] *= sc[lane];
      }
      chol_smem(L, p, ps, lane);
      // forward / backward substitution, column oriented (lane = row)
      for (int c = 0; c < p; c++) {
        if (lane == c) rhs[c] /= L[c * ps + c];
        __syncwarp();
        if (lane > c && lane < p) rhs[lane] -= L[lane * ps + c] * rhs[c];
        __syncwarp();
      }
      for (int c = p - 1; c >= 0; c--) {
        if (lane == c) rhs[c] /= L[c * ps + c];
        __syncwarp();
        if (lane < c) rhs[lane] -= L[c * ps + lane] * rhs[c];
        __syncwarp();
      }
      bool big = false;
      if (lane < p) {
        beta[lane] = rhs[lane] * sc[lane];
        big = fabs(beta[lane]) > kBetaLarge;
      }
      __syncwarp();
      if (__any_sync(0xffffffffu, big)) { ir.diverged(A.maxit); break; }
      const double dv = gbeta_pass(C, beta, alpha, r, log_alpha, true, lane);
      if (ir.stop_after_pass(dv, devc, A)) break;
    }
    // ---- post-loop block (src/DESeq2.cpp:429-455): W sums belong to the mu now in shared memory
    build_xtwx(C.D, S.WA, B, lane);
    if (lane < p) sc[lane] = rsqrt(B[lane * ps + lane] + lam[lane]);
    __syncwarp();
    if (lane < p)
      for (int b = 0; b < p; b++)
        L[lane * ps + b] = (B[lane * ps + b] + ((b == lane) ? lam[lane] : 0.0)) * sc[lane] * sc[b];
    chol_smem(L, p, ps, lane);
    chol_inverse_smem(L, Ainv, p, ps, lane);
    if (lane < p)
      for (int b = 0; b < p; b++) Ainv[lane * ps + b] *= sc[lane] * sc[b];
    __syncwarp();
    quad_forms(C.D, Ainv, S.q, lane);
    if (A.hat_diag != nullptr || A.mu_out != nullptr) {
      for (int j = lane; j < A.m; j += 32) {
        const double mu = S.r2[j];
        if (A.mu_out != nullptr) A.mu_out[off + j] = mu;
        if (A.hat_diag != nullptr) {
          double w = mu * rcp_fast(fma(alpha, mu, 1.0));
          if (A.use_weights) w *= S.wsm[j];
          A.hat_diag[off + j] = w * S.q[C.D.grouped ? C.D.gid[j] : j];
        }
      }
    }
    // sigma = Ainv * B * Ainv: T = Ainv B (row per lane), var_r = sum_k T[r][k] Ainv[k][r]
    double var = 0.0, cn = 0.0, cd = 0.0;
    if (lane < p) {
      for (int c = 0; c < p; c++) {
        double s = 0.0;
        for (int k = 0; k < p; k++) s = fma(Ainv[lane * ps + k], B[k * ps + c], s);
        Tm[lane * ps + c] = s;
      }
      double v = 0.0;
      for (int k = 0; k < p; k++) v = fma(Ainv[lane * ps + k], contrast[k], v);
      tmp[lane] = v;   // Ainv * contrast
    }
    __syncwarp();
    if (lane < p) {
      double sc_r = 0.0;
      for (int k = 0; k < p; k++) {
        var = fma(Tm[lane * ps + k], Ainv[k * ps + lane], var);
        sc_r = fma(Tm[lane * ps + k], tmp[k], sc_r);
      }
      cd = contrast[lane] * sc_r;
      cn = contrast[lane] * beta[lane];
      A.beta_out[(size_t)g + (size_t)A.n * lane] = beta[lane];
      A.beta_var[(size_t)g + (size_t)A.n * lane] = var;
    }
    cd = warp_allreduce_sum(cd);
    cn = warp_allreduce_sum(cn);
    if (lane == 0) {
      A.iter[g] = ir.it;
      A.contrast_num[g] = cn;
      A.contrast_denom[g] = sqrt(cd);
      A.deviance[g] = ir.dev;
    }
    __syncwarp();
  }
}

#include "fit_generic_seg.cuh"

struct GenLaunch {
  int mpad, ps, warps;
  size_t warp_doubles, smem;
  int rows_global;
};

// extra_doubles: the kernel's own part of the CTA's shared memory; extra_row: the part of it that has length m, which
// rows_global == 2 moves out of shared memory
bool plan_one(int m, int p, int G, int grouped, GenShape sh, size_t extra_doubles, size_t extra_row, GenLaunch& out) {
  out.mpad = (m + 3) & ~3;
  out.ps = p | 1;
  out.rows_global = sh.rows_global;
  out.warp_doubles = gen_warp_doubles(out.mpad, p, out.ps, G, grouped, sh);
  const size_t fixed =
      sh.rows_global == 2 ? ((size_t)(grouped ? G : 0) * out.ps + extra_doubles) * sizeof(double)
                          : ((size_t)(grouped ? G : m) * out.ps + (m + 1) / 2 + extra_doubles + extra_row) * sizeof(double);
  // the kernels' static shared memory (the log tables, 3104 bytes per ptxas -v) counts against the 227 KB per block
  const size_t cap = 227 * 1024 - 3104;
  int warps = 8;
  while (warps > 1 && fixed + warps * out.warp_doubles * sizeof(double) > cap) warps--;
  // several CTAs per SM need room for each: prefer 8-warp CTAs that fit at least twice (227 KB per SM)
  const size_t sm_cap = 227 * 1024;
  while (warps > 4 && 2 * (fixed + warps * out.warp_doubles * sizeof(double)) > sm_cap &&
         fixed + (warps - 1) * out.warp_doubles * sizeof(double) <= sm_cap / 2)
    warps--;
  out.warps = warps;
  out.smem = fixed + warps * out.warp_doubles * sizeof(double);
  return out.smem <= cap;
}

// Rows in shared memory whenever they fit.  Config 4 (m = 1000, two rows = 16 KB per warp) leaves 7 warps per SM; moving
// the rows to a per-warp slice of an L2-resident global scratch buffer (rows_global) doubles the resident warps, but
// the per-pass row reads turn from shared-memory into L2 latency and the kernel is not occupancy-bound.  The global
// rows remain for rows that do not fit in shared memory (and as the A/B switch B200NB_GENERIC_ROWS=global); when even
// one warp's m-long sums, the samplewise design or the row ids do not fit beside them, rows_global == 2 moves those
// too, so that every m has a plan.
bool plan(int m, int p, int G, int grouped, GenShape sh, size_t extra_doubles, size_t extra_row, GenLaunch& out) {
  const char* force = getenv("B200NB_GENERIC_ROWS");   // "smem" | "global": A/B switch
  if (force && (force[0] == 's' || force[0] == 'g')) {
    sh.rows_global = force[0] == 'g';
    if (plan_one(m, p, G, grouped, sh, extra_doubles, extra_row, out)) return true;
  }
  for (int level = 0; level <= 2; level++) {
    sh.rows_global = level;
    if (plan_one(m, p, G, grouped, sh, extra_doubles, extra_row, out)) return true;
  }
  return false;
}

// ---- segmented kernels: launch plan.  One CTA per SM of up to 16 warps; the kernels are compiled for 256 / 384 / 512
// threads (255 / 168 / 128 registers at most; 20 warps of the 92-register IRLS kernel were measured: no gain over 16).  B200NB_GENERIC_SEG=0 keeps the kernels above (A/B switch, read per launch),
// B200NB_GENERIC_WARPS=<n> caps the warps per CTA.
struct SegPlan {
  int warps, mpad, ps;
  size_t warp_bytes, smem;
};
bool seg_enabled(const SegLayout& L) {
  if (L.pos == nullptr) return false;
  const char* e = getenv("B200NB_GENERIC_SEG");
  return !(e && e[0] == '0');
}
bool plan_seg(size_t fixed, size_t warp_bytes, int max_warps, SegPlan& out) {
  const size_t cap = 227 * 1024 - 4096;   // the kernels' static shared memory (log tables, 3.1 KB) counts against the 227 KB
  if (fixed + warp_bytes > cap) return false;
  int warps = (int)((cap - fixed) / warp_bytes);
  if (warps > max_warps) warps = max_warps;
  const char* e = getenv("B200NB_GENERIC_WARPS");
  if (e && atoi(e) >= 1 && atoi(e) < warps) warps = atoi(e);
  out.warps = warps;
  out.warp_bytes = warp_bytes;
  out.smem = fixed + (size_t)warps * warp_bytes;
  return true;
}
template <int MAXT>
cudaError_t launch_disp_seg_t(const DispArgs& a, const SegPlan& P, cudaStream_t stream) {
  unsigned grid = 0;
  cudaError_t e = persistent_grid(reinterpret_cast<const void*>(fit_disp_seg_kernel<MAXT>), P.warps * 32, P.smem, P.warps,
                                  a.n, &grid);
  if (e != cudaSuccess) return e;
  fit_disp_seg_kernel<MAXT><<<grid, P.warps * 32, P.smem, stream>>>(a, P.mpad, P.ps, P.warp_bytes);
  return cudaGetLastError();
}
template <int MAXT>
cudaError_t launch_beta_seg_t(const BetaArgs& a, const SegPlan& P, cudaStream_t stream) {
  unsigned grid = 0;
  cudaError_t e = persistent_grid(reinterpret_cast<const void*>(fit_beta_seg_kernel<MAXT>), P.warps * 32, P.smem, P.warps,
                                  a.n, &grid);
  if (e != cudaSuccess) return e;
  fit_beta_seg_kernel<MAXT><<<grid, P.warps * 32, P.smem, stream>>>(a, P.mpad, P.ps, P.warp_bytes);
  return cudaGetLastError();
}

}  // namespace

// global row scratch: a small ring of grow-only device buffers (one per launch in flight)
namespace {
constexpr int kRowRing = 4;
void* g_rowbuf[kRowRing] = {};
size_t g_rowcap[kRowRing] = {};
unsigned int g_rownext = 0;
std::mutex g_rowmu;
}  // namespace
cudaError_t row_scratch(size_t bytes, double** out) {
  std::lock_guard<std::mutex> lk(g_rowmu);
  const int s = (int)(g_rownext++ % kRowRing);
  if (g_rowcap[s] < bytes) {
    if (g_rowbuf[s]) {
      cudaError_t e = cudaDeviceSynchronize();
      if (e != cudaSuccess) return e;
      cudaFree(g_rowbuf[s]);
      g_rowbuf[s] = nullptr;
      g_rowcap[s] = 0;
    }
    cudaError_t e = cudaMalloc(&g_rowbuf[s], bytes + bytes / 8);
    if (e != cudaSuccess) return e;
    g_rowcap[s] = bytes + bytes / 8;
  }
  *out = static_cast<double*>(g_rowbuf[s]);
  return cudaSuccess;
}

cudaError_t launch_fit_disp_generic(const DispArgs& a0, cudaStream_t stream) {
  DispArgs a = a0;
  if (a.grouped && !a.use_weights && a.grid == nullptr && seg_enabled(a.seg)) {
    SegPlan P;
    P.mpad = (a.m + 7) & ~7;
    P.ps = a.p | 1;
    const int sat = a.saturated && a.G == a.p;
    const size_t fixed = (size_t)a.G * P.ps * sizeof(double) + seg_table_bytes(a.seg.kmax, a.G) + pair_table_bytes(a.p);
    if (plan_seg(fixed, sdisp_warp_bytes(P.mpad, a.p, P.ps, a.G, a.seg.kmax, sat), 16, P)) {
      cudaError_t e = cudaMemsetAsync(a.scratch, 0, 4 * sizeof(unsigned int), stream);
      if (e != cudaSuccess) return e;
      a.counter = a.scratch;
      a.row_scratch = nullptr;
      if (P.warps <= 8) return launch_disp_seg_t<256>(a, P, stream);
      if (P.warps <= 12) return launch_disp_seg_t<384>(a, P, stream);
      return launch_disp_seg_t<512>(a, P, stream);
    }
  }
  GenLaunch L;
  GenShape sh{1, 0, a.use_weights != 0, 1, 3, 0};
  if (!plan(a.m, a.p, a.G, a.grouped, sh, 0, 0, L)) return cudaErrorInvalidValue;
  unsigned grid = 0;
  cudaError_t e = persistent_grid(reinterpret_cast<const void*>(fit_disp_generic_kernel), L.warps * 32, L.smem, L.warps, a.n, &grid);
  if (e != cudaSuccess) return e;
  a.row_scratch = nullptr;
  a.rows_global = sh.rows_global = L.rows_global;
  if (L.rows_global) {
    e = row_scratch((size_t)grid * L.warps * gen_global_doubles(L.mpad, a.grouped, sh) * sizeof(double), &a.row_scratch);
    if (e != cudaSuccess) return e;
  }
  e = cudaMemsetAsync(a.scratch, 0, 4 * sizeof(unsigned int), stream);
  if (e != cudaSuccess) return e;
  a.counter = a.scratch;
  fit_disp_generic_kernel<<<grid, L.warps * 32, L.smem, stream>>>(a, L.mpad, L.ps, L.warp_doubles);
  return cudaGetLastError();
}

cudaError_t launch_fit_beta_generic(const BetaArgs& a0, cudaStream_t stream) {
  BetaArgs a = a0;
  if (a.grouped && !a.use_weights && seg_enabled(a.seg)) {
    SegPlan P;
    P.mpad = (a.m + 7) & ~7;
    P.ps = a.p | 1;
    const size_t fixed = ((size_t)a.G * P.ps + (a.nf_is_vector ? 2 * P.mpad : 0) + 64 + 256) * sizeof(double) +
                         seg_table_bytes(a.seg.kmax, a.G) + pair_table_bytes(a.p);
    if (plan_seg(fixed, sbeta_warp_bytes(P.mpad, a.p, P.ps, a.G, a.seg.kmax, a.nf_is_vector), 16, P)) {
      cudaError_t e = cudaMemsetAsync(a.counter, 0, sizeof(unsigned int), stream);
      if (e != cudaSuccess) return e;
      a.row_scratch = nullptr;
      if (P.warps <= 8) return launch_beta_seg_t<256>(a, P, stream);
      if (P.warps <= 12) return launch_beta_seg_t<384>(a, P, stream);
      return launch_beta_seg_t<512>(a, P, stream);
    }
  }
  GenLaunch L;
  const int mpad = (a.m + 3) & ~3;
  GenShape sh{a.nf_is_vector ? 0 : 1, 1, a.use_weights != 0, 0, 2, 0};
  if (!plan(a.m, a.p, a.G, a.grouped, sh, 64, (size_t)mpad, L)) return cudaErrorInvalidValue;
  unsigned grid = 0;
  cudaError_t e = persistent_grid(reinterpret_cast<const void*>(fit_beta_generic_kernel), L.warps * 32, L.smem, L.warps, a.n, &grid);
  if (e != cudaSuccess) return e;
  a.row_scratch = nullptr;
  a.rows_global = sh.rows_global = L.rows_global;
  if (L.rows_global == 2) sh.has_r1 = 1;   // the log size factors move to a per-warp row with the other m-long arrays
  if (L.rows_global) {
    e = row_scratch((size_t)grid * L.warps * gen_global_doubles(L.mpad, a.grouped, sh) * sizeof(double), &a.row_scratch);
    if (e != cudaSuccess) return e;
  }
  e = cudaMemsetAsync(a.counter, 0, sizeof(unsigned int), stream);
  if (e != cudaSuccess) return e;
  fit_beta_generic_kernel<<<grid, L.warps * 32, L.smem, stream>>>(a, L.mpad, L.ps, L.warp_doubles);
  return cudaGetLastError();
}

}  // namespace nb
