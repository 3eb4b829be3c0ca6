// fit_disp.cu -- gene-wise Cox-Reid adjusted NB dispersion MLE/MAP on sm_90a, one warp per gene.
//
// Behavioural contract (WHAT): /root/reference/src/DESeq2.cpp:164-277 (fitDisp: Armijo back-tracking
// ascent on log alpha, accept / reject / kappa schedule replicated decision for decision), :31-158
// (log posterior and its first two derivatives, Cox-Reid term with weight-threshold row/column
// subsetting) and :469-513 (fitDispGrid).  The line-search and grid decisions are deseq_rules.cuh's.  HOW is new:
//   * the gene's row (counts, mu, weights) is staged once into shared memory with 128-bit loads;
//     every lane owns samples lane, lane+32, ...; all per-gene scalars are warp-uniform;
//   * one fused pass per proposal evaluates the log posterior AND its derivative (they share
//     log(1+mu*alpha) and 1/(1+mu*alpha)), so an accepted step costs one pass instead of the reference's
//     three (theta(kappa), lpnew, dlp) -- the values are the same because the reference re-evaluates the
//     same function at the same point (:225 vs :233);
//   * the identities log(mu+1/alpha) = log(1+mu*alpha) - log(alpha), mu*alpha/(1+mu*alpha) = alpha*wd,
//     y/(mu+1/alpha) = y*alpha/(1+mu*alpha) (wd = mu/(1+mu*alpha)) remove two logs/divisions per sample;
//   * counts are integers, so sum_j [lgamma(y_j + r) - lgamma(r)] = sum_k c_k log(r + k) and
//     sum_j [digamma(y_j + r) - digamma(r)] = sum_k c_k / (r + k) with c_k = sum_j w_j [y_j > k]:
//     for a gene whose largest count is below kTabMax the warp builds the c_k table once (shared-memory
//     histogram + suffix scan) and every evaluation then needs max(y)/32 logs per lane instead of one
//     lgamma/digamma pair per sample (TAB mode; exact, no lgamma cancellation).  Genes with larger counts
//     use the Stirling pair per sample, branch-free when every count is >= 10 (BIG mode), with an upward
//     shift loop otherwise (GEN mode, also taken for non-integer "counts");
//   * samples are processed four per lane per trip with clamped indices and 0/1 validity factors, giving
//     four independent dependency chains per lane (the FP64 pipe is latency-bound otherwise);
//   * X'WX, X'dWX are accumulated per lane and combined with xor-butterfly shuffles (bitwise identical in
//     every lane, so control flow stays warp-uniform); the p x p Cholesky runs in registers;
//   * genes are pulled from an atomic work queue by persistent warps (trip counts vary 1..maxit).
#include "deseq_rules.cuh"
#include "engine.h"
#include "smallp.cuh"

namespace nb {

namespace {

constexpr int kTabMax = 256;   // capacity of the per-warp factor table (counts 0 .. kTabMax-1 use TAB mode)
enum DispMode { MODE_TAB = 0, MODE_BIG = 1, MODE_GEN = 2 };

struct DispRow {
  const double* y;
  const double* mu;
  const double* w;    // only read when USE_W
  const double* x;    // shared, column-major with stride mpad
  const double* tab;  // c_k, k = 0 .. ntab-1 (TAB mode)
  int m, mpad, ntab;
};

struct DispScal {
  double prior_sigmasq, inv_sigmasq, weight_threshold;
  int use_prior, use_cr;
};

constexpr int pow2_ceil(int n) { int p = 1; while (p < n) p <<= 1; return p; }

// One fused pass: lp (and dlp when WANT_D) at log-alpha `a`.
// GL = lanes per gene: 32 (one warp per gene) or 16 / 8 (two / four genes per warp, fit_disp_grp.cuh) with
// `lane` the lane index inside the group; reductions then stay inside the group.
// IND: indicator design (smallp.cuh): no design products, the (a, a) Cox-Reid sums come from the (a, 0) sums.
template <int P, bool USE_W, bool WANT_D, int MODE, int GL = 32, bool IND = false>
__device__ __forceinline__ void disp_eval_mode(const DispRow& rv, const DispScal& sc, double a, double pm,
                                               double sum_wy, int lane, double& lp, double& dlp) {
  constexpr int NS = SymP<P>::N;
  const double alpha = exp_fast(a);   // a is confined to [-30, 10] by the line search / grid
  const double r = rcp_fast(alpha);
  double lg_r = 0.0, dg_r = 0.0;
  if (MODE != MODE_TAB) lgamma_digamma_pos(r, lg_r, dg_r);

  constexpr int NA = pow2_ceil(2 + 2 * NS);
  double acc[NA];
#pragma unroll
  for (int i = 0; i < NA; i++) acc[i] = 0.0;

  if (MODE == MODE_TAB) {
    // shared factor table: sum_k c_k log(r+k), sum_k c_k/(r+k)
#pragma unroll 2
    for (int k = lane; k < rv.ntab; k += GL) {
      const double ck = rv.tab[k];
      const double xk = r + (double)k;
      acc[0] = fma(ck, log_pos(xk), acc[0]);
      if (WANT_D) acc[1] = fma(-ck, rcp_fast(xk), acc[1]);
    }
  }

  const int mlast = rv.m - 1;
  for (int j0 = lane; j0 < rv.m; j0 += 4 * GL) {
#pragma unroll
    for (int u = 0; u < 4; u++) {
      if (GL != 32 && (j0 - lane) + GL * u >= rv.m) break;   // narrow groups: skip sweeps with no sample at all
      const int jr = j0 + GL * u;
      const int j = min(jr, mlast);
      double vw = (jr < rv.m) ? 1.0 : 0.0;
      const double y = rv.y[j], mu = rv.mu[j];
      // wd = 1/(1/mu + alpha) = mu/(1 + mu alpha); alpha wd (y/mu - 1) = alpha (y - mu)/(1 + mu alpha): 1/mu never needed
      const double onema = fma(mu, alpha, 1.0);
      const double wi = rcp_fast(onema);
      const double wd = mu * wi;
      const double l2 = log_pos(onema);
      const double xr = y + r;
      double t, d;
      if (MODE == MODE_TAB) {
        t = -xr * l2;
        d = l2 + alpha * (y - mu) * wi;
      } else {
        double lg, dg;
        if (MODE == MODE_BIG) lgamma_digamma_big(xr, lg, dg);
        else lgamma_digamma_pos(xr, lg, dg);
        t = (lg - lg_r) - xr * l2;
        d = (dg_r - dg) + l2 + alpha * (y - mu) * wi;
      }
      double wdm = wd * vw;
      if (USE_W) {
        const double wt = rv.w[j];
        if (!(wt > sc.weight_threshold)) wdm = 0.0;
        vw *= wt;
      }
      acc[0] = fma(vw, t, acc[0]);
      if (WANT_D) acc[1] = fma(vw, d, acc[1]);
      if (sc.use_cr) {
        const double dwd = -wdm * wd;
        double xv[P];
        load_design_row<P, IND>(rv.x, rv.mpad, j, xv);
#pragma unroll
        for (int aa = 0; aa < P; aa++)
#pragma unroll
          for (int bb = 0; bb <= aa; bb++) {
            if (IND && bb == aa && aa > 0) continue;
            const double xx = design_prod<P, IND>(xv, aa, bb);
            const int q = aa * (aa + 1) / 2 + bb;
            acc[2 + q] = fma(wdm, xx, acc[2 + q]);
            if (WANT_D) acc[2 + NS + q] = fma(dwd, xx, acc[2 + NS + q]);
          }
      }
    }
  }
  fill_diag_from_col0<P, IND>(acc + 2);
  if (WANT_D) fill_diag_from_col0<P, IND>(acc + 2 + NS);
  if constexpr (GL == 32) warp_allreduce_sum_rs<NA>(acc, lane);
  else if constexpr (NA <= GL) group_allreduce_sum_rs<NA, GL>(acc, lane);
  else group_allreduce_sum_n<NA, GL>(acc);

  double cr = 0.0, dcr = 0.0;
  if (sc.use_cr) {
    SymP<P> B, dB;
#pragma unroll
    for (int i = 0; i < NS; i++) {
      B.v[i] = acc[2 + i];
      dB.v[i] = acc[2 + NS + i];
    }
    if (USE_W) {
      // a column whose kept rows are all zero is dropped by the reference (:42): make it inert
#pragma unroll
      for (int k = 0; k < P; k++)
        if (B.get(k, k) == 0.0) B.at(k, k) = 1.0;
    }
    double det, tr;
    cr_det_trace<P, WANT_D>(B, dB, det, tr);
    // det > 0 for a positive definite X'WX; anything else takes libm's log for the reference's NaN / -inf
    cr = -0.5 * ((det > 2.3e-308 && det < 1.7e308) ? log_pos(det) : log(det));
    dcr = -0.5 * tr;
  }
  double prior = 0.0, dprior = 0.0;
  if (sc.use_prior) {
    const double dd = a - pm;
    prior = -0.5 * dd * dd * sc.inv_sigmasq;
    dprior = -dd * sc.inv_sigmasq;
  }
  lp = (acc[0] + a * sum_wy) + prior + cr;
  if (WANT_D) dlp = (r * r * acc[1] + dcr) * alpha + dprior;
}

// second derivative at `a` (once per gene): src/DESeq2.cpp:111-158.  In TAB mode the digamma / trigamma
// differences come from the factor table: psi(y+r)-psi(r) = sum_{k<y} 1/(r+k), psi'(y+r)-psi'(r) = -sum 1/(r+k)^2.
template <int P, bool USE_W, int GL = 32, bool IND = false>
__device__ __forceinline__ double disp_d2(const DispRow& rv, const DispScal& sc, int mode, double a, int lane) {
  constexpr int NS = SymP<P>::N;
  const double alpha = exp_fast(a);   // a is confined to [-30, 10] by the line search / grid
  const double r = rcp_fast(alpha);
  const double r2 = r * r;
  double dg_r = 0.0, tg_r = 0.0;
  if (mode != MODE_TAB) {
    dg_r = digamma_pos(r);
    tg_r = trigamma_pos(r);
  }
  double acc[2 + 3 * NS];
#pragma unroll
  for (int i = 0; i < 2 + 3 * NS; i++) acc[i] = 0.0;
  if (mode == MODE_TAB) {
    for (int k = lane; k < rv.ntab; k += GL) {
      const double ck = rv.tab[k];
      const double ik = rcp_fast(r + (double)k);
      acc[0] = fma(-ck, ik, acc[0]);
      acc[1] = fma(-ck * r2, ik * ik, acc[1]);
    }
  }
  for (int j = lane; j < rv.m; j += GL) {
    const double y = rv.y[j], mu = rv.mu[j];
    const double onema = fma(mu, alpha, 1.0);
    const double wi = rcp_fast(onema);
    const double wd = mu * wi;
    const double l2 = log_pos(onema);
    const double xr = y + r;
    // t1 = dg_r + l2 - mu a/(1+mu a) - psi(y+r) + y/(mu+r);  t2 = -r2 tg_r + mu^2 a/(1+mu a)^2 + r2 psi'(y+r) + r2 y/(mu+r)^2
    double t1 = l2 + alpha * (y - mu) * wi;
    double t2 = wd * wd * alpha + y * wi * wi;
    if (mode != MODE_TAB) {
      t1 += dg_r - digamma_pos(xr);
      t2 += r2 * (trigamma_pos(xr) - tg_r);
    }
    double wt = 1.0;
    if (USE_W) {
      wt = rv.w[j];
      t1 *= wt;
      t2 *= wt;
    }
    acc[0] += t1;
    acc[1] += t2;
    if (sc.use_cr) {
      double wdm = wd;
      if (USE_W) wdm = (wt > sc.weight_threshold) ? wd : 0.0;
      const double dwd = -wdm * wd;
      const double d2wd = 2.0 * wdm * wd * wd;
      double xv[P];
      load_design_row<P, IND>(rv.x, rv.mpad, j, xv);
#pragma unroll
      for (int aa = 0; aa < P; aa++)
#pragma unroll
        for (int bb = 0; bb <= aa; bb++) {
          if (IND && bb == aa && aa > 0) continue;
          const double xx = design_prod<P, IND>(xv, aa, bb);
          const int q = aa * (aa + 1) / 2 + bb;
          acc[2 + q] = fma(wdm, xx, acc[2 + q]);
          acc[2 + NS + q] = fma(dwd, xx, acc[2 + NS + q]);
          acc[2 + 2 * NS + q] = fma(d2wd, xx, acc[2 + 2 * NS + q]);
        }
    }
  }
#pragma unroll
  for (int i = 0; i < 3; i++) fill_diag_from_col0<P, IND>(acc + 2 + i * NS);
  group_allreduce_sum_n<2 + 3 * NS, GL>(acc);
  double cr2 = 0.0, dcr = 0.0;
  if (sc.use_cr) {
    SymP<P> B, dB, d2B, Bi;
#pragma unroll
    for (int i = 0; i < NS; i++) {
      B.v[i] = acc[2 + i];
      dB.v[i] = acc[2 + NS + i];
      d2B.v[i] = acc[2 + 2 * NS + i];
    }
    if (USE_W) {
#pragma unroll
      for (int k = 0; k < P; k++)
        if (B.get(k, k) == 0.0) B.at(k, k) = 1.0;
    }
    chol_factor<P>(B);
    chol_inverse<P>(B, Bi);
    double M[P][P];
    sym_mul_full<P>(Bi, dB, M);
    double tr1 = 0.0, tr2 = 0.0;
#pragma unroll
    for (int i = 0; i < P; i++) {
      tr1 += M[i][i];
#pragma unroll
      for (int k = 0; k < P; k++) tr2 = fma(M[i][k], M[k][i], tr2);
    }
    const double tr3 = sym_trace_prod<P>(Bi, d2B);
    cr2 = 0.5 * tr1 * tr1 - 0.5 * (tr1 * tr1 - tr2 + tr3);
    dcr = -0.5 * tr1;
  }
  const double ll2 = -2.0 * r2 * r * acc[0] + r2 * acc[1];
  const double dlp_noprior = (r2 * acc[0] + dcr) * alpha;
  const double prior2 = sc.use_prior ? -sc.inv_sigmasq : 0.0;
  return ((ll2 + cr2) * alpha * alpha + dlp_noprior) + prior2;
}

// ---------------------------------------------------------------- gene classification
// One warp per gene: largest / smallest count and integrality decide the evaluation mode; genes are appended to
// one list per mode so the persistent kernel can work through one mode at a time (keeps the instruction
// working set of an SM inside the instruction cache: a fused version stalls on instruction fetch).
// lists[mode * n + i], counts[mode].
// TAB genes ordered by the length of their count table, longest first (8 buckets of 32; used by the 8-lane kernels),
// so that genes which share a warp in the narrow-group kernels wait for tables of similar length, and the launch ends
// on the cheap genes.  classify_kernel records a bucket per TAB gene and counts the buckets; bucket_sort_kernel places
// the TAB list into a scratch list in bucket order (counting sort); the launcher copies it back over the TAB list.
constexpr int kTabBuckets = 8;
__global__ void __launch_bounds__(256) bucket_sort_kernel(const int* __restrict__ tab_list, const int* __restrict__ code,
                                                          const unsigned int* __restrict__ n_tab,
                                                          const unsigned int* __restrict__ bcount,
                                                          unsigned int* __restrict__ bfill, int* __restrict__ sorted) {
  const unsigned int n0 = *n_tab;
  unsigned int start[kTabBuckets];      // longest tables (highest bucket) first
  unsigned int run = 0;
#pragma unroll
  for (int b = kTabBuckets - 1; b >= 0; b--) {
    start[b] = run;
    run += bcount[b];
  }
  for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < n0; i += gridDim.x * blockDim.x) {
    const int g = tab_list[i];
    const int b = code[g];
    unsigned int base = 0;
#pragma unroll
    for (int k = 0; k < kTabBuckets; k++)
      if (k == b) base = start[k];
    sorted[base + atomicAdd(&bfill[b], 1u)] = g;
  }
}

__global__ void __launch_bounds__(256) classify_kernel(const void* y, int y_is_f64, int n, int m, long long ld,
                                                       int* lists, unsigned int* counts
                                                       , int* code, unsigned int* bcount
) {
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (g >= n) return;
  const size_t off = (size_t)g * ld;
  double ymax = 0.0, ymin = 1e300;
  bool integral = true;
  for (int j = lane; j < m; j += 32) {
    const double v = y_is_f64 ? static_cast<const double*>(y)[off + j] : (double)static_cast<const int32_t*>(y)[off + j];
    ymax = fmax(ymax, v);
    ymin = fmin(ymin, v);
    integral = integral && (v == floor(v));
  }
  ymax = warp_allreduce_max(ymax);
  ymin = -warp_allreduce_max(-ymin);
  integral = __all_sync(0xffffffffu, integral) && (ymin >= 0.0);
  int mode = MODE_GEN;
  if (integral && ymax < (double)kTabMax) mode = MODE_TAB;
  else if (ymin >= kShift) mode = MODE_BIG;
  if (lane == 0) {
    const unsigned int pos = atomicAdd(&counts[mode], 1u);
    lists[(size_t)mode * n + pos] = g;
    if (mode == MODE_TAB && code != nullptr) {   // bucket bookkeeping only for the 8-lane kernels (see the launcher)
      const int b = min(kTabBuckets - 1, (int)ymax / (kTabMax / kTabBuckets));
      code[g] = b;
      atomicAdd(&bcount[b], 1u);
    }
  }
}

struct DispWarpSmem {
  double *ys, *mus, *wsm, *tab;
};

// stage the row of gene g into the group's shared-memory slice (128-bit loads); lg = lane inside the group of GL lanes.
// Returns sum_j w_j y_j and max y.  `valid` false: the group has no gene this round -- nothing is loaded (the slice
// keeps the previous gene, which is fine to evaluate).
template <bool USE_W, int GL>
__device__ __forceinline__ void stage_row(const DispArgs& A, unsigned int g, bool valid, int mpad, int lg,
                                          const DispWarpSmem& S, double& sum_wy, double& ymax) {
  double sum_wy_l = 0.0, ymax_l = 0.0;
  const size_t off = (size_t)g * A.ld;
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
      const double2* m2 = reinterpret_cast<const double2*>(A.mu + off + j4);
      const double2 m0 = __ldg(m2), m1 = __ldg(m2 + 1);
      const double mv[4] = {m0.x, m0.y, m1.x, m1.y};
      double wv[4] = {1.0, 1.0, 1.0, 1.0};
      if (USE_W) {
        const double2* w2 = reinterpret_cast<const double2*>(A.w + off + j4);
        const double2 w0 = __ldg(w2), w1 = __ldg(w2 + 1);
        wv[0] = w0.x; wv[1] = w0.y; wv[2] = w1.x; wv[3] = w1.y;
      }
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const int j = j4 + q;
        S.ys[j] = yv[q];
        S.mus[j] = mv[q];
        if (USE_W) S.wsm[j] = wv[q];
        if (j < A.m) {
          sum_wy_l += wv[q] * yv[q];
          ymax_l = fmax(ymax_l, yv[q]);
        }
      }
    }
  }
  sum_wy = group_allreduce_sum<GL>(sum_wy_l);
  ymax = group_allreduce_max<GL>(ymax_l);
  __syncwarp();
}

// c_k = sum_j w_j [y_j > k], k = 0 .. ymax-1, for the group's gene: shared-memory histogram + suffix scan over the GL
// lanes (TAB mode)
template <bool USE_W, int GL>
__device__ __forceinline__ void build_table(const DispWarpSmem& S, int m, int lg) {
  for (int k = lg; k < kTabMax; k += GL) S.tab[k] = 0.0;
  __syncwarp();
  if (USE_W) {
    // weighted histogram in a FIXED order (bin k belongs to lane k % GL, which adds its samples in index order):
    // floating-point atomics would make c_k -- and with it `iter` on knife-edge genes -- vary from run to run
    for (int j = 0; j < m; j++) {
      const int v = (int)S.ys[j];
      if (v >= 1 && v <= kTabMax && ((v - 1) % GL) == lg) S.tab[v - 1] += S.wsm[j];
    }
  } else {
    for (int j = lg; j < m; j += GL) {
      const int v = (int)S.ys[j];
      if (v >= 1 && v <= kTabMax) atomicAdd(&S.tab[v - 1], 1.0);   // integer-valued sums: exact in any order
    }
  }
  __syncwarp();
  constexpr int PER = kTabMax / GL;
  double loc[PER];
  double run = 0.0;
#pragma unroll
  for (int q = PER - 1; q >= 0; q--) {
    run += S.tab[lg * PER + q];
    loc[q] = run;
  }
  double above = run;  // inclusive suffix scan over the lanes of the group
#pragma unroll
  for (int o = 1; o < GL; o <<= 1) {
    const double t = __shfl_down_sync(0xffffffffu, above, o, GL);
    if (lg + o < GL) above += t;
  }
  above -= run;
  __syncwarp();
#pragma unroll
  for (int q = 0; q < PER; q++) S.tab[lg * PER + q] = loc[q] + above;
  __syncwarp();
}

// the line search of one gene (deseq_rules.cuh::DispLineSearch) with a single evaluation site; t = -1 is the
// evaluation at the starting point, t >= 0 are the proposals
template <int P, bool USE_W, int MODE, bool IND>
__device__ __forceinline__ void line_search_gene(const DispArgs& A, const DispRow& rv, const DispScal& sc,
                                                 unsigned int g, double sum_wy, int lane) {
  const double pm = A.prior_mean[g];
  DispLineSearch ls(A.log_alpha_in[g], A.kappa_0);
  for (int t = -1; t < A.maxit; t++) {
    const double a_new = ls.propose();
    double lp_new, dlp_new;
    disp_eval_mode<P, USE_W, true, MODE, 32, IND>(rv, sc, a_new, pm, sum_wy, lane, lp_new, dlp_new);
    if (ls.take(lp_new, dlp_new, A)) break;
  }
  const double d2 = disp_d2<P, USE_W, 32, IND>(rv, sc, MODE, ls.a, lane);
  if (lane == 0) ls.store(A, g, d2);
}

#ifndef NB_LB_THREADS
#define NB_LB_THREADS 256
#define NB_LB_CTAS 2
#endif
template <int P, bool USE_W, bool IND>
__global__ void __launch_bounds__(NB_LB_THREADS, NB_LB_CTAS) fit_disp_kernel(const DispArgs A, int warps_per_cta, int mpad) {
  extern __shared__ __align__(16) double smem[];
  if (indicator_design<P>(A.x, A.m) != IND) return;   // the other variant of the launch fits this design
  init_log_table();
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  constexpr int NROW = USE_W ? 3 : 2;
  double* xs = smem;                                   // P * mpad
  double* rowbase = smem + (size_t)P * mpad + (size_t)warp * ((size_t)NROW * mpad + kTabMax);
  DispWarpSmem S{rowbase, rowbase + mpad, USE_W ? rowbase + 2 * mpad : nullptr, rowbase + (size_t)NROW * mpad};

  // stage the design matrix (column-major m x p -> column-major with padded stride)
  for (int idx = threadIdx.x; idx < P * A.m; idx += blockDim.x) {
    const int k = idx / A.m, j = idx - k * A.m;
    xs[k * mpad + j] = A.x[idx];
  }
  __syncthreads();

  DispRow rv{S.ys, S.mus, S.wsm, xs, S.tab, A.m, mpad, 0};
  const DispScal sc{A.prior_sigmasq, 1.0 / A.prior_sigmasq, A.weight_threshold, A.use_prior, A.use_cr};
  const unsigned int n0 = A.mode_counts[MODE_TAB], n1 = A.mode_counts[MODE_BIG];

  // persistent warps: genes come from one queue ordered TAB | BIG | GEN
  for (;;) {
    unsigned int q = 0;
    if (lane == 0) q = atomicAdd(A.counter, 1u);
    q = __shfl_sync(0xffffffffu, q, 0);
    if (q >= (unsigned int)A.n) break;
    int mode;
    unsigned int g;
    if (q < n0) { mode = MODE_TAB; g = A.mode_lists[q]; }
    else if (q < n0 + n1) { mode = MODE_BIG; g = A.mode_lists[(size_t)A.n + (q - n0)]; }
    else { mode = MODE_GEN; g = A.mode_lists[2 * (size_t)A.n + (q - n0 - n1)]; }

    double sum_wy, ymax;
    stage_row<USE_W, 32>(A, g, true, mpad, lane, S, sum_wy, ymax);
    if (mode == MODE_TAB) {
      build_table<USE_W, 32>(S, A.m, lane);
      rv.ntab = (int)ymax;
      line_search_gene<P, USE_W, MODE_TAB, IND>(A, rv, sc, g, sum_wy, lane);
    } else if (mode == MODE_BIG) {
      line_search_gene<P, USE_W, MODE_BIG, IND>(A, rv, sc, g, sum_wy, lane);
    } else {
      line_search_gene<P, USE_W, MODE_GEN, IND>(A, rv, sc, g, sum_wy, lane);
    }
    __syncwarp();
  }
}

#include "fit_disp_grp.cuh"

// fitDispGrid (src/DESeq2.cpp:492-510): rare path (non-converged genes only); generic evaluation mode
template <int P, bool USE_W>
__global__ void __launch_bounds__(256, 2) fit_disp_grid_kernel(const DispArgs A, int warps_per_cta, int mpad) {
  extern __shared__ __align__(16) double smem[];
  init_log_table();
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  constexpr int NROW = USE_W ? 3 : 2;
  double* xs = smem;
  double* rowbase = smem + (size_t)P * mpad + (size_t)warp * ((size_t)NROW * mpad + kTabMax);
  DispWarpSmem S{rowbase, rowbase + mpad, USE_W ? rowbase + 2 * mpad : nullptr, rowbase + (size_t)NROW * mpad};
  for (int idx = threadIdx.x; idx < P * A.m; idx += blockDim.x) {
    const int k = idx / A.m, j = idx - k * A.m;
    xs[k * mpad + j] = A.x[idx];
  }
  __syncthreads();
  DispRow rv{S.ys, S.mus, S.wsm, xs, S.tab, A.m, mpad, 0};
  const DispScal sc{A.prior_sigmasq, 1.0 / A.prior_sigmasq, A.weight_threshold, A.use_prior, A.use_cr};
  for (;;) {
    unsigned int g = 0;
    if (lane == 0) g = atomicAdd(A.counter, 1u);
    g = __shfl_sync(0xffffffffu, g, 0);
    if (g >= (unsigned int)A.n) break;
    double sum_wy, ymax;
    stage_row<USE_W, 32>(A, g, true, mpad, lane, S, sum_wy, ymax);
    const double pm = A.prior_mean[g];
    DispGridSearch gs(A);
    for (int t = 0; t < gs.evaluations(); t++) {
      const double a = gs.point(t);
      double lp, dummy;
      disp_eval_mode<P, USE_W, false, MODE_GEN>(rv, sc, a, pm, sum_wy, lane, lp, dummy);
      gs.take(t, a, lp);
    }
    if (lane == 0) A.log_alpha[g] = gs.a_best;
    __syncwarp();
  }
}

// launch the GL-lanes-per-gene kernel if its shared-memory slices fit; `launched` tells.  Both design variants are
// launched (the design lives on the device): the general one returns at once on an indicator design, and vice versa.
template <int P, bool USE_W, int GL>
cudaError_t launch_disp_grp(const DispArgs& a, int mpad, size_t xbytes, size_t rowbytes, cudaStream_t stream,
                            bool& launched) {
  constexpr int NG = 32 / GL, GW = GrpShape<GL>::threads / 32;
  const size_t gsmem = xbytes + (size_t)GW * NG * rowbytes;
  launched = false;
  if (gsmem > (size_t)227 * 1024 / GrpShape<GL>::ctas) return cudaSuccess;
  for (int ind = 0; ind < 2; ind++) {
    auto kg = ind ? fit_disp_grp_kernel<P, USE_W, GL, true> : fit_disp_grp_kernel<P, USE_W, GL, false>;
    unsigned grid = 0;
    cudaError_t e = persistent_grid(reinterpret_cast<const void*>(kg), GrpShape<GL>::threads, gsmem, GW * NG, a.n, &grid);
    if (e != cudaSuccess) return e;
    kg<<<grid, GrpShape<GL>::threads, gsmem, stream>>>(a, mpad);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  launched = true;
  return cudaSuccess;
}

// shared memory of the small-p kernels: the staged design (P rows of mpad) once per CTA, and per warp (or lane group)
// the NROW sample rows and the factor table
struct DispSmem {
  int mpad;
  size_t xbytes, rowbytes;
};
DispSmem disp_smem(int m, int p, bool use_w) {
  const int mpad = (m + 3) & ~3;
  const int nrow = use_w ? 3 : 2;
  return {mpad, (size_t)p * mpad * sizeof(double), ((size_t)nrow * mpad + kTabMax) * sizeof(double)};
}
constexpr size_t kDispSmemCap = 227 * 1024;
// a one-warp plan must also leave room for the kernels' static shared memory, which counts against the same 227 KB per
// block: the log tables, 3104 bytes (ptxas -v)
constexpr size_t kDispSmemCapOneWarp = kDispSmemCap - 3104;

template <int P, bool USE_W>
cudaError_t launch_disp_t(const DispArgs& a0, cudaStream_t stream) {
  DispArgs a = a0;
  const DispSmem L = disp_smem(a.m, P, USE_W);
  const int mpad = L.mpad;
  const size_t xbytes = L.xbytes, rowbytes = L.rowbytes;
  const size_t smem_cap = kDispSmemCap;
  int warps = NB_LB_THREADS / 32;
  while (warps > 1 && xbytes + warps * rowbytes > smem_cap / 2) warps >>= 1;   // aim for >= 2 CTAs/SM
  if (xbytes + warps * rowbytes > kDispSmemCapOneWarp) return cudaErrorInvalidValue;   // callers check fit_disp_smallp_fits
  const size_t smem = xbytes + warps * rowbytes;
  // scratch: [queue counter | 3 mode counters | 3 n gene lists]
  cudaError_t e = cudaMemsetAsync(a.scratch, 0, kDispScratchHead * sizeof(unsigned int), stream);
  if (e != cudaSuccess) return e;
  a.counter = a.scratch;
  a.mode_counts = a.scratch + 1;
  a.mode_lists = reinterpret_cast<int*>(a.scratch + kDispScratchHead);
  unsigned grid = 0;
  if (a.grid != nullptr) {   // fitDispGrid: one queue, no evaluation-mode classification, one gene per warp
    auto kg = fit_disp_grid_kernel<P, USE_W>;
    e = persistent_grid(reinterpret_cast<const void*>(kg), warps * 32, smem, warps, a.n, &grid);
    if (e != cudaSuccess) return e;
    kg<<<grid, warps * 32, smem, stream>>>(a, warps, mpad);
    return cudaGetLastError();
  }
  int* lists = reinterpret_cast<int*>(a.scratch + kDispScratchHead);
  int* code = lists + 3 * (size_t)a.n;
  int* sorted = lists + 4 * (size_t)a.n;
  // Table-length ordering of the TAB list only pays when four genes share a warp (8 lanes per gene: they wait for the
  // longest table of the four) and costs time at two genes per warp
  const int gl = group_lanes_disp(a.m);
  const bool buckets = gl == 8;
  classify_kernel<<<(a.n + 7) / 8, 256, 0, stream>>>(a.y, a.y_is_f64, a.n, a.m, a.ld, lists, a.scratch + 1,
                                                     buckets ? code : nullptr, a.scratch + 8);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  if (buckets) {
    bucket_sort_kernel<<<(a.n + 255) / 256 > 1184 ? 1184 : (a.n + 255) / 256, 256, 0, stream>>>(lists, code, a.scratch + 1 + MODE_TAB, a.scratch + 8, a.scratch + 16, sorted);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    // entries beyond the TAB count are never read by the kernels, so copying the whole n-entry region is harmless
    e = cudaMemcpyAsync(lists, sorted, sizeof(int) * (size_t)a.n, cudaMemcpyDeviceToDevice, stream);
    if (e != cudaSuccess) return e;
  }
  bool launched = false;
  if (gl == 8) e = launch_disp_grp<P, USE_W, 8>(a, mpad, xbytes, rowbytes, stream, launched);
  else if (gl == 16) e = launch_disp_grp<P, USE_W, 16>(a, mpad, xbytes, rowbytes, stream, launched);
  if (e != cudaSuccess || launched) return e;
  for (int ind = 0; ind < 2; ind++) {   // both design variants, as in launch_disp_grp
    auto kern = ind ? fit_disp_kernel<P, USE_W, true> : fit_disp_kernel<P, USE_W, false>;
    e = persistent_grid(reinterpret_cast<const void*>(kern), warps * 32, smem, warps, a.n, &grid);
    if (e != cudaSuccess) return e;
    kern<<<grid, warps * 32, smem, stream>>>(a, warps, mpad);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

template <bool USE_W>
cudaError_t launch_disp_p(const DispArgs& a, cudaStream_t stream) {
  switch (a.p) {
    case 1: return launch_disp_t<1, USE_W>(a, stream);
    case 2: return launch_disp_t<2, USE_W>(a, stream);
    case 3: return launch_disp_t<3, USE_W>(a, stream);
    case 4: return launch_disp_t<4, USE_W>(a, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

bool fit_disp_smallp_fits(int m, int p, int use_weights) {
  const DispSmem L = disp_smem(m, p, use_weights != 0);
  return L.xbytes + L.rowbytes <= kDispSmemCapOneWarp;
}

cudaError_t launch_fit_disp(const DispArgs& a, cudaStream_t stream) {
  if (a.n == 0) return cudaSuccess;
  return a.use_weights ? launch_disp_p<true>(a, stream) : launch_disp_p<false>(a, stream);
}

}  // namespace nb
