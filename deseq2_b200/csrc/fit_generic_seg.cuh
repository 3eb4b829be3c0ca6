// fit_generic_seg.cuh -- the general-p kernels for grouped designs without observation weights, "segmented" form.
// Included by fit_generic.cu (inside nb::{anonymous}); same contract as the kernels there
// (src/DESeq2.cpp:31-158, 164-277, 283-465), one warp per gene.
//
// Why a second form.  With long rows (config 4: m = 1000) the kernels of fit_generic.cu keep two fp64 rows plus
// G x 32 lane-private accumulator slots per set in shared memory: 30 KB per warp, 7 warps per SM, 254 registers --
// few warps are resident and every stall reason is a latency.  Here
//   * the samples are laid out sorted by design group, each lane owning a contiguous chunk of the sorted sequence
//     (engine.h::SegLayout, prepared once per call on the host): a lane meets one or two groups per pass, keeps the
//     per-group sums in REGISTERS and stores one value per segment (kmax x 32 slots instead of G x 32, no
//     read-modify-write of shared memory and no group-id load per sample);
//   * counts are kept as 16-bit values (a gene with a count beyond 65535, or with non-integer "counts", gathers y from
//     global memory through the inverse permutation); the IRLS kernel keeps no row of fitted means at all (the
//     post-loop block recomputes mu from the per-group linear predictor of the last pass, bit for bit);
//   * the factor table is 1024 16-bit counts (used while max y < 2 m) instead of 256 doubles;
//   * the saturated-design dispersion kernel carries no p x p matrices; the others factor with the reciprocal diagonal;
//   * the sample loops are specialised at compile time (factor table or not, second derivative or not), and the
//     per-group work sits in ONE divergent region ahead of the warp reductions.
// Config 4 then needs 13.6 KB (dispersion) / 9 KB (IRLS) per warp and the kernels run 16 warps per SM at <= 128
// registers.  Weights, the
// grid search and samplewise designs stay on the kernels of fit_generic.cu.  The device entry points also send long
// rows (m >= 400) of designs with p <= 4 here (capi.cu::long_rows).

// per-CTA shared-memory copies of SegLayout's small tables
struct SegTables {
  const unsigned short* seg_end;   // kmax x 32
  const unsigned char* gfirst;     // 32
  const unsigned char* glo;        // G
  const unsigned char* ghi;        // G
  int kmax;
};
__host__ __device__ inline size_t seg_table_bytes(int kmax, int G) {
  return ((size_t)kmax * 32 * 2 + 32 + 2 * (size_t)G + 15) & ~(size_t)15;
}
// copies the tables behind `dst` (16-byte aligned shared memory); every thread of the CTA calls it, then __syncthreads
__device__ __forceinline__ SegTables stage_seg_tables(const SegLayout& L, int G, unsigned char* dst) {
  unsigned short* se = reinterpret_cast<unsigned short*>(dst);
  unsigned char* gf = dst + (size_t)L.kmax * 32 * 2;
  unsigned char* lo = gf + 32;
  unsigned char* hi = lo + G;
  for (int i = threadIdx.x; i < L.kmax * 32; i += blockDim.x) se[i] = L.seg_end[i];
  for (int i = threadIdx.x; i < 32; i += blockDim.x) gf[i] = L.gfirst[i];
  for (int i = threadIdx.x; i < G; i += blockDim.x) {
    lo[i] = L.glo[i];
    hi[i] = L.ghi[i];
  }
  return SegTables{se, gf, lo, hi, L.kmax};
}

// sum of the segment values that belong to group `g` (lanes glo..ghi in lane order: a fixed summation order)
__device__ __forceinline__ double seg_group_sum(const SegTables& T, const double* seg, int g) {
  double s = 0.0;
  const int lo = T.glo[g], hi = T.ghi[g];
  for (int l = lo; l <= hi; l++) s += seg[(g - (int)T.gfirst[l]) * 32 + l];
  return s;
}
// the same for two or three slot arrays at once (one index computation per contributing lane)
template <bool THREE>
__device__ __forceinline__ void seg_group_sums(const SegTables& T, const double* sa, const double* sb, const double* sc, int g,
                                               double& a, double& b, double& c) {
  a = b = c = 0.0;
  const int lo = T.glo[g], hi = T.ghi[g];
  for (int l = lo; l <= hi; l++) {
    const int idx = (g - (int)T.gfirst[l]) * 32 + l;
    a += sa[idx];
    b += sb[idx];
    if (THREE) c += sc[idx];
  }
}

// (a, b), a >= b, of the lower-triangle entry `idx`: the p (p + 1) / 2 entries of X'WX are dealt to the 32 lanes
struct PairTable {
  const unsigned char* a;
  const unsigned char* b;
  int n;
};
__host__ __device__ inline size_t pair_table_bytes(int p) { return ((size_t)p * (p + 1) + 15) & ~(size_t)15; }
__device__ __forceinline__ PairTable stage_pair_table(int p, unsigned char* dst) {
  const int n = p * (p + 1) / 2;
  for (int idx = threadIdx.x; idx < n; idx += blockDim.x) {
    int a = 0, rem = idx;
    while (rem > a) {
      rem -= a + 1;
      a++;
    }
    dst[idx] = (unsigned char)a;
    dst[n + idx] = (unsigned char)rem;
  }
  return PairTable{dst, dst + n, n};
}
// M = sum_g W[g] x_g x_g' (full symmetric storage), one entry per lane and trip, sums kept in registers
__device__ __forceinline__ void build_xtwx_pairs(const Design& D, const PairTable& P, const double* W, double* M, int lane) {
  for (int idx = lane; idx < P.n; idx += 32) {
    const int a = P.a[idx], b = P.b[idx];
    double s = 0.0;
    for (int g = 0; g < D.G; g++) {
      const double* xr = D.xg + (size_t)g * D.ps;
      s = fma(W[g] * xr[a], xr[b], s);
    }
    M[a * D.ps + b] = s;
    M[b * D.ps + a] = s;
  }
  __syncwarp();
}

// In-place lower Cholesky as fit_generic.cu::chol_smem, with the reciprocal diagonal kept in dinv[0..p): one rsqrt per
// column instead of a square root and a division, and the triangular solves multiply instead of dividing.
__device__ __forceinline__ void chol_smem_d(double* A, double* dinv, int p, int ps, int lane) {
  for (int c = 0; c < p; c++) {
    __syncwarp();
    const double d = A[c * ps + c];
    const double il = rsqrt(d);
    __syncwarp();
    if (lane == c) {
      A[c * ps + c] = d * il;
      dinv[c] = il;
    }
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
__device__ __forceinline__ void chol_inverse_smem_d(const double* L, const double* dinv, double* inv, int p, int ps, int lane) {
  if (lane < p) {
    const int c = lane;
    for (int k = 0; k < c; k++) inv[k * ps + c] = 0.0;
    for (int k = c; k < p; k++) {
      double s = (k == c) ? 1.0 : 0.0;
      for (int i = c; i < k; i++) s -= L[k * ps + i] * inv[i * ps + c];
      inv[k * ps + c] = s * dinv[k];
    }
    for (int k = p - 1; k >= 0; k--) {
      double s = inv[k * ps + c];
      for (int i = k + 1; i < p; i++) s -= L[i * ps + k] * inv[i * ps + c];
      inv[k * ps + c] = s * dinv[k];
    }
  }
  __syncwarp();
}

// ================================================================ dispersion

// Factor table of the segmented dispersion kernel: c_k = #{j : y_j > k} as 16-bit counts (m <= 65535), kTabSeg entries.
// A table of T entries costs T / 32 log + reciprocal pairs per lane and evaluation, the lgamma / digamma pair it
// replaces about twice that per SAMPLE: the table pays while max(y) < 2 m, so long rows (config 4: m = 1000) take it
// up to max(y) = 1023 where the 256-entry fp64 table of fit_generic.cu left 23 % of the evaluations on the per-sample path.
constexpr int kTabSeg = 1024;
__host__ __device__ inline int seg_tab_limit(int m) {
  const int lim = 2 * m > 256 ? 2 * m : 256;
  return lim < kTabSeg ? lim : kTabSeg;
}

struct SDispWarp {
  double* mu;             // mpad, position order
  unsigned short* y16;    // mpad, position order (min(y, 65535); exact unless the gene gathers y from global memory)
  unsigned short* tab;    // kTabSeg
  double *segA, *segB, *segC;   // kmax x 32
  double *WA, *WB, *WC, *q;     // G (not saturated)
  double *M0, *M1, *M2, *M3;    // p x ps (not saturated)
  double* dv;                   // 32 (not saturated): reciprocal Cholesky diagonal
};
__host__ __device__ inline size_t sdisp_warp_bytes(int mpad, int p, int ps, int G, int kmax, int saturated) {
  const size_t Gp = (size_t)(G + 1) & ~(size_t)1;
  return 8 * ((size_t)mpad + 3 * (size_t)kmax * 32 + (saturated ? 0 : 4 * Gp + 4 * (size_t)p * ps + 32)) + 2 * (size_t)kTabSeg +
         2 * (size_t)mpad;
}
__device__ __forceinline__ SDispWarp sdisp_carve(double* base, int mpad, int p, int ps, int G, int kmax, int saturated) {
  SDispWarp S;
  const size_t Gp = (size_t)(G + 1) & ~(size_t)1;
  double* q = base;
  S.mu = q; q += mpad;
  S.segA = q; q += (size_t)kmax * 32;
  S.segB = q; q += (size_t)kmax * 32;
  S.segC = q; q += (size_t)kmax * 32;
  S.WA = S.WB = S.WC = S.q = S.M0 = S.M1 = S.M2 = S.M3 = S.dv = nullptr;
  if (!saturated) {
    S.WA = q; q += Gp;
    S.WB = q; q += Gp;
    S.WC = q; q += Gp;
    S.q = q; q += Gp;
    S.M0 = q; q += (size_t)p * ps;
    S.M1 = q; q += (size_t)p * ps;
    S.M2 = q; q += (size_t)p * ps;
    S.M3 = q; q += (size_t)p * ps;
    S.dv = q; q += 32;
  }
  S.tab = reinterpret_cast<unsigned short*>(q);
  S.y16 = S.tab + kTabSeg;
  return S;
}

// tab[k] = #{y == k + 1} (packed 16-bit counters, built with 32-bit shared-memory atomics) -> c_k = #{y > k}, in place.
// Lane l owns entries 32 l .. 32 l + 31 (16 words): its total, an exclusive suffix scan over the lanes, a second sweep.
__device__ __forceinline__ void seg_tab_suffix_sums(unsigned short* tab, int lane) {
  unsigned int* w = reinterpret_cast<unsigned int*>(tab) + lane * (kTabSeg / 64);
  unsigned int tot = 0;
#pragma unroll
  for (int q = 0; q < kTabSeg / 64; q++) {
    const unsigned int v = w[q];
    tot += (v & 0xffffu) + (v >> 16);
  }
  unsigned int above = tot;   // inclusive suffix sum over lanes >= lane
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int t = __shfl_down_sync(0xffffffffu, above, o);
    if (lane + o < 32) above += t;
  }
  unsigned int run = above - tot;   // counts in the lanes above
#pragma unroll
  for (int q = kTabSeg / 64 - 1; q >= 0; q--) {
    const unsigned int v = w[q];
    const unsigned int hi = run + (v >> 16);
    const unsigned int lo = hi + (v & 0xffffu);
    w[q] = (hi << 16) | lo;
    run = lo;
  }
  __syncwarp();
}

struct SDispCtx {
  Design D;
  SegTables T;
  PairTable P;
  SDispWarp S;
  const unsigned short* inv;   // global: sample at position q (genes whose counts do not fit the 16-bit row)
  const void* yrow;            // the gene's row of counts in global memory
  int y_is_f64, y_gather;
  double inv_sigmasq;
  int use_prior, use_cr;
  int tab_mode, ntab;
  int saturated;
  double sat_logdet;
  double sum_y;
};

// The sample pass: likelihood sums and the per-segment Cox-Reid weight sums.  TAB: the lgamma / digamma differences
// come from the factor table (integer counts below seg_tab_limit); else per sample.
template <bool TAB, bool WANT2>
__device__ __forceinline__ void sdisp_samples(const SDispCtx& C, double alpha, double r, double r2, int lane, double& s_ll,
                                              double& s_dl, double& s_d2) {
  const SDispWarp& S = C.S;
  const int m = C.D.m;
  double lg_r = 0.0, dg_r = 0.0, tg_r = 0.0;
  if (!TAB) {
    lgamma_digamma_pos(r, lg_r, dg_r);
    if (WANT2) tg_r = trigamma_pos(r);
  }
  int slot = lane;   // seg * 32 + lane of the lane's current segment
  int end = C.T.seg_end[lane];
  const int slot_last = (C.T.kmax - 1) * 32;
  double aW = 0.0, aB = 0.0, aC = 0.0;
  const double* mus = S.mu;
  const unsigned short* y16 = S.y16;
  for (int i = 1, j = lane; j < m; i++, j += 32) {
    const double mu = mus[j];
    double y;
    if (TAB || !C.y_gather) {
      y = (double)y16[j];
    } else {
      const int jj = C.inv[j];
      y = C.y_is_f64 ? static_cast<const double*>(C.yrow)[jj] : (double)static_cast<const int32_t*>(C.yrow)[jj];
    }
    // wd = 1/(1/mu + alpha) = mu/(1 + mu alpha); 1/mu never needed: y/mu - 1 = (y - mu)/mu cancels against wd
    const double onema = fma(mu, alpha, 1.0);
    const double wi = rcp_fast(onema);
    const double wd = mu * wi;
    const double l2 = log_pos(onema);
    const double xr = y + r;
    double t = -xr * l2;
    double d = l2 + alpha * (y - mu) * wi;
    double d2 = 0.0;
    if (WANT2) d2 = wd * wd * alpha + y * wi * wi;
    if (!TAB) {
      double lg, dg;
      lgamma_digamma_pos(xr, lg, dg);
      t += lg - lg_r;
      d += dg_r - dg;
      if (WANT2) d2 += r2 * (trigamma_pos(xr) - tg_r);
    }
    s_ll += t;
    s_dl += d;
    if (WANT2) s_d2 += d2;
    aW += wd;
    aB = fma(-wd, wd, aB);
    if (WANT2) aC = fma(2.0 * wd * wd, wd, aC);
    if (i == end) {   // last sample of this lane's current group: one store per sum
      S.segA[slot] = aW;
      S.segB[slot] = aB;
      if (WANT2) S.segC[slot] = aC;
      aW = aB = aC = 0.0;
      end = (slot < slot_last) ? (int)C.T.seg_end[slot + 32] : 0xffff;
      slot += 32;
    }
  }
}

// lp, dlp (and, when WANT2, the second derivative) at log-alpha a.  src/DESeq2.cpp:31-158.
template <bool WANT2>
__device__ __forceinline__ void sdisp_eval(const SDispCtx& C, double a, double pm, int lane, double& lp, double& dlp,
                                           double& d2lp) {
  const Design& D = C.D;
  const SDispWarp& S = C.S;
  const double alpha = exp_fast(a);   // a is confined to [-30, 10] by the line search
  const double r = rcp_fast(alpha);
  const double r2 = r * r;
  double s_ll = 0.0, s_dl = 0.0, s_d2 = 0.0;
  __syncwarp();   // the previous evaluation's reads of the segment slots are done
  if (C.tab_mode) {
    for (int k = lane; k < C.ntab; k += 32) {
      const double ck = (double)S.tab[k];
      const double xk = r + (double)k;
      const double ik = rcp_fast(xk);
      s_ll = fma(ck, log_pos(xk), s_ll);
      s_dl = fma(-ck, ik, s_dl);
      if (WANT2) s_d2 = fma(-ck * r2, ik * ik, s_d2);
    }
    sdisp_samples<true, WANT2>(C, alpha, r, r2, lane, s_ll, s_dl, s_d2);
  } else {
    sdisp_samples<false, WANT2>(C, alpha, r, r2, lane, s_ll, s_dl, s_d2);
  }
  __syncwarp();
  double red[3] = {s_ll, s_dl, s_d2};
  warp_allreduce_sum_n(red);
  double cr = 0.0, dcr = 0.0, cr2 = 0.0;
  if (C.use_cr) {
    // ONE divergent region (lane g owns group g), then warp-uniform code: with the group sums and the per-group terms
    // in two `if (lane < G)` blocks the compiler threaded the branches and the warp reached the reduction split in
    // two (ncu: every shuffle through the WARPSYNC.COLLECTIVE slow path, 25 % of the stall samples)
    double W = 0.0, dW = 0.0, d2W = 0.0;
    double rr[4] = {0.0, 0.0, 0.0, 0.0};
    if (lane < D.G) {
      seg_group_sums<WANT2>(C.T, S.segA, S.segB, S.segC, lane, W, dW, d2W);
      if (C.saturated) {
        const double iw = rcp_fast(W);
        const double q = dW * iw;
        rr[0] = log_pos(W);
        rr[1] = q;
        rr[2] = q * q;
        if (WANT2) rr[3] = d2W * iw;
      }
    }
    __syncwarp();
    if (C.saturated) {
      // log det B = 2 log|det X_g| + sum log W_g, tr(B^-1 dB) = sum dW/W, tr(B^-1 dB B^-1 dB) = sum (dW/W)^2,
      // tr(B^-1 d2B) = sum d2W/W
      warp_allreduce_sum_n(rr);
      cr = -0.5 * (rr[0] + C.sat_logdet);
      dcr = -0.5 * rr[1];
      if (WANT2) cr2 = 0.5 * rr[1] * rr[1] - 0.5 * (rr[1] * rr[1] - rr[2] + rr[3]);
    } else {
      if (lane < D.G) {
        S.WA[lane] = W;
        S.WB[lane] = dW;
        if (WANT2) S.WC[lane] = d2W;
      }
      __syncwarp();
      double* B = S.M0;
      build_xtwx_pairs(D, C.P, S.WA, B, lane);
      chol_smem_d(B, S.dv, D.p, D.ps, lane);
      double ld = (lane < D.p) ? log(B[lane * D.ps + lane]) : 0.0;
      ld = warp_allreduce_sum(ld);
      cr = -0.5 * (2.0 * ld);
      double* Bi = S.M1;
      chol_inverse_smem_d(B, S.dv, Bi, D.p, D.ps, lane);
      quad_forms(D, Bi, S.q, lane);
      double tr1 = 0.0, tr3 = 0.0;
      if (lane < D.G) {
        tr1 = S.WB[lane] * S.q[lane];
        if (WANT2) tr3 = S.WC[lane] * S.q[lane];
      }
      tr1 = warp_allreduce_sum(tr1);
      dcr = -0.5 * tr1;
      if (WANT2) {
        tr3 = warp_allreduce_sum(tr3);
        double* dB = S.M2;
        double* Mm = S.M3;
        build_xtwx_pairs(D, C.P, S.WB, dB, lane);
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
  lp = (red[0] + a * C.sum_y) + prior + cr;
  const double dlp_noprior = (r2 * red[1] + dcr) * alpha;
  dlp = dlp_noprior + dprior;
  if (WANT2) {
    const double ll2 = -2.0 * r2 * r * red[1] + r2 * red[2];
    d2lp = ((ll2 + cr2) * alpha * alpha + dlp_noprior) + (C.use_prior ? -C.inv_sigmasq : 0.0);
  }
}

template <int MAXT>
__global__ void __launch_bounds__(MAXT, 1) fit_disp_seg_kernel(const DispArgs A, int mpad, int ps, size_t warp_bytes) {
  extern __shared__ __align__(16) double smem[];
  init_log_table();
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  double* xg = smem;   // G x ps
  unsigned char* tabs = reinterpret_cast<unsigned char*>(xg + (size_t)A.G * ps);
  for (int i = threadIdx.x; i < A.G * ps; i += blockDim.x) xg[i] = A.xg[i];
  SDispCtx C;
  C.T = stage_seg_tables(A.seg, A.G, tabs);
  C.P = stage_pair_table(A.p, tabs + seg_table_bytes(A.seg.kmax, A.G));
  __syncthreads();
  C.D = Design{xg, nullptr, A.p, ps, A.G, 1, A.m};
  C.saturated = A.saturated && A.G == A.p;
  C.S = sdisp_carve(reinterpret_cast<double*>(tabs + seg_table_bytes(A.seg.kmax, A.G) + pair_table_bytes(A.p) +
                                              (size_t)warp * warp_bytes),
                    mpad, A.p, ps, A.G, A.seg.kmax, C.saturated);
  C.inv = A.seg.inv;
  C.y_is_f64 = A.y_is_f64;
  C.inv_sigmasq = 1.0 / A.prior_sigmasq;
  C.use_prior = A.use_prior;
  C.use_cr = A.use_cr;
  C.sat_logdet = A.sat_logdet;
  const SDispWarp& S = C.S;
  const int tab_limit = seg_tab_limit(A.m);

  for (;;) {
    unsigned int g = 0;
    if (lane == 0) g = atomicAdd(A.counter, 1u);
    g = __shfl_sync(0xffffffffu, g, 0);
    if (g >= (unsigned int)A.n) break;
    // ---- stage the row in position order
    const size_t off = (size_t)g * A.ld;
    C.yrow = A.y_is_f64 ? static_cast<const void*>(static_cast<const double*>(A.y) + off)
                        : static_cast<const void*>(static_cast<const int32_t*>(A.y) + off);
    double sy = 0.0, ym = 0.0, ymin = 0.0;
    bool integ = true;
    for (int j = lane; j < A.m; j += 32) {
      const double y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + j] : (double)static_cast<const int32_t*>(A.y)[off + j];
      const int q = A.seg.pos[j];
      S.mu[q] = A.mu[off + j];
      S.y16[q] = (unsigned short)fmin(fmax(y, 0.0), 65535.0);
      sy += y;
      ym = fmax(ym, y);
      ymin = fmin(ymin, y);
      integ = integ && (y == floor(y));
    }
    C.sum_y = warp_allreduce_sum(sy);
    const double ymax = warp_allreduce_max(ym);
    ymin = -warp_allreduce_max(-ymin);
    const bool counts = __all_sync(0xffffffffu, integ) && (ymin >= 0.0);
    C.y_gather = !(counts && ymax <= 65535.0);
    C.tab_mode = counts && (ymax < (double)tab_limit);
    C.ntab = 0;
    if (C.tab_mode) {
      unsigned int* tw = reinterpret_cast<unsigned int*>(S.tab);
      for (int k = lane; k < kTabSeg / 2; k += 32) tw[k] = 0u;
      __syncwarp();
      for (int j = lane; j < A.m; j += 32) {
        const int v = S.y16[j];
        if (v >= 1) atomicAdd(&tw[(v - 1) >> 1], 1u << (((v - 1) & 1) * 16));   // counts <= m <= 65535: no carry
      }
      __syncwarp();
      seg_tab_suffix_sums(S.tab, lane);
      C.ntab = (int)ymax;
    }
    const double pm = A.prior_mean[g];
    double lp_new, dlp_new, d2 = 0.0;
    DispLineSearch ls(A.log_alpha_in[g], A.kappa_0);
    for (int t = -1; t < A.maxit; t++) {   // t = -1: the evaluation at the starting point
      const double a_new = ls.propose();
      sdisp_eval<false>(C, a_new, pm, lane, lp_new, dlp_new, d2);
      if (ls.take(lp_new, dlp_new, A)) break;
    }
    sdisp_eval<true>(C, ls.a, pm, lane, lp_new, dlp_new, d2);
    if (lane == 0) ls.store(A, g, d2);
    __syncwarp();
  }
}

// ================================================================ beta (IRLS)

struct SBetaWarp {
  unsigned short* y16;   // mpad, position order (genes with counts that do not fit gather y from global memory)
  double *nf, *lnf;      // mpad each, position order: the gene's normalisation factors and their logs (nf matrix only)
  double *segA, *segB;   // kmax x 32
  double *WA, *WB, *eta, *eeta, *q;   // G
  double *M0, *M1, *M2, *M3;   // p x ps
  double *v0, *v1, *v2, *v3;   // 32
};
__host__ __device__ inline size_t sbeta_warp_bytes(int mpad, int p, int ps, int G, int kmax, int nf_is_vector) {
  const size_t Gp = (size_t)(G + 1) & ~(size_t)1;
  return 8 * ((nf_is_vector ? 0 : 2 * (size_t)mpad) + 2 * (size_t)kmax * 32 + 5 * Gp + 4 * (size_t)p * ps + 4 * 32) +
         2 * (size_t)mpad;
}
__device__ __forceinline__ SBetaWarp sbeta_carve(double* base, int mpad, int p, int ps, int G, int kmax, int nf_is_vector) {
  SBetaWarp S;
  const size_t Gp = (size_t)(G + 1) & ~(size_t)1;
  double* q = base;
  S.nf = nf_is_vector ? nullptr : q; q += nf_is_vector ? 0 : mpad;
  S.lnf = nf_is_vector ? nullptr : q; q += nf_is_vector ? 0 : mpad;
  S.segA = q; q += (size_t)kmax * 32;
  S.segB = q; q += (size_t)kmax * 32;
  S.WA = q; q += Gp;
  S.WB = q; q += Gp;
  S.eta = q; q += Gp;
  S.eeta = q; q += Gp;
  S.q = q; q += Gp;
  S.M0 = q; q += (size_t)p * ps;
  S.M1 = q; q += (size_t)p * ps;
  S.M2 = q; q += (size_t)p * ps;
  S.M3 = q; q += (size_t)p * ps;
  S.v0 = q; q += 32;
  S.v1 = q; q += 32;
  S.v2 = q; q += 32;
  S.v3 = q; q += 32;
  S.y16 = reinterpret_cast<unsigned short*>(q);
  return S;
}

struct SBetaCtx {
  Design D;
  SegTables T;
  PairTable P;
  SBetaWarp S;
  const double *nfp, *lnfp;    // position order: shared (size-factor vector) or the warp's rows
  const unsigned short* inv;   // global
  const void* yrow;
  int y_is_f64, y_gather;
  double minmu, log_minmu;
};

__device__ __forceinline__ double sbeta_y(const SBetaCtx& C, int j) {
  if (!C.y_gather) return (double)C.S.y16[j];
  const int jj = C.inv[j];
  return C.y_is_f64 ? static_cast<const double*>(C.yrow)[jj] : (double)static_cast<const int32_t*>(C.yrow)[jj];
}

// mu of a sample of group g: nf * exp(eta_g), the exponential taken once per group and pass (1 ulp from
// exp(eta_g + log nf), far below what the stop rule at 1e-8 can see); log mu = eta_g + log nf unless clamped
__device__ __forceinline__ double sbeta_exp(double e) { return (fabs(e) < 700.0) ? exp_fast(e) : exp(e); }

// one fused pass: eta per group -> mu, deviance part, per-group sums W = sum w, WZ = sum w z (src/DESeq2.cpp:324-373)
template <bool WANT_DEV>
__device__ __forceinline__ double sbeta_pass(const SBetaCtx& C, const double* beta, double alpha, double r, double log_alpha,
                                             int lane) {
  const Design& D = C.D;
  const SBetaWarp& S = C.S;
  __syncwarp();
  if (lane < D.G) {
    const double* xr = D.xg + (size_t)lane * D.ps;
    double e = 0.0;
    for (int k = 0; k < D.p; k++) e = fma(xr[k], beta[k], e);
    S.eta[lane] = e;
    S.eeta[lane] = sbeta_exp(e);
  }
  __syncwarp();
  int slot = lane;
  int end = C.T.seg_end[lane];
  const int slot_last = (C.T.kmax - 1) * 32;
  int g = C.T.gfirst[lane];
  double e = S.eta[g], ee = S.eeta[g];
  double aW = 0.0, aB = 0.0, dev = 0.0;
  for (int i = 1, j = lane; j < D.m; i++, j += 32) {
    const double mu = fmax(ee * C.nfp[j], C.minmu);
    const double y = sbeta_y(C, j);
    const double am = mu * alpha;
    const double u1 = 1.0 + am;
    const double iu1 = rcp_fast(u1);
    const double w = mu * iu1;
    double lmu_lnf = e;   // log(mu / nf)
    double lnf = 0.0;
    if (WANT_DEV || mu == C.minmu) lnf = C.lnfp[j];
    if (mu == C.minmu) lmu_lnf = C.log_minmu - lnf;
    const double z = lmu_lnf + fma(y, rcp_fast(mu), -1.0);
    if (WANT_DEV) {
      const double l1p = log_pos(u1) + (am - (u1 - 1.0)) * iu1;   // log1p(am)
      dev += fma(y, (lmu_lnf + lnf) + log_alpha, -(y + r) * l1p);
    }
    aW += w;
    aB = fma(w, z, aB);
    if (i == end) {
      S.segA[slot] = aW;
      S.segB[slot] = aB;
      aW = aB = 0.0;
      end = (slot < slot_last) ? (int)C.T.seg_end[slot + 32] : 0xffff;
      slot += 32;
      g = (g + 1 < D.G) ? g + 1 : g;
      e = S.eta[g];
      ee = S.eeta[g];
    }
  }
  __syncwarp();
  if (lane < D.G) {
    double wa, wb, unused;
    seg_group_sums<false>(C.T, S.segA, S.segB, nullptr, lane, wa, wb, unused);
    S.WA[lane] = wa;
    S.WB[lane] = wb;
  }
  __syncwarp();
  return WANT_DEV ? warp_allreduce_sum(dev) : 0.0;
}

template <int MAXT>
__global__ void __launch_bounds__(MAXT, 1) fit_beta_seg_kernel(const BetaArgs A, int mpad, int ps, size_t warp_bytes) {
  extern __shared__ __align__(16) double smem[];
  init_log_table();
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int p = A.p;
  double* xg = smem;                                         // G x ps
  double* nf_shared = xg + (size_t)A.G * ps;                 // mpad (size-factor vector only), position order
  double* lnf_shared = nf_shared + (A.nf_is_vector ? mpad : 0);   // mpad, their logs
  double* lam = lnf_shared + (A.nf_is_vector ? mpad : 0);    // 32
  double* contrast = lam + 32;                               // 32
  double* lfact = contrast + 32;                             // 256: log y! of small counts (the same lgamma_pos, bit for bit)
  unsigned char* tabs = reinterpret_cast<unsigned char*>(lfact + 256);
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lfact[i] = lgamma_pos((double)i + 1.0);
  for (int i = threadIdx.x; i < A.G * ps; i += blockDim.x) xg[i] = A.xg[i];
  if (A.nf_is_vector)
    for (int j = threadIdx.x; j < A.m; j += blockDim.x) {
      const int q = A.seg.pos[j];
      nf_shared[q] = A.nf[j];
      lnf_shared[q] = log(A.nf[j]);
    }
  for (int k = threadIdx.x; k < p; k += blockDim.x) {
    lam[k] = A.lambda[k];
    contrast[k] = A.contrast[k];
  }
  SBetaCtx C;
  C.T = stage_seg_tables(A.seg, A.G, tabs);
  C.P = stage_pair_table(p, tabs + seg_table_bytes(A.seg.kmax, A.G));
  __syncthreads();
  C.D = Design{xg, nullptr, p, ps, A.G, 1, A.m};
  C.S = sbeta_carve(reinterpret_cast<double*>(tabs + seg_table_bytes(A.seg.kmax, A.G) + pair_table_bytes(p) +
                                              (size_t)warp * warp_bytes),
                    mpad, p, ps, A.G, A.seg.kmax, A.nf_is_vector);
  C.inv = A.seg.inv;
  C.y_is_f64 = A.y_is_f64;
  C.minmu = A.minmu;
  C.log_minmu = log(A.minmu);
  C.nfp = A.nf_is_vector ? nf_shared : C.S.nf;
  C.lnfp = A.nf_is_vector ? lnf_shared : C.S.lnf;
  const SBetaWarp& S = C.S;
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
    C.yrow = A.y_is_f64 ? static_cast<const void*>(static_cast<const double*>(A.y) + off)
                        : static_cast<const void*>(static_cast<const int32_t*>(A.y) + off);
    bool fits = true;
    for (int j = lane; j < A.m; j += 32) {
      const double y = A.y_is_f64 ? static_cast<const double*>(A.y)[off + j] : (double)static_cast<const int32_t*>(A.y)[off + j];
      const int q = A.seg.pos[j];
      fits = fits && (y >= 0.0) && (y <= 65535.0) && (y == floor(y));
      S.y16[q] = (unsigned short)fmin(fmax(y, 0.0), 65535.0);
      if (!A.nf_is_vector) {
        const double f = A.nf[off + j];
        S.nf[q] = f;
        S.lnf[q] = log(f);
      }
    }
    C.y_gather = !__all_sync(0xffffffffu, fits);
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
        const double y = sbeta_y(C, j);
        const double lf = (y >= 0.0 && y < 256.0 && y == floor(y)) ? lfact[(int)y] : lgamma_pos(y + 1.0);
        c += lgamma_diff_g(y, r, lg_r) - lf;
      }
      devc = warp_allreduce_sum(c);
    }
    sbeta_pass<false>(C, beta, alpha, r, log_alpha, lane);
    IrlsProgress ir;
    for (int t = 0; t < A.maxit; t++) {
      ir.start_iteration();
      // normal equations (X'WX + Lambda) b = X'Wz, Jacobi-equilibrated Cholesky
      build_xtwx_pairs(C.D, C.P, S.WA, B, lane);
      if (lane < p) {
        double s = 0.0;
        for (int q = 0; q < A.G; q++) s = fma(S.WB[q], xg[(size_t)q * ps + lane], s);
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
      chol_smem_d(L, tmp, p, ps, lane);   // tmp: reciprocal diagonal
      // forward / backward substitution, column oriented (lane = row)
      for (int c = 0; c < p; c++) {
        if (lane == c) rhs[c] *= tmp[c];
        __syncwarp();
        if (lane > c && lane < p) rhs[lane] -= L[lane * ps + c] * rhs[c];
        __syncwarp();
      }
      for (int c = p - 1; c >= 0; c--) {
        if (lane == c) rhs[c] *= tmp[c];
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
      if (__any_sync(0xffffffffu, big)) { ir.diverged(A.maxit); break; }   // mu / eta stay those of the previous beta
      const double dv = sbeta_pass<true>(C, beta, alpha, r, log_alpha, lane);
      if (ir.stop_after_pass(dv, devc, A)) break;
    }
    // ---- post-loop block (src/DESeq2.cpp:429-455): the W sums and eta belong to the last pass
    build_xtwx_pairs(C.D, C.P, S.WA, B, lane);
    if (lane < p) sc[lane] = rsqrt(B[lane * ps + lane] + lam[lane]);
    __syncwarp();
    if (lane < p)
      for (int b = 0; b < p; b++)
        L[lane * ps + b] = (B[lane * ps + b] + ((b == lane) ? lam[lane] : 0.0)) * sc[lane] * sc[b];
    chol_smem_d(L, tmp, p, ps, lane);
    chol_inverse_smem_d(L, tmp, Ainv, p, ps, lane);
    if (lane < p)
      for (int b = 0; b < p; b++) Ainv[lane * ps + b] *= sc[lane] * sc[b];
    __syncwarp();
    quad_forms(C.D, Ainv, S.q, lane);
    if (A.hat_diag != nullptr || A.mu_out != nullptr) {
      for (int j = lane; j < A.m; j += 32) {   // sample order: coalesced stores
        const int q = A.seg.pos[j], gj = A.gid[j];
        const double mu = fmax(S.eeta[gj] * C.nfp[q], C.minmu);   // the last pass's mu, bit for bit
        if (A.mu_out != nullptr) A.mu_out[off + j] = mu;
        if (A.hat_diag != nullptr) A.hat_diag[off + j] = mu * rcp_fast(fma(alpha, mu, 1.0)) * S.q[gj];
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
