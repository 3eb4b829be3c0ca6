// fit_optim.cu -- the reference's fallback for rows the IRLS could not fit, on the device.
//
// WHAT (R/fitNbinomGLMs.R:203-227, 340-407): rows with iter == maxit (incl. the |beta| > 30 sentinel), NA coefficients
// or non-positive variances are re-fitted by maximising the penalised NB log-likelihood
//     logLike(p) + sum dnorm(p, 0, sqrt(1/lambda), log = TRUE)          (p on the log2 scale, box [-30, 30])
// with optim(method = "L-BFGS-B"), started from the IRLS result when it is usable and from the least-squares start
// values otherwise.  The objective is strictly concave in beta (log link, alpha > 0, ridge > 0), so its box-constrained
// maximiser is unique: any convergent method ends at the point L-BFGS-B converges to (optim stops at factr = 1e7, i.e.
// ~1e-5 in beta; this kernel iterates to ~1e-10).
// HOW: one warp per row, projected Newton on the natural-log scale (box +-30 ln 2, ridge lambda / ln(2)^2 -- the same
// objective): exact gradient X'[w (y - mu)/(1 + alpha mu)] - Lambda beta and Hessian
// -X' diag(w mu (1 + alpha y)/(1 + alpha mu)^2) X - Lambda from one pass over the samples, coordinates sitting on a bound
// with an outward gradient frozen (active set), the reduced system solved by Cholesky (diagonal damping if it fails),
// projected back-tracking until the objective increases (the full step when fp64 cannot resolve the gain), stopped
// when every free gradient entry is below 1e-10 of the size of its terms.  Rows are few (a handful per 50 000 genes),
// so nothing here is tuned: any p <= kMaxP, the p x p algebra by lane 0 in shared memory.
#include <math.h>

#include "engine.h"

namespace nb {
namespace {

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ double sample_y(const OptimArgs& A, size_t off, int j) {
  return A.y_is_f64 ? static_cast<const double*>(A.y)[off + j] : (double)static_cast<const int32_t*>(A.y)[off + j];
}

// objective only (beta-dependent part): sum w (y (eta + log nf) - (y + r) log1p(alpha mu)) - 1/2 sum lambda beta^2
__device__ double objective(const OptimArgs& A, size_t off, int lane, double alpha, double r, const double* beta) {
  // every read of beta comes before the warp_sum: once its shuffles are through, lane 0 may already be writing the
  // next trial point, and a lane reading it after that would return a different f than the others and leave the
  // back-tracking on its own branch (the warp's later shuffles then mix lanes of different calls)
  double pen = 0.0;
  for (int k = 0; k < A.p; k++) pen = fma(A.lambda[k] * beta[k], beta[k], pen);
  double acc = 0.0;
  for (int j = lane; j < A.m; j += 32) {
    double eta = 0.0;
    for (int k = 0; k < A.p; k++) eta = fma(__ldg(A.x + (size_t)k * A.m + j), beta[k], eta);
    const double nf = A.nf_is_vector ? __ldg(A.nf + j) : A.nf[off + j];
    const double le = eta + log(nf);
    const double mu = exp(le);
    const double y = sample_y(A, off, j);
    double t = y * le - (y + r) * log1p(alpha * mu);
    if (A.w != nullptr) t *= A.w[off + j];
    acc += t;
  }
  acc = warp_sum(acc);
  return acc - 0.5 * pen;
}

__global__ void __launch_bounds__(32) beta_optim_kernel(const OptimArgs A) {
  extern __shared__ __align__(16) double sm[];
  const int lane = threadIdx.x;
  const int p = A.p, mpad = (A.m + 3) & ~3;
  // A.row_scratch: the two rows of length m live in the CTA's slice of a global buffer, the rest in shared memory
  double* ge = A.row_scratch ? A.row_scratch + (size_t)blockIdx.x * 2 * mpad : sm;   // mpad: d f / d eta_j
  double* he = ge + mpad;            // mpad: -d2 f / d eta_j^2  (> 0)
  double* H = A.row_scratch ? sm : he + mpad;   // p x p: -Hessian (positive definite) of the reduced problem
  double* grad = H + (size_t)p * p;  // p
  double* beta = grad + p;           // p
  double* trial = beta + p;          // p
  double* gscale = trial;            // p: the stop rule's scale of each gradient entry (used before trial is)
  double* step = trial + p;          // p
  double* Lm = step + p;             // p x p: Cholesky factor
  int* active = reinterpret_cast<int*>(Lm + (size_t)p * p);   // p
  // genes strided over the grid: one per CTA when the grid covers every gene (shared-memory rows)
  for (int g = blockIdx.x; g < A.n; g += gridDim.x) {
  __syncwarp();
  const size_t off = (size_t)g * A.ld;
  const double alpha = A.alpha[g], r = 1.0 / alpha;
  const double U = A.bound;
  for (int k = lane; k < p; k += 32) {
    double b = A.beta_in[(size_t)g + (size_t)A.n * k];
    if (!(b == b)) b = 0.0;
    beta[k] = fmin(fmax(b, -U), U);
  }
  __syncwarp();
  double f = objective(A, off, lane, alpha, r, beta);
  int converged = 0, it = 0;
  for (; it < A.maxit; it++) {
    // ---- per-sample first and second derivative with respect to eta
    for (int j = lane; j < A.m; j += 32) {
      double eta = 0.0;
      for (int k = 0; k < p; k++) eta = fma(__ldg(A.x + (size_t)k * A.m + j), beta[k], eta);
      const double nf = A.nf_is_vector ? __ldg(A.nf + j) : A.nf[off + j];
      const double mu = exp(eta + log(nf));
      const double y = sample_y(A, off, j);
      const double u = 1.0 + alpha * mu;
      double g1, h1;
      if (isinf(mu)) {            // limit mu -> inf: (y - mu)/(1 + alpha mu) -> -1/alpha, curvature -> 0
        g1 = -r;
        h1 = 0.0;
      } else {
        g1 = (y - mu) / u;
        h1 = mu * (1.0 + alpha * y) / (u * u);
      }
      if (A.w != nullptr) {
        const double w = A.w[off + j];
        g1 *= w;
        h1 *= w;
      }
      ge[j] = g1;
      he[j] = h1;
    }
    __syncwarp();
    for (int a = 0; a < p; a++) {
      // gradient, and the size of its terms for the stop rule: |g1| + h1 >= w (y + mu) / (2 (1 + alpha mu)), the
      // magnitude the rounding of y - mu and of the sum is relative to
      double s = 0.0, sa = 0.0;
      for (int j = lane; j < A.m; j += 32) {
        const double xa = __ldg(A.x + (size_t)a * A.m + j);
        s = fma(xa, ge[j], s);
        sa = fma(fabs(xa), fabs(ge[j]) + he[j], sa);
      }
      s = warp_sum(s);
      sa = warp_sum(sa);
      if (lane == 0) {
        grad[a] = s - A.lambda[a] * beta[a];
        gscale[a] = 1.0 + sa + A.lambda[a] * fabs(beta[a]);
      }
      for (int b = 0; b <= a; b++) {
        double t = 0.0;
        for (int j = lane; j < A.m; j += 32)
          t = fma(__ldg(A.x + (size_t)a * A.m + j) * __ldg(A.x + (size_t)b * A.m + j), he[j], t);
        t = warp_sum(t);
        if (lane == 0) {
          if (a == b) t += A.lambda[a];
          H[(size_t)a * p + b] = t;
          H[(size_t)b * p + a] = t;
        }
      }
    }
    __syncwarp();
    // ---- active set, reduced Newton system, Cholesky (lane 0)
    int ok = 1;
    double gdot = 0.0, pg = 0.0;
    if (lane == 0) {
      for (int k = 0; k < p; k++) {
        const int act = (beta[k] >= U && grad[k] > 0.0) || (beta[k] <= -U && grad[k] < 0.0);
        active[k] = act;
        if (!act) pg = fmax(pg, fabs(grad[k]) / gscale[k]);
      }
      for (int k = 0; k < p; k++)
        if (active[k]) {
          for (int q = 0; q < p; q++) H[(size_t)k * p + q] = H[(size_t)q * p + k] = 0.0;
          H[(size_t)k * p + k] = 1.0;
        }
    }
    __syncwarp();
    // damped Cholesky of the reduced system into Lm (H is kept so that a retry with more damping is possible)
    if (lane == 0) {
      double tau = 0.0;
      for (int attempt = 0; attempt < 14; attempt++) {
        ok = 1;
        for (int c = 0; c < p && ok; c++) {
          for (int rr = c; rr < p; rr++) {
            double s = H[(size_t)rr * p + c];
            if (rr == c) s += tau * fmax(H[(size_t)c * p + c], 1e-300);
            for (int q = 0; q < c; q++) s -= Lm[(size_t)rr * p + q] * Lm[(size_t)c * p + q];
            if (rr == c) {
              if (!(s > 0.0) || isinf(s)) { ok = 0; break; }
              Lm[(size_t)c * p + c] = sqrt(s);
            } else {
              Lm[(size_t)rr * p + c] = s / Lm[(size_t)c * p + c];
            }
          }
        }
        if (ok) break;
        tau = (tau == 0.0) ? 1e-8 : tau * 100.0;
      }
      if (ok) {
        // solve L L' step = grad (active coordinates: 0)
        for (int k = 0; k < p; k++) {
          double s = active[k] ? 0.0 : grad[k];
          for (int q = 0; q < k; q++) s -= Lm[(size_t)k * p + q] * step[q];
          step[k] = s / Lm[(size_t)k * p + k];
        }
        for (int k = p - 1; k >= 0; k--) {
          double s = step[k];
          for (int q = k + 1; q < p; q++) s -= Lm[(size_t)q * p + k] * step[q];
          step[k] = s / Lm[(size_t)k * p + k];
        }
        for (int k = 0; k < p; k++) gdot += (active[k] ? 0.0 : grad[k]) * step[k];
      }
    }
    ok = __shfl_sync(0xffffffffu, ok, 0);
    gdot = __shfl_sync(0xffffffffu, gdot, 0);
    pg = __shfl_sync(0xffffffffu, pg, 0);
    __syncwarp();
    if (!ok || !(gdot == gdot)) break;                 // not even the damped system factors: give up (conv = 0)
    // projected gradient vanishes: every free entry below 1e-10 of the size of its own terms.  Relative to the terms,
    // not to |f|: f is dominated by y (eta + log nf) whatever the fit, so 1e-10 |f| can stop a row of large counts with
    // its coefficients units away from the maximiser
    if (pg <= 1e-10) { converged = 1; break; }
    // ---- projected back-tracking
    double t = 1.0, fnew = f;
    bool moved = false;
    for (int ls = 0; ls < 60; ls++) {
      for (int k = lane; k < p; k += 32) trial[k] = fmin(fmax(beta[k] + t * step[k], -U), U);
      __syncwarp();
      fnew = objective(A, off, lane, alpha, r, trial);
      if (fnew == fnew && !isinf(fnew) && fnew > f) { moved = true; break; }
      if (fnew == f && !isinf(f)) break;               // flat to rounding (not two -inf: a start whose means
                                                       // overflow has f = -inf, and shorter steps reach finite f)
      t *= 0.5;
    }
    if (!moved) {
      // No step length shows an increase: the gain of the Newton step (gdot / 2) is below what the fp64 objective
      // resolves, yet the gradient test above has not passed.  Near the maximiser the quadratic model is exact to
      // rounding, so take the full projected step unverified and let the gradient decide (maxit bounds the loop).
      for (int k = lane; k < p; k += 32) trial[k] = fmin(fmax(beta[k] + step[k], -U), U);
      __syncwarp();
      fnew = objective(A, off, lane, alpha, r, trial);
      if (!(fnew == fnew) || isinf(fnew)) break;       // not even that: give up (conv = 0)
    }
    __syncwarp();
    for (int k = lane; k < p; k += 32) beta[k] = trial[k];
    __syncwarp();
    f = fnew;
  }
  for (int k = lane; k < p; k += 32) A.beta_out[(size_t)g + (size_t)A.n * k] = beta[k];
  if (lane == 0) {
    A.converged[g] = converged;
    A.iter[g] = it;
  }
  }
}

}  // namespace

cudaError_t launch_beta_optim(const OptimArgs& a, cudaStream_t stream) {
  if (a.n == 0) return cudaSuccess;
  const int mpad = (a.m + 3) & ~3;
  size_t smem = ((size_t)2 * mpad + 2 * (size_t)a.p * a.p + 5 * (size_t)a.p + 2) * sizeof(double);
  OptimArgs b = a;
  b.row_scratch = nullptr;
  unsigned grid = (unsigned)a.n;
  if (smem > 200 * 1024) {
    // the two rows do not fit: they go to a global buffer, one slice per CTA, genes strided over at most 8 CTAs per SM
    smem -= (size_t)2 * mpad * sizeof(double);
    const unsigned cap = 8u * (unsigned)device_sm_count();
    if (grid > cap) grid = cap;
    cudaError_t e = row_scratch((size_t)grid * 2 * mpad * sizeof(double), &b.row_scratch);
    if (e != cudaSuccess) return e;
  }
  cudaError_t e = cudaFuncSetAttribute(beta_optim_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  beta_optim_kernel<<<grid, 32, smem, stream>>>(b);
  return cudaGetLastError();
}

}  // namespace nb
