// nb_logdens.cuh -- the engine's log negative-binomial density, shared by the kernels that report log-likelihoods:
// nb_loglik_kernel (fit_beta.cu, nbinomLogLike at the fitted mean) and iterate_loglik_kernel (sf_iterate.cuh, the
// objective of estimateSizeFactorsIterate).  Direct form, r = 1/alpha:
//   log dnbinom(y; mu, r) = [lgamma(y + r) - lgamma(r) - lgamma(y + 1)] + y (log mu + log alpha) - (y + r) log1p(mu alpha)
// The bracket does not depend on mu (lgamma_diff - log_factorial); nb_logdens_mu is the rest.
#pragma once
#include "nbmath.cuh"

namespace nb {
namespace {

// lgamma(y + r) - lgamma(r), accurate for large r (no catastrophic cancellation)
__device__ __forceinline__ double lgamma_diff(double y, double r, double lg_r) {
  if (r >= kShift) {
    const double xr = y + r;
    const double ixr = rcp_fast(xr), ir = rcp_fast(r);
    const double tail = stirling_tail(ixr, ixr * ixr) - stirling_tail(ir, ir * ir);
    return fma(y, log_pos(xr), fma(r - 0.5, log1p_pos(y * ir), -y)) + tail;
  }
  return lgamma_pos(y + r) - lg_r;
}

// lgamma(y + 1) for the mu-independent part of the deviance.  Counts
// below 256 read log(y!) from a per-CTA shared table filled once with the very same lgamma_pos(k + 1), so the value --
// and every result -- is bit-identical while one Stirling evaluation per sample and gene is saved.
__shared__ double s_lfact[256];
__device__ __forceinline__ void init_lfact_table() {   // call before the first log_factorial; contains a __syncthreads
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_lfact[i] = lgamma_pos((double)i + 1.0);
  __syncthreads();
}
__device__ __forceinline__ double log_factorial(double y) {
  return (y < 256.0 && y == floor(y)) ? s_lfact[(int)y] : lgamma_pos(y + 1.0);
}

// The mu-dependent part y (lmu + log alpha) - (y + r) log1p(mu alpha) for mu > 0, lmu = log(mu).  nb_loglik_kernel
// spells out the same three operations in place: routed through this function, ptxas gave it 76 instead of 64
// registers.
__device__ __forceinline__ double nb_logdens_mu(double y, double mu, double lmu, double alpha, double log_alpha,
                                                double r) {
  const double am = mu * alpha, u1 = 1.0 + am;
  const double l1p = log_pos(u1) + (am - (u1 - 1.0)) * rcp_fast(u1);
  return fma(y, lmu + log_alpha, -(y + r) * l1p);
}

}  // namespace
}  // namespace nb
