// transform.cuh -- the elementwise transforms of the normalized counts q = K / s_j (or K / nf_ij), gene-major in and out:
//   kTfVstParametric  getVarianceStabilizedData, fitType "parametric" (R/vst.R:153-155), a0 = asymptDisp, a1 = extraPois:
//                     log((1 + a1 + 2 a0 q + 2 sqrt(a0 q (1 + a1 + a0 q))) / (4 a0)) / log(2)
//   kTfVstMean        fitType "mean" (R/vst.R:185-189), alpha = the mean dispersion:
//                     (2 asinh(sqrt(alpha q)) - log(alpha) - log(4)) / log(2)
//   kTfLog2           normTransform with f = log2 (R/helper.R:428): log2(q + pc)
// Every entry is evaluated in R's operand order.  q is an IEEE division (not a multiply by 1/s), so it has the bits of
// counts / sf in R or numpy; the products and sums are __dmul_rn / __dadd_rn so that nvcc does not contract them into
// FMAs.  The per-call constants (1 + a1, 2 a0, 4 a0, log(alpha), log(4), log(2)) come from the host in double, so the
// only difference from R is the device's log / asinh / log2 (sqrt is correctly rounded).
// Memory-bound (12 B per entry for int32 counts): each CTA takes a block of whole rows and walks the block's entries
// with consecutive threads on consecutive samples, so reads and writes are coalesced along the sample axis and a small
// m (6, 12) keeps every lane busy.  Static shared memory only (included by size_factors.cu, launched through its
// launch_per_column with one CTA per block of rows).
#pragma once
#include "engine.h"

namespace nb {
namespace {

constexpr int kTfThreads = 256;
constexpr int kTfEntriesPerCta = kTfThreads * 8;   // ~8 entries per thread per CTA

template <class T>
__device__ __forceinline__ double tf_count(const T* y, size_t k) {
  return (double)__ldg(y + k);
}

template <int Mode, bool NF, class T>
__global__ void __launch_bounds__(kTfThreads) transform_kernel(const TransformArgs A, int rows_per_cta) {
  const T* __restrict__ y = static_cast<const T*>(A.y);
  const int r0 = blockIdx.x * rows_per_cta;
  const int rows = A.n - r0 < rows_per_cta ? A.n - r0 : rows_per_cta;
  const unsigned m = (unsigned)A.m;
  const unsigned total = (unsigned)rows * m;
  for (unsigned k = threadIdx.x; k < total; k += kTfThreads) {
    const unsigned di = k / m;
    const unsigned j = k - di * m;
    const size_t i = (size_t)r0 + di;
    const double s = NF ? __ldg(A.nf + i * A.ld + j) : __ldg(A.size_factors + j);
    const double q = tf_count(y, i * A.ld + j) / s;
    double v;
    if (Mode == kTfVstParametric) {
      // c0 = a0, c1 = 1 + a1, c2 = 2 a0, c3 = 4 a0
      const double aq = __dmul_rn(A.c0, q);
      const double root = sqrt(__dmul_rn(aq, __dadd_rn(A.c1, aq)));
      const double num = __dadd_rn(__dadd_rn(A.c1, __dmul_rn(A.c2, q)), __dmul_rn(2.0, root));
      v = log(num / A.c3) / A.ln2;
    } else if (Mode == kTfVstMean) {
      // c0 = alpha, c1 = log(alpha), c2 = log(4)
      v = __dadd_rn(__dadd_rn(__dmul_rn(2.0, asinh(sqrt(__dmul_rn(A.c0, q)))), -A.c1), -A.c2) / A.ln2;
    } else {
      // c0 = pc
      v = log2(__dadd_rn(q, A.c0));
    }
    A.out[i * A.ld_out + j] = v;
  }
}

// rows of one CTA: max(1, kTfEntriesPerCta / m)
inline int transform_rows_per_cta(int m) { return m >= kTfEntriesPerCta ? 1 : kTfEntriesPerCta / m; }

template <int Mode, bool NF>
void (*transform_kernel_for_type(const TransformArgs& a))(TransformArgs, int) {
  return a.y_is_f64 ? transform_kernel<Mode, NF, double> : transform_kernel<Mode, NF, int32_t>;
}

template <int Mode>
void (*transform_kernel_for_factors(const TransformArgs& a))(TransformArgs, int) {
  return a.nf != nullptr ? transform_kernel_for_type<Mode, true>(a) : transform_kernel_for_type<Mode, false>(a);
}

// the instantiation for a's mode, factors and count type
void (*transform_kernel_for(const TransformArgs& a))(TransformArgs, int) {
  switch (a.mode) {
    case kTfVstParametric: return transform_kernel_for_factors<kTfVstParametric>(a);
    case kTfVstMean: return transform_kernel_for_factors<kTfVstMean>(a);
    default: return transform_kernel_for_factors<kTfLog2>(a);
  }
}

}  // namespace
}  // namespace nb
