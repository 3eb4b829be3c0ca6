// smallp.cuh -- register-resident dense linear algebra for p x p symmetric systems, p <= 4,
// fully unrolled at compile time.  Replaces the Armadillo/LAPACK calls of the reference
// (qr_econ/solve/.i()/det/trace, /root/reference/src/DESeq2.cpp:45-46,83-85,129-134,344-356,398,439,452)
// on the per-gene normal equations.  Symmetric matrices are packed lower-triangular:
// element (a,b), a >= b, lives at a(a+1)/2 + b.
#pragma once
#include "nbmath.cuh"

namespace nb {

template <int P>
struct SymP {
  static constexpr int N = P * (P + 1) / 2;
  double v[N];
  __device__ __forceinline__ double& at(int a, int b) { return a >= b ? v[a * (a + 1) / 2 + b] : v[b * (b + 1) / 2 + a]; }
  __device__ __forceinline__ double get(int a, int b) const { return a >= b ? v[a * (a + 1) / 2 + b] : v[b * (b + 1) / 2 + a]; }
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int i = 0; i < N; i++) v[i] = 0.0;
  }
};

// ---------------------------------------------------------------- indicator designs
// A design whose column 0 is all 1.0 and whose other entries are all +0.0 or 1.0 (a factor design with an intercept:
// ~condition, ~batch + condition) makes every design product exact and predictable: x_a x_0 = x_a, x_a x_a = x_a,
// and x_a x_b is the AND of the two high words (1.0 = 0x3FF00000'00000000).  Each small-p kernel comes in two
// variants, both launched; each tests the design as it starts, and only the one that fits it runs.  The indicator
// variant forms the products without FP64 multiplies and takes the (a, a) sums of X'WX-type accumulators from the
// (a, 0) sums, which receive the same operations in the same order.  Every value is the general path's bit for bit.

// the warp reads the whole m x P design (column-major) from global memory; warp-uniform result.  The kernels call it
// first thing, so the variant of a launch that does not fit the design returns before any set-up.
template <int P>
__device__ __forceinline__ bool indicator_design(const double* x, int m) {
  bool ok = true;
  for (int idx = threadIdx.x & 31; idx < P * m; idx += 32) {
    const long long b = __double_as_longlong(x[idx]);
    ok = ok && (b == 0x3FF0000000000000LL || (idx >= m && b == 0));
  }
  return __all_sync(0xffffffffu, ok);
}

// design row of sample j; IND: x_0 = 1.0 is not loaded
template <int P, bool IND>
__device__ __forceinline__ void load_design_row(const double* xs, int mpad, int j, double (&xv)[P]) {
  xv[0] = IND ? 1.0 : xs[j];
#pragma unroll
  for (int k = 1; k < P; k++) xv[k] = xs[k * mpad + j];
}

// x_a x_b (b <= a) of a design row; IND: without an FP64 multiply
template <int P, bool IND>
__device__ __forceinline__ double design_prod(const double (&xv)[P], int a, int b) {
  if (!IND) return xv[a] * xv[b];
  if (b == 0 || b == a) return xv[a];
  return __hiloint2double(__double2hiint(xv[a]) & __double2hiint(xv[b]), 0);
}

// IND: the (a, a) entries of a packed accumulator, which the sample loop skips, are the (a, 0) entries
template <int P, bool IND>
__device__ __forceinline__ void fill_diag_from_col0(double* acc) {
  if (!IND) return;
#pragma unroll
  for (int a = 1; a < P; a++) acc[a * (a + 1) / 2 + a] = acc[a * (a + 1) / 2];
}

// in-place Cholesky A = L L' (lower, packed).  Returns false if a pivot is not positive (or NaN).
template <int P>
__device__ __forceinline__ bool chol_factor(SymP<P>& A) {
  bool ok = true;
#pragma unroll
  for (int c = 0; c < P; c++) {
    double d = A.at(c, c);
#pragma unroll
    for (int k = 0; k < c; k++) d = fma(-A.at(c, k), A.at(c, k), d);
    ok = ok && (d > 0.0);
    double l = sqrt(d);
    A.at(c, c) = l;
    double il = 1.0 / l;
#pragma unroll
    for (int r = c + 1; r < P; r++) {
      double s = A.at(r, c);
#pragma unroll
      for (int k = 0; k < c; k++) s = fma(-A.at(r, k), A.at(c, k), s);
      A.at(r, c) = s * il;
    }
  }
  return ok;
}

// solve L L' x = b in place
template <int P>
__device__ __forceinline__ void chol_solve(const SymP<P>& L, double (&b)[P]) {
#pragma unroll
  for (int r = 0; r < P; r++) {
    double s = b[r];
#pragma unroll
    for (int k = 0; k < r; k++) s = fma(-L.get(r, k), b[k], s);
    b[r] = s / L.get(r, r);
  }
#pragma unroll
  for (int r = P - 1; r >= 0; r--) {
    double s = b[r];
#pragma unroll
    for (int k = r + 1; k < P; k++) s = fma(-L.get(k, r), b[k], s);
    b[r] = s / L.get(r, r);
  }
}

// inverse of the factored matrix, symmetric packed
template <int P>
__device__ __forceinline__ void chol_inverse(const SymP<P>& L, SymP<P>& inv) {
#pragma unroll
  for (int c = 0; c < P; c++) {
    double e[P];
#pragma unroll
    for (int k = 0; k < P; k++) e[k] = (k == c) ? 1.0 : 0.0;
    chol_solve<P>(L, e);
#pragma unroll
    for (int r = c; r < P; r++) inv.at(r, c) = e[r];
  }
}

// det of the factored matrix = prod L_kk^2
template <int P>
__device__ __forceinline__ double chol_det(const SymP<P>& L) {
  double d = 1.0;
#pragma unroll
  for (int k = 0; k < P; k++) d *= L.get(k, k) * L.get(k, k);
  return d;
}

// trace(A * B) for symmetric packed A, B
template <int P>
__device__ __forceinline__ double sym_trace_prod(const SymP<P>& A, const SymP<P>& B) {
  double t = 0.0;
#pragma unroll
  for (int a = 0; a < P; a++) {
    t = fma(A.get(a, a), B.get(a, a), t);
#pragma unroll
    for (int b = 0; b < a; b++) t = fma(2.0 * A.get(a, b), B.get(a, b), t);
  }
  return t;
}

// full (non-symmetric) product M = A * B of two symmetric packed matrices
template <int P>
__device__ __forceinline__ void sym_mul_full(const SymP<P>& A, const SymP<P>& B, double (&M)[P][P]) {
#pragma unroll
  for (int i = 0; i < P; i++)
#pragma unroll
    for (int j = 0; j < P; j++) {
      double s = 0.0;
#pragma unroll
      for (int k = 0; k < P; k++) s = fma(A.get(i, k), B.get(k, j), s);
      M[i][j] = s;
    }
}

// Solve (A) x = b for SPD A with Jacobi equilibration (unit diagonal) before the Cholesky: removes the
// column-scaling part of the conditioning, which is what the reference's QR branch
// (src/DESeq2.cpp:344-356) buys over its normal-equation branch (:398) for badly scaled covariates.
// A is destroyed.  Returns false if not positive definite.
template <int P>
__device__ __forceinline__ bool spd_solve_equilibrated(SymP<P>& A, double (&b)[P]) {
  double s[P];
#pragma unroll
  for (int k = 0; k < P; k++) s[k] = rsqrt(A.get(k, k));
#pragma unroll
  for (int a = 0; a < P; a++) {
#pragma unroll
    for (int c = 0; c <= a; c++) A.at(a, c) *= s[a] * s[c];
    b[a] *= s[a];
  }
  bool ok = chol_factor<P>(A);
  chol_solve<P>(A, b);
#pragma unroll
  for (int k = 0; k < P; k++) b[k] *= s[k];
  return ok;
}

// Cox-Reid pieces for B = X'WX (SPD): det(B), and tr(B^-1 dB) when WANT_TR.
// p = 1, 2, 3 use the adjugate (no square roots, one reciprocal); larger p the Cholesky factor.
template <int P, bool WANT_TR>
__device__ __forceinline__ void cr_det_trace(const SymP<P>& B, const SymP<P>& dB, double& det, double& tr) {
  tr = 0.0;
  if constexpr (P == 1) {
    det = B.v[0];
    if (WANT_TR) tr = dB.v[0] * rcp_fast(det);
  } else if constexpr (P == 2) {
    const double b00 = B.v[0], b10 = B.v[1], b11 = B.v[2];
    det = fma(b00, b11, -b10 * b10);
    if (WANT_TR) tr = (fma(b11, dB.v[0], fma(b00, dB.v[2], -2.0 * b10 * dB.v[1]))) * rcp_fast(det);
  } else if constexpr (P == 3) {
    const double b00 = B.v[0], b10 = B.v[1], b11 = B.v[2], b20 = B.v[3], b21 = B.v[4], b22 = B.v[5];
    // cofactors (symmetric adjugate)
    const double c00 = fma(b11, b22, -b21 * b21);
    const double c10 = fma(b21, b20, -b10 * b22);
    const double c20 = fma(b10, b21, -b11 * b20);
    const double c11 = fma(b00, b22, -b20 * b20);
    const double c21 = fma(b10, b20, -b00 * b21);
    const double c22 = fma(b00, b11, -b10 * b10);
    det = fma(b00, c00, fma(b10, c10, b20 * c20));
    if (WANT_TR) {
      double t = c00 * dB.v[0];
      t = fma(c11, dB.v[2], t);
      t = fma(c22, dB.v[5], t);
      t = fma(2.0 * c10, dB.v[1], t);
      t = fma(2.0 * c20, dB.v[3], t);
      t = fma(2.0 * c21, dB.v[4], t);
      tr = t * rcp_fast(det);
    }
  } else {
    SymP<P> L = B;
    chol_factor<P>(L);
    det = chol_det<P>(L);
    if (WANT_TR) {
      SymP<P> Bi;
      chol_inverse<P>(L, Bi);
      tr = sym_trace_prod<P>(Bi, dB);
    }
  }
}

}  // namespace nb
