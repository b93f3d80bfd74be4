// cv::SVD::compute(A, w, u, vt, SVD::MODIFY_A | SVD::FULL_UV) for one 4x4 CV_32F matrix, as cv2 computes it bit for bit
// (LocalMapping::CreateNewMapPoints, LocalMapping.cc:465; the caller reads w and vt.row(3) only).
//
// The algorithm is a one-sided Jacobi sweep on the rows of At = A^T (the columns of A):
//   - squared row norms W and every inner product p accumulated in fp64 from fp32 operands, in index order;
//   - a pair is skipped when |p| <= eps * sqrt(W_i * W_j), eps = 2 * FLT_EPSILON;
//   - else gamma = hypot(2p, W_i - W_j), and the rotation's c and s are formed in fp64 from the larger of the two half-angle forms
//     and rounded to fp32.  The hypot is OpenCV's own template (lapack.cpp), not the C library's:
//     a > b ? a * sqrt(1 + (b/a)^2) : b > 0 ? b * sqrt(1 + (a/b)^2) : 0 on |a|, |b|, in fp64.  The two differ in the last bit of
//     gamma now and then, and one uniform random matrix in 1e7 to 1e8 then gets a different vt (tests/golden/orb_cv2_svd4.npz
//     holds such matrices, found by tools/svd4_hypot_search.cpp);
//   - both rows of At and of V are rotated in fp32 (t0 = c*x + s*y, t1 = -s*x + c*y, each product and sum rounded on its own), and
//     W_i, W_j are re-accumulated in fp64 from the rotated At rows;
//   - at most 30 sweeps, stopping after the first sweep without a rotation;
//   - W = sqrt of the re-accumulated squared norms (fp64), then a selection sort to descending W (strict <, so equal values keep
//     their order) that swaps V's rows along; w = (float)W.
// U (the normalised At rows, and FULL_UV's completion of the rows that belong to zero singular values) is not formed: no input
// to w or V depends on it.  tests/test_triangulate_svd.py compiles this header for the host and compares w and the whole of vt
// with cv2.SVDecomp, stored in tests/golden/orb_cv2_svd4.npz (and live where cv2 imports).
// On the device every operation is the _rn intrinsic, so no product is contracted whatever -fmad says; tests/test_float_math_gpu.py
// compares the device build with cv2 on the fixture and with the host build on fresh matrices.
#pragma once
#include "libm_glibc.cuh"

namespace pl {
namespace svd4_ops {
#ifdef __CUDA_ARCH__
PL_LIBM_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
PL_LIBM_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
PL_LIBM_HD double dmul(double a, double b) { return __dmul_rn(a, b); }
PL_LIBM_HD double dadd(double a, double b) { return __dadd_rn(a, b); }
PL_LIBM_HD double ddiv(double a, double b) { return __ddiv_rn(a, b); }
PL_LIBM_HD double dsqrt(double a) { return __dsqrt_rn(a); }
PL_LIBM_HD float d2f(double a) { return __double2float_rn(a); }
#else
PL_LIBM_HD float fmul(float a, float b) { return a * b; }
PL_LIBM_HD float fadd(float a, float b) { return a + b; }
PL_LIBM_HD double dmul(double a, double b) { return a * b; }
PL_LIBM_HD double dadd(double a, double b) { return a + b; }
PL_LIBM_HD double ddiv(double a, double b) { return a / b; }
PL_LIBM_HD double dsqrt(double a) { return sqrt(a); }
PL_LIBM_HD float d2f(double a) { return (float)a; }
#endif
// OpenCV's hypot<double> (lapack.cpp), in this operation order
PL_LIBM_HD double cv_hypot(double a, double b) {
  a = fabs(a); b = fabs(b);
  if (a > b) { b = ddiv(b, a); return dmul(a, dsqrt(dadd(1.0, dmul(b, b)))); }
  if (b > 0) { a = ddiv(a, b); return dmul(b, dsqrt(dadd(1.0, dmul(a, a)))); }
  return 0;
}
// sum of x_k * y_k in fp64, k = 0 .. 3 in order, from 0
PL_LIBM_HD double dot4(const float* x, const float* y) {
  double s = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) s = dadd(s, dmul((double)x[k], (double)y[k]));
  return s;
}
// (x, y) <- (c x + s y, -s x + c y) in fp32
PL_LIBM_HD void rotate4(float* x, float* y, float c, float s) {
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const float t0 = fadd(fmul(c, x[k]), fmul(s, y[k])), t1 = fadd(fmul(-s, x[k]), fmul(c, y[k]));
    x[k] = t0; y[k] = t1;
  }
}
}  // namespace svd4_ops

// A: row-major 4x4 (not modified).  w[4] descending; vt: row-major 4x4, rows = right singular vectors.
PL_LIBM_HD void svd4(const float* A, float* w, float* vt) {
  using namespace svd4_ops;
  float At[4][4], V[4][4];
  double W[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
#pragma unroll
    for (int k = 0; k < 4; k++) { At[i][k] = A[4 * k + i]; V[i][k] = i == k ? 1.f : 0.f; }
    W[i] = dot4(At[i], At[i]);
  }
  const double eps = (double)(2.0f * 1.1920928955078125e-07f);   // FLT_EPSILON * 2, an fp32 constant widened
  for (int iter = 0; iter < 30; iter++) {
    bool changed = false;
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
      for (int j = i + 1; j < 4; j++) {
        const double a = W[i], b = W[j];
        double p = dot4(At[i], At[j]);
        if (fabs(p) <= dmul(eps, dsqrt(dmul(a, b)))) continue;
        p = dmul(p, 2.0);
        const double beta = dadd(a, -b), gamma = cv_hypot(p, beta);
        float c, s;
        if (beta < 0) {
          const double delta = dmul(dadd(gamma, -beta), 0.5);
          s = d2f(dsqrt(ddiv(delta, gamma)));
          c = d2f(ddiv(p, dmul(dmul(gamma, (double)s), 2.0)));
        } else {
          c = d2f(dsqrt(ddiv(dadd(gamma, beta), dmul(gamma, 2.0))));
          s = d2f(ddiv(p, dmul(dmul(gamma, (double)c), 2.0)));
        }
        rotate4(At[i], At[j], c, s);
        W[i] = dot4(At[i], At[i]);
        W[j] = dot4(At[j], At[j]);
        rotate4(V[i], V[j], c, s);
        changed = true;
      }
    }
    if (!changed) break;
  }
#pragma unroll
  for (int i = 0; i < 4; i++) W[i] = dsqrt(dot4(At[i], At[i]));
  // selection sort to descending W; V's rows move along (compile-time indices only, so nothing leaves the registers)
#pragma unroll
  for (int i = 0; i < 3; i++) {
    int j = i;
    double wj = W[i];
#pragma unroll
    for (int k = i + 1; k < 4; k++) if (wj < W[k]) { j = k; wj = W[k]; }
#pragma unroll
    for (int k = i + 1; k < 4; k++) {
      if (k != j) continue;
      const double t = W[i]; W[i] = W[k]; W[k] = t;
#pragma unroll
      for (int m = 0; m < 4; m++) { const float v = V[i][m]; V[i][m] = V[k][m]; V[k][m] = v; }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    w[i] = d2f(W[i]);
#pragma unroll
    for (int k = 0; k < 4; k++) vt[4 * i + k] = V[i][k];
  }
}
}  // namespace pl
