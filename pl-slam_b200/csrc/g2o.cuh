// The g2o model the three optimisers evaluate, each formula once: lm.cu (pose-only LM, one CTA per frame), ba.cu (local BA,
// one CTA per window) and gba.cu (global BA, one grid-wide kernel per phase) differ only in how they drive these.
// Edges: EdgeSE3ProjectXYZ (Thirdparty/g2o/g2o/types/types_six_dof_expmap.h:90-94, .cpp:103-147) and EdgeLineProjectXYZ /
// EdgeLineProjectXYZOnlyPose (include/lineEdge.h:119-133,212-232) with g2o's numeric Jacobians (core/base_binary_edge.hpp:130-205,
// core/base_unary_edge.hpp:42-123); RobustKernelHuber (core/robust_kernel_impl.cpp:78-91); the blocks of BlockSolver_6_3
// (core/block_solver.hpp:353-486); OptimizationAlgorithmLevenberg's step control (core/optimization_algorithm_levenberg.cpp:61-189).
//
// The library builds with -fmad=false and these are bit-exact restatements: every expression keeps its operand order.
#pragma once
#include "se3.cuh"
namespace pl {

// Huber deltas: sqrt of the chi2 thresholds, held in a float as the reference declares them.
__host__ __device__ __forceinline__ double huber_delta_mono() { return (double)(float)sqrt(5.991); }  // Optimizer.cc:676,1013,1432
__host__ __device__ __forceinline__ double huber_delta_line() { return (double)(float)sqrt(3.84); }   // Optimizer.cc:318,678,1138,1434
__host__ __device__ __forceinline__ double huber_delta_gba() { return (double)(float)sqrt(5.99); }    // BundleAdjustment, Optimizer.cc:316

// RobustKernelHuber::robustify: rho0 = rho(e), rho1 = rho'(e) of the squared error e
__device__ __forceinline__ void huber(double e, double delta, double& rho0, double& rho1) {
  double dsqr = delta * delta;
  if (e <= dsqr) { rho0 = e; rho1 = 1.; }
  else { double s = sqrt(e); rho0 = 2 * s * delta - dsqr; rho1 = delta / s; }
}

// ---- point edge.  k = fx fy cx cy
// EdgeSE3ProjectXYZ::computeError: obs - cam_project(T X)
__device__ __forceinline__ void proj_error(const SE3& T, const double* X, const double k[4], double obs0, double obs1, double& e0, double& e1) {
  double c[3];
  se3_map(T, X, c);
  e0 = obs0 - (c[0] / c[2] * k[0] + k[2]);
  e1 = obs1 - (c[1] / c[2] * k[1] + k[3]);
}
// EdgeSE3ProjectXYZ::linearizeOplus: JA = d e / d X (2x3), JB = d e / d pose (2x6), both row-major
__device__ __forceinline__ void proj_jacobians(const SE3& T, const double* X, const double k[4], double* JA, double* JB) {
  double c[3], R[3][3];
  se3_map(T, X, c); quat_to_matrix(T.r, R);
  const double x = c[0], y = c[1], z = c[2], z_2 = z * z, fx = k[0], fy = k[1];
  const double t00 = fx, t02 = -x / z * fx, t11 = fy, t12 = -y / z * fy;
  for (int j = 0; j < 3; j++) {
    JA[j] = -1. / z * (t00 * R[0][j] + t02 * R[2][j]);
    JA[3 + j] = -1. / z * (t11 * R[1][j] + t12 * R[2][j]);
  }
  JB[0] = x * y / z_2 * fx; JB[1] = -(1 + (x * x / z_2)) * fx; JB[2] = y / z * fx; JB[3] = -1. / z * fx; JB[4] = 0; JB[5] = x / z_2 * fx;
  JB[6] = (1 + y * y / z_2) * fy; JB[7] = -x * y / z_2 * fy; JB[8] = -x / z * fy; JB[9] = 0; JB[10] = -1. / z * fy; JB[11] = y / z_2 * fy;
}

// ---- line edge: one end point X of a map line against the observed line function f (a b c)
// EdgeLineProjectXYZ::computeError: f . (cam_project(T X), 1)
__device__ __forceinline__ double line_error(const SE3& T, const double* X, const double k[4], const double* f) {
  double c[3];
  se3_map(T, X, c);
  const double u = c[0] / c[2] * k[0] + k[2], v = c[1] / c[2] * k[1] + k[3];
  return f[0] * u + f[1] * v + f[2];
}
// The poses g2o's numeric Jacobian evaluates: r = 2d + s -> exp(+-1e-9 e_d) * T (s = 0: +, s = 1: -), d = 0..5
__device__ __forceinline__ SE3 perturbed_pose(const SE3& T, int r) {
  double add[6] = {0, 0, 0, 0, 0, 0};
  add[r >> 1] = (r & 1) ? -1e-9 : 1e-9;
  return se3_mul(se3_exp(add), T);
}
// Central differences, scale 1 / (2 * 1e-9) written as the literal 5e8 (one ulp above g2o's computed scalar; DESIGN §5).
// The 6 pose columns, from the perturbed poses Tp[d] (+) and Tm[d] (-)
__device__ __forceinline__ void line_pose_jacobian(const SE3* Tp, const SE3* Tm, const double* X, const double k[4], const double* f, double* J) {
#pragma unroll 1
  for (int d = 0; d < 6; d++) J[d] = 5e8 * (line_error(Tp[d], X, k, f) - line_error(Tm[d], X, k, f));
}
// The 3 landmark columns
__device__ __forceinline__ void line_point_jacobian(const SE3& T, const double* X, const double k[4], const double* f, double* J) {
  for (int d = 0; d < 3; d++) {
    double Xp[3] = {X[0], X[1], X[2]}, Xm[3] = {X[0], X[1], X[2]};
    Xp[d] += 1e-9; Xm[d] += -1e-9;
    J[d] = 5e8 * (line_error(T, Xp, k, f) - line_error(T, Xm, k, f));
  }
}

// ---- quadratic form (BaseBinaryEdge::constructQuadraticForm) of an edge of dimension dim (2 point, 1 line) with scalar
// information w and error e: omr = -rho' w e, wgt = rho' w (rho' = 1 without a robust kernel)
__device__ __forceinline__ void edge_weights(int dim, double w, const double* e, bool robust, double delta, double omr[2], double& wgt) {
  const double e0 = e[0], e1 = dim == 2 ? e[1] : 0.0;
  omr[0] = -(w * e0); omr[1] = dim == 2 ? -(w * e1) : 0.0; wgt = w;
  if (robust) {
    double r0, r1;
    huber(dim == 2 ? e0 * (w * e0) + e1 * (w * e1) : e0 * (w * e0), delta, r0, r1);
    omr[0] *= r1; if (dim == 2) omr[1] *= r1; wgt = r1 * w;
  }
}
// Landmark block of one edge: H (3x3) += JA^T wgt JA, b (3) += JA^T omr
__device__ __forceinline__ void add_landmark_block(int dim, const double* JA, const double* omr, double wgt, double* H, double* b) {
  for (int a = 0; a < 3; a++) {
    double s = 0;
    for (int d = 0; d < dim; d++) s += JA[d * 3 + a] * omr[d];
    b[a] += s;
    for (int c = 0; c < 3; c++) { double h = 0; for (int d = 0; d < dim; d++) h += JA[d * 3 + a] * wgt * JA[d * 3 + c]; H[a * 3 + c] += h; }
  }
}
// Pose block of one edge: acc[0..21) += the upper triangle of JB^T wgt JB (row-major), acc[21..27) += JB^T omr
__device__ __forceinline__ void add_pose_block(int dim, const double* JB, const double* omr, double wgt, double* acc) {
  int q = 0;
  for (int a = 0; a < 6; a++)
    for (int c = a; c < 6; c++) { double h = 0; for (int d = 0; d < dim; d++) h += JB[d * 6 + a] * wgt * JB[d * 6 + c]; acc[q++] += h; }
  for (int a = 0; a < 6; a++) { double s = 0; for (int d = 0; d < dim; d++) s += JB[d * 6 + a] * omr[d]; acc[21 + a] += s; }
}
// Hpl of one edge, W (6x3) = JB^T wgt JA: entry (a, c), and the whole block
__device__ __forceinline__ double hpl_entry(int dim, const double* JA, const double* JB, double wgt, int a, int c) {
  double h = 0;
  for (int d = 0; d < dim; d++) h += JB[d * 6 + a] * wgt * JA[d * 3 + c];
  return h;
}
__device__ __forceinline__ void hpl_block(int dim, const double* JA, const double* JB, double wgt, double* W) {
  for (int a = 0; a < 6; a++)
    for (int c = 0; c < 3; c++) W[a * 3 + c] = hpl_entry(dim, JA, JB, wgt, a, c);
}
// (D + lambda I)^-1 of a landmark block D (3x3, row-major) by cofactors
__device__ __forceinline__ void inv3(const double* D, double lambda, double* Di) {
  const double a = D[0] + lambda, b = D[1], c = D[2], d = D[3], e = D[4] + lambda, f = D[5], g = D[6], h = D[7], i = D[8] + lambda;
  const double A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
  const double id = 1.0 / (a * A + b * B + c * C);
  Di[0] = A * id; Di[1] = -(b * i - c * h) * id; Di[2] = (b * f - c * e) * id;
  Di[3] = B * id; Di[4] = (a * i - c * g) * id; Di[5] = -(a * f - c * d) * id;
  Di[6] = C * id; Di[7] = -(a * h - b * g) * id; Di[8] = (a * e - b * d) * id;
}

// ---- Levenberg-Marquardt step control (OptimizationAlgorithmLevenberg::solve), on the host for the global BA.
// First iteration: lambda = tau * the largest |diagonal entry| of H, tau = 1e-5 (computeLambdaInit, :166-180)
__host__ __device__ __forceinline__ void lm_init(double max_diag, double& lambda, double& ni, int& nBad) {
  lambda = 1e-5 * max_diag; ni = 2; nBad = 0;
}
// One trial (:119-148): chi is the trial's chi2 (ignored unless solved), xlxb = x^T (lambda x + b).  Returns the gain ratio rho.
// The step is kept iff rho > 0 and the trial's chi2 is finite; then currentChi becomes that chi2, else the caller restores the
// state from before the step.
__host__ __device__ __forceinline__ double lm_trial(bool solved, double chi, double xlxb, double& lambda, double& ni, double& currentChi,
                                                    bool& kept) {
  const double tempChi = solved ? chi : 1.7976931348623157e308;
  const double rho = (currentChi - tempChi) / (xlxb + 1e-3);
  kept = rho > 0 && isfinite(tempChi);
  if (kept) {
    double alpha = 1. - pow((2 * rho - 1), 3.0);
    alpha = fmin(alpha, 2. / 3.);
    lambda *= fmax(1. / 3., alpha); ni = 2; currentChi = tempChi;
  } else {
    lambda *= ni; ni *= 2;
  }
  return rho;
}
// After the trials (:151-161, with the reference's added rule: stop after three iterations in a row that lower chi2 by under
// a thousandth).  trials = the trials run, rho = the last one's gain ratio.
__host__ __device__ __forceinline__ bool lm_stop(int trials, double rho, double iniChi, double currentChi, int& nBad) {
  if (trials == 10 || rho == 0) return true;
  if ((iniChi - currentChi) * 1e3 < iniChi) nBad++; else nBad = 0;
  return nBad >= 3;
}
}  // namespace pl
