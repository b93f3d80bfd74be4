// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_orb.cpp header for the rules).
//
// CPU restatement (fp64) of the reference's pose-only Levenberg–Marquardt:
//   Optimizer::PoseOptimization            src/Optimizer.cc:640-975
//   Optimizer::PoseOptimizationWithPoints  src/Optimizer.cc:977-1115
//   Optimizer::PoseOptimizationWithLines   src/Optimizer.cc:1117-1284
//   EdgeSE3ProjectXYZOnlyPose              Thirdparty/g2o/g2o/types/types_six_dof_expmap.{h:136-163,cpp:266-296}
//   EdgeLineProjectXYZOnlyPose             include/lineEdge.h:119-133 (numeric Jacobian: base_unary_edge.hpp:81-123)
//   OptimizationAlgorithmLevenberg::solve  Thirdparty/g2o/g2o/core/optimization_algorithm_levenberg.cpp:61-189
//   SparseOptimizer::optimize / activeRobustChi2   core/sparse_optimizer.cpp:354-419, :100-114
//   BlockSolver::buildSystem/setLambda/solve       core/block_solver.hpp:501-589, :354-365
//   BaseUnaryEdge::constructQuadraticForm          core/base_unary_edge.hpp:42-72
//   RobustKernelHuber::robustify                   core/robust_kernel_impl.cpp:78-91
//   SE3Quat (exp, map, operator*, normalizeRotation, to_homogeneous_matrix)   types/se3quat.h
//   LinearSolverDense (Eigen LDLT)                 solvers/linear_solver_dense.h:104-112
//   Converter::toSE3Quat / toCvMat                 src/Converter.cc:37-71
// Eigen (not vendored) is restated by hand: Quaterniond(Matrix3d), quaternion product, q*v, toRotationMatrix, and a
// 6x6 LDL^T without pivoting (Eigen pivots; for the SPD H+lambda*I systems here both give the solution to ~1e-12).
// Parity status: unpinned — the reference stores no expected values (SURVEY.md §4); the known-answer check is the
// testOpt.cpp recipe (ground-truth pose recovery), see tests/test_oracle_lm.py.
// g2o behaviours kept on purpose: edges keep the error of the LAST trial step even when that step was rejected
// (chi2() of inlier edges after optimize() is evaluated there); a failed factorisation keeps the previous x.

#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>
#include "se3.h"

namespace {

// 6x6 LDL^T; returns false if a pivot is not positive (LinearSolverDense: _cholesky.isPositive())
bool solve6(const double H[6][6], const double b[6], double x[6]) {
  double L[6][6] = {{0}}, D[6];
  for (int j = 0; j < 6; j++) {
    double d = H[j][j];
    for (int k = 0; k < j; k++) d -= L[j][k] * L[j][k] * D[k];
    if (!(d > 0)) return false;
    D[j] = d;
    L[j][j] = 1;
    for (int i = j + 1; i < 6; i++) {
      double s = H[i][j];
      for (int k = 0; k < j; k++) s -= L[i][k] * L[j][k] * D[k];
      L[i][j] = s / d;
    }
  }
  double y[6];
  for (int i = 0; i < 6; i++) { double s = b[i]; for (int k = 0; k < i; k++) s -= L[i][k] * y[k]; y[i] = s; }
  for (int i = 0; i < 6; i++) y[i] /= D[i];
  for (int i = 5; i >= 0; i--) { double s = y[i]; for (int k = i + 1; k < 6; k++) s -= L[k][i] * x[k]; x[i] = s; }
  return true;
}

struct Problem {
  double fx, fy, cx, cy;
  int np, nl;
  const float* pt_obs; const float* pt_w; const float* pt_X;
  const double* ln_f; const double* ln_X;
  // per-edge state
  std::vector<double> pe;        // point errors [np][2]
  std::vector<double> le;        // line endpoint errors [nl][2] (start, end), component 0 only
  std::vector<uint8_t> p_active, l_active;   // level 0
  bool p_robust, l_robust;
  // Rounding variants, for tests that need results which do not hang on the last bits of a sum (oracle_pose_optimization_ex):
  // the line Jacobians' central-difference scale (g2o's 1 / (2 * 1e-9), or the literal 5e8 that k_pose_opt uses, one ulp
  // higher), and the order the chi2 and H / b sums are formed in (sequential, or k_pose_opt's: see device_sum).
  double jac_scale = 1.0 / (2 * 1e-9);
  bool device_order = false;
};
const double kDeltaMono = (double)(float)std::sqrt(5.991);   // const float deltaMono = sqrt(5.991)
const double kDeltaLine = (double)(float)std::sqrt(3.84);

inline void huber(double e, double delta, double rho[3]) {
  double dsqr = delta * delta;
  if (e <= dsqr) { rho[0] = e; rho[1] = 1.; rho[2] = 0.; }
  else { double s = std::sqrt(e); rho[0] = 2 * s * delta - dsqr; rho[1] = delta / s; rho[2] = -0.5 * rho[1] / e; }
}
// k_pose_opt's summation order: edge i goes to thread i % 128, which adds its edges in index order (points before lines);
// v[t * n + k] holds thread t's partial k.  The CTA then reduces with butterflies inside each warp (xor 16, 8, 4, 2, 1) and adds
// the four warp totals in warp order.
constexpr int kDevThreads = 128;
void device_sum(std::vector<double>& v, int n, double* out) {
  std::vector<double> nv(v.size());
  for (int o = 16; o > 0; o >>= 1) {
    for (int t = 0; t < kDevThreads; t++) for (int k = 0; k < n; k++) nv[t * n + k] = v[t * n + k] + v[(t ^ o) * n + k];
    v.swap(nv);
  }
  for (int k = 0; k < n; k++) { double s = 0; for (int w = 0; w < kDevThreads / 32; w++) s += v[32 * w * n + k]; out[k] = s; }
}
inline void point_error(const Problem& P, const SE3& T, int i, double e[2]) {
  double X[3] = {(double)P.pt_X[3 * i], (double)P.pt_X[3 * i + 1], (double)P.pt_X[3 * i + 2]}, c[3];
  se3_map(T, X, c);
  double px = c[0] / c[2], py = c[1] / c[2];
  e[0] = (double)P.pt_obs[2 * i] - (px * P.fx + P.cx);
  e[1] = (double)P.pt_obs[2 * i + 1] - (py * P.fy + P.cy);
}
inline double line_error(const Problem& P, const SE3& T, int i, int end) {
  double c[3];
  se3_map(T, P.ln_X + 6 * i + 3 * end, c);
  double u = c[0] / c[2] * P.fx + P.cx, v = c[1] / c[2] * P.fy + P.cy;
  const double* l = P.ln_f + 3 * i;
  return l[0] * u + l[1] * v + l[2];
}
void compute_active_errors(Problem& P, const SE3& T) {
  for (int i = 0; i < P.np; i++) if (P.p_active[i]) point_error(P, T, i, &P.pe[2 * i]);
  for (int i = 0; i < P.nl; i++) if (P.l_active[i]) { P.le[2 * i] = line_error(P, T, i, 0); P.le[2 * i + 1] = line_error(P, T, i, 1); }
}
double active_robust_chi2(const Problem& P) {
  double chi = 0, rho[3];
  if (P.device_order) {
    std::vector<double> v(kDevThreads, 0.0);
    for (int i = 0; i < P.np; i++) if (P.p_active[i]) {
      double w = (double)P.pt_w[i];
      double c2 = P.pe[2 * i] * (w * P.pe[2 * i]) + P.pe[2 * i + 1] * (w * P.pe[2 * i + 1]);
      if (P.p_robust) { huber(c2, kDeltaMono, rho); v[i % kDevThreads] += rho[0]; } else v[i % kDevThreads] += c2;
    }
    for (int i = 0; i < P.nl; i++) if (P.l_active[i])
      for (int e = 0; e < 2; e++) {
        double c2 = P.le[2 * i + e] * P.le[2 * i + e];
        if (P.l_robust) { huber(c2, kDeltaLine, rho); v[i % kDevThreads] += rho[0]; } else v[i % kDevThreads] += c2;
      }
    device_sum(v, 1, &chi);
    return chi;
  }
  for (int i = 0; i < P.np; i++) if (P.p_active[i]) {
    double w = (double)P.pt_w[i];
    double c2 = P.pe[2 * i] * (w * P.pe[2 * i]) + P.pe[2 * i + 1] * (w * P.pe[2 * i + 1]);
    if (P.p_robust) { huber(c2, kDeltaMono, rho); chi += rho[0]; } else chi += c2;
  }
  for (int i = 0; i < P.nl; i++) if (P.l_active[i])
    for (int e = 0; e < 2; e++) {
      double c2 = P.le[2 * i + e] * P.le[2 * i + e];
      if (P.l_robust) { huber(c2, kDeltaLine, rho); chi += rho[0]; } else chi += c2;
    }
  return chi;
}
void build_system(const Problem& P, const SE3& T, double H[6][6], double b[6]) {
  memset(H, 0, sizeof(double) * 36);
  memset(b, 0, sizeof(double) * 6);
  double rho[3];
  std::vector<double> v(P.device_order ? kDevThreads * 27 : 0, 0.0);   // device order: per thread 21 unique H entries + 6 of b
  for (int i = 0; i < P.np; i++) if (P.p_active[i]) {
    double X[3] = {(double)P.pt_X[3 * i], (double)P.pt_X[3 * i + 1], (double)P.pt_X[3 * i + 2]}, c[3];
    se3_map(T, X, c);
    double x = c[0], y = c[1], invz = 1.0 / c[2], invz_2 = invz * invz;
    double J[2][6];
    J[0][0] = x * y * invz_2 * P.fx; J[0][1] = -(1 + (x * x * invz_2)) * P.fx; J[0][2] = y * invz * P.fx;
    J[0][3] = -invz * P.fx; J[0][4] = 0; J[0][5] = x * invz_2 * P.fx;
    J[1][0] = (1 + y * y * invz_2) * P.fy; J[1][1] = -x * y * invz_2 * P.fy; J[1][2] = -x * invz * P.fy;
    J[1][3] = 0; J[1][4] = -invz * P.fy; J[1][5] = y * invz_2 * P.fy;
    double w = (double)P.pt_w[i];
    const double* e = &P.pe[2 * i];
    double r1 = 1.0;
    if (P.p_robust) { huber(e[0] * (w * e[0]) + e[1] * (w * e[1]), kDeltaMono, rho); r1 = rho[1]; }
    if (P.device_order) {
      double* acc = &v[(size_t)(i % kDevThreads) * 27];
      int k = 0;
      for (int a = 0; a < 6; a++)
        for (int c2 = a; c2 < 6; c2++) acc[k++] += J[0][a] * (r1 * w) * J[0][c2] + J[1][a] * (r1 * w) * J[1][c2];
      for (int a = 0; a < 6; a++) acc[21 + a] -= r1 * (J[0][a] * (w * e[0]) + J[1][a] * (w * e[1]));
      continue;
    }
    for (int a = 0; a < 6; a++) {
      b[a] -= r1 * (J[0][a] * (w * e[0]) + J[1][a] * (w * e[1]));
      for (int c2 = 0; c2 < 6; c2++) H[a][c2] += J[0][a] * (r1 * w) * J[0][c2] + J[1][a] * (r1 * w) * J[1][c2];
    }
  }
  if (P.nl > 0) {
    // numeric Jacobian: central differences, delta = 1e-9, through oplus (exp(d)*T); scale 1 / (2 delta) unless a variant asks
    const double delta = 1e-9, scalar = P.jac_scale;
    SE3 Tp[6], Tm[6];
    for (int d = 0; d < 6; d++) {
      double add[6] = {0, 0, 0, 0, 0, 0};
      add[d] = delta; Tp[d] = se3_mul(se3_exp(add), T);
      add[d] = -delta; Tm[d] = se3_mul(se3_exp(add), T);
    }
    for (int i = 0; i < P.nl; i++) if (P.l_active[i])
      for (int e = 0; e < 2; e++) {
        double J[6];
        for (int d = 0; d < 6; d++) J[d] = scalar * (line_error(P, Tp[d], i, e) - line_error(P, Tm[d], i, e));
        double err = P.le[2 * i + e], r1 = 1.0;
        if (P.l_robust) { huber(err * err, kDeltaLine, rho); r1 = rho[1]; }
        if (P.device_order) {
          double* acc = &v[(size_t)(i % kDevThreads) * 27];
          int k = 0;
          for (int a = 0; a < 6; a++)
            for (int c2 = a; c2 < 6; c2++) acc[k++] += J[a] * r1 * J[c2];
          for (int a = 0; a < 6; a++) acc[21 + a] -= r1 * (J[a] * err);
          continue;
        }
        for (int a = 0; a < 6; a++) {
          b[a] -= r1 * (J[a] * err);
          for (int c2 = 0; c2 < 6; c2++) H[a][c2] += J[a] * r1 * J[c2];
        }
      }
  }
  if (P.device_order) {      // the kernel keeps the upper triangle and mirrors it
    double s[27];
    device_sum(v, 27, s);
    int k = 0;
    for (int a = 0; a < 6; a++) for (int c2 = a; c2 < 6; c2++) { H[a][c2] = s[k]; H[c2][a] = s[k]; k++; }
    for (int a = 0; a < 6; a++) b[a] = s[21 + a];
  }
}

// SparseOptimizer::optimize(iterations) with OptimizationAlgorithmLevenberg; T = vertex estimate (in/out);
// Terr = pose at which the active edges' stored errors were last evaluated.
void optimize(Problem& P, SE3& T, SE3& Terr, int iterations, int* its_done) {
  double lambda = 0, ni = 2, x[6] = {0, 0, 0, 0, 0, 0};
  int nBad = 0;
  bool any = false;
  for (int i = 0; i < P.np; i++) any |= (P.p_active[i] != 0);
  for (int i = 0; i < P.nl; i++) any |= (P.l_active[i] != 0);
  if (!any) return;  // "0 vertices to optimize": optimize() returns -1 without touching anything
  for (int it = 0; it < iterations; it++) {
    if (its_done) (*its_done)++;
    compute_active_errors(P, T); Terr = T;
    double currentChi = active_robust_chi2(P), tempChi = currentChi, iniChi = currentChi;
    double H[6][6], b[6];
    build_system(P, T, H, b);
    if (it == 0) {
      double md = 0;
      for (int j = 0; j < 6; j++) md = std::max(std::fabs(H[j][j]), md);
      lambda = 1e-5 * md; ni = 2; nBad = 0;
    }
    double rho = 0;
    int qmax = 0;
    do {
      SE3 backup = T;
      double Hl[6][6];
      memcpy(Hl, H, sizeof(Hl));
      for (int j = 0; j < 6; j++) Hl[j][j] += lambda;
      bool ok2 = solve6(Hl, b, x);
      T = se3_mul(se3_exp(x), T);
      compute_active_errors(P, T); Terr = T;
      tempChi = active_robust_chi2(P);
      if (!ok2) tempChi = std::numeric_limits<double>::max();
      rho = (currentChi - tempChi);
      double scale = 0;
      for (int j = 0; j < 6; j++) scale += x[j] * (lambda * x[j] + b[j]);
      scale += 1e-3;
      rho /= scale;
      if (rho > 0 && std::isfinite(tempChi)) {
        double alpha = 1. - std::pow((2 * rho - 1), 3);
        alpha = std::min(alpha, 2. / 3.);
        double scaleFactor = std::max(1. / 3., alpha);
        lambda *= scaleFactor; ni = 2; currentChi = tempChi;
      } else {
        lambda *= ni; ni *= 2; T = backup;
      }
      qmax++;
    } while (rho < 0 && qmax < 10);
    if (qmax == 10 || rho == 0) break;
    if ((iniChi - currentChi) * 1e3 < iniChi) nBad++; else nBad = 0;
    if (nBad >= 3) break;
  }
}
}  // namespace

// variant (0 = the reference): bit 0 = line Jacobian scale 5e8 instead of 1 / (2 * 1e-9), bit 1 = k_pose_opt's summation order.
// A problem whose result is the same under every variant does not sit on a rounding-level LM decision (DESIGN.md §5).
extern "C" int oracle_pose_optimization_ex(int mode, const float* Tcw_in, const float* K, int np, const float* pt_obs,
                                           const float* pt_inv_sigma2, const float* pt_Xw, int nl, const double* line_func,
                                           const double* line_Xw, float* Tcw_out, uint8_t* pt_outlier,
                                           uint8_t* line_outlier, int* iterations_out, int variant) {
  if (mode == 1) nl = 0;
  if (mode == 2) np = 0;
  Problem P;
  P.fx = K[0]; P.fy = K[1]; P.cx = K[2]; P.cy = K[3];
  P.np = np; P.nl = nl; P.pt_obs = pt_obs; P.pt_w = pt_inv_sigma2; P.pt_X = pt_Xw; P.ln_f = line_func; P.ln_X = line_Xw;
  P.pe.assign(2 * (size_t)np + 2, 0.0); P.le.assign(2 * (size_t)nl + 2, 0.0);
  P.p_active.assign(np + 1, 1); P.l_active.assign(nl + 1, 1);
  P.p_robust = true; P.l_robust = true;
  if (variant & 1) P.jac_scale = 5e8;
  P.device_order = (variant & 2) != 0;
  for (int i = 0; i < np; i++) pt_outlier[i] = 0;
  for (int i = 0; i < nl; i++) line_outlier[i] = 0;
  memcpy(Tcw_out, Tcw_in, 16 * sizeof(float));
  if (iterations_out) *iterations_out = 0;
  if (mode == 2 ? (nl < 3) : (np < 3)) return 0;
  const float chi2Mono = 5.991f, chi2LEnd = 3.84f;
  const SE3 T0 = se3_from_cv(Tcw_in);
  SE3 T = T0, Terr = T0;
  int nBad = 0, nLineBad = 0;
  for (int it = 0; it < 4; it++) {
    T = T0;
    optimize(P, T, Terr, 10, iterations_out);
    nBad = 0;
    for (int i = 0; i < np; i++) {
      if (pt_outlier[i]) point_error(P, T, i, &P.pe[2 * i]);  // e->computeError() at the current estimate
      double w = (double)pt_inv_sigma2[i];
      const float chi2 = (float)(P.pe[2 * i] * (w * P.pe[2 * i]) + P.pe[2 * i + 1] * (w * P.pe[2 * i + 1]));
      if (chi2 > chi2Mono) { pt_outlier[i] = 1; P.p_active[i] = 0; nBad++; }
      else { pt_outlier[i] = 0; P.p_active[i] = 1; }
    }
    if (it == 2) P.p_robust = false;
    nLineBad = 0;
    for (int i = 0; i < nl; i++) {
      if (line_outlier[i]) { P.le[2 * i] = line_error(P, T, i, 0); P.le[2 * i + 1] = line_error(P, T, i, 1); }
      const float c_s = (float)(P.le[2 * i] * P.le[2 * i]), c_e = (float)(P.le[2 * i + 1] * P.le[2 * i + 1]);
      if (c_s > chi2LEnd || c_e > chi2LEnd) { line_outlier[i] = 1; P.l_active[i] = 0; nLineBad++; }
      else { line_outlier[i] = 0; P.l_active[i] = 1; }
    }
    if (it == 2) P.l_robust = false;
    if (np + 2 * nl < 10) break;
  }
  (void)Terr;
  se3_to_cv(T, Tcw_out);
  return mode == 2 ? nl - nLineBad : np - nBad;
}

extern "C" int oracle_pose_optimization(int mode, const float* Tcw_in, const float* K, int np, const float* pt_obs,
                                        const float* pt_inv_sigma2, const float* pt_Xw, int nl, const double* line_func,
                                        const double* line_Xw, float* Tcw_out, uint8_t* pt_outlier,
                                        uint8_t* line_outlier, int* iterations_out) {
  return oracle_pose_optimization_ex(mode, Tcw_in, K, np, pt_obs, pt_inv_sigma2, pt_Xw, nl, line_func, line_Xw, Tcw_out, pt_outlier,
                                     line_outlier, iterations_out, 0);
}
