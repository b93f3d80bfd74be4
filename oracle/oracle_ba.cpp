// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_orb.cpp header for the rules).
//
// CPU restatement (fp64) of the reference's local bundle adjustment with lines:
//   Optimizer::LocalBundleAdjustmentWithLine   src/Optimizer.cc:1645-2100  (points-only twin :1308-1642 = n_le == 0)
//   EdgeSE3ProjectXYZ (analytic Jacobians)     Thirdparty/g2o/g2o/types/types_six_dof_expmap.{h:82-120,cpp:103-139}
//   EdgeLineProjectXYZ (numeric Jacobians)     include/lineEdge.h:212-232, core/base_binary_edge.hpp:130-205
//   BaseBinaryEdge::constructQuadraticForm     core/base_binary_edge.hpp:54-123
//   BlockSolver_6_3 Schur path                 core/block_solver.hpp:353-486, buildSystem :501-560, setLambda :563-589
//   OptimizationAlgorithmLevenberg             core/optimization_algorithm_levenberg.cpp:61-189
//   LinearSolverEigen (SimplicialLDLT)         solvers/linear_solver_eigen.h:94-124  -> dense LDL^T here (same solution)
//   VertexSBAPointXYZ::oplusImpl (x += dx)     types/types_sba.h
// Reference quirks reproduced literally (SURVEY.md §8a a21): end-point line edges use the CURRENT keyframe's intrinsics
// (K_end) instead of the observing keyframe's (Optimizer.cc:1939-1942); the final line check reads the START-point edge
// twice (:2030-2031) and pairs observation i with the keyframe of observation i/2 (vpLineEdgeKF is pushed twice per
// observation, :1924,1948).  Parity status: unpinned (no expected values in the reference); known-answer test =
// recovery of the ground-truth structure on synthetic windows (tests/test_oracle_ba.py).
//
// oracle_global_ba: Optimizer::BundleAdjustment with lines (src/Optimizer.cc:275-638, called by GlobalBundleAdjustemnt :41-58):
// the same graph types and the same Levenberg-Marquardt, ONE optimize(nIterations) call, no outlier rounds; Huber deltas
// sqrt(5.99) (points, :316) and sqrt(3.84) (line end points, :318) only if bRobust; line information = identity (invSigma = 1,
// :278); every line edge uses the OBSERVING keyframe's intrinsics (:472-475,526-529); edges are inserted points first, then
// all start-point edges, then all end-point edges (:321-536).

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>
#include "se3.h"

namespace {
const double kDeltaMono = (double)(float)std::sqrt(5.991);   // const float thHuberMono = sqrt(5.991)
const double kDeltaLine = (double)(float)std::sqrt(3.84);

inline void huber(double e, double delta, double& r0, double& r1) {
  double dsqr = delta * delta;
  if (e <= dsqr) { r0 = e; r1 = 1.; } else { double s = std::sqrt(e); r0 = 2 * s * delta - dsqr; r1 = delta / s; }
}
inline bool inv3(const double* D, double* Di) {  // Eigen Matrix3d::inverse(): cofactors / determinant
  const double a = D[0], b = D[1], c = D[2], d = D[3], e = D[4], f = D[5], g = D[6], h = D[7], i = D[8];
  const double A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
  const double det = a * A + b * B + c * C;
  const double id = 1.0 / det;
  Di[0] = A * id; Di[1] = -(b * i - c * h) * id; Di[2] = (b * f - c * e) * id;
  Di[3] = B * id; Di[4] = (a * i - c * g) * id; Di[5] = -(a * f - c * d) * id;
  Di[6] = C * id; Di[7] = -(a * h - b * g) * id; Di[8] = (a * e - b * d) * id;
  return std::isfinite(id);
}
bool ldlt_solve(std::vector<double>& A, int n, const double* b, double* x) {  // dense LDL^T, no pivoting
  std::vector<double> D(n);
  for (int j = 0; j < n; j++) {
    double d = A[(size_t)j * n + j];
    for (int k = 0; k < j; k++) d -= A[(size_t)j * n + k] * A[(size_t)j * n + k] * D[k];
    if (d == 0 || !std::isfinite(d)) return false;
    D[j] = d;
    for (int i = j + 1; i < n; i++) {
      double s = A[(size_t)i * n + j];
      for (int k = 0; k < j; k++) s -= A[(size_t)i * n + k] * A[(size_t)j * n + k] * D[k];
      A[(size_t)i * n + j] = s / d;
    }
  }
  std::vector<double> y(n);
  for (int i = 0; i < n; i++) { double s = b[i]; for (int k = 0; k < i; k++) s -= A[(size_t)i * n + k] * y[k]; y[i] = s; }
  for (int i = 0; i < n; i++) y[i] /= D[i];
  for (int i = n - 1; i >= 0; i--) { double s = y[i]; for (int k = i + 1; k < n; k++) s -= A[(size_t)k * n + i] * x[k]; x[i] = s; }
  return true;
}

struct BA {
  int n_kf, n_pt, n_ln, n_pe, n_le;
  std::vector<SE3> T; std::vector<uint8_t> fixed; const float* K; double Kend[4];
  std::vector<double> X;            // landmarks: points then line start/end (3 each): n_lm = n_pt + 2*n_ln
  const int *pe_kf, *pe_pt; const float *pe_obs, *pe_w;
  const int *le_kf, *le_ln; const double* le_f;
  std::vector<double> perr, lerr;   // stored errors: [n_pe][2], [n_le][2] (start,end)
  std::vector<uint8_t> p_lvl, l_lvl;   // level (1 = excluded)
  bool p_robust = true, l_robust = true;
  double info_line = 0.5;           // invSigma = 0.5 (Optimizer.cc:1647)
  double delta_p = kDeltaMono, delta_l = kDeltaLine;
  bool end_uses_Kend = true;        // local BA quirk (Optimizer.cc:1939-1942); global BA: the observing keyframe's own K
  bool start_uses_Kend = false;     // never in the reference: a deliberately wrong camera model for the tests (see oracle_local_ba)
  bool starts_first = false;        // global BA inserts all start-point edges, then all end-point edges
  volatile const int* stop = nullptr;
  int n_lm() const { return n_pt + 2 * n_ln; }
  bool terminate() const { return stop && *stop; }
};

inline void cam(const double c[3], const double* K, double& u, double& v) { u = c[0] / c[2] * K[0] + K[2]; v = c[1] / c[2] * K[1] + K[3]; }
inline void Kd(const float* K, int kf, double* o) { for (int i = 0; i < 4; i++) o[i] = (double)K[4 * kf + i]; }

void point_err(const BA& P, const SE3& T, const double* X, int e, double* out) {
  double c[3], k[4], u, v;
  se3_map(T, X, c); Kd(P.K, P.pe_kf[e], k); cam(c, k, u, v);
  out[0] = (double)P.pe_obs[2 * e] - u; out[1] = (double)P.pe_obs[2 * e + 1] - v;
}
double line_err(const BA& P, const SE3& T, const double* X, int e, int end) {
  double c[3], k[4], u, v;
  se3_map(T, X, c);
  const bool use_Kend = end == 0 ? P.start_uses_Kend : P.end_uses_Kend;
  if (!use_Kend) Kd(P.K, P.le_kf[e], k); else for (int i = 0; i < 4; i++) k[i] = P.Kend[i];
  cam(c, k, u, v);
  const double* l = P.le_f + 3 * e;
  return l[0] * u + l[1] * v + l[2];
}
inline const double* lm_point(const BA& P, int pt) { return &P.X[3 * pt]; }
inline const double* lm_line(const BA& P, int ln, int end) { return &P.X[3 * (P.n_pt + 2 * ln + end)]; }

void compute_active_errors(BA& P) {
  for (int e = 0; e < P.n_pe; e++) if (!P.p_lvl[e]) point_err(P, P.T[P.pe_kf[e]], lm_point(P, P.pe_pt[e]), e, &P.perr[2 * e]);
  for (int e = 0; e < P.n_le; e++) if (!P.l_lvl[e])
    for (int end = 0; end < 2; end++) P.lerr[2 * e + end] = line_err(P, P.T[P.le_kf[e]], lm_line(P, P.le_ln[e], end), e, end);
}
double active_chi2(const BA& P) {
  double chi = 0, r0, r1;
  for (int e = 0; e < P.n_pe; e++) if (!P.p_lvl[e]) {
    double w = (double)P.pe_w[e], c2 = P.perr[2 * e] * (w * P.perr[2 * e]) + P.perr[2 * e + 1] * (w * P.perr[2 * e + 1]);
    if (P.p_robust) { huber(c2, P.delta_p, r0, r1); chi += r0; } else chi += c2;
  }
  for (int pass = 0; pass < (P.starts_first ? 2 : 1); pass++)
    for (int e = 0; e < P.n_le; e++) if (!P.l_lvl[e])
      for (int end = (P.starts_first ? pass : 0); end < (P.starts_first ? pass + 1 : 2); end++) {
        double c2 = P.lerr[2 * e + end] * (P.info_line * P.lerr[2 * e + end]);
        if (P.l_robust) { huber(c2, P.delta_l, r0, r1); chi += r0; } else chi += c2;
      }
  return chi;
}

// normal equations in dense form over the ACTIVE free poses and ACTIVE landmarks
struct System {
  std::vector<int> pose_slot, lm_slot;       // -1 = not in the system
  int np = 0, nl = 0;
  std::vector<double> Hpp, bp;                // [np][36] diagonal blocks, [np*6]
  std::vector<double> Hll, bl;                // [nl][9], [nl*3]
  struct PL { int p, l; double B[18]; };      // Hpl block (6x3) of one edge with a free pose
  std::vector<PL> pl;
};

void build_system(BA& P, System& S) {
  const int nlm = P.n_lm();
  S.pose_slot.assign(P.n_kf, -1); S.lm_slot.assign(nlm, -1);
  std::vector<uint8_t> pa(P.n_kf, 0), la(nlm, 0);
  for (int e = 0; e < P.n_pe; e++) if (!P.p_lvl[e]) { pa[P.pe_kf[e]] = 1; la[P.pe_pt[e]] = 1; }
  for (int e = 0; e < P.n_le; e++) if (!P.l_lvl[e]) { pa[P.le_kf[e]] = 1; la[P.n_pt + 2 * P.le_ln[e]] = 1; la[P.n_pt + 2 * P.le_ln[e] + 1] = 1; }
  S.np = S.nl = 0;
  for (int k = 0; k < P.n_kf; k++) if (pa[k] && !P.fixed[k]) S.pose_slot[k] = S.np++;
  for (int l = 0; l < nlm; l++) if (la[l]) S.lm_slot[l] = S.nl++;
  S.Hpp.assign((size_t)S.np * 36, 0); S.bp.assign((size_t)S.np * 6, 0);
  S.Hll.assign((size_t)S.nl * 9, 0); S.bl.assign((size_t)S.nl * 3, 0);
  S.pl.clear();
  // perturbed poses for the numeric (line) Jacobians
  std::vector<SE3> Tp, Tm;
  if (P.n_le > 0) {
    Tp.resize((size_t)P.n_kf * 6); Tm.resize((size_t)P.n_kf * 6);
    for (int k = 0; k < P.n_kf; k++)
      for (int d = 0; d < 6; d++) {
        double add[6] = {0, 0, 0, 0, 0, 0};
        add[d] = 1e-9; Tp[(size_t)k * 6 + d] = se3_mul(se3_exp(add), P.T[k]);
        add[d] = -1e-9; Tm[(size_t)k * 6 + d] = se3_mul(se3_exp(add), P.T[k]);
      }
  }
  auto accumulate = [&](int kf, int lm, const double* A /*D x 3*/, const double* B /*D x 6*/, const double* omega_r, double wgt, int D) {
    // from = landmark (A), to = pose (B); weightedOmega = wgt * I_D (information is a multiple of identity)
    const int ls = S.lm_slot[lm], ps = S.pose_slot[kf];
    for (int a = 0; a < 3; a++) {
      double s = 0; for (int d = 0; d < D; d++) s += A[d * 3 + a] * omega_r[d];
      S.bl[(size_t)ls * 3 + a] += s;
      for (int c = 0; c < 3; c++) { double h = 0; for (int d = 0; d < D; d++) h += A[d * 3 + a] * wgt * A[d * 3 + c]; S.Hll[(size_t)ls * 9 + a * 3 + c] += h; }
    }
    if (ps >= 0) {
      for (int a = 0; a < 6; a++) {
        double s = 0; for (int d = 0; d < D; d++) s += B[d * 6 + a] * omega_r[d];
        S.bp[(size_t)ps * 6 + a] += s;
        for (int c = 0; c < 6; c++) { double h = 0; for (int d = 0; d < D; d++) h += B[d * 6 + a] * wgt * B[d * 6 + c]; S.Hpp[(size_t)ps * 36 + a * 6 + c] += h; }
      }
      System::PL blk; blk.p = ps; blk.l = ls;
      for (int a = 0; a < 6; a++) for (int c = 0; c < 3; c++) { double h = 0; for (int d = 0; d < D; d++) h += B[d * 6 + a] * wgt * A[d * 3 + c]; blk.B[a * 3 + c] = h; }
      S.pl.push_back(blk);
    }
  };
  double r0, r1;
  for (int e = 0; e < P.n_pe; e++) if (!P.p_lvl[e]) {
    const int kf = P.pe_kf[e];
    const SE3& T = P.T[kf];
    double c[3], k[4], R[3][3];
    se3_map(T, lm_point(P, P.pe_pt[e]), c); Kd(P.K, kf, k); quat_to_matrix(T.r, R);
    const double x = c[0], y = c[1], z = c[2], z_2 = z * z, fx = k[0], fy = k[1];
    double tmp[2][3] = {{fx, 0, -x / z * fx}, {0, fy, -y / z * fy}}, A[6], B[12];
    for (int i = 0; i < 2; i++) for (int j = 0; j < 3; j++) { double s = 0; for (int m = 0; m < 3; m++) s += tmp[i][m] * R[m][j]; A[i * 3 + j] = -1. / z * s; }
    B[0] = x * y / z_2 * fx; B[1] = -(1 + (x * x / z_2)) * fx; B[2] = y / z * fx; B[3] = -1. / z * fx; B[4] = 0; B[5] = x / z_2 * fx;
    B[6] = (1 + y * y / z_2) * fy; B[7] = -x * y / z_2 * fy; B[8] = -x / z * fy; B[9] = 0; B[10] = -1. / z * fy; B[11] = y / z_2 * fy;
    const double w = (double)P.pe_w[e], e0 = P.perr[2 * e], e1 = P.perr[2 * e + 1];
    double omr[2] = {-(w * e0), -(w * e1)}, wgt = w;
    if (P.p_robust) { huber(e0 * (w * e0) + e1 * (w * e1), P.delta_p, r0, r1); omr[0] *= r1; omr[1] *= r1; wgt = r1 * w; }
    accumulate(kf, P.pe_pt[e], A, B, omr, wgt, 2);
  }
  for (int pass = 0; pass < (P.starts_first ? 2 : 1); pass++)
  for (int e = 0; e < P.n_le; e++) if (!P.l_lvl[e])
    for (int end = (P.starts_first ? pass : 0); end < (P.starts_first ? pass + 1 : 2); end++) {
      const int kf = P.le_kf[e], lm = P.n_pt + 2 * P.le_ln[e] + end;
      const double* X = &P.X[3 * lm];
      double A[3], B[6];   // only error component 0 is non-constant
      for (int d = 0; d < 3; d++) {
        double Xp[3] = {X[0], X[1], X[2]}, Xm[3] = {X[0], X[1], X[2]};
        Xp[d] += 1e-9; Xm[d] += -1e-9;
        A[d] = 5e8 * (line_err(P, P.T[kf], Xp, e, end) - line_err(P, P.T[kf], Xm, e, end));
      }
      for (int d = 0; d < 6; d++) B[d] = 5e8 * (line_err(P, Tp[(size_t)kf * 6 + d], X, e, end) - line_err(P, Tm[(size_t)kf * 6 + d], X, e, end));
      const double er = P.lerr[2 * e + end], w = P.info_line;
      double omr[1] = {-(w * er)}, wgt = w;
      if (P.l_robust) { huber(er * (w * er), P.delta_l, r0, r1); omr[0] *= r1; wgt = r1 * w; }
      accumulate(kf, lm, A, B, omr, wgt, 1);
    }
}

// BlockSolver::solve (Schur) with H + lambda on every diagonal; x = [poses (np*6) | landmarks (nl*3)]
bool solve_system(const System& S, double lambda, std::vector<double>& x) {
  const int n = S.np * 6;
  std::vector<double> Hs((size_t)n * n, 0.0), bs(S.bp), Dinv((size_t)S.nl * 9), Dinvb((size_t)S.nl * 3);
  for (int p = 0; p < S.np; p++)
    for (int a = 0; a < 6; a++) for (int c = 0; c < 6; c++) Hs[(size_t)(p * 6 + a) * n + p * 6 + c] = S.Hpp[(size_t)p * 36 + a * 6 + c] + (a == c ? lambda : 0.0);
  for (int l = 0; l < S.nl; l++) {
    double D[9];
    for (int i = 0; i < 9; i++) D[i] = S.Hll[(size_t)l * 9 + i];
    D[0] += lambda; D[4] += lambda; D[8] += lambda;
    inv3(D, &Dinv[(size_t)l * 9]);
    for (int a = 0; a < 3; a++) Dinvb[(size_t)l * 3 + a] = Dinv[(size_t)l * 9 + a * 3] * S.bl[(size_t)l * 3] + Dinv[(size_t)l * 9 + a * 3 + 1] * S.bl[(size_t)l * 3 + 1] + Dinv[(size_t)l * 9 + a * 3 + 2] * S.bl[(size_t)l * 3 + 2];
  }
  // group pose-landmark blocks by landmark
  std::vector<std::vector<int>> by_l(S.nl);
  for (int i = 0; i < (int)S.pl.size(); i++) by_l[S.pl[i].l].push_back(i);
  for (int l = 0; l < S.nl; l++) {
    // several edges may connect the same (pose, landmark) pair: g2o sums them into one Hpl block first
    std::vector<int> poses; std::vector<std::vector<double>> blocks;
    for (int i : by_l[l]) {
      int p = S.pl[i].p, at = -1;
      for (size_t q = 0; q < poses.size(); q++) if (poses[q] == p) at = (int)q;
      if (at < 0) { poses.push_back(p); blocks.emplace_back(S.pl[i].B, S.pl[i].B + 18); }
      else for (int t = 0; t < 18; t++) blocks[at][t] += S.pl[i].B[t];
    }
    const double* Di = &Dinv[(size_t)l * 9];
    for (size_t i1 = 0; i1 < poses.size(); i1++) {
      const double* Bi = blocks[i1].data();
      double BD[18];
      for (int a = 0; a < 6; a++) for (int c = 0; c < 3; c++) BD[a * 3 + c] = Bi[a * 3] * Di[c] + Bi[a * 3 + 1] * Di[3 + c] + Bi[a * 3 + 2] * Di[6 + c];
      for (int a = 0; a < 6; a++) bs[(size_t)poses[i1] * 6 + a] -= Bi[a * 3] * Dinvb[(size_t)l * 3] + Bi[a * 3 + 1] * Dinvb[(size_t)l * 3 + 1] + Bi[a * 3 + 2] * Dinvb[(size_t)l * 3 + 2];
      for (size_t i2 = 0; i2 < poses.size(); i2++) {
        const double* Bj = blocks[i2].data();
        for (int a = 0; a < 6; a++) for (int c = 0; c < 6; c++)
          Hs[(size_t)(poses[i1] * 6 + a) * n + poses[i2] * 6 + c] -= BD[a * 3] * Bj[c * 3] + BD[a * 3 + 1] * Bj[c * 3 + 1] + BD[a * 3 + 2] * Bj[c * 3 + 2];
      }
    }
  }
  x.assign((size_t)n + (size_t)S.nl * 3, 0.0);
  if (n > 0 && !ldlt_solve(Hs, n, bs.data(), x.data())) return false;
  std::vector<double> cl(S.bl);
  for (const System::PL& b : S.pl)
    for (int c = 0; c < 3; c++) { double s = 0; for (int a = 0; a < 6; a++) s += b.B[a * 3 + c] * x[(size_t)b.p * 6 + a]; cl[(size_t)b.l * 3 + c] -= s; }
  for (int l = 0; l < S.nl; l++)
    for (int a = 0; a < 3; a++) x[(size_t)n + l * 3 + a] = Dinv[(size_t)l * 9 + a * 3] * cl[(size_t)l * 3] + Dinv[(size_t)l * 9 + a * 3 + 1] * cl[(size_t)l * 3 + 1] + Dinv[(size_t)l * 9 + a * 3 + 2] * cl[(size_t)l * 3 + 2];
  return true;
}

int optimize(BA& P, int iterations) {
  double lambda = 0, ni = 2;
  int nBad = 0, done = 0;
  System S;
  std::vector<double> x;
  for (int it = 0; it < iterations && !P.terminate(); it++) {
    done++;
    compute_active_errors(P);
    double currentChi = active_chi2(P), tempChi = currentChi, iniChi = currentChi;
    build_system(P, S);
    if (S.np + S.nl == 0) return done;
    if (it == 0) {
      double md = 0;
      for (int p = 0; p < S.np; p++) for (int j = 0; j < 6; j++) md = std::max(std::fabs(S.Hpp[(size_t)p * 36 + j * 7]), md);
      for (int l = 0; l < S.nl; l++) for (int j = 0; j < 3; j++) md = std::max(std::fabs(S.Hll[(size_t)l * 9 + j * 4]), md);
      lambda = 1e-5 * md; ni = 2; nBad = 0;
      x.assign((size_t)S.np * 6 + (size_t)S.nl * 3, 0.0);
    }
    double rho = 0;
    int qmax = 0;
    do {
      std::vector<SE3> Tb = P.T; std::vector<double> Xb = P.X;
      std::vector<double> xn;
      bool ok2 = solve_system(S, lambda, xn);
      if (ok2) x = xn;
      for (int k = 0; k < P.n_kf; k++) if (S.pose_slot[k] >= 0) P.T[k] = se3_mul(se3_exp(&x[(size_t)S.pose_slot[k] * 6]), P.T[k]);
      for (int l = 0; l < P.n_lm(); l++) if (S.lm_slot[l] >= 0) for (int a = 0; a < 3; a++) P.X[3 * l + a] += x[(size_t)S.np * 6 + (size_t)S.lm_slot[l] * 3 + a];
      compute_active_errors(P);
      tempChi = active_chi2(P);
      if (!ok2) tempChi = std::numeric_limits<double>::max();
      rho = currentChi - tempChi;
      double scale = 0;
      for (int p = 0; p < S.np * 6; p++) scale += x[p] * (lambda * x[p] + S.bp[p]);
      for (int l = 0; l < S.nl * 3; l++) scale += x[(size_t)S.np * 6 + l] * (lambda * x[(size_t)S.np * 6 + l] + S.bl[l]);
      scale += 1e-3;
      rho /= scale;
      if (rho > 0 && std::isfinite(tempChi)) {
        double alpha = 1. - std::pow((2 * rho - 1), 3);
        alpha = std::min(alpha, 2. / 3.);
        lambda *= std::max(1. / 3., alpha); ni = 2; currentChi = tempChi;
      } else { lambda *= ni; ni *= 2; P.T = Tb; P.X = Xb; }
      qmax++;
    } while (rho < 0 && qmax < 10 && !P.terminate());
    if (qmax == 10 || rho == 0) break;
    if ((iniChi - currentChi) * 1e3 < iniChi) nBad++; else nBad = 0;
    if (nBad >= 3) break;
  }
  return done;
}
}  // namespace

extern "C" int oracle_local_ba(int n_kf, const float* kf_Tcw, const uint8_t* kf_fixed, const float* kf_K, const float* K_end,
                               int n_pt, const float* pt_Xw, int n_ln, const double* ln_Xw, int n_pe, const int* pe_kf,
                               const int* pe_pt, const float* pe_obs, const float* pe_inv_sigma2, int n_le, const int* le_kf,
                               const int* le_ln, const double* le_func, const int* stop_flag, float* kf_Tcw_out,
                               float* pt_Xw_out, double* ln_Xw_out, uint8_t* pe_erase, uint8_t* le_erase, int* le_erase_kf,
                               int* iterations_out, int line_cameras, double* gate_gap) {
  // line_cameras: 0 = the reference (start points: observing keyframe's K, end points: K_end).  The tests' "wrong camera"
  // models, which an implementation must be told apart from: 1 = end points with the observing K, 2 = start points with K_end.
  // gate_gap (may be NULL): the smallest relative distance |chi2 - gate| / gate of any edge from its chi2 gate (5.991 points,
  // 3.84 line end points) at the two classifications; an implementation that sums in another order can only agree on the
  // masks if this is well above rounding level.
  BA P;
  P.n_kf = n_kf; P.n_pt = n_pt; P.n_ln = n_ln; P.n_pe = n_pe; P.n_le = n_le;
  P.T.resize(n_kf); P.fixed.assign(kf_fixed, kf_fixed + n_kf); P.K = kf_K;
  for (int i = 0; i < 4; i++) P.Kend[i] = (double)K_end[i];
  P.end_uses_Kend = line_cameras != 1; P.start_uses_Kend = line_cameras == 2;
  for (int k = 0; k < n_kf; k++) P.T[k] = se3_from_cv(kf_Tcw + 16 * k);
  P.X.resize((size_t)3 * (n_pt + 2 * n_ln));
  for (int i = 0; i < 3 * n_pt; i++) P.X[i] = (double)pt_Xw[i];
  for (int i = 0; i < 6 * n_ln; i++) P.X[3 * n_pt + i] = ln_Xw[i];
  P.pe_kf = pe_kf; P.pe_pt = pe_pt; P.pe_obs = pe_obs; P.pe_w = pe_inv_sigma2; P.le_kf = le_kf; P.le_ln = le_ln; P.le_f = le_func;
  P.perr.assign((size_t)2 * n_pe + 2, 0); P.lerr.assign((size_t)2 * n_le + 2, 0);
  P.p_lvl.assign(n_pe + 1, 0); P.l_lvl.assign(n_le + 1, 0);
  P.stop = stop_flag;
  int its = 0;
  double gap = std::numeric_limits<double>::infinity();
  auto near = [&](double c2, double gate) { gap = std::min(gap, std::fabs(c2 - gate) / gate); };
  if (!(stop_flag && *stop_flag)) {
    its += optimize(P, 5);
    bool more = !(stop_flag && *stop_flag);
    if (more) {
      for (int e = 0; e < n_pe; e++) {
        double w = (double)pe_inv_sigma2[e], c2 = P.perr[2 * e] * (w * P.perr[2 * e]) + P.perr[2 * e + 1] * (w * P.perr[2 * e + 1]);
        double c[3]; se3_map(P.T[pe_kf[e]], lm_point(P, pe_pt[e]), c);
        if (c2 > 5.991 || !(c[2] > 0.0)) P.p_lvl[e] = 1;
        near(c2, 5.991);
      }
      P.p_robust = false;
      for (int e = 0; e < n_le; e++) {
        double c1 = P.lerr[2 * e] * (P.info_line * P.lerr[2 * e]), c2 = P.lerr[2 * e + 1] * (P.info_line * P.lerr[2 * e + 1]);
        if (c1 > 3.84 || c2 > 3.84) P.l_lvl[e] = 1;
        near(c1, 3.84); near(c2, 3.84);
      }
      P.l_robust = false;
      its += optimize(P, 10);
    }
    for (int e = 0; e < n_pe; e++) {
      double w = (double)pe_inv_sigma2[e], c2 = P.perr[2 * e] * (w * P.perr[2 * e]) + P.perr[2 * e + 1] * (w * P.perr[2 * e + 1]);
      double c[3]; se3_map(P.T[pe_kf[e]], lm_point(P, pe_pt[e]), c);
      pe_erase[e] = (c2 > 5.991 || !(c[2] > 0.0)) ? 1 : 0;
      near(c2, 5.991);
    }
    for (int e = 0; e < n_le; e++) {
      double c1 = P.lerr[2 * e] * (P.info_line * P.lerr[2 * e]);   // e1 and e2 both read the START-point edge (:2030-2031)
      le_erase[e] = (c1 > 3.84) ? 1 : 0;
      near(c1, 3.84);
      le_erase_kf[e] = le_kf[e / 2];                                // vpLineEdgeKF[i] with the double push (:1924,1948)
    }
  } else {
    memset(pe_erase, 0, n_pe); memset(le_erase, 0, n_le);
    for (int e = 0; e < n_le; e++) le_erase_kf[e] = le_kf[e / 2];
  }
  for (int k = 0; k < n_kf; k++) {
    if (kf_fixed[k] || its == 0) memcpy(kf_Tcw_out + 16 * k, kf_Tcw + 16 * k, 64);   // fixed / never optimised: untouched
    else se3_to_cv(P.T[k], kf_Tcw_out + 16 * k);
  }
  for (int i = 0; i < 3 * n_pt; i++) pt_Xw_out[i] = (float)P.X[i];
  for (int i = 0; i < 6 * n_ln; i++) ln_Xw_out[i] = (double)(float)P.X[3 * n_pt + i];   // via Converter::toCvMat (float) -> Vector6d
  if (iterations_out) *iterations_out = its;
  if (gate_gap) *gate_gap = gap;
  return 0;
}

extern "C" int oracle_global_ba(int n_kf, const float* kf_Tcw, const uint8_t* kf_fixed, const float* kf_K, int n_pt, const float* pt_Xw,
                                int n_ln, const double* ln_Xw, int n_pe, const int* pe_kf, const int* pe_pt, const float* pe_obs,
                                const float* pe_inv_sigma2, int n_le, const int* le_kf, const int* le_ln, const double* le_func,
                                int n_iterations, int robust, const int* stop_flag, float* kf_Tcw_out, float* pt_Xw_out, double* ln_Xw_out,
                                int* iterations_out) {
  BA P;
  P.n_kf = n_kf; P.n_pt = n_pt; P.n_ln = n_ln; P.n_pe = n_pe; P.n_le = n_le;
  P.T.resize(n_kf); P.fixed.assign(kf_fixed, kf_fixed + n_kf); P.K = kf_K;
  for (int i = 0; i < 4; i++) P.Kend[i] = 0;
  for (int k = 0; k < n_kf; k++) P.T[k] = se3_from_cv(kf_Tcw + 16 * k);
  P.X.resize((size_t)3 * (n_pt + 2 * n_ln));
  for (int i = 0; i < 3 * n_pt; i++) P.X[i] = (double)pt_Xw[i];
  for (int i = 0; i < 6 * n_ln; i++) P.X[3 * n_pt + i] = ln_Xw[i];
  P.pe_kf = pe_kf; P.pe_pt = pe_pt; P.pe_obs = pe_obs; P.pe_w = pe_inv_sigma2; P.le_kf = le_kf; P.le_ln = le_ln; P.le_f = le_func;
  P.perr.assign((size_t)2 * n_pe + 2, 0); P.lerr.assign((size_t)2 * n_le + 2, 0);
  P.p_lvl.assign(n_pe + 1, 0); P.l_lvl.assign(n_le + 1, 0);
  P.stop = stop_flag;
  P.p_robust = P.l_robust = robust != 0;
  P.info_line = 1.0;
  P.delta_p = (double)(float)std::sqrt(5.99); P.delta_l = (double)(float)std::sqrt(3.84);
  P.end_uses_Kend = false; P.starts_first = true;
  const int its = optimize(P, n_iterations);
  // landmarks without any observation are not part of the graph (vbNotIncludedMP, :411-416): their input comes back
  std::vector<uint8_t> seen((size_t)n_pt + 2 * n_ln + 1, 0);
  for (int e = 0; e < n_pe; e++) seen[pe_pt[e]] = 1;
  for (int e = 0; e < n_le; e++) { seen[n_pt + 2 * le_ln[e]] = 1; seen[n_pt + 2 * le_ln[e] + 1] = 1; }
  for (int k = 0; k < n_kf; k++) se3_to_cv(P.T[k], kf_Tcw_out + 16 * k);      // every keyframe gets SetPose(toCvMat(estimate)) (:549-556)
  for (int i = 0; i < n_pt; i++) for (int a = 0; a < 3; a++) pt_Xw_out[3 * i + a] = seen[i] ? (float)P.X[3 * i + a] : pt_Xw[3 * i + a];
  for (int i = 0; i < 6 * n_ln; i++) ln_Xw_out[i] = (double)(float)P.X[3 * n_pt + i];
  if (iterations_out) *iterations_out = its;
  return 0;
}
