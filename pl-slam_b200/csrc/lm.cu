// Pose-only Levenberg–Marquardt for batches of frames on sm_90a (fp64).
//
// Replaces Optimizer::PoseOptimization / PoseOptimizationWithPoints / PoseOptimizationWithLines
// (reference src/Optimizer.cc:640-1284) and the g2o machinery they drive: OptimizationAlgorithmLevenberg::solve
// (Thirdparty/g2o/g2o/core/optimization_algorithm_levenberg.cpp:61-189), BlockSolver::buildSystem/setLambda/solve
// (core/block_solver.hpp:354-365,501-589), BaseUnaryEdge::constructQuadraticForm / numeric linearizeOplus
// (core/base_unary_edge.hpp:42-123), RobustKernelHuber (core/robust_kernel_impl.cpp:78-91), SE3Quat
// (types/se3quat.h), EdgeSE3ProjectXYZOnlyPose (types/types_six_dof_expmap.cpp:266-296),
// EdgeLineProjectXYZOnlyPose (include/lineEdge.h:119-133), LinearSolverDense (solvers/linear_solver_dense.h).
//
// One CTA (128 threads) per problem; grid = number of problems in the batch.  Per LM iteration every thread
// linearises its edges (analytic 2x6 for points; central differences, delta=1e-9, through exp(d)*T for line
// end-points exactly like g2o's numeric Jacobian — the 12 perturbed poses are built once per iteration by 12
// threads), accumulates its share of J^T W J (21 unique entries) and J^T W r (6) in registers, and the CTA reduces
// them with warp shuffles + one shared-memory hop.  Thread 0 factorises the 6x6 system (LDL^T), applies the LM
// step-control logic and broadcasts the decision.  No graph objects, no per-edge allocation, no virtual calls.

#include "common.cuh"
#include "g2o.cuh"
#include <vector>

namespace pl {

__device__ bool solve6(const double* H /*6x6 row-major*/, const double* b, double lambda, double* x) {
  double L[6][6], D[6];
  for (int j = 0; j < 6; j++) {
    double d = H[j * 6 + j] + lambda;
    for (int k = 0; k < j; k++) d -= L[j][k] * L[j][k] * D[k];
    if (!(d > 0)) return false;
    D[j] = d;
    for (int i = j + 1; i < 6; i++) {
      double s = H[i * 6 + j];
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
struct PoseArgs {
  int mode;                       // 0 points+lines, 1 points only, 2 lines only
  const float* Tcw_in;            // [B][16]
  const float* K;                 // [B][4] fx fy cx cy
  const int* np; int capP;        // [B]
  const float* pt_obs;            // [B][capP][2]
  const float* pt_w;              // [B][capP]   mvInvLevelSigma2[octave]
  const float* pt_X;              // [B][capP][3]
  const int* nl; int capL;
  const double* ln_f;             // [B][capL][3]  mvKeyLineFunctions
  const double* ln_X;             // [B][capL][6]  MapLine::mWorldPos
  float* Tcw_out;                 // [B][16]
  uint8_t* pt_outlier;            // [B][capP]
  uint8_t* ln_outlier;            // [B][capL]
  int* inliers;                   // [B]
  int* iterations;                // [B] (may be NULL) total LM iterations executed
  double* pe;                     // scratch [B][capP][2]
  double* le;                     // scratch [B][capL][2]
};

constexpr int LM_THREADS = 128;
constexpr int NRED = 28;  // 21 H + 6 b + 1 spare

struct LmShared {
  SE3 T, T0, backup, Tp[6], Tm[6];
  double red[LM_THREADS / 32][NRED];
  double H[36], b[6], x[6];
  double lambda, ni, rho, currentChi, iniChi, chi;
  int nBad, qmax, flag, any;
};

template <int n>
__device__ __forceinline__ void block_reduce(LmShared& S, double* v, int tid) {
  // v[0..n) per thread -> S.red[0][0..n) total (all threads must call)
  const int lane = tid & 31, wid = tid >> 5;
#pragma unroll
  for (int k = 0; k < n; k++) v[k] = warp_sum(v[k]);
  __syncthreads();
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < n; k++) S.red[wid][k] = v[k];
  }
  __syncthreads();
  if (tid < n) { double s = 0; for (int w = 0; w < LM_THREADS / 32; w++) s += S.red[w][tid]; S.red[0][tid] = s; }
  __syncthreads();
}

__global__ void __launch_bounds__(LM_THREADS) k_pose_opt(PoseArgs A) {
  __shared__ LmShared S;
  const int b = blockIdx.x, tid = threadIdx.x;
  const double kDeltaMono = huber_delta_mono(), kDeltaLine = huber_delta_line();
  int np = min(A.np[b], A.capP), nl = min(A.nl[b], A.capL);
  if (A.mode == 1) nl = 0;
  if (A.mode == 2) np = 0;
  const double cam[4] = {A.K[4 * b], A.K[4 * b + 1], A.K[4 * b + 2], A.K[4 * b + 3]};
  const float* obs = A.pt_obs + (long long)b * A.capP * 2;
  const float* pw = A.pt_w + (long long)b * A.capP;
  const float* pX = A.pt_X + (long long)b * A.capP * 3;
  const double* lf = A.ln_f + (long long)b * A.capL * 3;
  const double* lX = A.ln_X + (long long)b * A.capL * 6;
  uint8_t* pout = A.pt_outlier + (long long)b * A.capP;
  uint8_t* lout = A.ln_outlier + (long long)b * A.capL;
  double* pe = A.pe + (long long)b * A.capP * 2;
  double* le = A.le + (long long)b * A.capL * 2;
  float* Tout = A.Tcw_out + 16 * b;

  for (int i = tid; i < np; i += LM_THREADS) pout[i] = 0;
  for (int i = tid; i < nl; i += LM_THREADS) lout[i] = 0;
  if (tid < 16) Tout[tid] = A.Tcw_in[16 * b + tid];
  if (tid == 0 && A.iterations) A.iterations[b] = 0;
  if (A.mode == 2 ? (nl < 3) : (np < 3)) { if (tid == 0) A.inliers[b] = 0; return; }
  if (tid == 0) { S.T0 = se3_from_cv(A.Tcw_in + 16 * b); for (int j = 0; j < 6; j++) S.x[j] = 0; }
  __syncthreads();

  auto point_err = [&](const SE3& T, int i, double& e0, double& e1) {
    const double X[3] = {(double)pX[3 * i], (double)pX[3 * i + 1], (double)pX[3 * i + 2]};
    proj_error(T, X, cam, (double)obs[2 * i], (double)obs[2 * i + 1], e0, e1);
  };
  auto line_err = [&](const SE3& T, int i, int e) { return line_error(T, lX + 6 * i + 3 * e, cam, lf + 3 * i); };
  bool p_robust = true, l_robust = true;
  // computeActiveErrors + activeRobustChi2 at pose S.T; result in S.red[0][0]
  auto errors_and_chi2 = [&]() {
    const SE3 T = S.T;
    double chi = 0, r0, r1;
    for (int i = tid; i < np; i += LM_THREADS) if (!pout[i]) {
      double e0, e1;
      point_err(T, i, e0, e1);
      pe[2 * i] = e0; pe[2 * i + 1] = e1;
      double w = (double)pw[i], c2 = e0 * (w * e0) + e1 * (w * e1);
      if (p_robust) { huber(c2, kDeltaMono, r0, r1); chi += r0; } else chi += c2;
    }
    for (int i = tid; i < nl; i += LM_THREADS) if (!lout[i])
      for (int e = 0; e < 2; e++) {
        double er = line_err(T, i, e);
        le[2 * i + e] = er;
        double c2 = er * er;
        if (l_robust) { huber(c2, kDeltaLine, r0, r1); chi += r0; } else chi += c2;
      }
    double v[1] = {chi};
    block_reduce<1>(S, v, tid);
  };

  int nBadPts = 0, nBadLines = 0, total_its = 0;
  // The loops are NOT unrolled on purpose: unrolled and unswitched on the two robust flags the kernel grows to ~150 k SASS
  // instructions (over 2 MB of code) and stalls on instruction fetch.
#pragma unroll 1
  for (int round = 0; round < 4; round++) {
    // ---- optimizer.optimize(10) on the level-0 edges, starting from the frame's initial pose
    int cnt = 0;
    for (int i = tid; i < np; i += LM_THREADS) cnt += !pout[i];
    for (int i = tid; i < nl; i += LM_THREADS) cnt += !lout[i];
    const int anyActive = __syncthreads_or(cnt > 0);
    if (tid == 0) { S.T = S.T0; S.nBad = 0; }
    __syncthreads();
    if (anyActive) {
#pragma unroll 1
      for (int it = 0; it < 10; it++) {
        total_its++;
        errors_and_chi2();
        if (tid == 0) { S.currentChi = S.red[0][0]; S.iniChi = S.currentChi; }
        if (nl > 0 && tid < 12) {  // perturbed poses for the numeric Jacobian
          const SE3 Tn = perturbed_pose(S.T, tid);
          if (tid & 1) S.Tm[tid >> 1] = Tn; else S.Tp[tid >> 1] = Tn;
        }
        __syncthreads();
        // ---- buildSystem
        double acc[NRED];
#pragma unroll
        for (int k = 0; k < NRED; k++) acc[k] = 0;
        {
          const SE3 T = S.T;
          double r0, r1;
          for (int i = tid; i < np; i += LM_THREADS) if (!pout[i]) {
            // EdgeSE3ProjectXYZOnlyPose::linearizeOplus (types_six_dof_expmap.cpp:266-296) multiplies by invz and invz_2 where
            // EdgeSE3ProjectXYZ (proj_jacobians, :103-139) divides by z and z_2; the two round differently, so this one stays.
            double X[3] = {(double)pX[3 * i], (double)pX[3 * i + 1], (double)pX[3 * i + 2]}, c[3];
            se3_map(T, X, c);
            const double x = c[0], y = c[1], invz = 1.0 / c[2], invz_2 = invz * invz, fx = cam[0], fy = cam[1];
            double J0[6], J1[6];
            J0[0] = x * y * invz_2 * fx; J0[1] = -(1 + (x * x * invz_2)) * fx; J0[2] = y * invz * fx;
            J0[3] = -invz * fx; J0[4] = 0; J0[5] = x * invz_2 * fx;
            J1[0] = (1 + y * y * invz_2) * fy; J1[1] = -x * y * invz_2 * fy; J1[2] = -x * invz * fy;
            J1[3] = 0; J1[4] = -invz * fy; J1[5] = y * invz_2 * fy;
            const double w = (double)pw[i], e0 = pe[2 * i], e1 = pe[2 * i + 1];
            r1 = 1.0;
            if (p_robust) huber(e0 * (w * e0) + e1 * (w * e1), kDeltaMono, r0, r1);
            int k = 0;
#pragma unroll
            for (int a = 0; a < 6; a++) {
#pragma unroll
              for (int c2 = a; c2 < 6; c2++) acc[k++] += J0[a] * (r1 * w) * J0[c2] + J1[a] * (r1 * w) * J1[c2];
            }
#pragma unroll
            for (int a = 0; a < 6; a++) acc[21 + a] -= r1 * (J0[a] * (w * e0) + J1[a] * (w * e1));
          }
          for (int i = tid; i < nl; i += LM_THREADS) if (!lout[i])
            for (int e = 0; e < 2; e++) {
              double J[6];
              line_pose_jacobian(S.Tp, S.Tm, lX + 6 * i + 3 * e, cam, lf + 3 * i, J);
              const double err = le[2 * i + e];
              r1 = 1.0;
              if (l_robust) huber(err * err, kDeltaLine, r0, r1);
              int k = 0;
#pragma unroll
              for (int a = 0; a < 6; a++) {
#pragma unroll
                for (int c2 = a; c2 < 6; c2++) acc[k++] += J[a] * r1 * J[c2];
              }
#pragma unroll
              for (int a = 0; a < 6; a++) acc[21 + a] -= r1 * (J[a] * err);
            }
        }
        block_reduce<27>(S, acc, tid);
        if (tid == 0) {
          int k = 0;
          for (int a = 0; a < 6; a++) for (int c2 = a; c2 < 6; c2++) { S.H[a * 6 + c2] = S.red[0][k]; S.H[c2 * 6 + a] = S.red[0][k]; k++; }
          for (int a = 0; a < 6; a++) S.b[a] = S.red[0][21 + a];
          if (it == 0) {
            double md = 0;
            for (int j = 0; j < 6; j++) md = fmax(fabs(S.H[j * 6 + j]), md);
            lm_init(md, S.lambda, S.ni, S.nBad);
          }
          S.rho = 0; S.qmax = 0;
        }
        __syncthreads();
        // ---- trial steps
#pragma unroll 1
        while (true) {
          if (tid == 0) {
            S.backup = S.T;
            S.flag = solve6(S.H, S.b, S.lambda, S.x) ? 1 : 0;
            S.T = se3_mul(se3_exp(S.x), S.T);
          }
          __syncthreads();
          errors_and_chi2();
          if (tid == 0) {
            double scale = 0;
            for (int j = 0; j < 6; j++) scale += S.x[j] * (S.lambda * S.x[j] + S.b[j]);
            bool kept;
            S.rho = lm_trial(S.flag, S.red[0][0], scale, S.lambda, S.ni, S.currentChi, kept);
            if (!kept) S.T = S.backup;
            S.qmax++;
            S.flag = (S.rho < 0 && S.qmax < 10) ? 1 : 0;  // repeat?
          }
          __syncthreads();
          if (!S.flag) break;
        }
        if (tid == 0) S.any = lm_stop(S.qmax, S.rho, S.iniChi, S.currentChi, S.nBad);
        __syncthreads();
        if (S.any) break;
      }
    }
    __syncthreads();
    // ---- classification (Optimizer.cc:866-959): stored error for inliers, recomputed error for outliers
    {
      const SE3 T = S.T;
      int bad = 0, lbad = 0;
      for (int i = tid; i < np; i += LM_THREADS) {
        if (pout[i]) { double e0, e1; point_err(T, i, e0, e1); pe[2 * i] = e0; pe[2 * i + 1] = e1; }
        const double w = (double)pw[i], e0 = pe[2 * i], e1 = pe[2 * i + 1];
        const float chi2 = (float)(e0 * (w * e0) + e1 * (w * e1));
        if (chi2 > 5.991f) { pout[i] = 1; bad++; } else pout[i] = 0;
      }
      for (int i = tid; i < nl; i += LM_THREADS) {
        if (lout[i]) { le[2 * i] = line_err(T, i, 0); le[2 * i + 1] = line_err(T, i, 1); }
        const float cs = (float)(le[2 * i] * le[2 * i]), ce = (float)(le[2 * i + 1] * le[2 * i + 1]);
        if (cs > 3.84f || ce > 3.84f) { lout[i] = 1; lbad++; } else lout[i] = 0;
      }
      double v[2] = {(double)bad, (double)lbad};
      block_reduce<2>(S, v, tid);
      nBadPts = (int)S.red[0][0]; nBadLines = (int)S.red[0][1];
      __syncthreads();
    }
    if (round == 2) { p_robust = false; l_robust = false; }
    if (np + 2 * nl < 10) break;
  }
  if (tid == 0) {
    se3_to_cv(S.T, Tout);
    A.inliers[b] = (A.mode == 2) ? nl - nBadLines : np - nBadPts;
    if (A.iterations) A.iterations[b] = total_its;
  }
}
}  // namespace pl

using namespace pl;

extern "C" int pl_pose_optimization_dev(int mode, int B, const float* Tcw_in, const float* K, const int* n_points,
                                        int cap_points, const float* pt_obs, const float* pt_inv_sigma2,
                                        const float* pt_Xw, const int* n_lines, int cap_lines, const double* line_func,
                                        const double* line_Xw, float* Tcw_out, uint8_t* pt_outlier,
                                        uint8_t* line_outlier, int* inliers, int* iterations, double* scratch,
                                        void* stream) {
  PL_ARG(mode >= 0 && mode <= 2 && B > 0 && Tcw_in && K && n_points && n_lines && Tcw_out && inliers && scratch);
  PL_ARG(cap_points >= 1 && cap_lines >= 1 && pt_obs && pt_inv_sigma2 && pt_Xw && line_func && line_Xw && pt_outlier && line_outlier);
  PoseArgs A;
  A.mode = mode; A.Tcw_in = Tcw_in; A.K = K; A.np = n_points; A.capP = cap_points; A.pt_obs = pt_obs; A.pt_w = pt_inv_sigma2;
  A.pt_X = pt_Xw; A.nl = n_lines; A.capL = cap_lines; A.ln_f = line_func; A.ln_X = line_Xw; A.Tcw_out = Tcw_out;
  A.pt_outlier = pt_outlier; A.ln_outlier = line_outlier; A.inliers = inliers; A.iterations = iterations;
  A.pe = scratch; A.le = scratch + (size_t)B * cap_points * 2;
  k_pose_opt<<<B, LM_THREADS, 0, (cudaStream_t)stream>>>(A);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

extern "C" size_t pl_pose_optimization_scratch_doubles(int B, int cap_points, int cap_lines) {
  return (size_t)B * ((size_t)cap_points * 2 + (size_t)cap_lines * 2);
}

extern "C" int pl_pose_optimization(int mode, const float* Tcw_in, const float* K, int n_points, const float* pt_obs,
                                    const float* pt_inv_sigma2, const float* pt_Xw, int n_lines,
                                    const double* line_func, const double* line_Xw, float* Tcw_out,
                                    uint8_t* pt_outlier, uint8_t* line_outlier, int* iterations) {
  PL_ARG(Tcw_in && K && Tcw_out && n_points >= 0 && n_lines >= 0);
  int rc = require_device(); if (rc) return rc;
  const int cp = std::max(n_points, 1), cl = std::max(n_lines, 1);
  Staging s;
  float* dT = s.in(Tcw_in, 16); float* dK = s.in(K, 4); int* dnp = s.in(&n_points, 1); int* dnl = s.in(&n_lines, 1);
  float* dobs = s.in(pt_obs, (size_t)n_points * 2); float* dw = s.in(pt_inv_sigma2, n_points); float* dX = s.in(pt_Xw, (size_t)n_points * 3);
  double* dlf = s.in(line_func, (size_t)n_lines * 3); double* dlX = s.in(line_Xw, (size_t)n_lines * 6);
  int inl = 0, its = 0;
  float* dTo = s.out(Tcw_out, 16); int* dinl = s.out(&inl, 1); int* dits = s.out(&its, 1);
  // the kernel writes only the masks of the edges the mode optimises (mode 1: points, mode 2: lines); the other one is the
  // caller's and stays untouched, as the reference leaves mvbLineOutlier / mvbOutlier alone in those modes
  uint8_t* dpo = mode != 2 && pt_outlier ? s.out(pt_outlier, n_points, cp) : s.out<uint8_t>(cp);
  uint8_t* dlo = mode != 1 && line_outlier ? s.out(line_outlier, n_lines, cl) : s.out<uint8_t>(cl);
  double* scr = s.out<double>(pl_pose_optimization_scratch_doubles(1, cp, cl));
  if ((rc = s.status()) ||
      (rc = pl_pose_optimization_dev(mode, 1, dT, dK, dnp, cp, dobs, dw, dX, dnl, cl, dlf, dlX, dTo, dpo, dlo, dinl, dits, scr, nullptr)) ||
      (rc = s.fetch()))
    return rc;
  if (iterations) *iterations = its;
  return inl;
}
