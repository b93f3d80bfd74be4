// Local bundle adjustment with points and line end-points on sm_90a (fp64).
//
// Replaces Optimizer::LocalBundleAdjustmentWithLine (reference src/Optimizer.cc:1645-2100; the points-only twin
// :1308-1642 is the n_line_edges == 0 case) together with the g2o machinery it drives: BlockSolver_6_3 with the Schur
// complement over the marginalised landmarks (core/block_solver.hpp:353-486,501-589), OptimizationAlgorithmLevenberg
// (core/optimization_algorithm_levenberg.cpp:61-189), EdgeSE3ProjectXYZ (types/types_six_dof_expmap.cpp:103-139),
// EdgeLineProjectXYZ with g2o's numeric Jacobians (include/lineEdge.h:212-232, core/base_binary_edge.hpp:130-205),
// Huber kernels, and the reference's outlier gating / erase lists (Optimizer.cc:1957-2043).
//
// One persistent CTA (512 threads) runs a whole problem: no graph objects, edges are flat arrays with two CSR
// indices (by landmark, by keyframe) built by the host wrapper.  Per LM iteration: residuals + per-edge Jacobians
// (thread per edge), landmark blocks Hll/bl (thread per landmark, fixed edge order), pose blocks Hpp/bp (warp per
// keyframe, fixed order), then per trial: 3x3 inverses, Schur complement accumulated per landmark into the dense
// reduced pose system (fp64 atomics), in-CTA dense LDL^T, landmark back-substitution, state update, step control.
// A different keyframe's LBA is an independent problem ("replicas only" across GPUs, SURVEY.md §8e).

#include "common.cuh"
#include <mutex>
#include "se3.cuh"
#include <vector>
#include <algorithm>

namespace pl {

constexpr int BA_THREADS = 512;

struct BAArgs {
  int n_kf, n_pt, n_ln, n_pe, n_le;
  const float* kf_Tcw; const uint8_t* kf_fixed; const float* kf_K; float K_end[4];
  const float* pt_Xw; const double* ln_Xw;
  const int* pe_kf; const int* pe_pt; const float* pe_obs; const float* pe_w;
  const int* le_kf; const int* le_ln; const double* le_f;
  const int* lm_start; const int* lm_edges;     // CSR by landmark; edge code: point edge e -> e, line edge (e,end) -> n_pe + 2e + end
  const int* kf_start; const int* kf_edges;     // CSR by keyframe (same edge codes)
  const volatile int* stop;                     // may be NULL
  // outputs
  float* kf_Tcw_out; float* pt_Xw_out; double* ln_Xw_out; uint8_t* pe_erase; uint8_t* le_erase; int* le_erase_kf; int* iterations;
  // scratch
  SE3* T; SE3* Tb; SE3* Tp; SE3* Tm;            // [n_kf], [n_kf], [n_kf*6], [n_kf*6]
  double* X; double* Xb;                        // [n_lm*3]
  double* err;                                  // [n_pe*2 + n_le*2]
  uint8_t* lvl;                                 // [n_pe + n_le]
  double* JA; double* JB; double* omr; double* wgt;   // per edge code: A[6], B[12], omega_r[2], weight
  int* pose_slot; int* lm_slot;
  double* Hpp; double* bp; double* Hll; double* bl; double* Dinv; double* Dinvb;
  double* Hs; double* bs; double* x; double* Dd;      // Hs [n*n], bs [n], x [n + nl*3], Dd [n]
};

struct BAShared {
  double red[BA_THREADS / 32];
  double lambda, ni, rho, currentChi, iniChi, scale_acc;
  int np, nl, nBad, qmax, flag, stop_it, ok2;
};

__device__ __forceinline__ double block_sum(BAShared& S, double v, int tid) {
  v = warp_sum(v);
  __syncthreads();
  if ((tid & 31) == 0) S.red[tid >> 5] = v;
  __syncthreads();
  double s = 0;
  for (int w = 0; w < BA_THREADS / 32; w++) s += S.red[w];
  __syncthreads();
  return s;
}
__device__ __forceinline__ double block_max(BAShared& S, double v, int tid) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((tid & 31) == 0) S.red[tid >> 5] = v;
  __syncthreads();
  double s = 0;
  for (int w = 0; w < BA_THREADS / 32; w++) s = fmax(s, S.red[w]);
  __syncthreads();
  return s;
}
__device__ __forceinline__ void inv3(const double* D, double lambda, double* Di) {
  const double a = D[0] + lambda, b = D[1], c = D[2], d = D[3], e = D[4] + lambda, f = D[5], g = D[6], h = D[7], i = D[8] + lambda;
  const double A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
  const double id = 1.0 / (a * A + b * B + c * C);
  Di[0] = A * id; Di[1] = -(b * i - c * h) * id; Di[2] = (b * f - c * e) * id;
  Di[3] = B * id; Di[4] = (a * i - c * g) * id; Di[5] = -(a * f - c * d) * id;
  Di[6] = C * id; Di[7] = -(a * h - b * g) * id; Di[8] = (a * e - b * d) * id;
}

__device__ __forceinline__ void edge_decode(const BAArgs& A, int code, int& kf, int& lm, int& dim, int& e, int& end) {
  if (code < A.n_pe) { e = code; end = 0; dim = 2; kf = A.pe_kf[e]; lm = A.pe_pt[e]; }
  else { const int c = code - A.n_pe; e = c >> 1; end = c & 1; dim = 1; kf = A.le_kf[e]; lm = A.n_pt + 2 * A.le_ln[e] + end; }
}
__device__ __forceinline__ void cam_K(const BAArgs& A, int kf, int end_edge, double* k) {
  if (end_edge) { for (int i = 0; i < 4; i++) k[i] = (double)A.K_end[i]; }
  else { for (int i = 0; i < 4; i++) k[i] = (double)A.kf_K[4 * kf + i]; }
}
__device__ __forceinline__ double line_err_at(const BAArgs& A, const SE3& T, const double* X, int e, int end) {
  double c[3], k[4];
  se3_map(T, X, c);
  cam_K(A, A.le_kf[e], end, k);
  const double u = c[0] / c[2] * k[0] + k[2], v = c[1] / c[2] * k[1] + k[3];
  return A.le_f[3 * e] * u + A.le_f[3 * e + 1] * v + A.le_f[3 * e + 2];
}

// computeActiveErrors + activeRobustChi2
__device__ double errors_and_chi2(const BAArgs& A, BAShared& S, bool p_robust, bool l_robust, int tid) {
  const double kDeltaMono = (double)(float)sqrt(5.991), kDeltaLine = (double)(float)sqrt(3.84);
  double chi = 0, r0, r1;
  for (int e = tid; e < A.n_pe; e += BA_THREADS) if (!A.lvl[e]) {
    double c[3], k[4];
    se3_map(A.T[A.pe_kf[e]], A.X + 3 * A.pe_pt[e], c);
    cam_K(A, A.pe_kf[e], 0, k);
    const double e0 = (double)A.pe_obs[2 * e] - (c[0] / c[2] * k[0] + k[2]), e1 = (double)A.pe_obs[2 * e + 1] - (c[1] / c[2] * k[1] + k[3]);
    A.err[2 * e] = e0; A.err[2 * e + 1] = e1;
    const double w = (double)A.pe_w[e], c2 = e0 * (w * e0) + e1 * (w * e1);
    if (p_robust) { huber(c2, kDeltaMono, r0, r1); chi += r0; } else chi += c2;
  }
  for (int e = tid; e < A.n_le; e += BA_THREADS) if (!A.lvl[A.n_pe + e])
    for (int end = 0; end < 2; end++) {
      const double er = line_err_at(A, A.T[A.le_kf[e]], A.X + 3 * (A.n_pt + 2 * A.le_ln[e] + end), e, end);
      A.err[2 * A.n_pe + 2 * e + end] = er;
      const double c2 = er * (0.5 * er);
      if (l_robust) { huber(c2, kDeltaLine, r0, r1); chi += r0; } else chi += c2;
    }
  return block_sum(S, chi, tid);
}

// one optimizer.optimize(iterations) call on the level-0 edges.  (Unlike k_pose_opt, this kernel is ONE CTA per problem with the SM
// to itself: keeping the LM loops rolled and this function out of line shrinks it from 81 k to 21 k SASS instructions but makes
// the 20+40-keyframe window markedly slower, so the inlined, unrolled form stays.)
__device__ int ba_optimize(const BAArgs& A, BAShared& S, int iterations, bool p_robust, bool l_robust, int tid) {
  const double kDeltaMono = (double)(float)sqrt(5.991), kDeltaLine = (double)(float)sqrt(3.84);
  const int n_lm = A.n_pt + 2 * A.n_ln, n_edges = A.n_pe + 2 * A.n_le;
  // ---- active sets and slots (initializeOptimization)
  for (int k = tid; k < A.n_kf; k += BA_THREADS) {
    int act = 0;
    for (int j = A.kf_start[k]; j < A.kf_start[k + 1] && !act; j++) { int c = A.kf_edges[j]; act = !A.lvl[c < A.n_pe ? c : A.n_pe + ((c - A.n_pe) >> 1)]; }
    A.pose_slot[k] = (act && !A.kf_fixed[k]) ? 1 : -1;
  }
  for (int l = tid; l < n_lm; l += BA_THREADS) {
    int act = 0;
    for (int j = A.lm_start[l]; j < A.lm_start[l + 1] && !act; j++) { int c = A.lm_edges[j]; act = !A.lvl[c < A.n_pe ? c : A.n_pe + ((c - A.n_pe) >> 1)]; }
    A.lm_slot[l] = act ? 1 : -1;
  }
  __syncthreads();
  if (tid == 0) {
    int np = 0, nl = 0;
    for (int k = 0; k < A.n_kf; k++) if (A.pose_slot[k] > 0) A.pose_slot[k] = np++;
    for (int l = 0; l < n_lm; l++) if (A.lm_slot[l] > 0) A.lm_slot[l] = nl++;
    S.np = np; S.nl = nl;
  }
  __syncthreads();
  const int np = S.np, nl = S.nl, n = np * 6;
  if (np + nl == 0) return 0;
  for (int i = tid; i < n + nl * 3; i += BA_THREADS) A.x[i] = 0.0;
  int done = 0;
  for (int it = 0; it < iterations; it++) {
    if (A.stop && *A.stop) break;                       // SparseOptimizer::terminate()
    done++;
    const double chi0 = errors_and_chi2(A, S, p_robust, l_robust, tid);
    if (tid == 0) { S.currentChi = chi0; S.iniChi = chi0; }
    // ---- perturbed poses for the numeric (line) Jacobians
    if (A.n_le > 0)
      for (int i = tid; i < A.n_kf * 12; i += BA_THREADS) {
        const int k = i / 12, r = i - k * 12, d = r >> 1;
        double add[6] = {0, 0, 0, 0, 0, 0};
        add[d] = (r & 1) ? -1e-9 : 1e-9;
        const SE3 Tn = se3_mul(se3_exp(add), A.T[k]);
        if (r & 1) A.Tm[k * 6 + d] = Tn; else A.Tp[k * 6 + d] = Tn;
      }
    __syncthreads();
    // ---- per-edge linearisation
    for (int code = tid; code < n_edges; code += BA_THREADS) {
      int kf, lm, dim, e, end;
      edge_decode(A, code, kf, lm, dim, e, end);
      if (A.lvl[code < A.n_pe ? e : A.n_pe + e]) continue;
      double* JA = A.JA + 6 * (size_t)code; double* JB = A.JB + 12 * (size_t)code;
      double r0, r1 = 1.0;
      if (dim == 2) {
        const SE3 T = A.T[kf];
        double c[3], k[4], R[3][3];
        se3_map(T, A.X + 3 * lm, c); cam_K(A, kf, 0, k); quat_to_matrix(T.r, R);
        const double x = c[0], y = c[1], z = c[2], z_2 = z * z, fx = k[0], fy = k[1];
        const double t00 = fx, t02 = -x / z * fx, t11 = fy, t12 = -y / z * fy;
        for (int j = 0; j < 3; j++) {
          JA[j] = -1. / z * (t00 * R[0][j] + t02 * R[2][j]);
          JA[3 + j] = -1. / z * (t11 * R[1][j] + t12 * R[2][j]);
        }
        JB[0] = x * y / z_2 * fx; JB[1] = -(1 + (x * x / z_2)) * fx; JB[2] = y / z * fx; JB[3] = -1. / z * fx; JB[4] = 0; JB[5] = x / z_2 * fx;
        JB[6] = (1 + y * y / z_2) * fy; JB[7] = -x * y / z_2 * fy; JB[8] = -x / z * fy; JB[9] = 0; JB[10] = -1. / z * fy; JB[11] = y / z_2 * fy;
        const double w = (double)A.pe_w[e], e0 = A.err[2 * e], e1 = A.err[2 * e + 1];
        double o0 = -(w * e0), o1 = -(w * e1), wg = w;
        if (p_robust) { huber(e0 * (w * e0) + e1 * (w * e1), kDeltaMono, r0, r1); o0 *= r1; o1 *= r1; wg = r1 * w; }
        A.omr[2 * (size_t)code] = o0; A.omr[2 * (size_t)code + 1] = o1; A.wgt[code] = wg;
      } else {
        const double* X = A.X + 3 * lm;
        for (int d = 0; d < 3; d++) {
          double Xp[3] = {X[0], X[1], X[2]}, Xm[3] = {X[0], X[1], X[2]};
          Xp[d] += 1e-9; Xm[d] += -1e-9;
          JA[d] = 5e8 * (line_err_at(A, A.T[kf], Xp, e, end) - line_err_at(A, A.T[kf], Xm, e, end));
        }
        for (int d = 0; d < 6; d++) JB[d] = 5e8 * (line_err_at(A, A.Tp[kf * 6 + d], X, e, end) - line_err_at(A, A.Tm[kf * 6 + d], X, e, end));
        const double er = A.err[2 * A.n_pe + 2 * e + end], w = 0.5;
        double o0 = -(w * er), wg = w;
        if (l_robust) { huber(er * (w * er), kDeltaLine, r0, r1); o0 *= r1; wg = r1 * w; }
        A.omr[2 * (size_t)code] = o0; A.omr[2 * (size_t)code + 1] = 0; A.wgt[code] = wg;
      }
    }
    __syncthreads();
    // ---- landmark blocks (thread per landmark, edges in CSR order)
    for (int l = tid; l < n_lm; l += BA_THREADS) {
      const int ls = A.lm_slot[l];
      if (ls < 0) continue;
      double H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, b[3] = {0, 0, 0};
      for (int j = A.lm_start[l]; j < A.lm_start[l + 1]; j++) {
        const int code = A.lm_edges[j];
        if (A.lvl[code < A.n_pe ? code : A.n_pe + ((code - A.n_pe) >> 1)]) continue;
        const int dim = code < A.n_pe ? 2 : 1;
        const double* JA = A.JA + 6 * (size_t)code;
        const double wg = A.wgt[code];
        for (int a = 0; a < 3; a++) {
          double s = 0;
          for (int d = 0; d < dim; d++) s += JA[d * 3 + a] * A.omr[2 * (size_t)code + d];
          b[a] += s;
          for (int c = 0; c < 3; c++) { double h = 0; for (int d = 0; d < dim; d++) h += JA[d * 3 + a] * wg * JA[d * 3 + c]; H[a * 3 + c] += h; }
        }
      }
      for (int i = 0; i < 9; i++) A.Hll[(size_t)ls * 9 + i] = H[i];
      for (int i = 0; i < 3; i++) A.bl[(size_t)ls * 3 + i] = b[i];
    }
    // ---- pose blocks (warp per keyframe)
    for (int k = tid >> 5; k < A.n_kf; k += BA_THREADS / 32) {
      const int ps = A.pose_slot[k];
      if (ps < 0) continue;
      const int lane = tid & 31;
      double acc[27];
#pragma unroll
      for (int i = 0; i < 27; i++) acc[i] = 0;
      for (int j = A.kf_start[k] + lane; j < A.kf_start[k + 1]; j += 32) {
        const int code = A.kf_edges[j];
        if (A.lvl[code < A.n_pe ? code : A.n_pe + ((code - A.n_pe) >> 1)]) continue;
        const int dim = code < A.n_pe ? 2 : 1;
        const double* JB = A.JB + 12 * (size_t)code;
        const double wg = A.wgt[code];
        int q = 0;
        for (int a = 0; a < 6; a++)
          for (int c = a; c < 6; c++) { double h = 0; for (int d = 0; d < dim; d++) h += JB[d * 6 + a] * wg * JB[d * 6 + c]; acc[q++] += h; }
        for (int a = 0; a < 6; a++) { double s = 0; for (int d = 0; d < dim; d++) s += JB[d * 6 + a] * A.omr[2 * (size_t)code + d]; acc[21 + a] += s; }
      }
#pragma unroll
      for (int i = 0; i < 27; i++) acc[i] = warp_sum(acc[i]);
      if (lane == 0) {
        int q = 0;
        for (int a = 0; a < 6; a++) for (int c = a; c < 6; c++) { A.Hpp[(size_t)ps * 36 + a * 6 + c] = acc[q]; A.Hpp[(size_t)ps * 36 + c * 6 + a] = acc[q]; q++; }
        for (int a = 0; a < 6; a++) A.bp[(size_t)ps * 6 + a] = acc[21 + a];
      }
    }
    __syncthreads();
    if (it == 0) {
      double md = 0;
      for (int i = tid; i < np * 6; i += BA_THREADS) md = fmax(md, fabs(A.Hpp[(size_t)(i / 6) * 36 + (i % 6) * 7]));
      for (int i = tid; i < nl * 3; i += BA_THREADS) md = fmax(md, fabs(A.Hll[(size_t)(i / 3) * 9 + (i % 3) * 4]));
      md = block_max(S, md, tid);
      if (tid == 0) { S.lambda = 1e-5 * md; S.ni = 2; S.nBad = 0; }
    }
    if (tid == 0) { S.rho = 0; S.qmax = 0; }
    __syncthreads();
    // ---- trial steps
    while (true) {
      const double lambda = S.lambda;
      for (int k = tid; k < A.n_kf; k += BA_THREADS) A.Tb[k] = A.T[k];
      for (int i = tid; i < n_lm * 3; i += BA_THREADS) A.Xb[i] = A.X[i];
      for (int l = tid; l < nl; l += BA_THREADS) {
        double Di[9];
        inv3(A.Hll + (size_t)l * 9, lambda, Di);
        for (int i = 0; i < 9; i++) A.Dinv[(size_t)l * 9 + i] = Di[i];
        for (int a = 0; a < 3; a++) A.Dinvb[(size_t)l * 3 + a] = Di[a * 3] * A.bl[(size_t)l * 3] + Di[a * 3 + 1] * A.bl[(size_t)l * 3 + 1] + Di[a * 3 + 2] * A.bl[(size_t)l * 3 + 2];
      }
      for (int i = tid; i < n * n; i += BA_THREADS) A.Hs[i] = 0.0;
      __syncthreads();
      for (int i = tid; i < np * 36; i += BA_THREADS) {
        const int p = i / 36, a = (i % 36) / 6, c = i % 6;
        A.Hs[(size_t)(p * 6 + a) * n + p * 6 + c] = A.Hpp[i] + (a == c ? lambda : 0.0);
      }
      for (int i = tid; i < n; i += BA_THREADS) A.bs[i] = A.bp[i];
      __syncthreads();
      // Schur complement, one thread per landmark
      for (int l = tid; l < n_lm; l += BA_THREADS) {
        const int ls = A.lm_slot[l];
        if (ls < 0) continue;
        const double* Di = A.Dinv + (size_t)ls * 9;
        const double* Db = A.Dinvb + (size_t)ls * 3;
        for (int j1 = A.lm_start[l]; j1 < A.lm_start[l + 1]; j1++) {
          const int c1 = A.lm_edges[j1];
          if (A.lvl[c1 < A.n_pe ? c1 : A.n_pe + ((c1 - A.n_pe) >> 1)]) continue;
          const int k1 = c1 < A.n_pe ? A.pe_kf[c1] : A.le_kf[(c1 - A.n_pe) >> 1];
          const int p1 = A.pose_slot[k1];
          if (p1 < 0) continue;
          const int d1 = c1 < A.n_pe ? 2 : 1;
          const double *JA1 = A.JA + 6 * (size_t)c1, *JB1 = A.JB + 12 * (size_t)c1;
          const double w1 = A.wgt[c1];
          double B1[18], BD[18];   // Hpl block = B^T w A (6x3); BD = Hpl * Dinv
          for (int a = 0; a < 6; a++) for (int c = 0; c < 3; c++) { double h = 0; for (int d = 0; d < d1; d++) h += JB1[d * 6 + a] * w1 * JA1[d * 3 + c]; B1[a * 3 + c] = h; }
          for (int a = 0; a < 6; a++) for (int c = 0; c < 3; c++) BD[a * 3 + c] = B1[a * 3] * Di[c] + B1[a * 3 + 1] * Di[3 + c] + B1[a * 3 + 2] * Di[6 + c];
          for (int a = 0; a < 6; a++) atomicAdd(&A.bs[p1 * 6 + a], -(B1[a * 3] * Db[0] + B1[a * 3 + 1] * Db[1] + B1[a * 3 + 2] * Db[2]));
          for (int j2 = A.lm_start[l]; j2 < A.lm_start[l + 1]; j2++) {
            const int c2 = A.lm_edges[j2];
            if (A.lvl[c2 < A.n_pe ? c2 : A.n_pe + ((c2 - A.n_pe) >> 1)]) continue;
            const int k2 = c2 < A.n_pe ? A.pe_kf[c2] : A.le_kf[(c2 - A.n_pe) >> 1];
            const int p2 = A.pose_slot[k2];
            if (p2 < 0) continue;
            const int d2 = c2 < A.n_pe ? 2 : 1;
            const double *JA2 = A.JA + 6 * (size_t)c2, *JB2 = A.JB + 12 * (size_t)c2;
            const double w2 = A.wgt[c2];
            for (int a = 0; a < 6; a++)
              for (int c = 0; c < 6; c++) {
                double s = 0;
                for (int m = 0; m < 3; m++) { double b2 = 0; for (int d = 0; d < d2; d++) b2 += JB2[d * 6 + c] * w2 * JA2[d * 3 + m]; s += BD[a * 3 + m] * b2; }
                atomicAdd(&A.Hs[(size_t)(p1 * 6 + a) * n + p2 * 6 + c], -s);
              }
          }
        }
      }
      __syncthreads();
      // dense LDL^T of Hs (lower triangle, in place), no pivoting
      if (tid == 0) S.ok2 = 1;
      __syncthreads();
      for (int j = 0; j < n; j++) {
        if (tid == 0) {
          double d = A.Hs[(size_t)j * n + j];
          for (int k = 0; k < j; k++) d -= A.Hs[(size_t)j * n + k] * A.Hs[(size_t)j * n + k] * A.Dd[k];
          if (d == 0 || !isfinite(d)) S.ok2 = 0;
          A.Dd[j] = d;
        }
        __syncthreads();
        if (!S.ok2) break;
        const double d = A.Dd[j];
        for (int i = j + 1 + tid; i < n; i += BA_THREADS) {
          double s = A.Hs[(size_t)i * n + j];
          for (int k = 0; k < j; k++) s -= A.Hs[(size_t)i * n + k] * A.Hs[(size_t)j * n + k] * A.Dd[k];
          A.Hs[(size_t)i * n + j] = s / d;
        }
        __syncthreads();
      }
      if (S.ok2 && tid == 0) {   // triangular solves (n is a few hundred at most)
        double* y = A.bs;        // in place
        for (int i = 0; i < n; i++) { double s = y[i]; for (int k = 0; k < i; k++) s -= A.Hs[(size_t)i * n + k] * y[k]; y[i] = s; }
        for (int i = 0; i < n; i++) y[i] /= A.Dd[i];
        for (int i = n - 1; i >= 0; i--) { double s = y[i]; for (int k = i + 1; k < n; k++) s -= A.Hs[(size_t)k * n + i] * A.x[k]; A.x[i] = s; }
      }
      __syncthreads();
      if (S.ok2) {   // landmark part: xl = Dinv (bl - Hpl^T xp)
        for (int l = tid; l < n_lm; l += BA_THREADS) {
          const int ls = A.lm_slot[l];
          if (ls < 0) continue;
          double cl[3] = {A.bl[(size_t)ls * 3], A.bl[(size_t)ls * 3 + 1], A.bl[(size_t)ls * 3 + 2]};
          for (int j1 = A.lm_start[l]; j1 < A.lm_start[l + 1]; j1++) {
            const int c1 = A.lm_edges[j1];
            if (A.lvl[c1 < A.n_pe ? c1 : A.n_pe + ((c1 - A.n_pe) >> 1)]) continue;
            const int k1 = c1 < A.n_pe ? A.pe_kf[c1] : A.le_kf[(c1 - A.n_pe) >> 1];
            const int p1 = A.pose_slot[k1];
            if (p1 < 0) continue;
            const int d1 = c1 < A.n_pe ? 2 : 1;
            const double *JA1 = A.JA + 6 * (size_t)c1, *JB1 = A.JB + 12 * (size_t)c1;
            const double w1 = A.wgt[c1];
            for (int c = 0; c < 3; c++) {
              double s = 0;
              for (int a = 0; a < 6; a++) { double h = 0; for (int d = 0; d < d1; d++) h += JB1[d * 6 + a] * w1 * JA1[d * 3 + c]; s += h * A.x[p1 * 6 + a]; }
              cl[c] -= s;
            }
          }
          const double* Di = A.Dinv + (size_t)ls * 9;
          for (int a = 0; a < 3; a++) A.x[n + ls * 3 + a] = Di[a * 3] * cl[0] + Di[a * 3 + 1] * cl[1] + Di[a * 3 + 2] * cl[2];
        }
      }
      __syncthreads();
      // update (with the previous x when the factorisation failed, like g2o)
      for (int k = tid; k < A.n_kf; k += BA_THREADS) if (A.pose_slot[k] >= 0) A.T[k] = se3_mul(se3_exp(A.x + (size_t)A.pose_slot[k] * 6), A.T[k]);
      for (int l = tid; l < n_lm; l += BA_THREADS) if (A.lm_slot[l] >= 0) for (int a = 0; a < 3; a++) A.X[3 * l + a] += A.x[n + A.lm_slot[l] * 3 + a];
      __syncthreads();
      double tempChi = errors_and_chi2(A, S, p_robust, l_robust, tid);
      double sc = 0;
      for (int i = tid; i < n; i += BA_THREADS) sc += A.x[i] * (lambda * A.x[i] + A.bp[i]);
      for (int i = tid; i < nl * 3; i += BA_THREADS) sc += A.x[n + i] * (lambda * A.x[n + i] + A.bl[i]);
      sc = block_sum(S, sc, tid);
      if (tid == 0) {
        if (!S.ok2) tempChi = 1.7976931348623157e308;
        double rho = (S.currentChi - tempChi) / (sc + 1e-3);
        if (rho > 0 && isfinite(tempChi)) {
          double alpha = 1. - pow((2 * rho - 1), 3.0);
          alpha = fmin(alpha, 2. / 3.);
          S.lambda *= fmax(1. / 3., alpha); S.ni = 2; S.currentChi = tempChi; S.flag = 0;
        } else { S.lambda *= S.ni; S.ni *= 2; S.flag = 1; }
        S.rho = rho; S.qmax++;
      }
      __syncthreads();
      if (S.flag) {   // rejected: restore the state
        for (int k = tid; k < A.n_kf; k += BA_THREADS) A.T[k] = A.Tb[k];
        for (int i = tid; i < n_lm * 3; i += BA_THREADS) A.X[i] = A.Xb[i];
      }
      __syncthreads();
      const bool again = S.rho < 0 && S.qmax < 10 && !(A.stop && *A.stop);
      __syncthreads();
      if (!again) break;
    }
    if (tid == 0) {
      int stop = 0;
      if (S.qmax == 10 || S.rho == 0) stop = 1;
      else { if ((S.iniChi - S.currentChi) * 1e3 < S.iniChi) S.nBad++; else S.nBad = 0; if (S.nBad >= 3) stop = 1; }
      S.stop_it = stop;
    }
    __syncthreads();
    if (S.stop_it) break;
  }
  return done;
}

__global__ void __launch_bounds__(BA_THREADS) k_local_ba(BAArgs A) {
  __shared__ BAShared S;
  const int tid = threadIdx.x;
  const int n_lm = A.n_pt + 2 * A.n_ln;
  for (int k = tid; k < A.n_kf; k += BA_THREADS) A.T[k] = se3_from_cv(A.kf_Tcw + 16 * k);
  for (int i = tid; i < 3 * A.n_pt; i += BA_THREADS) A.X[i] = (double)A.pt_Xw[i];
  for (int i = tid; i < 6 * A.n_ln; i += BA_THREADS) A.X[3 * A.n_pt + i] = A.ln_Xw[i];
  for (int i = tid; i < A.n_pe + A.n_le; i += BA_THREADS) A.lvl[i] = 0;
  for (int i = tid; i < 2 * (A.n_pe + A.n_le); i += BA_THREADS) A.err[i] = 0;
  __syncthreads();
  int its = 0;
  const bool stop0 = A.stop && *A.stop;
  if (!stop0) {
    its += ba_optimize(A, S, 5, true, true, tid);
    __syncthreads();
    const bool more = !(A.stop && *A.stop);
    if (more) {
      for (int e = tid; e < A.n_pe; e += BA_THREADS) {
        const double w = (double)A.pe_w[e], c2 = A.err[2 * e] * (w * A.err[2 * e]) + A.err[2 * e + 1] * (w * A.err[2 * e + 1]);
        double c[3];
        se3_map(A.T[A.pe_kf[e]], A.X + 3 * A.pe_pt[e], c);
        if (c2 > 5.991 || !(c[2] > 0.0)) A.lvl[e] = 1;
      }
      for (int e = tid; e < A.n_le; e += BA_THREADS) {
        const double a = A.err[2 * A.n_pe + 2 * e], b = A.err[2 * A.n_pe + 2 * e + 1];
        if (a * (0.5 * a) > 3.84 || b * (0.5 * b) > 3.84) A.lvl[A.n_pe + e] = 1;
      }
      __syncthreads();
      its += ba_optimize(A, S, 10, false, false, tid);
      __syncthreads();
    }
    for (int e = tid; e < A.n_pe; e += BA_THREADS) {
      const double w = (double)A.pe_w[e], c2 = A.err[2 * e] * (w * A.err[2 * e]) + A.err[2 * e + 1] * (w * A.err[2 * e + 1]);
      double c[3];
      se3_map(A.T[A.pe_kf[e]], A.X + 3 * A.pe_pt[e], c);
      A.pe_erase[e] = (c2 > 5.991 || !(c[2] > 0.0)) ? 1 : 0;
    }
    for (int e = tid; e < A.n_le; e += BA_THREADS) {
      const double a = A.err[2 * A.n_pe + 2 * e];
      A.le_erase[e] = (a * (0.5 * a) > 3.84) ? 1 : 0;           // START-point edge read twice (Optimizer.cc:2030-2031)
      A.le_erase_kf[e] = A.le_kf[e / 2];                        // vpLineEdgeKF double push (Optimizer.cc:1924,1948)
    }
  } else {
    for (int e = tid; e < A.n_pe; e += BA_THREADS) A.pe_erase[e] = 0;
    for (int e = tid; e < A.n_le; e += BA_THREADS) { A.le_erase[e] = 0; A.le_erase_kf[e] = A.le_kf[e / 2]; }
  }
  __syncthreads();
  for (int k = tid; k < A.n_kf; k += BA_THREADS) {
    if (A.kf_fixed[k] || its == 0) { for (int i = 0; i < 16; i++) A.kf_Tcw_out[16 * k + i] = A.kf_Tcw[16 * k + i]; }
    else se3_to_cv(A.T[k], A.kf_Tcw_out + 16 * k);
  }
  for (int i = tid; i < 3 * A.n_pt; i += BA_THREADS) A.pt_Xw_out[i] = (float)A.X[i];
  for (int i = tid; i < 6 * A.n_ln; i += BA_THREADS) A.ln_Xw_out[i] = (double)(float)A.X[3 * A.n_pt + i];
  if (tid == 0 && A.iterations) *A.iterations = its;
  (void)n_lm;
}
}  // namespace pl

using namespace pl;

extern "C" int pl_local_ba(const PLBAProblem* p, const int* stop_flag_dev, float* kf_Tcw_out, float* pt_Xw_out,
                           double* ln_Xw_out, uint8_t* pe_erase, uint8_t* le_erase, int* le_erase_kf, int* iterations) {
  PL_ARG(p && kf_Tcw_out && p->n_kf >= 1 && p->n_pt >= 0 && p->n_ln >= 0 && p->n_pe >= 0 && p->n_le >= 0);
  PL_ARG(p->kf_Tcw && p->kf_fixed && p->kf_K);
  int rc = require_device();
  if (rc) return rc;
  const int n_kf = p->n_kf, n_pt = p->n_pt, n_ln = p->n_ln, n_pe = p->n_pe, n_le = p->n_le;
  const int n_lm = n_pt + 2 * n_ln, n_edges = n_pe + 2 * n_le;
  for (int e = 0; e < n_pe; e++) PL_ARG(p->pe_kf[e] >= 0 && p->pe_kf[e] < n_kf && p->pe_pt[e] >= 0 && p->pe_pt[e] < n_pt);
  for (int e = 0; e < n_le; e++) PL_ARG(p->le_kf[e] >= 0 && p->le_kf[e] < n_kf && p->le_ln[e] >= 0 && p->le_ln[e] < n_ln);
  // CSR by landmark and by keyframe, edges kept in insertion order (= g2o's active-edge order)
  std::vector<int> lm_start(n_lm + 1, 0), kf_start(n_kf + 1, 0), lm_edges(std::max(n_edges, 1)), kf_edges(std::max(n_edges, 1));
  auto lm_of = [&](int code) { return code < n_pe ? p->pe_pt[code] : n_pt + 2 * p->le_ln[(code - n_pe) >> 1] + ((code - n_pe) & 1); };
  auto kf_of = [&](int code) { return code < n_pe ? p->pe_kf[code] : p->le_kf[(code - n_pe) >> 1]; };
  for (int c = 0; c < n_edges; c++) { lm_start[lm_of(c) + 1]++; kf_start[kf_of(c) + 1]++; }
  for (int i = 0; i < n_lm; i++) lm_start[i + 1] += lm_start[i];
  for (int i = 0; i < n_kf; i++) kf_start[i + 1] += kf_start[i];
  { std::vector<int> a(lm_start.begin(), lm_start.end() - 1), b(kf_start.begin(), kf_start.end() - 1);
    for (int c = 0; c < n_edges; c++) { lm_edges[a[lm_of(c)]++] = c; kf_edges[b[kf_of(c)]++] = c; } }
  int n_free = 0;
  for (int k = 0; k < n_kf; k++) n_free += !p->kf_fixed[k];
  const size_t n = (size_t)n_free * 6;
  // Device workspace: ONE cached block per process, sub-allocated by a bump pointer (57 cudaMalloc + cudaFree pairs per call are
  // slow inside a process that holds tens of GB of other allocations: cudaFree synchronises and unmaps).
  // Calls are serialised by the mutex (the reference runs one LocalMapping thread); the block only grows.
  static std::mutex ws_mu;
  static char* ws_base = nullptr; static size_t ws_cap = 0; static int ws_dev = -1;
  std::lock_guard<std::mutex> ws_lock(ws_mu);
  int dev = 0; cudaGetDevice(&dev);
  bool fail = false, dry = true;
  size_t off = 0;
  auto dalloc = [&](size_t bytes) -> void* { void* d = dry ? nullptr : (void*)(ws_base + off); off += (std::max<size_t>(bytes, 16) + 255) & ~(size_t)255; return d; };
  auto up = [&](const void* h, size_t bytes) -> void* { void* d = dalloc(bytes); if (!dry && h && bytes && cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice) != cudaSuccess) fail = true; return d; };
  BAArgs A;
  for (int pass = 0; pass < 2; pass++) {
    dry = pass == 0;
    if (!dry && cudaMemset(ws_base, 0, off) != cudaSuccess) { fail = true; break; }     // off = this problem's extent, from the dry pass
    off = 0;
    A.n_kf = n_kf; A.n_pt = n_pt; A.n_ln = n_ln; A.n_pe = n_pe; A.n_le = n_le;
    A.kf_Tcw = (const float*)up(p->kf_Tcw, 64 * (size_t)n_kf); A.kf_fixed = (const uint8_t*)up(p->kf_fixed, n_kf);
    A.kf_K = (const float*)up(p->kf_K, 16 * (size_t)n_kf);
    for (int i = 0; i < 4; i++) A.K_end[i] = p->K_end[i];
    A.pt_Xw = (const float*)up(p->pt_Xw, 12 * (size_t)n_pt); A.ln_Xw = (const double*)up(p->ln_Xw, 48 * (size_t)n_ln);
    A.pe_kf = (const int*)up(p->pe_kf, 4 * (size_t)n_pe); A.pe_pt = (const int*)up(p->pe_pt, 4 * (size_t)n_pe);
    A.pe_obs = (const float*)up(p->pe_obs, 8 * (size_t)n_pe); A.pe_w = (const float*)up(p->pe_inv_sigma2, 4 * (size_t)n_pe);
    A.le_kf = (const int*)up(p->le_kf, 4 * (size_t)n_le); A.le_ln = (const int*)up(p->le_ln, 4 * (size_t)n_le);
    A.le_f = (const double*)up(p->le_func, 24 * (size_t)n_le);
    A.lm_start = (const int*)up(lm_start.data(), 4 * (size_t)(n_lm + 1)); A.lm_edges = (const int*)up(lm_edges.data(), 4 * (size_t)std::max(n_edges, 1));
    A.kf_start = (const int*)up(kf_start.data(), 4 * (size_t)(n_kf + 1)); A.kf_edges = (const int*)up(kf_edges.data(), 4 * (size_t)std::max(n_edges, 1));
    A.stop = stop_flag_dev;
    A.kf_Tcw_out = (float*)dalloc(64 * (size_t)n_kf); A.pt_Xw_out = (float*)dalloc(12 * (size_t)n_pt); A.ln_Xw_out = (double*)dalloc(48 * (size_t)n_ln);
    A.pe_erase = (uint8_t*)dalloc(n_pe); A.le_erase = (uint8_t*)dalloc(n_le); A.le_erase_kf = (int*)dalloc(4 * (size_t)n_le); A.iterations = (int*)dalloc(4);
    A.T = (SE3*)dalloc(sizeof(SE3) * n_kf); A.Tb = (SE3*)dalloc(sizeof(SE3) * n_kf);
    A.Tp = (SE3*)dalloc(sizeof(SE3) * n_kf * 6); A.Tm = (SE3*)dalloc(sizeof(SE3) * n_kf * 6);
    A.X = (double*)dalloc(24 * (size_t)n_lm); A.Xb = (double*)dalloc(24 * (size_t)n_lm);
    A.err = (double*)dalloc(16 * (size_t)(n_pe + n_le)); A.lvl = (uint8_t*)dalloc(n_pe + n_le);
    A.JA = (double*)dalloc(48 * (size_t)n_edges); A.JB = (double*)dalloc(96 * (size_t)n_edges);
    A.omr = (double*)dalloc(16 * (size_t)n_edges); A.wgt = (double*)dalloc(8 * (size_t)n_edges);
    A.pose_slot = (int*)dalloc(4 * (size_t)n_kf); A.lm_slot = (int*)dalloc(4 * (size_t)n_lm);
    A.Hpp = (double*)dalloc(288 * (size_t)n_free); A.bp = (double*)dalloc(48 * (size_t)n_free);
    A.Hll = (double*)dalloc(72 * (size_t)n_lm); A.bl = (double*)dalloc(24 * (size_t)n_lm);
    A.Dinv = (double*)dalloc(72 * (size_t)n_lm); A.Dinvb = (double*)dalloc(24 * (size_t)n_lm);
    A.Hs = (double*)dalloc(8 * n * n); A.bs = (double*)dalloc(8 * n); A.x = (double*)dalloc(8 * (n + 3 * (size_t)n_lm)); A.Dd = (double*)dalloc(8 * n);
    if (dry && (off > ws_cap || dev != ws_dev)) {       // grow (or move to the current device)
      if (ws_base) cudaFree(ws_base);
      ws_base = nullptr; ws_cap = 0; ws_dev = dev;
      const size_t want = off + off / 4;
      if (cudaMalloc((void**)&ws_base, want) != cudaSuccess) { ws_base = nullptr; fail = true; break; }
      ws_cap = want;
    }
  }
  int ret = PL_OK;
  if (fail) { set_error("local BA: device allocation failed"); ret = PL_ERR_CUDA; }
  else {
    k_local_ba<<<1, BA_THREADS>>>(A);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(kf_Tcw_out, A.kf_Tcw_out, 64 * (size_t)n_kf, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && n_pt && pt_Xw_out) e = cudaMemcpy(pt_Xw_out, A.pt_Xw_out, 12 * (size_t)n_pt, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && n_ln && ln_Xw_out) e = cudaMemcpy(ln_Xw_out, A.ln_Xw_out, 48 * (size_t)n_ln, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && n_pe && pe_erase) e = cudaMemcpy(pe_erase, A.pe_erase, n_pe, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && n_le && le_erase) e = cudaMemcpy(le_erase, A.le_erase, n_le, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && n_le && le_erase_kf) e = cudaMemcpy(le_erase_kf, A.le_erase_kf, 4 * (size_t)n_le, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && iterations) e = cudaMemcpy(iterations, A.iterations, 4, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { set_error("local BA: %s", cudaGetErrorString(e)); ret = PL_ERR_CUDA; }
  }
  return ret;
}
