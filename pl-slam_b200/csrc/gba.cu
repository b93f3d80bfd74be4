// Global bundle adjustment with points and line end points on sm_90a (fp64), multi-CTA.
//
// Replaces Optimizer::BundleAdjustment(vpKFs, vpMP, vpML, nIterations, pbStopFlag, nLoopKF, bRobust) of the reference
// (src/Optimizer.cc:275-638; GlobalBundleAdjustemnt :41-58 gathers the whole map and calls it) with the g2o machinery behind
// it: BlockSolver_6_3 + Schur complement (core/block_solver.hpp:353-589), OptimizationAlgorithmLevenberg
// (core/optimization_algorithm_levenberg.cpp:61-189), EdgeSE3ProjectXYZ (analytic Jacobians), EdgeLineProjectXYZ (g2o's
// numeric Jacobians, include/lineEdge.h:212-232), Huber kernels when bRobust.  Differences from the LOCAL BA the reference
// runs (ba.cu): one optimize(nIterations), no outlier rounds; Huber deltas sqrt(5.99) / sqrt(3.84) (:316-318); line
// information = identity (:278); every line edge uses the observing keyframe's own intrinsics (:472-475, :526-529);
// insertion order = point edges, then all start-point edges, then all end-point edges.
//
// ba.cu solves a local window inside ONE CTA with a dense reduced system.  The whole map does not fit that shape, so here
// every phase is its own grid-wide kernel and the host only steers the Levenberg-Marquardt loop (three scalars per trial):
//   k_gba_errors / k_gba_linearize   thread per edge
//   k_gba_lm_blocks / k_gba_hpl      thread per landmark / per (landmark, pose) block
//   k_gba_pose_blocks                warp per keyframe
//   k_gba_schur                      warp per NON-ZERO 6x6 block of the reduced pose system: the contributions of the landmarks
//                                    both keyframes observe are listed per block by the host once (the structure never changes)
//                                    and summed in landmark order - no atomics, the result is bit-reproducible
//   k_chol_potrf / trsm / syrk       right-looking blocked Cholesky of the dense reduced system, 32x32 tiles, FMA
//   k_gba_trisolve, k_gba_backsub, k_gba_update
// Sums over edges (chi2, the gain ratio's scale) are two-stage reductions with a fixed grid: deterministic as well.

#include "common.cuh"
#include "se3.cuh"
#include <algorithm>
#include <cmath>
#include <limits>
#include <vector>

namespace pl {
namespace gba {

constexpr int NB = 32;                      // Cholesky tile
constexpr int RED_BLOCKS = 296, RED_THREADS = 256;

struct G {
  int n_kf, n_pt, n_ln, n_pe, n_le, n_lm, n_edges, np, nl, n, npad, n_plb, n_blk;
  const float* kf_Tcw; const float* kf_K; const float* pt_Xw; const double* ln_Xw;
  const int* ed_kf; const int* ed_lm;       // per edge code: point edge e -> e, line edge (e, end) -> n_pe + end * n_le + e
  const float* pe_obs; const float* pe_w; const double* le_f;
  const int *lm_start, *lm_edges, *kf_start, *kf_edges;         // CSR by landmark / keyframe, edges in code (= insertion) order
  const int *pose_slot, *lm_slot;
  const int *plb_start, *plb_edges, *plb_pose, *plb_lm;         // unique (landmark, free pose) blocks Hpl, landmark-major
  const int* lm_plb_start;                                      // [nl + 1]
  const int *pose_plb_start, *pose_plb;                         // blocks of one pose, landmark order
  const int *blk_start, *blk_row, *blk_col, *ent_a, *ent_b;     // non-zero blocks of the reduced system and their contributions
  SE3 *T, *Tp, *Tm; double* X;
  double *err, *JA, *JB, *omr, *wgt, *W, *WD;
  double *Hpp, *bp, *Hll, *bl, *Dinv, *Dinvb, *Hs, *bs, *x;
  double* part; double* scal; int* flag;
  double delta_p, delta_l, info_line; int robust;
};

__device__ __forceinline__ double block_sum256(double v, double* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0;
  if (threadIdx.x == 0) for (int w = 0; w < RED_THREADS / 32; w++) s += red[w];
  __syncthreads();
  return s;                                  // valid in thread 0
}

__device__ __forceinline__ void cam_K(const G& A, int kf, double* k) { for (int i = 0; i < 4; i++) k[i] = (double)A.kf_K[4 * kf + i]; }
__device__ __forceinline__ double line_err_at(const G& A, const SE3& T, const double* X, int kf, int e) {
  double c[3], k[4];
  se3_map(T, X, c);
  cam_K(A, kf, k);
  const double u = c[0] / c[2] * k[0] + k[2], v = c[1] / c[2] * k[1] + k[3];
  return A.le_f[3 * e] * u + A.le_f[3 * e + 1] * v + A.le_f[3 * e + 2];
}

__global__ void k_gba_init(G A) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < A.n_kf) A.T[i] = se3_from_cv(A.kf_Tcw + 16 * i);
  if (i < 3 * A.n_pt) A.X[i] = (double)A.pt_Xw[i];
  if (i < 6 * A.n_ln) A.X[3 * A.n_pt + i] = A.ln_Xw[i];
}

// computeActiveErrors + activeRobustChi2: per-block partial sums (fixed grid), final sum by k_gba_reduce
__global__ void __launch_bounds__(RED_THREADS) k_gba_errors(G A) {
  __shared__ double red[RED_THREADS / 32];
  double chi = 0, r0, r1;
  for (int code = blockIdx.x * RED_THREADS + threadIdx.x; code < A.n_edges; code += RED_BLOCKS * RED_THREADS) {
    const int kf = A.ed_kf[code], lm = A.ed_lm[code];
    double c2;
    if (code < A.n_pe) {
      double c[3], k[4];
      se3_map(A.T[kf], A.X + 3 * lm, c);
      cam_K(A, kf, k);
      const double e0 = (double)A.pe_obs[2 * code] - (c[0] / c[2] * k[0] + k[2]), e1 = (double)A.pe_obs[2 * code + 1] - (c[1] / c[2] * k[1] + k[3]);
      A.err[2 * (size_t)code] = e0; A.err[2 * (size_t)code + 1] = e1;
      const double w = (double)A.pe_w[code];
      c2 = e0 * (w * e0) + e1 * (w * e1);
      if (A.robust) { huber(c2, A.delta_p, r0, r1); c2 = r0; }
    } else {
      const double er = line_err_at(A, A.T[kf], A.X + 3 * lm, kf, (code - A.n_pe) % A.n_le);
      A.err[2 * (size_t)code] = er; A.err[2 * (size_t)code + 1] = 0;
      c2 = er * (A.info_line * er);
      if (A.robust) { huber(c2, A.delta_l, r0, r1); c2 = r0; }
    }
    chi += c2;
  }
  const double s = block_sum256(chi, red);
  if (threadIdx.x == 0) A.part[blockIdx.x] = s;
}
// scale = x^T (lambda x + b) over poses and landmarks
__global__ void __launch_bounds__(RED_THREADS) k_gba_scale(G A, double lambda) {
  __shared__ double red[RED_THREADS / 32];
  double sc = 0;
  const int tot = A.n + 3 * A.nl;
  for (int i = blockIdx.x * RED_THREADS + threadIdx.x; i < tot; i += RED_BLOCKS * RED_THREADS) {
    const double b = i < A.n ? A.bp[i] : A.bl[i - A.n];
    sc += A.x[i] * (lambda * A.x[i] + b);
  }
  const double s = block_sum256(sc, red);
  if (threadIdx.x == 0) A.part[blockIdx.x] = s;
}
__global__ void __launch_bounds__(RED_THREADS) k_gba_maxdiag(G A) {
  __shared__ double red[RED_THREADS / 32];
  double md = 0;
  for (int i = blockIdx.x * RED_THREADS + threadIdx.x; i < A.n + 3 * A.nl; i += RED_BLOCKS * RED_THREADS)
    md = fmax(md, i < A.n ? fabs(A.Hpp[(size_t)(i / 6) * 36 + (i % 6) * 7]) : fabs(A.Hll[(size_t)((i - A.n) / 3) * 9 + ((i - A.n) % 3) * 4]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) md = fmax(md, __shfl_xor_sync(0xffffffffu, md, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = md;
  __syncthreads();
  if (threadIdx.x == 0) { for (int w = 0; w < RED_THREADS / 32; w++) md = fmax(md, red[w]); A.part[blockIdx.x] = md; }
}
__global__ void k_gba_reduce(G A, int slot, int is_max) {     // one thread: RED_BLOCKS partials in index order
  double s = 0;
  for (int i = 0; i < RED_BLOCKS; i++) s = is_max ? fmax(s, A.part[i]) : s + A.part[i];
  A.scal[slot] = s;
}

__global__ void k_gba_perturb(G A) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n_kf * 12) return;
  const int k = i / 12, r = i - k * 12, d = r >> 1;
  double add[6] = {0, 0, 0, 0, 0, 0};
  add[d] = (r & 1) ? -1e-9 : 1e-9;
  const SE3 Tn = se3_mul(se3_exp(add), A.T[k]);
  if (r & 1) A.Tm[k * 6 + d] = Tn; else A.Tp[k * 6 + d] = Tn;
}

__global__ void k_gba_linearize(G A) {
  const int code = blockIdx.x * blockDim.x + threadIdx.x;
  if (code >= A.n_edges) return;
  const int kf = A.ed_kf[code], lm = A.ed_lm[code];
  double* JA = A.JA + 6 * (size_t)code; double* JB = A.JB + 12 * (size_t)code;
  double r0, r1 = 1.0;
  if (code < A.n_pe) {
    const SE3 T = A.T[kf];
    double c[3], k[4], R[3][3];
    se3_map(T, A.X + 3 * lm, c); cam_K(A, kf, k); quat_to_matrix(T.r, R);
    const double x = c[0], y = c[1], z = c[2], z_2 = z * z, fx = k[0], fy = k[1];
    const double t00 = fx, t02 = -x / z * fx, t11 = fy, t12 = -y / z * fy;
    for (int j = 0; j < 3; j++) {
      JA[j] = -1. / z * (t00 * R[0][j] + t02 * R[2][j]);
      JA[3 + j] = -1. / z * (t11 * R[1][j] + t12 * R[2][j]);
    }
    JB[0] = x * y / z_2 * fx; JB[1] = -(1 + (x * x / z_2)) * fx; JB[2] = y / z * fx; JB[3] = -1. / z * fx; JB[4] = 0; JB[5] = x / z_2 * fx;
    JB[6] = (1 + y * y / z_2) * fy; JB[7] = -x * y / z_2 * fy; JB[8] = -x / z * fy; JB[9] = 0; JB[10] = -1. / z * fy; JB[11] = y / z_2 * fy;
    const double w = (double)A.pe_w[code], e0 = A.err[2 * (size_t)code], e1 = A.err[2 * (size_t)code + 1];
    double o0 = -(w * e0), o1 = -(w * e1), wg = w;
    if (A.robust) { huber(e0 * (w * e0) + e1 * (w * e1), A.delta_p, r0, r1); o0 *= r1; o1 *= r1; wg = r1 * w; }
    A.omr[2 * (size_t)code] = o0; A.omr[2 * (size_t)code + 1] = o1; A.wgt[code] = wg;
  } else {
    const int e = (code - A.n_pe) % A.n_le;
    const double* X = A.X + 3 * lm;
    for (int d = 0; d < 3; d++) {
      double Xp[3] = {X[0], X[1], X[2]}, Xm[3] = {X[0], X[1], X[2]};
      Xp[d] += 1e-9; Xm[d] += -1e-9;
      JA[d] = 5e8 * (line_err_at(A, A.T[kf], Xp, kf, e) - line_err_at(A, A.T[kf], Xm, kf, e));
    }
    for (int d = 0; d < 6; d++) JB[d] = 5e8 * (line_err_at(A, A.Tp[kf * 6 + d], X, kf, e) - line_err_at(A, A.Tm[kf * 6 + d], X, kf, e));
    const double er = A.err[2 * (size_t)code], w = A.info_line;
    double o0 = -(w * er), wg = w;
    if (A.robust) { huber(er * (w * er), A.delta_l, r0, r1); o0 *= r1; wg = r1 * w; }
    A.omr[2 * (size_t)code] = o0; A.omr[2 * (size_t)code + 1] = 0; A.wgt[code] = wg;
  }
}

__global__ void k_gba_lm_blocks(G A) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= A.n_lm) return;
  const int ls = A.lm_slot[l];
  if (ls < 0) return;
  double H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, b[3] = {0, 0, 0};
  for (int j = A.lm_start[l]; j < A.lm_start[l + 1]; j++) {
    const int code = A.lm_edges[j], dim = code < A.n_pe ? 2 : 1;
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

__global__ void k_gba_pose_blocks(G A) {     // warp per keyframe
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (k >= A.n_kf) return;
  const int ps = A.pose_slot[k];
  if (ps < 0) return;
  double acc[27];
#pragma unroll
  for (int i = 0; i < 27; i++) acc[i] = 0;
  for (int j = A.kf_start[k] + lane; j < A.kf_start[k + 1]; j += 32) {
    const int code = A.kf_edges[j], dim = code < A.n_pe ? 2 : 1;
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

// Hpl of one (landmark, pose) pair: B^T w A summed over its edges (normally one)
__global__ void k_gba_hpl(G A) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= A.n_plb) return;
  double W[18];
  for (int i = 0; i < 18; i++) W[i] = 0;
  for (int j = A.plb_start[b]; j < A.plb_start[b + 1]; j++) {
    const int code = A.plb_edges[j], dim = code < A.n_pe ? 2 : 1;
    const double *JA = A.JA + 6 * (size_t)code, *JB = A.JB + 12 * (size_t)code;
    const double wg = A.wgt[code];
    for (int a = 0; a < 6; a++) for (int c = 0; c < 3; c++) { double h = 0; for (int d = 0; d < dim; d++) h += JB[d * 6 + a] * wg * JA[d * 3 + c]; W[a * 3 + c] += h; }
  }
  for (int i = 0; i < 18; i++) A.W[(size_t)b * 18 + i] = W[i];
}

__device__ __forceinline__ void inv3(const double* D, double lambda, double* Di) {
  const double a = D[0] + lambda, b = D[1], c = D[2], d = D[3], e = D[4] + lambda, f = D[5], g = D[6], h = D[7], i = D[8] + lambda;
  const double A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
  const double id = 1.0 / (a * A + b * B + c * C);
  Di[0] = A * id; Di[1] = -(b * i - c * h) * id; Di[2] = (b * f - c * e) * id;
  Di[3] = B * id; Di[4] = (a * i - c * g) * id; Di[5] = -(a * f - c * d) * id;
  Di[6] = C * id; Di[7] = -(a * h - b * g) * id; Di[8] = (a * e - b * d) * id;
}
__global__ void k_gba_dinv(G A, double lambda) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= A.nl) return;
  double Di[9];
  inv3(A.Hll + (size_t)l * 9, lambda, Di);
  for (int i = 0; i < 9; i++) A.Dinv[(size_t)l * 9 + i] = Di[i];
  const double* bl = A.bl + (size_t)l * 3;
  for (int a = 0; a < 3; a++) A.Dinvb[(size_t)l * 3 + a] = Di[a * 3] * bl[0] + Di[a * 3 + 1] * bl[1] + Di[a * 3 + 2] * bl[2];
  for (int b = A.lm_plb_start[l]; b < A.lm_plb_start[l + 1]; b++) {
    const double* W = A.W + (size_t)b * 18;
    double* WD = A.WD + (size_t)b * 18;
    for (int a = 0; a < 6; a++) for (int c = 0; c < 3; c++) WD[a * 3 + c] = W[a * 3] * Di[c] + W[a * 3 + 1] * Di[3 + c] + W[a * 3 + 2] * Di[6 + c];
  }
}

// reduced pose system, lower block triangle: block (r, c) = [r == c](Hpp_r + lambda I) - sum_l Hpl(r,l) Dinv_l Hpl(c,l)^T
__global__ void k_gba_schur(G A, double lambda) {
  const int blk = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (blk >= A.n_blk) return;
  const int r = A.blk_row[blk], c = A.blk_col[blk];
  for (int el = lane; el < 36; el += 32) {
    const int a = el / 6, b = el % 6;
    double s = (r == c) ? A.Hpp[(size_t)r * 36 + el] + (a == b ? lambda : 0.0) : 0.0;
    for (int j = A.blk_start[blk]; j < A.blk_start[blk + 1]; j++) {
      const double* WD = A.WD + (size_t)A.ent_a[j] * 18 + a * 3;
      const double* W = A.W + (size_t)A.ent_b[j] * 18 + b * 3;
      s -= WD[0] * W[0] + WD[1] * W[1] + WD[2] * W[2];
    }
    A.Hs[(size_t)(r * 6 + a) * A.npad + c * 6 + b] = s;
  }
}
__global__ void k_gba_rhs(G A) {        // bs = bp - sum_l Hpl Dinv bl; padding rows: identity
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.npad) return;
  if (i >= A.n) { A.Hs[(size_t)i * A.npad + i] = 1.0; A.bs[i] = 0.0; return; }
  const int p = i / 6, a = i % 6;
  double s = A.bp[i];
  for (int j = A.pose_plb_start[p]; j < A.pose_plb_start[p + 1]; j++) {
    const int b = A.pose_plb[j];
    const double* W = A.W + (size_t)b * 18 + a * 3;
    const double* Db = A.Dinvb + (size_t)A.plb_lm[b] * 3;
    s -= W[0] * Db[0] + W[1] * Db[1] + W[2] * Db[2];
  }
  A.bs[i] = s;
}

// ---- blocked Cholesky (lower, row-major, leading dimension ld), right-looking: potrf(k), trsm(column k), syrk(trailing)
__global__ void __launch_bounds__(32) k_chol_potrf(double* H, int ld, int k, int* flag) {
  __shared__ double a[NB][NB + 1];
  const int lane = threadIdx.x;
  double* D = H + (size_t)k * NB * ld + (size_t)k * NB;
  for (int r = 0; r < NB; r++) a[r][lane] = D[(size_t)r * ld + lane];
  __syncwarp();
  for (int j = 0; j < NB; j++) {
    double d = a[j][j];
    if (!(d > 0.0) || !isfinite(d)) { if (lane == 0) *flag = 1; d = 1.0; }
    d = sqrt(d);
    __syncwarp();
    if (lane == j) a[j][j] = d;
    if (lane > j) a[lane][j] /= d;
    __syncwarp();
    if (lane > j) { const double lj = a[lane][j]; for (int c = j + 1; c <= lane; c++) a[lane][c] = fma(-lj, a[c][j], a[lane][c]); }
    __syncwarp();
  }
  for (int r = 0; r < NB; r++) if (lane <= r) D[(size_t)r * ld + lane] = a[r][lane];
}
__global__ void __launch_bounds__(128) k_chol_trsm(double* H, int ld, int k, int nbk) {
  __shared__ double L[NB][NB + 1];
  __shared__ double t[4][NB][NB + 1];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const double* D = H + (size_t)k * NB * ld + (size_t)k * NB;
  for (int r = w; r < NB; r += 4) L[r][lane] = D[(size_t)r * ld + lane];
  __syncthreads();
  const int tile = k + 1 + blockIdx.x * 4 + w;
  if (tile >= nbk) return;
  double* P = H + (size_t)tile * NB * ld + (size_t)k * NB;
  for (int r = 0; r < NB; r++) t[w][r][lane] = P[(size_t)r * ld + lane];
  __syncwarp();
  for (int j = 0; j < NB; j++) {      // row `lane` of the tile: x L^T = a
    double s = t[w][lane][j];
    for (int c = 0; c < j; c++) s = fma(-t[w][lane][c], L[j][c], s);
    t[w][lane][j] = s / L[j][j];
  }
  __syncwarp();
  for (int r = 0; r < NB; r++) P[(size_t)r * ld + lane] = t[w][r][lane];
}
__global__ void __launch_bounds__(256) k_chol_syrk(double* H, int ld, int k) {
  const int I = k + 1 + blockIdx.y, J = k + 1 + blockIdx.x;
  if (I < J) return;
  __shared__ double a[NB][NB + 1], b[NB][NB + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const double* PA = H + (size_t)I * NB * ld + (size_t)k * NB;
  const double* PB = H + (size_t)J * NB * ld + (size_t)k * NB;
  for (int i = threadIdx.x; i < NB * NB; i += 256) { a[i >> 5][i & 31] = PA[(size_t)(i >> 5) * ld + (i & 31)]; b[i >> 5][i & 31] = PB[(size_t)(i >> 5) * ld + (i & 31)]; }
  __syncthreads();
  double c00 = 0, c01 = 0, c10 = 0, c11 = 0;
#pragma unroll 8
  for (int m = 0; m < NB; m++) {
    const double a0 = a[ty][m], a1 = a[ty + 16][m], b0 = b[tx][m], b1 = b[tx + 16][m];
    c00 = fma(a0, b0, c00); c01 = fma(a0, b1, c01); c10 = fma(a1, b0, c10); c11 = fma(a1, b1, c11);
  }
  double* C = H + (size_t)I * NB * ld + (size_t)J * NB;
  C[(size_t)ty * ld + tx] -= c00; C[(size_t)ty * ld + tx + 16] -= c01;
  C[(size_t)(ty + 16) * ld + tx] -= c10; C[(size_t)(ty + 16) * ld + tx + 16] -= c11;
}

// L y = b, L^T x = y with the factor of the reduced system; one CTA.  Nothing is written when the factorisation failed
// (g2o keeps the previous increment in that case).
__global__ void __launch_bounds__(1024) k_gba_trisolve(G A) {
  if (*A.flag) return;
  __shared__ double L[NB][NB + 1];
  __shared__ double yk[NB];
  const int tid = threadIdx.x, lane = tid & 31, nbk = A.npad / NB, ld = A.npad;
  double* y = A.bs;
  for (int kb = 0; kb < nbk; kb++) {
    const int k0 = kb * NB;
    L[tid >> 5][lane] = A.Hs[(size_t)(k0 + (tid >> 5)) * ld + k0 + lane];
    __syncthreads();
    if (tid < 32) {
      double v = y[k0 + lane];
      for (int j = 0; j < NB; j++) {
        const double yj = __shfl_sync(0xffffffffu, v, j) / L[j][j];
        if (lane == j) v = yj;
        if (lane > j) v -= L[lane][j] * yj;
      }
      yk[lane] = v; y[k0 + lane] = v;
    }
    __syncthreads();
    for (int r = k0 + NB + tid; r < A.npad; r += 1024) {
      const double* row = A.Hs + (size_t)r * ld + k0;
      double s = 0;
#pragma unroll 8
      for (int c = 0; c < NB; c++) s = fma(row[c], yk[c], s);
      y[r] -= s;
    }
    __syncthreads();
  }
  for (int kb = nbk - 1; kb >= 0; kb--) {
    const int k0 = kb * NB;
    L[tid >> 5][lane] = A.Hs[(size_t)(k0 + (tid >> 5)) * ld + k0 + lane];
    __syncthreads();
    if (tid < 32) {
      double v = y[k0 + lane];
      for (int j = NB - 1; j >= 0; j--) {
        const double xj = __shfl_sync(0xffffffffu, v, j) / L[j][j];
        if (lane == j) v = xj;
        if (lane < j) v -= L[j][lane] * xj;
      }
      yk[lane] = v; y[k0 + lane] = v;
    }
    __syncthreads();
    for (int c = tid; c < k0; c += 1024) {
      double s = 0;
#pragma unroll 8
      for (int r = 0; r < NB; r++) s = fma(A.Hs[(size_t)(k0 + r) * ld + c], yk[r], s);
      y[c] -= s;
    }
    __syncthreads();
  }
  for (int i = tid; i < A.n; i += 1024) A.x[i] = y[i];
}
// landmark part: xl = Dinv (bl - Hpl^T xp)
__global__ void k_gba_backsub(G A) {
  if (*A.flag) return;
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= A.nl) return;
  double cl[3] = {A.bl[(size_t)l * 3], A.bl[(size_t)l * 3 + 1], A.bl[(size_t)l * 3 + 2]};
  for (int b = A.lm_plb_start[l]; b < A.lm_plb_start[l + 1]; b++) {
    const double* W = A.W + (size_t)b * 18;
    const double* xp = A.x + (size_t)A.plb_pose[b] * 6;
    for (int c = 0; c < 3; c++) { double s = 0; for (int a = 0; a < 6; a++) s += W[a * 3 + c] * xp[a]; cl[c] -= s; }
  }
  const double* Di = A.Dinv + (size_t)l * 9;
  for (int a = 0; a < 3; a++) A.x[A.n + l * 3 + a] = Di[a * 3] * cl[0] + Di[a * 3 + 1] * cl[1] + Di[a * 3 + 2] * cl[2];
}
__global__ void k_gba_update(G A) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < A.n_kf && A.pose_slot[i] >= 0) A.T[i] = se3_mul(se3_exp(A.x + (size_t)A.pose_slot[i] * 6), A.T[i]);
  if (i < A.n_lm && A.lm_slot[i] >= 0) for (int a = 0; a < 3; a++) A.X[3 * i + a] += A.x[A.n + A.lm_slot[i] * 3 + a];
}
__global__ void k_gba_finish(G A, float* kf_out, float* pt_out, double* ln_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < A.n_kf) se3_to_cv(A.T[i], kf_out + 16 * i);         // every keyframe gets SetPose(toCvMat(estimate)) (:549-556)
  if (i < A.n_pt) for (int a = 0; a < 3; a++) pt_out[3 * i + a] = A.lm_slot[i] >= 0 ? (float)A.X[3 * i + a] : A.pt_Xw[3 * i + a];
  if (i < 6 * A.n_ln) ln_out[i] = (double)(float)A.X[3 * A.n_pt + i];
}

}  // namespace gba
}  // namespace pl

using namespace pl;
using namespace pl::gba;

namespace {
inline int cdiv(long long a, int b) { return (int)((a + b - 1) / b); }
}  // namespace

extern "C" int pl_global_ba(const PLBAProblem* p, int n_iterations, int robust, const int* stop_flag_host, float* kf_Tcw_out,
                            float* pt_Xw_out, double* ln_Xw_out, int* iterations, float* solve_ms) {
  PL_ARG(p && kf_Tcw_out && p->n_kf >= 1 && p->n_pt >= 0 && p->n_ln >= 0 && p->n_pe >= 0 && p->n_le >= 0 && n_iterations >= 0);
  PL_ARG(p->kf_Tcw && p->kf_fixed && p->kf_K);
  int rc = require_device();
  if (rc) return rc;
  const int n_kf = p->n_kf, n_pt = p->n_pt, n_ln = p->n_ln, n_pe = p->n_pe, n_le = p->n_le;
  const int n_lm = n_pt + 2 * n_ln, n_edges = n_pe + 2 * n_le;
  for (int e = 0; e < n_pe; e++) PL_ARG(p->pe_kf[e] >= 0 && p->pe_kf[e] < n_kf && p->pe_pt[e] >= 0 && p->pe_pt[e] < n_pt);
  for (int e = 0; e < n_le; e++) PL_ARG(p->le_kf[e] >= 0 && p->le_kf[e] < n_kf && p->le_ln[e] >= 0 && p->le_ln[e] < n_ln);
  // ---- structure (never changes during the optimisation: no edge levels in the global BA)
  std::vector<int> ed_kf(std::max(n_edges, 1)), ed_lm(std::max(n_edges, 1));
  for (int e = 0; e < n_pe; e++) { ed_kf[e] = p->pe_kf[e]; ed_lm[e] = p->pe_pt[e]; }
  for (int end = 0; end < 2; end++) for (int e = 0; e < n_le; e++) { ed_kf[n_pe + end * n_le + e] = p->le_kf[e]; ed_lm[n_pe + end * n_le + e] = n_pt + 2 * p->le_ln[e] + end; }
  std::vector<int> lm_start(n_lm + 1, 0), kf_start(n_kf + 1, 0), lm_edges(std::max(n_edges, 1)), kf_edges(std::max(n_edges, 1));
  for (int c = 0; c < n_edges; c++) { lm_start[ed_lm[c] + 1]++; kf_start[ed_kf[c] + 1]++; }
  for (int i = 0; i < n_lm; i++) lm_start[i + 1] += lm_start[i];
  for (int i = 0; i < n_kf; i++) kf_start[i + 1] += kf_start[i];
  { std::vector<int> a(lm_start.begin(), lm_start.end() - 1), b(kf_start.begin(), kf_start.end() - 1);
    for (int c = 0; c < n_edges; c++) { lm_edges[a[ed_lm[c]]++] = c; kf_edges[b[ed_kf[c]]++] = c; } }
  std::vector<int> pose_slot(n_kf, -1), lm_slot(std::max(n_lm, 1), -1);
  int np = 0, nl = 0;
  for (int k = 0; k < n_kf; k++) if (!p->kf_fixed[k] && kf_start[k + 1] > kf_start[k]) pose_slot[k] = np++;
  for (int l = 0; l < n_lm; l++) if (lm_start[l + 1] > lm_start[l]) lm_slot[l] = nl++;
  const int n = np * 6, npad = std::max(NB, (n + NB - 1) / NB * NB), nbk = npad / NB;
  // (landmark, free pose) blocks, landmark-major; contributions to the reduced system grouped by its non-zero blocks
  std::vector<int> plb_start(1, 0), plb_edges, plb_pose, plb_lm, lm_plb_start(nl + 1, 0);
  for (int l = 0; l < n_lm; l++) {
    const int ls = lm_slot[l];
    if (ls < 0) continue;
    const size_t first = plb_pose.size();
    std::vector<std::vector<int>> ed;
    for (int j = lm_start[l]; j < lm_start[l + 1]; j++) {
      const int code = lm_edges[j], ps = pose_slot[ed_kf[code]];
      if (ps < 0) continue;
      size_t at = first;
      while (at < plb_pose.size() && plb_pose[at] != ps) at++;
      if (at == plb_pose.size()) { plb_pose.push_back(ps); plb_lm.push_back(ls); ed.emplace_back(); }
      ed[at - first].push_back(code);
    }
    for (auto& v : ed) { plb_edges.insert(plb_edges.end(), v.begin(), v.end()); plb_start.push_back((int)plb_edges.size()); }
    lm_plb_start[ls + 1] = (int)plb_pose.size();
  }
  for (int l = 0; l < nl; l++) lm_plb_start[l + 1] = std::max(lm_plb_start[l + 1], lm_plb_start[l]);
  const int n_plb = (int)plb_pose.size();
  std::vector<int> pose_plb_start(np + 1, 0), pose_plb(std::max(n_plb, 1));
  for (int b = 0; b < n_plb; b++) pose_plb_start[plb_pose[b] + 1]++;
  for (int i = 0; i < np; i++) pose_plb_start[i + 1] += pose_plb_start[i];
  { std::vector<int> a(pose_plb_start.begin(), pose_plb_start.end() - 1); for (int b = 0; b < n_plb; b++) pose_plb[a[plb_pose[b]]++] = b; }
  struct Ent { long long key; int a, b; };
  std::vector<Ent> ents;
  for (int k = 0; k < np; k++) ents.push_back({(long long)k * np + k, -1, -1});        // every diagonal block exists (Hpp + lambda)
  for (int l = 0; l < nl; l++)
    for (int i1 = lm_plb_start[l]; i1 < lm_plb_start[l + 1]; i1++)
      for (int i2 = lm_plb_start[l]; i2 < lm_plb_start[l + 1]; i2++)
        if (plb_pose[i1] >= plb_pose[i2]) ents.push_back({(long long)plb_pose[i1] * np + plb_pose[i2], i1, i2});
  std::stable_sort(ents.begin(), ents.end(), [](const Ent& x, const Ent& y) { return x.key < y.key; });
  std::vector<int> blk_start, blk_row, blk_col, ent_a, ent_b;
  for (size_t i = 0; i < ents.size(); i++) {
    if (i == 0 || ents[i].key != ents[i - 1].key) { blk_start.push_back((int)ent_a.size()); blk_row.push_back((int)(ents[i].key / np)); blk_col.push_back((int)(ents[i].key % np)); }
    if (ents[i].a >= 0) { ent_a.push_back(ents[i].a); ent_b.push_back(ents[i].b); }
  }
  const int n_blk = (int)blk_row.size();
  blk_start.push_back((int)ent_a.size());
  std::vector<Ent>().swap(ents);

  std::vector<void*> frees;
  bool fail = false;
  auto dalloc = [&](size_t bytes) -> void* { void* d = nullptr; if (cudaMalloc(&d, std::max<size_t>(bytes, 16)) != cudaSuccess) { fail = true; return nullptr; } frees.push_back(d); return d; };
  auto up = [&](const void* h, size_t bytes) -> void* { void* d = dalloc(bytes); if (d && h && bytes) cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice); return d; };
  auto upv = [&](const std::vector<int>& v) -> const int* { return (const int*)up(v.data(), 4 * v.size()); };
  G A;
  A.n_kf = n_kf; A.n_pt = n_pt; A.n_ln = n_ln; A.n_pe = n_pe; A.n_le = std::max(n_le, 1); A.n_lm = n_lm; A.n_edges = n_edges;
  A.np = np; A.nl = nl; A.n = n; A.npad = npad; A.n_plb = n_plb; A.n_blk = n_blk;
  A.kf_Tcw = (const float*)up(p->kf_Tcw, 64 * (size_t)n_kf); A.kf_K = (const float*)up(p->kf_K, 16 * (size_t)n_kf);
  A.pt_Xw = (const float*)up(p->pt_Xw, 12 * (size_t)n_pt); A.ln_Xw = (const double*)up(p->ln_Xw, 48 * (size_t)n_ln);
  A.ed_kf = upv(ed_kf); A.ed_lm = upv(ed_lm);
  A.pe_obs = (const float*)up(p->pe_obs, 8 * (size_t)n_pe); A.pe_w = (const float*)up(p->pe_inv_sigma2, 4 * (size_t)n_pe);
  A.le_f = (const double*)up(p->le_func, 24 * (size_t)n_le);
  A.lm_start = upv(lm_start); A.lm_edges = upv(lm_edges); A.kf_start = upv(kf_start); A.kf_edges = upv(kf_edges);
  A.pose_slot = upv(pose_slot); A.lm_slot = upv(lm_slot);
  if (plb_edges.empty()) plb_edges.push_back(0);
  if (plb_pose.empty()) { plb_pose.push_back(0); plb_lm.push_back(0); }
  if (ent_a.empty()) { ent_a.push_back(0); ent_b.push_back(0); }
  if (blk_row.empty()) { blk_row.push_back(0); blk_col.push_back(0); }
  A.plb_start = upv(plb_start); A.plb_edges = upv(plb_edges); A.plb_pose = upv(plb_pose); A.plb_lm = upv(plb_lm);
  A.lm_plb_start = upv(lm_plb_start); A.pose_plb_start = upv(pose_plb_start); A.pose_plb = upv(pose_plb);
  A.blk_start = upv(blk_start); A.blk_row = upv(blk_row); A.blk_col = upv(blk_col); A.ent_a = upv(ent_a); A.ent_b = upv(ent_b);
  A.T = (SE3*)dalloc(sizeof(SE3) * n_kf); SE3* Tb = (SE3*)dalloc(sizeof(SE3) * n_kf);
  A.Tp = (SE3*)dalloc(sizeof(SE3) * n_kf * 6); A.Tm = (SE3*)dalloc(sizeof(SE3) * n_kf * 6);
  A.X = (double*)dalloc(24 * (size_t)n_lm); double* Xb = (double*)dalloc(24 * (size_t)n_lm);
  A.err = (double*)dalloc(16 * (size_t)n_edges); A.JA = (double*)dalloc(48 * (size_t)n_edges); A.JB = (double*)dalloc(96 * (size_t)n_edges);
  A.omr = (double*)dalloc(16 * (size_t)n_edges); A.wgt = (double*)dalloc(8 * (size_t)n_edges);
  A.W = (double*)dalloc(144 * (size_t)std::max(n_plb, 1)); A.WD = (double*)dalloc(144 * (size_t)std::max(n_plb, 1));
  A.Hpp = (double*)dalloc(288 * (size_t)std::max(np, 1)); A.bp = (double*)dalloc(48 * (size_t)std::max(np, 1));
  A.Hll = (double*)dalloc(72 * (size_t)std::max(nl, 1)); A.bl = (double*)dalloc(24 * (size_t)std::max(nl, 1));
  A.Dinv = (double*)dalloc(72 * (size_t)std::max(nl, 1)); A.Dinvb = (double*)dalloc(24 * (size_t)std::max(nl, 1));
  A.Hs = (double*)dalloc(8 * (size_t)npad * npad); A.bs = (double*)dalloc(8 * (size_t)npad);
  A.x = (double*)dalloc(8 * ((size_t)n + 3 * (size_t)nl + 8));
  A.part = (double*)dalloc(8 * RED_BLOCKS); A.scal = (double*)dalloc(64); A.flag = (int*)dalloc(4);
  float* d_kf_out = (float*)dalloc(64 * (size_t)n_kf); float* d_pt_out = (float*)dalloc(12 * (size_t)n_pt); double* d_ln_out = (double*)dalloc(48 * (size_t)n_ln);
  A.robust = robust ? 1 : 0; A.info_line = 1.0;
  A.delta_p = (double)(float)std::sqrt(5.99); A.delta_l = (double)(float)std::sqrt(3.84);
  int ret = PL_OK, done = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  auto terminate = [&]() { return stop_flag_host && *(volatile const int*)stop_flag_host; };
  auto sum_to = [&](int slot, int is_max) { k_gba_reduce<<<1, 1>>>(A, slot, is_max); count_launch(); };
  auto chi2 = [&](double& out) -> cudaError_t {
    k_gba_errors<<<RED_BLOCKS, RED_THREADS>>>(A); sum_to(0, 0); count_launch();
    return cudaMemcpy(&out, A.scal, 8, cudaMemcpyDeviceToHost);
  };
  if (fail) { set_error("global BA: device allocation failed (reduced system %d x %d)", npad, npad); ret = PL_ERR_CUDA; }
  else {
    cudaError_t e = cudaSuccess;
    cudaEventCreate(&ev0); cudaEventCreate(&ev1);
    cudaEventRecord(ev0, 0);
    const int big = std::max(std::max(n_kf * 12, 3 * n_pt), std::max(6 * n_ln, std::max(n_lm, n_edges)));
    k_gba_init<<<cdiv(big, 256), 256>>>(A); count_launch();
    cudaMemset(A.x, 0, 8 * ((size_t)n + 3 * (size_t)nl + 8));
    double lambda = 0, ni = 2;
    int nBad = 0;
    for (int it = 0; it < n_iterations && !terminate() && e == cudaSuccess && np + nl > 0; it++) {
      done++;
      double currentChi = 0;
      e = chi2(currentChi);
      if (e != cudaSuccess) break;
      const double iniChi = currentChi;
      double tempChi = currentChi;
      if (n_le > 0) { k_gba_perturb<<<cdiv(n_kf * 12, 128), 128>>>(A); count_launch(); }
      k_gba_linearize<<<cdiv(n_edges, 128), 128>>>(A);
      k_gba_lm_blocks<<<cdiv(n_lm, 128), 128>>>(A);
      k_gba_pose_blocks<<<cdiv((long long)n_kf * 32, 128), 128>>>(A);
      if (n_plb) k_gba_hpl<<<cdiv(n_plb, 128), 128>>>(A);
      count_launch(4);
      if (it == 0) {
        k_gba_maxdiag<<<RED_BLOCKS, RED_THREADS>>>(A); sum_to(2, 1); count_launch();
        double md = 0;
        e = cudaMemcpy(&md, A.scal + 2, 8, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) break;
        lambda = 1e-5 * md; ni = 2; nBad = 0;
      }
      double rho = 0;
      int qmax = 0;
      do {
        cudaMemcpyAsync(Tb, A.T, sizeof(SE3) * n_kf, cudaMemcpyDeviceToDevice, 0);
        cudaMemcpyAsync(Xb, A.X, 24 * (size_t)n_lm, cudaMemcpyDeviceToDevice, 0);
        cudaMemsetAsync(A.Hs, 0, 8 * (size_t)npad * npad, 0);
        cudaMemsetAsync(A.flag, 0, 4, 0);
        if (nl) { k_gba_dinv<<<cdiv(nl, 128), 128>>>(A, lambda); count_launch(); }
        if (np) {
          k_gba_schur<<<cdiv((long long)n_blk * 32, 128), 128>>>(A, lambda);
          k_gba_rhs<<<cdiv(npad, 128), 128>>>(A);
          count_launch(2);
          for (int k = 0; k < nbk; k++) {
            k_chol_potrf<<<1, 32>>>(A.Hs, npad, k, A.flag);
            count_launch();
            const int m = nbk - k - 1;
            if (m > 0) {
              k_chol_trsm<<<cdiv(m, 4), 128>>>(A.Hs, npad, k, nbk);
              k_chol_syrk<<<dim3(m, m), 256>>>(A.Hs, npad, k);
              count_launch(2);
            }
          }
          k_gba_trisolve<<<1, 1024>>>(A); count_launch();
        }
        if (nl) { k_gba_backsub<<<cdiv(nl, 128), 128>>>(A); count_launch(); }
        k_gba_update<<<cdiv(std::max(n_kf, n_lm), 128), 128>>>(A); count_launch();
        k_gba_errors<<<RED_BLOCKS, RED_THREADS>>>(A); sum_to(0, 0);
        k_gba_scale<<<RED_BLOCKS, RED_THREADS>>>(A, lambda); sum_to(1, 0);
        count_launch(2);
        double sc[2]; int bad = 0;
        e = cudaMemcpy(sc, A.scal, 16, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(&bad, A.flag, 4, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) break;
        tempChi = bad ? std::numeric_limits<double>::max() : sc[0];
        rho = (currentChi - tempChi) / (sc[1] + 1e-3);
        if (rho > 0 && std::isfinite(tempChi)) {
          double alpha = 1. - std::pow((2 * rho - 1), 3);
          alpha = std::min(alpha, 2. / 3.);
          lambda *= std::max(1. / 3., alpha); ni = 2; currentChi = tempChi;
        } else {
          lambda *= ni; ni *= 2;
          cudaMemcpyAsync(A.T, Tb, sizeof(SE3) * n_kf, cudaMemcpyDeviceToDevice, 0);
          cudaMemcpyAsync(A.X, Xb, 24 * (size_t)n_lm, cudaMemcpyDeviceToDevice, 0);
        }
        qmax++;
      } while (rho < 0 && qmax < 10 && !terminate());
      if (e != cudaSuccess) break;
      if (qmax == 10 || rho == 0) break;
      if ((iniChi - currentChi) * 1e3 < iniChi) nBad++; else nBad = 0;
      if (nBad >= 3) break;
    }
    if (e == cudaSuccess) {
      k_gba_finish<<<cdiv(std::max(std::max(n_kf, n_pt), 6 * n_ln), 128), 128>>>(A, d_kf_out, d_pt_out, d_ln_out); count_launch();
      cudaEventRecord(ev1, 0);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(kf_Tcw_out, d_kf_out, 64 * (size_t)n_kf, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && n_pt && pt_Xw_out) e = cudaMemcpy(pt_Xw_out, d_pt_out, 12 * (size_t)n_pt, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && n_ln && ln_Xw_out) e = cudaMemcpy(ln_Xw_out, d_ln_out, 48 * (size_t)n_ln, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && solve_ms) cudaEventElapsedTime(solve_ms, ev0, ev1);
    if (e != cudaSuccess) { set_error("global BA: %s", cudaGetErrorString(e)); ret = PL_ERR_CUDA; }
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
  }
  if (iterations) *iterations = done;
  for (void* d : frees) cudaFree(d);
  return ret;
}
