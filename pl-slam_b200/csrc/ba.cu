// Local bundle adjustment with points and line end-points on sm_90a (fp64).
//
// Replaces Optimizer::LocalBundleAdjustmentWithLine (reference src/Optimizer.cc:1645-2100; the points-only twin
// :1308-1642 is the n_line_edges == 0 case) together with the g2o machinery it drives: BlockSolver_6_3 with the Schur
// complement over the marginalised landmarks (core/block_solver.hpp:353-486,501-589), OptimizationAlgorithmLevenberg
// (core/optimization_algorithm_levenberg.cpp:61-189), EdgeSE3ProjectXYZ (types/types_six_dof_expmap.cpp:103-139),
// EdgeLineProjectXYZ with g2o's numeric Jacobians (include/lineEdge.h:212-232, core/base_binary_edge.hpp:130-205),
// Huber kernels, and the reference's outlier gating / erase lists (Optimizer.cc:1957-2043).
//
// One persistent CTA (512 threads) runs a whole problem (a window; a launch runs W of them, blockIdx.x = window): no graph
// objects, edges are flat arrays with two CSR indices (by landmark, by keyframe) that the CTA builds first.  Per LM iteration: residuals + per-edge Jacobians
// (thread per edge), landmark blocks Hll/bl (thread per landmark, fixed edge order), pose blocks Hpp/bp (warp per
// keyframe, fixed order), then per trial: 3x3 inverses, Schur complement accumulated per landmark into the dense
// reduced pose system (fp64 atomics), in-CTA dense LDL^T, landmark back-substitution, state update, step control.
// A different keyframe's LBA is an independent problem ("replicas only" across GPUs, SURVEY.md §8e).

#include "common.cuh"
#include <mutex>
#include "g2o.cuh"
#include <algorithm>
#include <climits>

namespace pl {

constexpr int BA_THREADS = 512, BA_WARPS = BA_THREADS / 32;

// Byte offsets of one window's scratch, from the capacities; windows are `window` bytes apart.
struct BALayout {
  size_t cur_lm, cur_kf, rank_lm, rank_kf, lm_start, lm_edges, kf_start, kf_edges, T, Tb, Tp, Tm, X, Xb, err, lvl, JA, JB, omr, wgt,
         pose_slot, lm_slot, Hpp, bp, Hll, bl, Dinv, Dinvb, Hs, bs, x, Dd, window;
};
// cap_free bounds the window's free keyframes: the reduced system (n = 6 cap_free) and the pose blocks.
static BALayout ba_layout(int cap_kf, int cap_free, int cap_pt, int cap_ln, int cap_pe, int cap_le) {
  const size_t kf = cap_kf, lm = cap_pt + 2 * (size_t)cap_ln, e = cap_pe + 2 * (size_t)cap_le, le = cap_pe + (size_t)cap_le;
  const size_t n = 6 * (size_t)cap_free;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  BALayout L;
  L.cur_lm = take(4 * BA_WARPS * lm); L.cur_kf = take(4 * BA_WARPS * kf); L.rank_lm = take(4 * e); L.rank_kf = take(4 * e);
  L.lm_start = take(4 * (lm + 1)); L.lm_edges = take(4 * e); L.kf_start = take(4 * (kf + 1)); L.kf_edges = take(4 * e);
  L.T = take(sizeof(SE3) * kf); L.Tb = take(sizeof(SE3) * kf); L.Tp = take(sizeof(SE3) * kf * 6); L.Tm = take(sizeof(SE3) * kf * 6);
  L.X = take(24 * lm); L.Xb = take(24 * lm); L.err = take(16 * le); L.lvl = take(le);
  L.JA = take(48 * e); L.JB = take(96 * e); L.omr = take(16 * e); L.wgt = take(8 * e);
  L.pose_slot = take(4 * kf); L.lm_slot = take(4 * lm);
  L.Hpp = take(288 * (size_t)cap_free); L.bp = take(48 * (size_t)cap_free); L.Hll = take(72 * lm); L.bl = take(24 * lm); L.Dinv = take(72 * lm); L.Dinvb = take(24 * lm);
  L.Hs = take(8 * n * n); L.bs = take(8 * n); L.x = take(8 * (n + 3 * lm)); L.Dd = take(8 * n);
  L.window = off;
  return L;
}

struct BABatch {
  PLBAWindows P; PLBAOut O; const volatile int* stop; char* scratch; BALayout L;
};

// Window blockIdx.x of a launch: its counts (in shared memory), and its rows of the inputs and outputs and its scratch, each
// pointer computed where it is used from the launch's parameters, which stay in the constant bank.
// Edge code: point edge e -> e, line edge (e, end) -> n_pe + 2e + end.  CSR by landmark (lm_start, lm_edges) and by keyframe
// (kf_start, kf_edges); CSR build: cur_lm [BA_WARPS][n_lm], cur_kf [BA_WARPS][n_kf], rank_lm / rank_kf [n_edges].  Scratch
// sizes: T, Tb [n_kf]; Tp, Tm [n_kf*6]; X, Xb [n_lm*3]; err [n_pe*2 + n_le*2]; lvl [n_pe + n_le]; per edge code JA [6], JB [12],
// omr [2], wgt; Hs [n*n], bs [n], x [n + nl*3], Dd [n].
struct BAArgs {
  const BABatch& B;
  const int* cnt;
  __device__ __forceinline__ int w() const { return blockIdx.x; }
  __device__ __forceinline__ size_t rk() const { return (size_t)(w() * B.P.cap_kf); }
  __device__ __forceinline__ size_t rp() const { return (size_t)(w() * B.P.cap_pt); }
  __device__ __forceinline__ size_t rl() const { return (size_t)(w() * B.P.cap_ln); }
  __device__ __forceinline__ size_t rpe() const { return (size_t)(w() * B.P.cap_pe); }
  __device__ __forceinline__ size_t rle() const { return (size_t)(w() * B.P.cap_le); }
  template <typename V> __device__ __forceinline__ V* ws(size_t off) const { return (V*)(B.scratch + (size_t)w() * B.L.window + off); }
  __device__ __forceinline__ int n_kf() const { return cnt[0]; }
  __device__ __forceinline__ int n_pt() const { return cnt[1]; }
  __device__ __forceinline__ int n_ln() const { return cnt[2]; }
  __device__ __forceinline__ int n_pe() const { return cnt[3]; }
  __device__ __forceinline__ int n_le() const { return cnt[4]; }
  __device__ __forceinline__ const float* kf_Tcw() const { return B.P.kf_Tcw + 16 * rk(); }
  __device__ __forceinline__ const uint8_t* kf_fixed() const { return B.P.kf_fixed + rk(); }
  __device__ __forceinline__ const float* kf_K() const { return B.P.kf_K + 4 * rk(); }
  __device__ __forceinline__ const float* K_end() const { return B.P.K_end + 4 * (size_t)w(); }
  __device__ __forceinline__ const float* pt_Xw() const { return B.P.pt_Xw + 3 * rp(); }
  __device__ __forceinline__ const double* ln_Xw() const { return B.P.ln_Xw + 6 * rl(); }
  __device__ __forceinline__ const int* pe_kf() const { return B.P.pe_kf + rpe(); }
  __device__ __forceinline__ const int* pe_pt() const { return B.P.pe_pt + rpe(); }
  __device__ __forceinline__ const float* pe_obs() const { return B.P.pe_obs + 2 * rpe(); }
  __device__ __forceinline__ const float* pe_w() const { return B.P.pe_inv_sigma2 + rpe(); }
  __device__ __forceinline__ const int* le_kf() const { return B.P.le_kf + rle(); }
  __device__ __forceinline__ const int* le_ln() const { return B.P.le_ln + rle(); }
  __device__ __forceinline__ const double* le_f() const { return B.P.le_func + 3 * rle(); }
  __device__ __forceinline__ const volatile int* stop() const { return B.stop; }
  __device__ __forceinline__ float* kf_Tcw_out() const { return B.O.kf_Tcw + 16 * rk(); }
  __device__ __forceinline__ float* pt_Xw_out() const { return B.O.pt_Xw + 3 * rp(); }
  __device__ __forceinline__ double* ln_Xw_out() const { return B.O.ln_Xw + 6 * rl(); }
  __device__ __forceinline__ uint8_t* pe_erase() const { return B.O.pe_erase + rpe(); }
  __device__ __forceinline__ uint8_t* le_erase() const { return B.O.le_erase + rle(); }
  __device__ __forceinline__ int* le_erase_kf() const { return B.O.le_erase_kf + rle(); }
  __device__ __forceinline__ int* iterations() const { return B.O.iterations + w(); }
  __device__ __forceinline__ int* cur_lm() const { return ws<int>(B.L.cur_lm); }
  __device__ __forceinline__ int* cur_kf() const { return ws<int>(B.L.cur_kf); }
  __device__ __forceinline__ int* rank_lm() const { return ws<int>(B.L.rank_lm); }
  __device__ __forceinline__ int* rank_kf() const { return ws<int>(B.L.rank_kf); }
  __device__ __forceinline__ int* lm_start() const { return ws<int>(B.L.lm_start); }
  __device__ __forceinline__ int* lm_edges() const { return ws<int>(B.L.lm_edges); }
  __device__ __forceinline__ int* kf_start() const { return ws<int>(B.L.kf_start); }
  __device__ __forceinline__ int* kf_edges() const { return ws<int>(B.L.kf_edges); }
  __device__ __forceinline__ SE3* T() const { return ws<SE3>(B.L.T); }
  __device__ __forceinline__ SE3* Tb() const { return ws<SE3>(B.L.Tb); }
  __device__ __forceinline__ SE3* Tp() const { return ws<SE3>(B.L.Tp); }
  __device__ __forceinline__ SE3* Tm() const { return ws<SE3>(B.L.Tm); }
  __device__ __forceinline__ double* X() const { return ws<double>(B.L.X); }
  __device__ __forceinline__ double* Xb() const { return ws<double>(B.L.Xb); }
  __device__ __forceinline__ double* err() const { return ws<double>(B.L.err); }
  __device__ __forceinline__ uint8_t* lvl() const { return ws<uint8_t>(B.L.lvl); }
  __device__ __forceinline__ uint8_t& edge_lvl(int c) const { return lvl()[c < n_pe() ? c : n_pe() + ((c - n_pe()) >> 1)]; }   // by edge code
  __device__ __forceinline__ double* JA() const { return ws<double>(B.L.JA); }
  __device__ __forceinline__ double* JB() const { return ws<double>(B.L.JB); }
  __device__ __forceinline__ double* omr() const { return ws<double>(B.L.omr); }
  __device__ __forceinline__ double* wgt() const { return ws<double>(B.L.wgt); }
  __device__ __forceinline__ int* pose_slot() const { return ws<int>(B.L.pose_slot); }
  __device__ __forceinline__ int* lm_slot() const { return ws<int>(B.L.lm_slot); }
  __device__ __forceinline__ double* Hpp() const { return ws<double>(B.L.Hpp); }
  __device__ __forceinline__ double* bp() const { return ws<double>(B.L.bp); }
  __device__ __forceinline__ double* Hll() const { return ws<double>(B.L.Hll); }
  __device__ __forceinline__ double* bl() const { return ws<double>(B.L.bl); }
  __device__ __forceinline__ double* Dinv() const { return ws<double>(B.L.Dinv); }
  __device__ __forceinline__ double* Dinvb() const { return ws<double>(B.L.Dinvb); }
  __device__ __forceinline__ double* Hs() const { return ws<double>(B.L.Hs); }
  __device__ __forceinline__ double* bs() const { return ws<double>(B.L.bs); }
  __device__ __forceinline__ double* x() const { return ws<double>(B.L.x); }
  __device__ __forceinline__ double* Dd() const { return ws<double>(B.L.Dd); }
};

struct BAShared {
  double red[BA_WARPS];
  int wsum[BA_WARPS];
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
__device__ __forceinline__ void edge_decode(const BAArgs& A, int code, int& kf, int& lm, int& dim, int& e, int& end) {
  if (code < A.n_pe()) { e = code; end = 0; dim = 2; kf = A.pe_kf()[e]; lm = A.pe_pt()[e]; }
  else { const int c = code - A.n_pe(); e = c >> 1; end = c & 1; dim = 1; kf = A.le_kf()[e]; lm = A.n_pt() + 2 * A.le_ln()[e] + end; }
}
__device__ __forceinline__ void cam_K(const BAArgs& A, int kf, int end_edge, double* k) {
  if (end_edge) { for (int i = 0; i < 4; i++) k[i] = (double)A.K_end()[i]; }
  else { for (int i = 0; i < 4; i++) k[i] = (double)A.kf_K()[4 * kf + i]; }
}

__device__ __forceinline__ int edge_lm(const BAArgs& A, int c) {
  return c < A.n_pe() ? A.pe_pt()[c] : A.n_pt() + 2 * A.le_ln()[(c - A.n_pe()) >> 1] + ((c - A.n_pe()) & 1);
}
__device__ __forceinline__ int edge_kf(const BAArgs& A, int c) { return c < A.n_pe() ? A.pe_kf()[c] : A.le_kf()[(c - A.n_pe()) >> 1]; }

// computeActiveErrors + activeRobustChi2
__device__ double errors_and_chi2(const BAArgs& A, BAShared& S, bool p_robust, bool l_robust, int tid) {
  const double kDeltaMono = huber_delta_mono(), kDeltaLine = huber_delta_line();
  double chi = 0, r0, r1;
  for (int e = tid; e < A.n_pe(); e += BA_THREADS) if (!A.lvl()[e]) {
    double k[4], e0, e1;
    cam_K(A, A.pe_kf()[e], 0, k);
    proj_error(A.T()[A.pe_kf()[e]], A.X() + 3 * A.pe_pt()[e], k, (double)A.pe_obs()[2 * e], (double)A.pe_obs()[2 * e + 1], e0, e1);
    A.err()[2 * e] = e0; A.err()[2 * e + 1] = e1;
    const double w = (double)A.pe_w()[e], c2 = e0 * (w * e0) + e1 * (w * e1);
    if (p_robust) { huber(c2, kDeltaMono, r0, r1); chi += r0; } else chi += c2;
  }
  for (int e = tid; e < A.n_le(); e += BA_THREADS) if (!A.lvl()[A.n_pe() + e])
    for (int end = 0; end < 2; end++) {
      double k[4];
      cam_K(A, A.le_kf()[e], end, k);
      const double er = line_error(A.T()[A.le_kf()[e]], A.X() + 3 * (A.n_pt() + 2 * A.le_ln()[e] + end), k, A.le_f() + 3 * e);
      A.err()[2 * A.n_pe() + 2 * e + end] = er;
      const double c2 = er * (0.5 * er);
      if (l_robust) { huber(c2, kDeltaLine, r0, r1); chi += r0; } else chi += c2;
    }
  return block_sum(S, chi, tid);
}

// one optimizer.optimize(iterations) call on the level-0 edges.  (Unlike k_pose_opt, this kernel is ONE CTA per problem with the SM
// to itself: keeping the LM loops rolled and this function out of line shrinks it from 81 k to 21 k SASS instructions but makes
// the 20+40-keyframe window markedly slower, so the inlined, unrolled form stays.)
__device__ int ba_optimize(const BAArgs& A, BAShared& S, int iterations, bool p_robust, bool l_robust, int tid) {
  const double kDeltaMono = huber_delta_mono(), kDeltaLine = huber_delta_line();
  const int n_lm = A.n_pt() + 2 * A.n_ln(), n_edges = A.n_pe() + 2 * A.n_le();
  // ---- active sets and slots (initializeOptimization)
  for (int k = tid; k < A.n_kf(); k += BA_THREADS) {
    int act = 0;
    for (int j = A.kf_start()[k]; j < A.kf_start()[k + 1] && !act; j++) act = !A.edge_lvl(A.kf_edges()[j]);
    A.pose_slot()[k] = (act && !A.kf_fixed()[k]) ? 1 : -1;
  }
  for (int l = tid; l < n_lm; l += BA_THREADS) {
    int act = 0;
    for (int j = A.lm_start()[l]; j < A.lm_start()[l + 1] && !act; j++) act = !A.edge_lvl(A.lm_edges()[j]);
    A.lm_slot()[l] = act ? 1 : -1;
  }
  __syncthreads();
  if (tid == 0) {
    int np = 0, nl = 0;
    for (int k = 0; k < A.n_kf(); k++) if (A.pose_slot()[k] > 0) A.pose_slot()[k] = np++;
    for (int l = 0; l < n_lm; l++) if (A.lm_slot()[l] > 0) A.lm_slot()[l] = nl++;
    S.np = np; S.nl = nl;
  }
  __syncthreads();
  const int np = S.np, nl = S.nl, n = np * 6;
  if (np + nl == 0) return 0;
  for (int i = tid; i < n + nl * 3; i += BA_THREADS) A.x()[i] = 0.0;
  int done = 0;
  for (int it = 0; it < iterations; it++) {
    if (A.stop() && *A.stop()) break;                       // SparseOptimizer::terminate()
    done++;
    const double chi0 = errors_and_chi2(A, S, p_robust, l_robust, tid);
    if (tid == 0) { S.currentChi = chi0; S.iniChi = chi0; }
    // ---- perturbed poses for the numeric (line) Jacobians
    if (A.n_le() > 0)
      for (int i = tid; i < A.n_kf() * 12; i += BA_THREADS) {
        const int k = i / 12, r = i - k * 12;
        const SE3 Tn = perturbed_pose(A.T()[k], r);
        if (r & 1) A.Tm()[k * 6 + (r >> 1)] = Tn; else A.Tp()[k * 6 + (r >> 1)] = Tn;
      }
    __syncthreads();
    // ---- per-edge linearisation
    for (int code = tid; code < n_edges; code += BA_THREADS) {
      int kf, lm, dim, e, end;
      edge_decode(A, code, kf, lm, dim, e, end);
      if (A.edge_lvl(code)) continue;
      double* JA = A.JA() + 6 * (size_t)code; double* JB = A.JB() + 12 * (size_t)code;
      double k[4], omr[2], wg;
      cam_K(A, kf, end, k);
      if (dim == 2) {
        proj_jacobians(A.T()[kf], A.X() + 3 * lm, k, JA, JB);
        edge_weights(2, (double)A.pe_w()[e], A.err() + 2 * e, p_robust, kDeltaMono, omr, wg);
      } else {
        line_point_jacobian(A.T()[kf], A.X() + 3 * lm, k, A.le_f() + 3 * e, JA);
        line_pose_jacobian(A.Tp() + kf * 6, A.Tm() + kf * 6, A.X() + 3 * lm, k, A.le_f() + 3 * e, JB);
        edge_weights(1, 0.5, A.err() + 2 * A.n_pe() + 2 * e + end, l_robust, kDeltaLine, omr, wg);
      }
      A.omr()[2 * (size_t)code] = omr[0]; A.omr()[2 * (size_t)code + 1] = omr[1]; A.wgt()[code] = wg;
    }
    __syncthreads();
    // ---- landmark blocks (thread per landmark, edges in CSR order)
    for (int l = tid; l < n_lm; l += BA_THREADS) {
      const int ls = A.lm_slot()[l];
      if (ls < 0) continue;
      double H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, b[3] = {0, 0, 0};
      for (int j = A.lm_start()[l]; j < A.lm_start()[l + 1]; j++) {
        const int code = A.lm_edges()[j];
        if (A.edge_lvl(code)) continue;
        add_landmark_block(code < A.n_pe() ? 2 : 1, A.JA() + 6 * (size_t)code, A.omr() + 2 * (size_t)code, A.wgt()[code], H, b);
      }
      for (int i = 0; i < 9; i++) A.Hll()[(size_t)ls * 9 + i] = H[i];
      for (int i = 0; i < 3; i++) A.bl()[(size_t)ls * 3 + i] = b[i];
    }
    // ---- pose blocks (warp per keyframe)
    for (int k = tid >> 5; k < A.n_kf(); k += BA_THREADS / 32) {
      const int ps = A.pose_slot()[k];
      if (ps < 0) continue;
      const int lane = tid & 31;
      double acc[27];
#pragma unroll
      for (int i = 0; i < 27; i++) acc[i] = 0;
      for (int j = A.kf_start()[k] + lane; j < A.kf_start()[k + 1]; j += 32) {
        const int code = A.kf_edges()[j];
        if (A.edge_lvl(code)) continue;
        add_pose_block(code < A.n_pe() ? 2 : 1, A.JB() + 12 * (size_t)code, A.omr() + 2 * (size_t)code, A.wgt()[code], acc);
      }
#pragma unroll
      for (int i = 0; i < 27; i++) acc[i] = warp_sum(acc[i]);
      if (lane == 0) {
        int q = 0;
        for (int a = 0; a < 6; a++) for (int c = a; c < 6; c++) { A.Hpp()[(size_t)ps * 36 + a * 6 + c] = acc[q]; A.Hpp()[(size_t)ps * 36 + c * 6 + a] = acc[q]; q++; }
        for (int a = 0; a < 6; a++) A.bp()[(size_t)ps * 6 + a] = acc[21 + a];
      }
    }
    __syncthreads();
    if (it == 0) {
      double md = 0;
      for (int i = tid; i < np * 6; i += BA_THREADS) md = fmax(md, fabs(A.Hpp()[(size_t)(i / 6) * 36 + (i % 6) * 7]));
      for (int i = tid; i < nl * 3; i += BA_THREADS) md = fmax(md, fabs(A.Hll()[(size_t)(i / 3) * 9 + (i % 3) * 4]));
      md = block_max(S, md, tid);
      if (tid == 0) lm_init(md, S.lambda, S.ni, S.nBad);
    }
    if (tid == 0) { S.rho = 0; S.qmax = 0; }
    __syncthreads();
    // ---- trial steps
    while (true) {
      const double lambda = S.lambda;
      for (int k = tid; k < A.n_kf(); k += BA_THREADS) A.Tb()[k] = A.T()[k];
      for (int i = tid; i < n_lm * 3; i += BA_THREADS) A.Xb()[i] = A.X()[i];
      for (int l = tid; l < nl; l += BA_THREADS) {
        double Di[9];
        inv3(A.Hll() + (size_t)l * 9, lambda, Di);
        for (int i = 0; i < 9; i++) A.Dinv()[(size_t)l * 9 + i] = Di[i];
        for (int a = 0; a < 3; a++) A.Dinvb()[(size_t)l * 3 + a] = Di[a * 3] * A.bl()[(size_t)l * 3] + Di[a * 3 + 1] * A.bl()[(size_t)l * 3 + 1] + Di[a * 3 + 2] * A.bl()[(size_t)l * 3 + 2];
      }
      for (int i = tid; i < n * n; i += BA_THREADS) A.Hs()[i] = 0.0;
      __syncthreads();
      for (int i = tid; i < np * 36; i += BA_THREADS) {
        const int p = i / 36, a = (i % 36) / 6, c = i % 6;
        A.Hs()[(size_t)(p * 6 + a) * n + p * 6 + c] = A.Hpp()[i] + (a == c ? lambda : 0.0);
      }
      for (int i = tid; i < n; i += BA_THREADS) A.bs()[i] = A.bp()[i];
      __syncthreads();
      // Schur complement, one thread per landmark
      for (int l = tid; l < n_lm; l += BA_THREADS) {
        const int ls = A.lm_slot()[l];
        if (ls < 0) continue;
        const double* Di = A.Dinv() + (size_t)ls * 9;
        const double* Db = A.Dinvb() + (size_t)ls * 3;
        for (int j1 = A.lm_start()[l]; j1 < A.lm_start()[l + 1]; j1++) {
          const int c1 = A.lm_edges()[j1];
          if (A.edge_lvl(c1)) continue;
          const int p1 = A.pose_slot()[edge_kf(A, c1)];
          if (p1 < 0) continue;
          double B1[18], BD[18];   // Hpl block (6x3); BD = Hpl * Dinv
          hpl_block(c1 < A.n_pe() ? 2 : 1, A.JA() + 6 * (size_t)c1, A.JB() + 12 * (size_t)c1, A.wgt()[c1], B1);
          for (int a = 0; a < 6; a++) for (int c = 0; c < 3; c++) BD[a * 3 + c] = B1[a * 3] * Di[c] + B1[a * 3 + 1] * Di[3 + c] + B1[a * 3 + 2] * Di[6 + c];
          for (int a = 0; a < 6; a++) atomicAdd(&A.bs()[p1 * 6 + a], -(B1[a * 3] * Db[0] + B1[a * 3 + 1] * Db[1] + B1[a * 3 + 2] * Db[2]));
          for (int j2 = A.lm_start()[l]; j2 < A.lm_start()[l + 1]; j2++) {
            const int c2 = A.lm_edges()[j2];
            if (A.edge_lvl(c2)) continue;
            const int p2 = A.pose_slot()[edge_kf(A, c2)];
            if (p2 < 0) continue;
            const int d2 = c2 < A.n_pe() ? 2 : 1;
            const double *JA2 = A.JA() + 6 * (size_t)c2, *JB2 = A.JB() + 12 * (size_t)c2;
            const double w2 = A.wgt()[c2];
            for (int a = 0; a < 6; a++)
              for (int c = 0; c < 6; c++) {
                double s = 0;
                for (int m = 0; m < 3; m++) s += BD[a * 3 + m] * hpl_entry(d2, JA2, JB2, w2, c, m);
                atomicAdd(&A.Hs()[(size_t)(p1 * 6 + a) * n + p2 * 6 + c], -s);
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
          double d = A.Hs()[(size_t)j * n + j];
          for (int k = 0; k < j; k++) d -= A.Hs()[(size_t)j * n + k] * A.Hs()[(size_t)j * n + k] * A.Dd()[k];
          if (d == 0 || !isfinite(d)) S.ok2 = 0;
          A.Dd()[j] = d;
        }
        __syncthreads();
        if (!S.ok2) break;
        const double d = A.Dd()[j];
        for (int i = j + 1 + tid; i < n; i += BA_THREADS) {
          double s = A.Hs()[(size_t)i * n + j];
          for (int k = 0; k < j; k++) s -= A.Hs()[(size_t)i * n + k] * A.Hs()[(size_t)j * n + k] * A.Dd()[k];
          A.Hs()[(size_t)i * n + j] = s / d;
        }
        __syncthreads();
      }
      if (S.ok2 && tid == 0) {   // triangular solves (n is a few hundred at most)
        double* y = A.bs();        // in place
        for (int i = 0; i < n; i++) { double s = y[i]; for (int k = 0; k < i; k++) s -= A.Hs()[(size_t)i * n + k] * y[k]; y[i] = s; }
        for (int i = 0; i < n; i++) y[i] /= A.Dd()[i];
        for (int i = n - 1; i >= 0; i--) { double s = y[i]; for (int k = i + 1; k < n; k++) s -= A.Hs()[(size_t)k * n + i] * A.x()[k]; A.x()[i] = s; }
      }
      __syncthreads();
      if (S.ok2) {   // landmark part: xl = Dinv (bl - Hpl^T xp)
        for (int l = tid; l < n_lm; l += BA_THREADS) {
          const int ls = A.lm_slot()[l];
          if (ls < 0) continue;
          double cl[3] = {A.bl()[(size_t)ls * 3], A.bl()[(size_t)ls * 3 + 1], A.bl()[(size_t)ls * 3 + 2]};
          for (int j1 = A.lm_start()[l]; j1 < A.lm_start()[l + 1]; j1++) {
            const int c1 = A.lm_edges()[j1];
            if (A.edge_lvl(c1)) continue;
            const int p1 = A.pose_slot()[edge_kf(A, c1)];
            if (p1 < 0) continue;
            const int d1 = c1 < A.n_pe() ? 2 : 1;
            const double *JA1 = A.JA() + 6 * (size_t)c1, *JB1 = A.JB() + 12 * (size_t)c1;
            const double w1 = A.wgt()[c1];
            for (int c = 0; c < 3; c++) {
              double s = 0;
              for (int a = 0; a < 6; a++) s += hpl_entry(d1, JA1, JB1, w1, a, c) * A.x()[p1 * 6 + a];
              cl[c] -= s;
            }
          }
          const double* Di = A.Dinv() + (size_t)ls * 9;
          for (int a = 0; a < 3; a++) A.x()[n + ls * 3 + a] = Di[a * 3] * cl[0] + Di[a * 3 + 1] * cl[1] + Di[a * 3 + 2] * cl[2];
        }
      }
      __syncthreads();
      // update (with the previous x when the factorisation failed, like g2o)
      for (int k = tid; k < A.n_kf(); k += BA_THREADS) if (A.pose_slot()[k] >= 0) A.T()[k] = se3_mul(se3_exp(A.x() + (size_t)A.pose_slot()[k] * 6), A.T()[k]);
      for (int l = tid; l < n_lm; l += BA_THREADS) if (A.lm_slot()[l] >= 0) for (int a = 0; a < 3; a++) A.X()[3 * l + a] += A.x()[n + A.lm_slot()[l] * 3 + a];
      __syncthreads();
      const double tempChi = errors_and_chi2(A, S, p_robust, l_robust, tid);
      double sc = 0;
      for (int i = tid; i < n; i += BA_THREADS) sc += A.x()[i] * (lambda * A.x()[i] + A.bp()[i]);
      for (int i = tid; i < nl * 3; i += BA_THREADS) sc += A.x()[n + i] * (lambda * A.x()[n + i] + A.bl()[i]);
      sc = block_sum(S, sc, tid);
      if (tid == 0) {
        bool kept;
        S.rho = lm_trial(S.ok2, tempChi, sc, S.lambda, S.ni, S.currentChi, kept);
        S.flag = !kept; S.qmax++;
      }
      __syncthreads();
      if (S.flag) {   // rejected: restore the state
        for (int k = tid; k < A.n_kf(); k += BA_THREADS) A.T()[k] = A.Tb()[k];
        for (int i = tid; i < n_lm * 3; i += BA_THREADS) A.X()[i] = A.Xb()[i];
      }
      __syncthreads();
      const bool again = S.rho < 0 && S.qmax < 10 && !(A.stop() && *A.stop());
      __syncthreads();
      if (!again) break;
    }
    if (tid == 0) S.stop_it = lm_stop(S.qmax, S.rho, S.iniChi, S.currentChi, S.nBad);
    __syncthreads();
    if (S.stop_it) break;
  }
  return done;
}

// The reference's point gate (Optimizer.cc:1957-1964 marks level 1, :2010-2016 erases): chi2 over 5.991 or not in front of the camera
__device__ __forceinline__ bool point_gated(const BAArgs& A, int e) {
  const double w = (double)A.pe_w()[e], c2 = A.err()[2 * e] * (w * A.err()[2 * e]) + A.err()[2 * e + 1] * (w * A.err()[2 * e + 1]);
  double c[3];
  se3_map(A.T()[A.pe_kf()[e]], A.X() + 3 * A.pe_pt()[e], c);
  return c2 > 5.991 || !(c[2] > 0.0);
}

// a[0 .. n) -> its exclusive prefix sums, a contiguous chunk per thread
__device__ void block_exclusive_scan(BAShared& S, int* a, int n, int tid) {
  const int per = (n + BA_THREADS - 1) / BA_THREADS, lo = min(tid * per, n), hi = min(lo + per, n), lane = tid & 31;
  int s = 0;
  for (int i = lo; i < hi; i++) s += a[i];
  int incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  if (lane == 31) S.wsum[tid >> 5] = incl;
  __syncthreads();
  int run = incl - s;
  for (int v = 0; v < (tid >> 5); v++) run += S.wsum[v];
  for (int i = lo; i < hi; i++) { const int t = a[i]; a[i] = run; run += t; }
  __syncthreads();
}

// The CSR indices by landmark and by keyframe, each list in edge-code order (= g2o's active-edge order: the landmark and pose
// sums run in it).  Stable counting sort: warp v ranks the edges of the v-th contiguous slice of codes among the slice's edges
// with the same key (__match_any_sync inside a 32-edge step, a per-warp cursor per key across steps); then each key's list
// holds the slices' edges in slice order.
__device__ void build_csr(const BAArgs& A, BAShared& S, int tid) {
  const int n_lm = A.n_pt() + 2 * A.n_ln(), n_edges = A.n_pe() + 2 * A.n_le(), per = (n_edges + BA_WARPS - 1) / BA_WARPS;
  for (int i = tid; i < BA_WARPS * n_lm; i += BA_THREADS) A.cur_lm()[i] = 0;
  for (int i = tid; i < BA_WARPS * A.n_kf(); i += BA_THREADS) A.cur_kf()[i] = 0;
  __syncthreads();
  {
    const int v = tid >> 5, lane = tid & 31, lo = v * per, hi = min(lo + per, n_edges);
    int* cl = A.cur_lm() + (size_t)v * n_lm;
    int* ck = A.cur_kf() + (size_t)v * A.n_kf();
    const unsigned below = (1u << lane) - 1u;
    for (int b = lo; b < hi; b += 32) {
      const int c = b + lane;
      const bool in = c < hi;
      const int l = in ? edge_lm(A, c) : -1, k = in ? edge_kf(A, c) : -1;
      const unsigned ml = __match_any_sync(0xffffffffu, l), mk = __match_any_sync(0xffffffffu, k);
      const int bl = in ? cl[l] : 0, bk = in ? ck[k] : 0;
      __syncwarp();
      if (in) {
        const int rl = __popc(ml & below), rk = __popc(mk & below);
        A.rank_lm()[c] = bl + rl; A.rank_kf()[c] = bk + rk;
        if (rl == __popc(ml) - 1) cl[l] = bl + rl + 1;
        if (rk == __popc(mk) - 1) ck[k] = bk + rk + 1;
      }
      __syncwarp();
    }
  }
  __syncthreads();
  for (int l = tid; l < n_lm; l += BA_THREADS) { int s = 0; for (int v = 0; v < BA_WARPS; v++) s += A.cur_lm()[(size_t)v * n_lm + l]; A.lm_start()[l] = s; }
  for (int k = tid; k < A.n_kf(); k += BA_THREADS) { int s = 0; for (int v = 0; v < BA_WARPS; v++) s += A.cur_kf()[(size_t)v * A.n_kf() + k]; A.kf_start()[k] = s; }
  if (tid == 0) { A.lm_start()[n_lm] = 0; A.kf_start()[A.n_kf()] = 0; }
  __syncthreads();
  block_exclusive_scan(S, A.lm_start(), n_lm + 1, tid);
  block_exclusive_scan(S, A.kf_start(), A.n_kf() + 1, tid);
  for (int l = tid; l < n_lm; l += BA_THREADS) {          // per-slice counts -> the slices' first positions in the list
    int run = A.lm_start()[l];
    for (int v = 0; v < BA_WARPS; v++) { int* p = A.cur_lm() + (size_t)v * n_lm + l; const int t = *p; *p = run; run += t; }
  }
  for (int k = tid; k < A.n_kf(); k += BA_THREADS) {
    int run = A.kf_start()[k];
    for (int v = 0; v < BA_WARPS; v++) { int* p = A.cur_kf() + (size_t)v * A.n_kf() + k; const int t = *p; *p = run; run += t; }
  }
  __syncthreads();
  for (int c = tid; c < n_edges; c += BA_THREADS) {
    const int v = c / per;
    A.lm_edges()[A.cur_lm()[(size_t)v * n_lm + edge_lm(A, c)] + A.rank_lm()[c]] = c;
    A.kf_edges()[A.cur_kf()[(size_t)v * A.n_kf() + edge_kf(A, c)] + A.rank_kf()[c]] = c;
  }
  __syncthreads();
}

// One CTA per window (blockIdx.x).  A window whose counts or edge indices are out of range writes its status, iterations = 0
// and nothing else.
__global__ void __launch_bounds__(BA_THREADS) k_local_ba(const __grid_constant__ BABatch Bt) {
  __shared__ BAShared S;
  __shared__ int cnt[5];
  const int tid = threadIdx.x, w = blockIdx.x;
  const PLBAWindows& P = Bt.P;
  const int n_kf = P.n_kf[w], n_pt = P.n_pt[w], n_ln = P.n_ln[w], n_pe = P.n_pe[w], n_le = P.n_le[w];
  const int rpe = w * P.cap_pe, rle = w * P.cap_le;   // the window's first edge rows
  int status = (n_kf < 0 || n_kf > P.cap_kf || n_pt < 0 || n_pt > P.cap_pt || n_ln < 0 || n_ln > P.cap_ln || n_pe < 0 ||
                n_pe > P.cap_pe || n_le < 0 || n_le > P.cap_le) ? 1 : 0;
  if (!status) {
    int bad = 0;
    for (int e = tid; e < n_pe; e += BA_THREADS) {
      const int k = P.pe_kf[rpe + e], p = P.pe_pt[rpe + e];
      bad |= k < 0 || k >= n_kf || p < 0 || p >= n_pt;
    }
    for (int e = tid; e < n_le; e += BA_THREADS) {
      const int k = P.le_kf[rle + e], l = P.le_ln[rle + e];
      bad |= k < 0 || k >= n_kf || l < 0 || l >= n_ln;
    }
    status = __syncthreads_or(bad) ? 2 : 0;
  }
  if (tid == 0) Bt.O.status[w] = status;
  if (status) {
    if (tid == 0) Bt.O.iterations[w] = 0;
    return;
  }
  if (tid == 0) { cnt[0] = n_kf; cnt[1] = n_pt; cnt[2] = n_ln; cnt[3] = n_pe; cnt[4] = n_le; }
  __syncthreads();
  const BAArgs A{Bt, cnt};
  build_csr(A, S, tid);
  const int n_lm = A.n_pt() + 2 * A.n_ln();
  for (int k = tid; k < A.n_kf(); k += BA_THREADS) A.T()[k] = se3_from_cv(A.kf_Tcw() + 16 * k);
  for (int i = tid; i < 3 * A.n_pt(); i += BA_THREADS) A.X()[i] = (double)A.pt_Xw()[i];
  for (int i = tid; i < 6 * A.n_ln(); i += BA_THREADS) A.X()[3 * A.n_pt() + i] = A.ln_Xw()[i];
  for (int i = tid; i < A.n_pe() + A.n_le(); i += BA_THREADS) A.lvl()[i] = 0;
  for (int i = tid; i < 2 * (A.n_pe() + A.n_le()); i += BA_THREADS) A.err()[i] = 0;
  __syncthreads();
  int its = 0;
  const bool stop0 = A.stop() && *A.stop();
  if (!stop0) {
    its += ba_optimize(A, S, 5, true, true, tid);
    __syncthreads();
    const bool more = !(A.stop() && *A.stop());
    if (more) {
      for (int e = tid; e < A.n_pe(); e += BA_THREADS) if (point_gated(A, e)) A.lvl()[e] = 1;
      for (int e = tid; e < A.n_le(); e += BA_THREADS) {
        const double a = A.err()[2 * A.n_pe() + 2 * e], b = A.err()[2 * A.n_pe() + 2 * e + 1];
        if (a * (0.5 * a) > 3.84 || b * (0.5 * b) > 3.84) A.lvl()[A.n_pe() + e] = 1;
      }
      __syncthreads();
      its += ba_optimize(A, S, 10, false, false, tid);
      __syncthreads();
    }
    for (int e = tid; e < A.n_pe(); e += BA_THREADS) A.pe_erase()[e] = point_gated(A, e) ? 1 : 0;
    for (int e = tid; e < A.n_le(); e += BA_THREADS) {
      const double a = A.err()[2 * A.n_pe() + 2 * e];
      A.le_erase()[e] = (a * (0.5 * a) > 3.84) ? 1 : 0;           // START-point edge read twice (Optimizer.cc:2030-2031)
      A.le_erase_kf()[e] = A.le_kf()[e / 2];                        // vpLineEdgeKF double push (Optimizer.cc:1924,1948)
    }
  } else {
    for (int e = tid; e < A.n_pe(); e += BA_THREADS) A.pe_erase()[e] = 0;
    for (int e = tid; e < A.n_le(); e += BA_THREADS) { A.le_erase()[e] = 0; A.le_erase_kf()[e] = A.le_kf()[e / 2]; }
  }
  __syncthreads();
  for (int k = tid; k < A.n_kf(); k += BA_THREADS) {
    if (A.kf_fixed()[k] || its == 0) { for (int i = 0; i < 16; i++) A.kf_Tcw_out()[16 * k + i] = A.kf_Tcw()[16 * k + i]; }
    else se3_to_cv(A.T()[k], A.kf_Tcw_out() + 16 * k);
  }
  for (int i = tid; i < 3 * A.n_pt(); i += BA_THREADS) A.pt_Xw_out()[i] = (float)A.X()[i];
  for (int i = tid; i < 6 * A.n_ln(); i += BA_THREADS) A.ln_Xw_out()[i] = (double)(float)A.X()[3 * A.n_pt() + i];
  if (tid == 0 && A.iterations()) *A.iterations() = its;
  (void)n_lm;
}
}  // namespace pl

using namespace pl;

// PL_OK if these capacities are within the limits in plslam_b200.h.  pl_local_ba_dev passes cap_free = cap_kf (any keyframe
// of a window may be free); pl_local_ba sizes the reduced system by its window's free keyframes, as it always did.
static int ba_caps_ok(int W, int cap_kf, int cap_free, int cap_pt, int cap_ln, int cap_pe, int cap_le) {
  const long long lim = 1 << 24;
  if (W < 0 || cap_free < 1 || cap_free > 7723) return PL_ERR_ARG;
  for (int c : {cap_kf, cap_pt, cap_ln, cap_pe, cap_le}) if (c < 1 || c > lim) return PL_ERR_ARG;
  for (int c : {cap_kf, cap_pt, cap_ln, cap_pe, cap_le}) if ((long long)W * c > INT_MAX) return PL_ERR_ARG;
  return PL_OK;
}

extern "C" size_t pl_local_ba_scratch_bytes(int W, int cap_kf, int cap_pt, int cap_ln, int cap_pe, int cap_le) {
  if (ba_caps_ok(W, cap_kf, cap_kf, cap_pt, cap_ln, cap_pe, cap_le)) return 0;
  return (size_t)W * ba_layout(cap_kf, cap_kf, cap_pt, cap_ln, cap_pe, cap_le).window;
}

static int ba_launch(const PLBAWindows& P, const int* stop_flag_dev, const PLBAOut& O, void* scratch, const BALayout& L, void* stream) {
  BABatch Bt;
  Bt.P = P; Bt.O = O; Bt.stop = stop_flag_dev; Bt.scratch = (char*)scratch; Bt.L = L;
  k_local_ba<<<P.W, BA_THREADS, 0, (cudaStream_t)stream>>>(Bt);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

extern "C" int pl_local_ba_dev(const PLBAWindows* windows, const int* stop_flag_dev, const PLBAOut* out, void* scratch, void* stream) {
  PL_ARG(windows && out && windows->W >= 0);
  const PLBAWindows& P = *windows;
  if (P.W == 0) return PL_OK;
  PL_ARG(!ba_caps_ok(P.W, P.cap_kf, P.cap_kf, P.cap_pt, P.cap_ln, P.cap_pe, P.cap_le));
  PL_ARG(P.n_kf && P.n_pt && P.n_ln && P.n_pe && P.n_le && P.kf_Tcw && P.kf_fixed && P.kf_K && P.K_end && P.pt_Xw && P.ln_Xw);
  PL_ARG(P.pe_kf && P.pe_pt && P.pe_obs && P.pe_inv_sigma2 && P.le_kf && P.le_ln && P.le_func);
  PL_ARG(out->kf_Tcw && out->pt_Xw && out->ln_Xw && out->pe_erase && out->le_erase && out->le_erase_kf && out->iterations && out->status);
  PL_ARG(scratch && ((uintptr_t)scratch & 15) == 0);
  PL_TRY(require_device());
  return ba_launch(P, stop_flag_dev, *out, scratch, ba_layout(P.cap_kf, P.cap_kf, P.cap_pt, P.cap_ln, P.cap_pe, P.cap_le), stream);
}

// The W = 1 case of pl_local_ba_dev on host arrays.
extern "C" int pl_local_ba(const PLBAProblem* p, const int* stop_flag_dev, float* kf_Tcw_out, float* pt_Xw_out,
                           double* ln_Xw_out, uint8_t* pe_erase, uint8_t* le_erase, int* le_erase_kf, int* iterations) {
  PL_ARG(p && kf_Tcw_out && p->n_kf >= 1 && p->n_pt >= 0 && p->n_ln >= 0 && p->n_pe >= 0 && p->n_le >= 0);
  PL_ARG(p->kf_Tcw && p->kf_fixed && p->kf_K);
  int rc = require_device();
  if (rc) return rc;
  const int n_kf = p->n_kf, n_pt = p->n_pt, n_ln = p->n_ln, n_pe = p->n_pe, n_le = p->n_le;
  for (int e = 0; e < n_pe; e++) PL_ARG(p->pe_kf[e] >= 0 && p->pe_kf[e] < n_kf && p->pe_pt[e] >= 0 && p->pe_pt[e] < n_pt);
  for (int e = 0; e < n_le; e++) PL_ARG(p->le_kf[e] >= 0 && p->le_kf[e] < n_kf && p->le_ln[e] >= 0 && p->le_ln[e] < n_ln);
  const int cap_pt = std::max(n_pt, 1), cap_ln = std::max(n_ln, 1), cap_pe = std::max(n_pe, 1), cap_le = std::max(n_le, 1);
  int n_free = 0;
  for (int k = 0; k < n_kf; k++) n_free += !p->kf_fixed[k];
  const int cap_free = std::max(n_free, 1);
  PL_ARG(!ba_caps_ok(1, n_kf, cap_free, cap_pt, cap_ln, cap_pe, cap_le));
  const int counts[5] = {n_kf, n_pt, n_ln, n_pe, n_le};
  const BALayout layout = ba_layout(n_kf, cap_free, cap_pt, cap_ln, cap_pe, cap_le);
  const size_t scratch_bytes = layout.window;
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
  PLBAWindows P;
  PLBAOut O;
  void* scratch = nullptr;
  for (int pass = 0; pass < 2 && !fail; pass++) {
    dry = pass == 0;
    off = 0;
    const int* dn = (const int*)up(counts, sizeof(counts));
    P.W = 1; P.cap_kf = n_kf; P.cap_pt = cap_pt; P.cap_ln = cap_ln; P.cap_pe = cap_pe; P.cap_le = cap_le;
    P.n_kf = dn; P.n_pt = dn + 1; P.n_ln = dn + 2; P.n_pe = dn + 3; P.n_le = dn + 4;
    P.kf_Tcw = (const float*)up(p->kf_Tcw, 64 * (size_t)n_kf); P.kf_fixed = (const uint8_t*)up(p->kf_fixed, n_kf);
    P.kf_K = (const float*)up(p->kf_K, 16 * (size_t)n_kf); P.K_end = (const float*)up(p->K_end, 16);
    P.pt_Xw = (const float*)up(p->pt_Xw, 12 * (size_t)n_pt); P.ln_Xw = (const double*)up(p->ln_Xw, 48 * (size_t)n_ln);
    P.pe_kf = (const int*)up(p->pe_kf, 4 * (size_t)n_pe); P.pe_pt = (const int*)up(p->pe_pt, 4 * (size_t)n_pe);
    P.pe_obs = (const float*)up(p->pe_obs, 8 * (size_t)n_pe); P.pe_inv_sigma2 = (const float*)up(p->pe_inv_sigma2, 4 * (size_t)n_pe);
    P.le_kf = (const int*)up(p->le_kf, 4 * (size_t)n_le); P.le_ln = (const int*)up(p->le_ln, 4 * (size_t)n_le);
    P.le_func = (const double*)up(p->le_func, 24 * (size_t)n_le);
    O.kf_Tcw = (float*)dalloc(64 * (size_t)n_kf); O.pt_Xw = (float*)dalloc(12 * (size_t)n_pt); O.ln_Xw = (double*)dalloc(48 * (size_t)n_ln);
    O.pe_erase = (uint8_t*)dalloc(n_pe); O.le_erase = (uint8_t*)dalloc(n_le); O.le_erase_kf = (int*)dalloc(4 * (size_t)n_le);
    O.iterations = (int*)dalloc(4); O.status = (int*)dalloc(4);
    scratch = dalloc(scratch_bytes);
    if (dry && (off > ws_cap || dev != ws_dev)) {       // grow (or move to the current device)
      if (ws_base) cudaFree(ws_base);
      ws_base = nullptr; ws_cap = 0; ws_dev = dev;
      const size_t want = off + off / 4;
      if (cudaMalloc((void**)&ws_base, want) != cudaSuccess) { ws_base = nullptr; fail = true; break; }
      ws_cap = want;
    }
  }
  if (fail) { set_error("local BA: device allocation or copy failed"); return PL_ERR_CUDA; }
  if ((rc = ba_launch(P, stop_flag_dev, O, scratch, layout, nullptr))) return rc;
  cudaError_t e = cudaDeviceSynchronize();
  int status = 0;
  if (e == cudaSuccess) e = cudaMemcpy(&status, O.status, 4, cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemcpy(kf_Tcw_out, O.kf_Tcw, 64 * (size_t)n_kf, cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && n_pt && pt_Xw_out) e = cudaMemcpy(pt_Xw_out, O.pt_Xw, 12 * (size_t)n_pt, cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && n_ln && ln_Xw_out) e = cudaMemcpy(ln_Xw_out, O.ln_Xw, 48 * (size_t)n_ln, cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && n_pe && pe_erase) e = cudaMemcpy(pe_erase, O.pe_erase, n_pe, cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && n_le && le_erase) e = cudaMemcpy(le_erase, O.le_erase, n_le, cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && n_le && le_erase_kf) e = cudaMemcpy(le_erase_kf, O.le_erase_kf, 4 * (size_t)n_le, cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && iterations) e = cudaMemcpy(iterations, O.iterations, 4, cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) { set_error("local BA: %s", cudaGetErrorString(e)); return PL_ERR_CUDA; }
  if (status) { set_error("local BA: window refused on the device (status %d)", status); return PL_ERR_ARG; }   // checked above
  return PL_OK;
}
