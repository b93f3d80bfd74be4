// Triangulation, gates and neighbour-order commit of LocalMapping::CreateNewMapPoints (src/LocalMapping.cc:417-574, monocular) for
// the pairs that pl_orb_search_for_triangulation_dev found, on the device (DESIGN.md §8f.5).
//
//   k_tri_gates   one thread per (problem, idx1) slot, blocks of kGateSlots slots of one problem: the problem's status, then for a
//                 slot that holds a match the reference's per-pair body in its order - normalised rays and the parallax gate
//                 (:433-455), the linear triangulation with cv::SVD (:457-473, svd4.cuh), depth in both cameras (:489-497),
//                 reprojection in both keyframes at each keypoint's octave (:499-555), the scale-consistency gate (:557-574).
//                 Stereo branches are not restated (mvuRight < 0 throughout, DESIGN.md §9).
//   k_tri_commit  one CTA per problem: a slot that passed at problem p is dropped iff an earlier problem with the same kf1 passed at
//                 the same idx1 - the reference's "idx1 received a map point at an earlier neighbour", by induction over the
//                 neighbours - and nnew[p] counts the rest.  A function of gate results alone: no scratch, deterministic.
//
// Every reference expression keeps its C++ promotions and its cv::Mat order (DESIGN.md §8f.5): cv::gemm's fp32 order for Rwc * xn,
// fp64 for Mat::dot and cv::norm, MatExpr's fp64 addWeighted for the rows of A, M / s as M * (float)(1.0 / s) + 0.  Every operation
// is an _rn intrinsic, so nothing is contracted.
#include "common.cuh"
#include "search.cuh"
#include "svd4.cuh"
#include "tri_math.cuh"

namespace pl {

namespace {
using namespace tri;
constexpr int kGateSlots = 128;      // slots (threads) per k_tri_gates block
constexpr int kCommitThreads = 256;

enum : int8_t { kNoPair = -1, kCommitted = 0, kDropped = 1, kParallax = 2, kWZero = 3, kBehind1 = 4, kBehind2 = 5, kReproj1 = 6,
                kReproj2 = 7, kScale = 8 };

struct TriGateArgs {
  PLTriKeyframes K; PLTriProblems Q;
  const int* matches12; const int* search_status; float ratio_factor;
  float* x3D; int8_t* code; int* status;
};

// the reprojection test of :510-516 / :538-543: true when the squared error exceeds 5.991 sigma^2
__device__ __forceinline__ bool reproj_fails(const float* T, const float* Kc, float z, const float* x, float kx, float ky, float sigma2) {
  const float xc = cam(T, 0, x), yc = cam(T, 1, x), invz = inv_d(z);
  const float u = fadd(fmul(fmul(Kc[0], xc), invz), Kc[2]), v = fadd(fmul(fmul(Kc[1], yc), invz), Kc[3]);
  const float ex = fsub(u, kx), ey = fsub(v, ky);
  return (double)fadd(fmul(ex, ex), fmul(ey, ey)) > __dmul_rn(5.991, (double)sigma2);
}
// cv::norm(x - O) rounded to fp32
__device__ __forceinline__ float dist(const float* x, const float* O) {
  const float d[3] = {fsub(x[0], O[0]), fsub(x[1], O[1]), fsub(x[2], O[2])};
  return __double2float_rn(__dsqrt_rn(ddot3(d, d)));
}

// The gates of :433-574 for one pair; x3D is written when every gate passes.
__device__ int8_t gate_pair(const PLKeyPoint& kp1, const PLKeyPoint& kp2, const float* T1, const float* T2, const float* K1,
                            const float* K2, const float* O1, const float* O2, const float* sf, const float* sigma2, float ratio_factor,
                            float* x3D) {
  // Frame: invfx = 1.0f / fx (Frame.cc:123), copied into the KeyFrame
  const float xn1[3] = {fmul(fsub(kp1.x, K1[2]), __fdiv_rn(1.f, K1[0])), fmul(fsub(kp1.y, K1[3]), __fdiv_rn(1.f, K1[1])), 1.f};
  const float xn2[3] = {fmul(fsub(kp2.x, K2[2]), __fdiv_rn(1.f, K2[0])), fmul(fsub(kp2.y, K2[3]), __fdiv_rn(1.f, K2[1])), 1.f};
  // ray = Rwc * xn, Rwc = Rcw^T, cv::gemm's fp32 order
  float ray1[3], ray2[3];
#pragma unroll
  for (int i = 0; i < 3; i++) {
    ray1[i] = fadd(fadd(fmul(T1[i], xn1[0]), fmul(T1[4 + i], xn1[1])), fmul(T1[8 + i], xn1[2]));
    ray2[i] = fadd(fadd(fmul(T2[i], xn2[0]), fmul(T2[4 + i], xn2[1])), fmul(T2[8 + i], xn2[2]));
  }
  const float cosp = __double2float_rn(__ddiv_rn(ddot3(ray1, ray2), __dmul_rn(__dsqrt_rn(ddot3(ray1, ray1)), __dsqrt_rn(ddot3(ray2, ray2)))));
  // cosParallaxStereo = cosParallaxRays + 1 on both sides (monocular); 0.9998 is a double
  if (!(cosp < fadd(cosp, 1.f) && cosp > 0.f && (double)cosp < 0.9998)) return kParallax;
  // A.row(r) = xn * Tcw.row(2) - Tcw.row(k): MatExpr -> addWeighted(a, s, b, -1, 0), fp64 then one rounding
  float A[16];
#pragma unroll
  for (int c = 0; c < 4; c++) {
    A[c] = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)xn1[0], (double)T1[8 + c]), -(double)T1[c]), 0.0));
    A[4 + c] = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)xn1[1], (double)T1[8 + c]), -(double)T1[4 + c]), 0.0));
    A[8 + c] = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)xn2[0], (double)T2[8 + c]), -(double)T2[c]), 0.0));
    A[12 + c] = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)xn2[1], (double)T2[8 + c]), -(double)T2[4 + c]), 0.0));
  }
  float w[4], vt[16];
  svd4(A, w, vt);
  if (vt[15] == 0.f) return kWZero;
  // x3D.rowRange(0,3) / x3D.at<float>(3): convertTo with alpha = (float)(1.0 / w), beta = 0
  const float s = inv_d(vt[15]);
  const float x[3] = {fadd(fmul(vt[12], s), 0.f), fadd(fmul(vt[13], s), 0.f), fadd(fmul(vt[14], s), 0.f)};
  const float z1 = cam(T1, 2, x);
  if (z1 <= 0.f) return kBehind1;
  const float z2 = cam(T2, 2, x);
  if (z2 <= 0.f) return kBehind2;
  if (reproj_fails(T1, K1, z1, x, kp1.x, kp1.y, sigma2[kp1.octave])) return kReproj1;
  if (reproj_fails(T2, K2, z2, x, kp2.x, kp2.y, sigma2[kp2.octave])) return kReproj2;
  const float dist1 = dist(x, O1), dist2 = dist(x, O2);
  if (dist1 == 0.f || dist2 == 0.f) return kScale;
  const float ratio_dist = __fdiv_rn(dist2, dist1), ratio_oct = __fdiv_rn(sf[kp1.octave], sf[kp2.octave]);
  if (fmul(ratio_dist, ratio_factor) < ratio_oct || ratio_dist > fmul(ratio_oct, ratio_factor)) return kScale;
  x3D[0] = x[0]; x3D[1] = x[1]; x3D[2] = x[2];
  return kCommitted;
}

// grid (P, ceil(cap / kGateSlots)): block (p, c) takes slots c * kGateSlots .. of problem p.  Every block that holds slots of a
// problem decides the problem's status from the same reads, so a problem is written completely or not at all; block (p, 0)
// writes status[p].
__global__ void __launch_bounds__(kGateSlots) k_tri_gates(const __grid_constant__ TriGateArgs A) {
  const PLTriKeyframes& K = A.K; const PLTriProblems& Q = A.Q;
  const int p = blockIdx.x, tid = threadIdx.x;
  const int ss = A.search_status[p];
  int st = ss;
  const int k1 = Q.kf1[p], k2 = Q.kf2[p];
  int n1 = 0, n2 = 0;
  long long oo = 0;
  if (!st && (k1 < 0 || k1 >= K.n_kf || k2 < 0 || k2 >= K.n_kf)) st = 1;
  if (!st) {
    n1 = K.n[k1]; n2 = K.n[k2];
    if (n1 < 0 || n1 > K.cap || n2 < 0 || n2 > K.cap) st = 2;
  }
  if (!st) {
    oo = Q.out_offset[p];
    if (oo < 0 || oo + n1 > Q.n_out) st = 1;
  }
  // a block past the problem's slots has nothing to write; block (p, 0) always stays, to write the status
  if (blockIdx.y > 0 && (st || (int)blockIdx.y * kGateSlots >= n1)) return;
  if (!st) {     // status 4: a matches12 entry outside -1 .. n2 - 1 (each block of the problem reads all n1 entries, from L2)
    bool ok = true;
    for (int i = tid; i < n1; i += kGateSlots) { const int m = A.matches12[oo + i]; ok = ok && m >= -1 && m < n2; }
    if (!__syncthreads_and(ok)) st = 4;
  }
  if (blockIdx.y == 0 && tid == 0) A.status[p] = st;
  if (st) return;
  const int idx1 = blockIdx.y * kGateSlots + tid;
  if (idx1 >= n1) return;
  const long long slot = oo + idx1;
  const int idx2 = A.matches12[slot];
  if (idx2 < 0) { A.code[slot] = kNoPair; return; }
  const long long r1 = (long long)k1 * K.cap, r2 = (long long)k2 * K.cap;
  A.code[slot] = gate_pair(K.keys_un[r1 + idx1], K.keys_un[r2 + idx2], K.Tcw + 16LL * k1, K.Tcw + 16LL * k2, K.K + 4LL * k1,
                           K.K + 4LL * k2, K.Ow + 3LL * k1, K.Ow + 3LL * k2, K.scale_factors, K.level_sigma2, A.ratio_factor,
                           A.x3D + 3 * slot);
}

struct TriCommitArgs { PLTriKeyframes K; PLTriProblems Q; int8_t* code; const int* status; int* nnew; };

// One CTA per problem.  Problem p only turns its own passed slots from kCommitted to kDropped, and reads the slots of earlier
// problems, for which both values mean "passed the gates", so the CTAs need no ordering among themselves.
__global__ void __launch_bounds__(kCommitThreads) k_tri_commit(const __grid_constant__ TriCommitArgs A) {
  __shared__ int s_n;
  const int p = blockIdx.x, tid = threadIdx.x;
  if (A.status[p]) return;
  const int k1 = A.Q.kf1[p], n1 = A.K.n[k1];
  const long long oo = A.Q.out_offset[p];
  if (tid == 0) s_n = 0;
  __syncthreads();
  int mine = 0;
  for (int i = tid; i < n1; i += kCommitThreads) {
    if (A.code[oo + i] != kCommitted) continue;
    bool dropped = false;
    for (int q = 0; q < p && !dropped; q++) {
      if (A.Q.kf1[q] != k1 || A.status[q]) continue;
      const int8_t c = A.code[(long long)A.Q.out_offset[q] + i];
      dropped = c == kCommitted || c == kDropped;
    }
    if (dropped) A.code[oo + i] = kDropped; else mine++;
  }
  if (mine) atomicAdd(&s_n, mine);
  __syncthreads();
  if (tid == 0) A.nnew[p] = s_n;
}
}  // namespace

}  // namespace pl

using namespace pl;

extern "C" int pl_orb_triangulate_dev(const PLTriKeyframes* kfs, const PLTriProblems* problems, const int* matches12,
                                      const int* search_status, float scale_factor, float* x3D, int8_t* code, int* nnew, int* status,
                                      void* stream) {
  PL_TRY(orb_tri_args_ok(kfs, problems, matches12, nnew, status));
  const PLTriProblems& Q = *problems;
  if (Q.P == 0) return PL_OK;
  PL_ARG(search_status && (Q.n_out == 0 || (x3D && code)));
  const PLTriKeyframes& K = *kfs;
  PL_TRY(require_device());
  const TriGateArgs G{K, Q, matches12, search_status, 1.5f * scale_factor, x3D, code, status};
  k_tri_gates<<<dim3(Q.P, (K.cap + kGateSlots - 1) / kGateSlots), kGateSlots, 0, (cudaStream_t)stream>>>(G);
  PL_LAUNCH_CHECK();
  const TriCommitArgs Cm{K, Q, code, status, nnew};
  k_tri_commit<<<Q.P, kCommitThreads, 0, (cudaStream_t)stream>>>(Cm);
  PL_LAUNCH_CHECK();
  return PL_OK;
}
