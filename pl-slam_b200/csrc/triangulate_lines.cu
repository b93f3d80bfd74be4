// The three-view line triangulation, gates and commit of LocalMapping::CreateNewMapLinesConstraint (src/LocalMapping.cc:966-1439,
// monocular) for the matches of a pl_lsd_search_for_triangulation_dev batch, on the device (DESIGN.md §8f.6).
//
//   k_line_tri_gates   one thread per (group, entry pair, ikl) slot, blocks of kLineGateSlots slots of one pair: the group's status,
//                      then for a slot that holds a triple whose three slots are free at the snapshot the reference's per-triple
//                      body in its order - the epipolar-plane test through F21 (:1063-1079), the direction test (:1083-1114), the
//                      two 4x4 SVD triangulations (:1118-1171, svd4.cuh), parallax (:1176-1205), distance and length against the
//                      entry's median depth (:1207-1227), depth (:1229-1252), reprojection (:1254-1331) and overlap (:1333-1416).
//   k_line_tri_commit  one CTA per group: the pairs in order, ikl ascending within a pair, against the taken state of kf_cur and of
//                      each entry's positional keyframe in shared memory, seeded from has_ml (:1044, :1428-1430).
//
// Every reference expression keeps its C++ promotions and its cv::Mat order (DESIGN.md §8f.6): cv::gemm's fp32 order for products
// without a transposed operand, fp64 accumulation for klF.t() * M (GEMM_1_T), cv::solve's small-matrix fp64 formula for
// K.inv() * x and its fp32 LU for (K2.t()).inv() * t21x, cv::invert's fp64 formula for K1.inv(), fp32 Mat::cross and subtraction,
// fp64 Mat::dot and cv::norm, MatExpr's fp64 addWeighted for s * M.row(2) - M.row(k), M / s and M /= s as M * (float)(1.0 / s) + 0.
// Every operation is an _rn intrinsic, so nothing is contracted.
#include "common.cuh"
#include "search.cuh"
#include "svd4.cuh"
#include "tri_math.cuh"

namespace pl {

namespace {
using namespace tri;
constexpr int kLineGateSlots = 128;      // slots (threads) per k_line_tri_gates block
constexpr int kLineCommitThreads = 128;
constexpr int kMaxE = PL_TRI_LINE_MAX_ENTRIES;
constexpr int kMaxPairs = kMaxE * (kMaxE - 1) / 2;
constexpr int kRoles = 1 + kMaxE;        // taken state: kf_cur, then each entry's positional keyframe
constexpr double kPI = 3.1415926;        // LocalMapping.cc:28 (#define PI), not M_PI

enum : int8_t { kNoTriple = -1, kCommitted = 0, kHeld = 1, kTaken = 2, kEpipolar = 3, kZeroNorm = 4, kCosSita = 5, kWZero = 6,
                kParallax = 7, kNear = 8, kLong = 9, kBehind = 10, kReproj1 = 11, kOverlap1 = 14 };

struct KeyLineRec {  // cv::line_descriptor::KeyLine (68 B)
  float angle; int class_id; int octave; float ptx, pty; float response; float size;
  float startPointX, startPointY, endPointX, endPointY, sPointInOctaveX, sPointInOctaveY, ePointInOctaveX, ePointInOctaveY;
  float lineLength; int numOfPixels;
};
static_assert(sizeof(KeyLineRec) == 68, "KeyLine record");

struct LineTriArgs {
  PLTriLineKeyframes K; PLTriLineGeometry Gm; PLTriProblems Q; PLTriLineGroups Gr;
  const int* matches; const int* nmatches; const int* search_status;
  int8_t* code; float* line3D; int* nnew; int* status;
};

__device__ __forceinline__ double dsum3(double a, double b, double c) { return __dadd_rn(__dadd_rn(a, b), c); }
// C = A * B for row-major 3x3 fp32 matrices, cv::gemm's small-matrix order ((a0 b0 + a1 b1) + a2 b2); bt: B is given transposed
__device__ void gemm33(const float* A, const float* B, float* C, bool bt) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      const float b0 = bt ? B[3 * c] : B[c], b1 = bt ? B[3 * c + 1] : B[3 + c], b2 = bt ? B[3 * c + 2] : B[6 + c];
      C[3 * r + c] = fadd(fadd(fmul(A[3 * r], b0), fmul(A[3 * r + 1], b1)), fmul(A[3 * r + 2], b2));
    }
}
// y = A x (A 3x3 row-major; at: A given transposed), cv::gemm's order
__device__ __forceinline__ void gemv3(const float* A, const float* x, float* y, bool at = false) {
#pragma unroll
  for (int r = 0; r < 3; r++) {
    const float a0 = at ? A[r] : A[3 * r], a1 = at ? A[3 + r] : A[3 * r + 1], a2 = at ? A[6 + r] : A[3 * r + 2];
    y[r] = fadd(fadd(fmul(a0, x[0]), fmul(a1, x[1])), fmul(a2, x[2]));
  }
}
// Mat::cross of two CV_32F 3-vectors: c0 = a1 b2 - a2 b1, c1 = a2 b0 - a0 b2, c2 = a0 b1 - a1 b0, each operation rounded
__device__ __forceinline__ void cross3(const float* a, const float* b, float* c) {
  c[0] = fsub(fmul(a[1], b[2]), fmul(a[2], b[1]));
  c[1] = fsub(fmul(a[2], b[0]), fmul(a[0], b[2]));
  c[2] = fsub(fmul(a[0], b[1]), fmul(a[1], b[0]));
}
__device__ __forceinline__ double dm(float a, float b) { return __dmul_rn((double)a, (double)b); }
// det3 of cv::invert / cv::solve (lapack.cpp) on a CV_32F matrix, fp64
__device__ __forceinline__ double det3(const float* S) {
  return __dadd_rn(__dsub_rn(__dmul_rn((double)S[0], __dsub_rn(dm(S[4], S[8]), dm(S[5], S[7]))),
                             __dmul_rn((double)S[1], __dsub_rn(dm(S[3], S[8]), dm(S[5], S[6])))),
                   __dmul_rn((double)S[2], __dsub_rn(dm(S[3], S[7]), dm(S[4], S[6]))));
}
// the camera matrix mK = [fx 0 cx; 0 fy cy; 0 0 1]
__device__ __forceinline__ void kmat(const float* k, float* M) {
  M[0] = k[0]; M[1] = 0.f; M[2] = k[2]; M[3] = 0.f; M[4] = k[1]; M[5] = k[3]; M[6] = 0.f; M[7] = 0.f; M[8] = 1.f;
}
// K.inv() (cv::invert, DECOMP_LU, n = 3, CV_32F): the adjugate in fp64 times 1 / det3, each entry rounded; zeros when det3 == 0
__device__ void inv3(const float* S, float* D) {
  double d = det3(S);
  if (d == 0.0) { for (int k = 0; k < 9; k++) D[k] = 0.f; return; }
  d = __ddiv_rn(1.0, d);
  const int a[9][4] = {{4, 8, 5, 7}, {2, 7, 1, 8}, {1, 5, 2, 4}, {5, 6, 3, 8}, {0, 8, 2, 6}, {2, 3, 0, 5}, {3, 7, 4, 6}, {1, 6, 0, 7},
                       {0, 4, 1, 3}};
  for (int k = 0; k < 9; k++) D[k] = __double2float_rn(__dmul_rn(__dsub_rn(dm(S[a[k][0]], S[a[k][1]]), dm(S[a[k][2]], S[a[k][3]])), d));
}
// K.inv() * x for a 3-vector x: MatExpr turns it into cv::solve(K, x, DECOMP_LU), whose n = 3, one-column CV_32F path is Cramer's
// rule in fp64 (lapack.cpp); zeros when det3 == 0
__device__ void solve3(const float* S, const float* b, float* x) {
  double d = det3(S);
  if (d == 0.0) { x[0] = x[1] = x[2] = 0.f; return; }
  d = __ddiv_rn(1.0, d);
  const double t0 = __dmul_rn(d, __dadd_rn(__dsub_rn(__dmul_rn((double)b[0], __dsub_rn(dm(S[4], S[8]), dm(S[5], S[7]))),
                                                     __dmul_rn((double)S[1], __dsub_rn(dm(b[1], S[8]), dm(S[5], b[2])))),
                                           __dmul_rn((double)S[2], __dsub_rn(dm(b[1], S[7]), dm(S[4], b[2])))));
  const double t1 = __dmul_rn(d, __dadd_rn(__dsub_rn(__dmul_rn((double)S[0], __dsub_rn((double)fmul(b[1], S[8]), dm(S[5], b[2]))),
                                                     __dmul_rn((double)b[0], __dsub_rn(dm(S[3], S[8]), dm(S[5], S[6])))),
                                           __dmul_rn((double)S[2], __dsub_rn(dm(S[3], b[2]), dm(b[1], S[6])))));
  const double t2 = __dmul_rn(d, __dadd_rn(__dsub_rn(__dmul_rn((double)S[0], __dsub_rn(dm(S[4], b[2]), dm(b[1], S[7]))),
                                                     __dmul_rn((double)S[1], __dsub_rn(dm(S[3], b[2]), dm(b[1], S[6])))),
                                           __dmul_rn((double)b[0], __dsub_rn(dm(S[3], S[7]), dm(S[4], S[6])))));
  x[0] = __double2float_rn(t0); x[1] = __double2float_rn(t1); x[2] = __double2float_rn(t2);
}
// cv::solve(A, B, X, DECOMP_LU) for a 3x3 CV_32F A and a 3-column B: LUImpl in fp32 (partial pivoting on the larger |a|, pivot
// below 10 FLT_EPSILON = singular, then X = 0), A and B overwritten
__device__ void lu_solve3(float* A, float* B) {
  for (int i = 0; i < 3; i++) {
    int k = i;
    for (int j = i + 1; j < 3; j++)
      if (fabsf(A[3 * j + i]) > fabsf(A[3 * k + i])) k = j;
    if (fabsf(A[3 * k + i]) < 10.f * 1.1920928955078125e-07f) { for (int q = 0; q < 9; q++) B[q] = 0.f; return; }
    if (k != i) {
      for (int j = i; j < 3; j++) { const float t = A[3 * i + j]; A[3 * i + j] = A[3 * k + j]; A[3 * k + j] = t; }
      for (int j = 0; j < 3; j++) { const float t = B[3 * i + j]; B[3 * i + j] = B[3 * k + j]; B[3 * k + j] = t; }
    }
    const float d = __fdiv_rn(-1.f, A[3 * i + i]);
    for (int j = i + 1; j < 3; j++) {
      const float alpha = fmul(A[3 * j + i], d);
      for (int q = i + 1; q < 3; q++) A[3 * j + q] = fadd(A[3 * j + q], fmul(alpha, A[3 * i + q]));
      for (int q = 0; q < 3; q++) B[3 * j + q] = fadd(B[3 * j + q], fmul(alpha, B[3 * i + q]));
    }
  }
  for (int i = 2; i >= 0; i--)
    for (int j = 0; j < 3; j++) {
      float s = B[3 * i + j];
      for (int q = i + 1; q < 3; q++) s = fsub(s, fmul(A[3 * i + q], B[3 * q + j]));
      B[3 * i + j] = __fdiv_rn(s, A[3 * i + i]);
    }
}
// cv::norm of a CV_32F vector rounded to fp32: sqrt of the fp64 sum of squares from 0, in index order
__device__ __forceinline__ float fnorm3(const float* v) { return __double2float_rn(__dsqrt_rn(ddot3(v, v))); }
// v *= (float)(1.0 / s) + 0: Mat /= double (convertTo with alpha = 1 / s, beta = 0)
__device__ __forceinline__ void scale3(float* v, float s) {
  const float a = inv_d(s);
  v[0] = fadd(fmul(v[0], a), 0.f); v[1] = fadd(fmul(v[1], a), 0.f); v[2] = fadd(fmul(v[2], a), 0.f);
}
// Result = (float)(Th_.dot(lineVector2) / (norm(Th_) * norm(lineVector2))) for Th = F21 * (x, y, 1), Th_ = (-Th1, Th0)
__device__ float epipolar(const float* F21, float x, float y, const float* lv) {
  const float r[3] = {x, y, 1.f};
  float th[3];
  gemv3(F21, r, th);
  const float t0 = -th[1], t1 = th[0];
  const double dot = __dadd_rn(__dmul_rn((double)t0, (double)lv[0]), __dmul_rn((double)t1, (double)lv[1]));
  const double nt = __dsqrt_rn(__dadd_rn(__dmul_rn((double)t0, (double)t0), __dmul_rn((double)t1, (double)t1)));
  const double nl = __dsqrt_rn(__dadd_rn(__dmul_rn((double)lv[0], (double)lv[0]), __dmul_rn((double)lv[1], (double)lv[1])));
  return __double2float_rn(__ddiv_rn(dot, __dmul_rn(nt, nl)));
}
// L = K.inv() * (sx, sy, 1) x K.inv() * (ex, ey, 1)
__device__ void plane_normal(const float* Km, const KeyLineRec& kl, float* L) {
  const float s[3] = {kl.startPointX, kl.startPointY, 1.f}, e[3] = {kl.endPointX, kl.endPointY, 1.f};
  float s_[3], e_[3];
  solve3(Km, s, s_); solve3(Km, e, e_);
  cross3(s_, e_, L);
}
// One endpoint's linear triangulation: rows 0, 1 = klF3^T M3, klF2^T M2 (given), rows 2, 3 = x M1.row(2) - M1.row(0), y M1.row(2)
// - M1.row(1) (addWeighted, fp64, one rounding), cv::SVD, then vt.row(3) / vt(3,3).  False when vt(3,3) == 0.
__device__ bool endpoint(const float* r01, const float* M1, float x, float y, float* X) {
  float A[16];
#pragma unroll
  for (int c = 0; c < 8; c++) A[c] = r01[c];
#pragma unroll
  for (int c = 0; c < 4; c++) {
    A[8 + c] = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)x, (double)M1[8 + c]), -(double)M1[c]), 0.0));
    A[12 + c] = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)y, (double)M1[8 + c]), -(double)M1[4 + c]), 0.0));
  }
  float w[4], vt[16];
  svd4(A, w, vt);
  if (vt[15] == 0.f) return false;
  const float s = inv_d(vt[15]);
  X[0] = fadd(fmul(vt[12], s), 0.f); X[1] = fadd(fmul(vt[13], s), 0.f); X[2] = fadd(fmul(vt[14], s), 0.f);
  return true;
}
// (float)(normal1.dot(normal2) / (dist1 * dist2)), the product of the two fp32 distances rounded to fp32
__device__ __forceinline__ float cos_parallax(const float* n1, const float* n2, float d1, float d2) {
  return __double2float_rn(__ddiv_rn(ddot3(n1, n2), (double)fmul(d1, d2)));
}
__device__ __forceinline__ void diff3(const float* a, const float* b, float* d) {
  d[0] = fsub(a[0], b[0]); d[1] = fsub(a[1], b[1]); d[2] = fsub(a[2], b[2]);
}
// true when one endpoint's parallax against views 2 and 3 is too small (cosParallax >= 0.99998)
__device__ bool parallax_fails(const float* X, const float* O1, const float* O2, const float* O3) {
  float n1[3], n2[3], n3[3];
  diff3(X, O1, n1); diff3(X, O2, n2); diff3(X, O3, n3);
  const float d1 = fnorm3(n1), d2 = fnorm3(n2), d3 = fnorm3(n3);
  return (double)cos_parallax(n1, n2, d1, d2) >= 0.99998 || (double)cos_parallax(n1, n3, d1, d3) >= 0.99998;
}
// the projection (u, v) of X in a camera (:1258-1263), fp32 after the fp64 dot products
__device__ __forceinline__ void project(const float* T, const float* k, float z, const float* X, float& u, float& v) {
  const float x = cam(T, 0, X), y = cam(T, 1, X), invz = inv_d(z);
  u = fadd(fmul(fmul(k[0], x), invz), k[2]);
  v = fadd(fmul(fmul(k[1], y), invz), k[3]);
}
// (err * err) > 3.84 * sigma2 with err = f0 u + f1 v + f2 in fp64
__device__ __forceinline__ bool reproj_fails(const double* f, float u, float v, float sigma2) {
  const double err = __dadd_rn(__dadd_rn(__dmul_rn(f[0], (double)u), __dmul_rn(f[1], (double)v)), f[2]);
  return __dmul_rn(err, err) > __dmul_rn(3.84, (double)sigma2);
}
// std::min / std::max on floats as the reference calls them: min(a, b) = b < a ? b : a, max(a, b) = a < b ? b : a
__device__ __forceinline__ float smin(float a, float b) { return b < a ? b : a; }
__device__ __forceinline__ float smax(float a, float b) { return a < b ? b : a; }
// the overlap test of one view (:1335-1360): along y when PI/4 < |angle| < 3 PI/4, else along x; IEEE quotients (0 / 0 is NaN,
// which passes the "< 0.85" tests as it does in the reference)
__device__ bool overlap_fails(const KeyLineRec& kl, float us, float vs, float ue, float ve) {
  const double a = (double)fabsf(kl.angle);
  const bool ydir = a < 3.0 * kPI / 4.0 && a > 1.0 * kPI / 4.0;
  const float ps = ydir ? vs : us, pe = ydir ? ve : ue;
  const float ks = ydir ? kl.startPointY : kl.startPointX, ke = ydir ? kl.endPointY : kl.endPointX;
  if (smin(pe, ps) > smax(ks, ke) || smin(ks, ke) > smax(pe, ps)) return true;
  const float hi = smin(smax(pe, ps), smax(ks, ke)), lo = smax(smin(pe, ps), smin(ks, ke));
  const float r1 = __fdiv_rn(fsub(hi, lo), fsub(smax(pe, ps), smin(pe, ps)));
  const float r2 = __fdiv_rn(fsub(hi, lo), fsub(smax(ks, ke), smin(ks, ke)));
  return (double)r1 < 0.85 || (double)r2 < 0.85;
}

// The constants of one entry pair (i, j) of a group, the same for every ikl: the reference forms them per triple, with the same
// operands and the same arithmetic, so forming them once per block gives the same values.
struct PairConsts {
  float F21[9], R12[9], R13[9], M1[12], M2[12], M3[12], K1[9], K2[9], K3[9];
};

// M = K * Tcw.rowRange(0, 3) (3x3 times 3x4), cv::gemm's order
__device__ void proj_matrix(const float* Km, const float* T, float* M) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++)
      M[4 * r + c] = fadd(fadd(fmul(Km[3 * r], T[c]), fmul(Km[3 * r + 1], T[4 + c])), fmul(Km[3 * r + 2], T[8 + c]));
}

__device__ void pair_consts(const PLTriLineGeometry& Gm, int k1, int k2, int k3, PairConsts& P) {
  const float *T1 = Gm.Tcw + 16LL * k1, *T2 = Gm.Tcw + 16LL * k2, *T3 = Gm.Tcw + 16LL * k3;
  const float R1[9] = {T1[0], T1[1], T1[2], T1[4], T1[5], T1[6], T1[8], T1[9], T1[10]};
  const float R2[9] = {T2[0], T2[1], T2[2], T2[4], T2[5], T2[6], T2[8], T2[9], T2[10]};
  const float R3[9] = {T3[0], T3[1], T3[2], T3[4], T3[5], T3[6], T3[8], T3[9], T3[10]};
  const float t1[3] = {T1[3], T1[7], T1[11]}, t2[3] = {T2[3], T2[7], T2[11]};
  kmat(Gm.K + 4LL * k1, P.K1); kmat(Gm.K + 4LL * k2, P.K2); kmat(Gm.K + 4LL * k3, P.K3);
  // R21 = Rcw2 * Rwc1; t21 = Rcw2 * (Rwc2 * tcw2 - Rwc1 * tcw1): two gemms, cv::subtract in fp32, a gemm
  float R21[9], a[3], b[3], d[3], t21[3];
  gemm33(R2, R1, R21, true);
  gemv3(R2, t2, a, true); gemv3(R1, t1, b, true);
  diff3(a, b, d);
  gemv3(R2, d, t21);
  // F21 = (K2.t()).inv() * t21x * R21 * K1.inv() = ((solve(K2^T, t21x) * R21) * invert(K1))
  float KT[9] = {P.K2[0], P.K2[3], P.K2[6], P.K2[1], P.K2[4], P.K2[7], P.K2[2], P.K2[5], P.K2[8]};
  float S[9] = {0.f, -t21[2], t21[1], t21[2], 0.f, -t21[0], -t21[1], t21[0], 0.f};
  lu_solve3(KT, S);
  float SR[9], K1i[9];
  gemm33(S, R21, SR, false);
  inv3(P.K1, K1i);
  gemm33(SR, K1i, P.F21, false);
  gemm33(R1, R2, P.R12, true);
  gemm33(R1, R3, P.R13, true);
  proj_matrix(P.K1, T1, P.M1); proj_matrix(P.K2, T2, P.M2); proj_matrix(P.K3, T3, P.M3);
}

// klF.t() * M for a line function narrowed to fp32 and a 3x4 M: cv::gemm with GEMM_1_T accumulates in fp64 from 0, then rounds
__device__ __forceinline__ void klf_row(const double* f, const float* M, float* row) {
  const float k0 = __double2float_rn(f[0]), k1 = __double2float_rn(f[1]), k2 = __double2float_rn(f[2]);
#pragma unroll
  for (int c = 0; c < 4; c++) row[c] = __double2float_rn(dsum3(dm(k0, M[c]), dm(k1, M[4 + c]), dm(k2, M[8 + c])));
}

// The gates of :1063-1416 for one triple; line3D is written when every gate passes.
__device__ int8_t gate_triple(const PairConsts& P, const PLTriLineGeometry& Gm, int k1, int k2, int k3, const KeyLineRec& l1,
                              const KeyLineRec& l2, const KeyLineRec& l3, const double* f1, const double* f2, const double* f3,
                              float median, float* line3D) {
  // :1065-1079 the epipolar plane
  const float lv2[2] = {__double2float_rn(-f2[1]), __double2float_rn(f2[0])};
  const float res1 = epipolar(P.F21, l1.startPointX, l1.startPointY, lv2);
  const float res2 = epipolar(P.F21, l1.endPointX, l1.endPointY, lv2);
  if ((double)fabsf(res1) > 0.996 || (double)fabsf(res2) > 0.996) return kEpipolar;
  // :1083-1114 the direction test
  float L1[3], L2[3], L3[3], a[3], b[3], tw[3];
  plane_normal(P.K1, l1, L1); plane_normal(P.K2, l2, L2); plane_normal(P.K3, l3, L3);
  gemv3(P.R12, L2, a); gemv3(P.R13, L3, b);
  cross3(a, b, tw);
  float nrm = fnorm3(tw);
  if (nrm == 0.f) return kZeroNorm;
  scale3(tw, nrm);
  nrm = fnorm3(L1);
  scale3(L1, nrm);
  if (nrm == 0.f) return kZeroNorm;
  const float cos_sita = __double2float_rn(fabs(ddot3(L1, tw)));
  if ((double)cos_sita > 0.0087) return kCosSita;
  // :1118-1171 both endpoints
  float r01[8], s3[3], e3[3];
  klf_row(f3, P.M3, r01); klf_row(f2, P.M2, r01 + 4);
  if (!endpoint(r01, P.M1, l1.startPointX, l1.startPointY, s3)) return kWZero;
  if (!endpoint(r01, P.M1, l1.endPointX, l1.endPointY, e3)) return kWZero;
  // :1176-1205 parallax
  const float *O1 = Gm.Ow + 3LL * k1, *O2 = Gm.Ow + 3LL * k2, *O3 = Gm.Ow + 3LL * k3;
  if (parallax_fails(s3, O1, O2, O3) || parallax_fails(e3, O1, O2, O3)) return kParallax;
  // :1207-1227 against pKF2's median depth
  float v[3];
  diff3(s3, O1, v);
  if ((double)__fdiv_rn(fnorm3(v), median) < 0.3) return kNear;
  diff3(s3, O2, v);
  if ((double)__fdiv_rn(fnorm3(v), median) < 0.3) return kNear;
  diff3(e3, s3, v);
  if ((double)__fdiv_rn(fnorm3(v), median) > 1.0) return kLong;
  // :1229-1252 depth
  const float *T1 = Gm.Tcw + 16LL * k1, *T2 = Gm.Tcw + 16LL * k2, *T3 = Gm.Tcw + 16LL * k3;
  const float zs1 = cam(T1, 2, s3);
  if (zs1 <= 0.f) return kBehind;
  const float ze1 = cam(T1, 2, e3);
  if (ze1 <= 0.f) return kBehind;
  const float zs2 = cam(T2, 2, s3);
  if (zs2 <= 0.f) return kBehind;
  const float ze2 = cam(T2, 2, e3);
  if (ze2 <= 0.f) return kBehind;
  const float zs3 = cam(T3, 2, s3);
  if (zs3 <= 0.f) return kBehind;
  const float ze3 = cam(T3, 2, e3);
  if (ze3 <= 0.f) return kBehind;
  // :1254-1331 reprojection, each view at its keyline's octave
  const float* T[3] = {T1, T2, T3};
  const int kk[3] = {k1, k2, k3};
  const KeyLineRec* kl[3] = {&l1, &l2, &l3};
  const double* f[3] = {f1, f2, f3};
  const float zs[3] = {zs1, zs2, zs3}, ze[3] = {ze1, ze2, ze3};
  float us[3], vs[3], ue[3], ve[3];
  for (int w = 0; w < 3; w++) {
    const float* kc = Gm.K + 4LL * kk[w];
    const float sigma2 = Gm.level_sigma2_line[kl[w]->octave];
    project(T[w], kc, zs[w], s3, us[w], vs[w]);
    if (reproj_fails(f[w], us[w], vs[w], sigma2)) return (int8_t)(kReproj1 + w);
    project(T[w], kc, ze[w], e3, ue[w], ve[w]);
    if (reproj_fails(f[w], ue[w], ve[w], sigma2)) return (int8_t)(kReproj1 + w);
  }
  // :1333-1416 overlap
  for (int w = 0; w < 3; w++)
    if (overlap_fails(*kl[w], us[w], vs[w], ue[w], ve[w])) return (int8_t)(kOverlap1 + w);
  line3D[0] = s3[0]; line3D[1] = s3[1]; line3D[2] = s3[2]; line3D[3] = e3[0]; line3D[4] = e3[1]; line3D[5] = e3[2];
  return kCommitted;
}

// (i, j) of pair index p among the E (E - 1) / 2 pairs i < j in the reference's order
__device__ __forceinline__ void pair_of(int p, int E, int& i, int& j) {
  i = 0;
  while (p >= E - 1 - i) { p -= E - 1 - i; i++; }
  j = i + 1 + p;
}

struct GroupView { int kc, e0, nE, ncur; long long oo; };

// Status of group g (plslam_b200.h, pl_lsd_triangulate_dev), the same in every thread of the block; every thread must call it.
__device__ int group_status(const LineTriArgs& A, int g, GroupView& v) {
  const PLTriLineKeyframes& K = A.K; const PLTriProblems& Q = A.Q; const PLTriLineGroups& Gr = A.Gr;
  v.kc = Gr.kf_cur[g]; v.e0 = Gr.entry_start[g]; v.nE = Gr.n_entries[g]; v.ncur = 0; v.oo = Gr.out_offset[g];
  int st = 0;
  if (v.nE < 0 || v.nE > kMaxE) st = 2;
  else if (v.e0 < 0 || (long long)v.e0 + v.nE > Gr.n_entry_list) st = 1;
  for (int e = 0; e < v.nE && !st; e++) {
    const int p = Gr.entry_problem[v.e0 + e];
    if (p < 0 || p >= Q.P) st = 1;
  }
  for (int e = 0; e < v.nE && !st; e++) st = A.search_status[Gr.entry_problem[v.e0 + e]];
  const auto in_table = [&](int k) { return k >= 0 && k < K.n_kf; };
  const auto count_ok = [&](int k) { return K.n[k] >= 0 && K.n[k] <= K.cap; };
  if (!st && !in_table(v.kc)) st = 1;
  for (int e = 0; e < v.nE && !st; e++) {
    const int p = Gr.entry_problem[v.e0 + e];
    if (!in_table(Gr.entry_kf[v.e0 + e]) || !in_table(Q.kf1[p]) || !in_table(Q.kf2[p])) st = 1;
  }
  if (!st && !count_ok(v.kc)) st = 2;
  for (int e = 0; e < v.nE && !st; e++) {
    const int p = Gr.entry_problem[v.e0 + e];
    if (!count_ok(Gr.entry_kf[v.e0 + e]) || !count_ok(Q.kf1[p]) || !count_ok(Q.kf2[p])) st = 2;
  }
  if (!st) {
    v.ncur = K.n[v.kc];
    const long long np = (long long)v.nE * (v.nE - 1) / 2;
    if (v.oo < 0 || v.oo + np * v.ncur > Gr.n_out) st = 1;
  }
  for (int e = 0; e < v.nE && !st; e++) {
    const int p = Gr.entry_problem[v.e0 + e];
    const long long qo = Q.out_offset[p];
    if (qo < 0 || qo + K.n[Q.kf1[p]] > Q.n_out) st = 1;
  }
  for (int e = 0; e < v.nE && !st; e++)
    if (Q.kf1[Gr.entry_problem[v.e0 + e]] != v.kc) st = 3;
  if (!st) {   // status 4: a matches entry outside -1 .. n[kf2] - 1 (every block of the group reads them, from L2)
    bool ok = true;
    for (int e = 0; e < v.nE; e++) {
      const int p = Gr.entry_problem[v.e0 + e], n2 = K.n[Q.kf2[p]];
      const int* m = A.matches + Q.out_offset[p];
      for (int i = threadIdx.x; i < v.ncur; i += blockDim.x) ok = ok && m[i] >= -1 && m[i] < n2;
    }
    if (!__syncthreads_and(ok)) st = 4;
  } else {
    __syncthreads_and(true);
  }
  return st;
}

// grid (G, kMaxPairs, ceil(cap / kLineGateSlots)): block (g, p, c) takes keylines c * kLineGateSlots .. of pair p of group g.  Every
// block decides the group's status from the same reads, so a group is written completely or not at all; block (g, 0, 0) writes
// status[g].
__global__ void __launch_bounds__(kLineGateSlots) k_line_tri_gates(const __grid_constant__ LineTriArgs A) {
  __shared__ PairConsts s_pc;
  const int g = blockIdx.x, pr = blockIdx.y, tid = threadIdx.x;
  GroupView v;
  const int st = group_status(A, g, v);
  if (blockIdx.y == 0 && blockIdx.z == 0 && tid == 0) A.status[g] = st;
  if (st) return;
  const int np = v.nE * (v.nE - 1) / 2;
  if (pr >= np || (int)blockIdx.z * kLineGateSlots >= v.ncur) return;
  int i, j;
  pair_of(pr, v.nE, i, j);
  const PLTriLineGroups& Gr = A.Gr; const PLTriLineGeometry& Gm = A.Gm; const PLTriLineKeyframes& K = A.K;
  const int pi = Gr.entry_problem[v.e0 + i], pj = Gr.entry_problem[v.e0 + j];
  const int k1 = v.kc, k2 = Gr.entry_kf[v.e0 + i], k3 = Gr.entry_kf[v.e0 + j];
  if (tid == 0) pair_consts(Gm, k1, k2, k3, s_pc);
  __syncthreads();
  const int ikl = blockIdx.z * kLineGateSlots + tid;
  if (ikl >= v.ncur) return;
  const long long slot = v.oo + (long long)pr * v.ncur + ikl;
  const int idx1 = A.matches[A.Q.out_offset[pi] + ikl], idx2 = A.matches[A.Q.out_offset[pj] + ikl];
  const int n2 = K.n[k2], n3 = K.n[k3];
  // :973 / :999 an entry without matches; :1041 no triple
  if (A.nmatches[pi] == 0 || A.nmatches[pj] == 0 || idx1 == -1 || idx2 == -1 || idx1 >= n2 || idx2 >= n3) {
    A.code[slot] = kNoTriple; return;
  }
  const long long r1 = (long long)k1 * K.cap + ikl, r2 = (long long)k2 * K.cap + idx1, r3 = (long long)k3 * K.cap + idx2;
  if (K.has_ml[r1] || K.has_ml[r2] || K.has_ml[r3]) { A.code[slot] = kHeld; return; }     // :1044 at the snapshot
  const KeyLineRec* kl = (const KeyLineRec*)Gm.keylines;
  A.code[slot] = gate_triple(s_pc, Gm, k1, k2, k3, kl[r1], kl[r2], kl[r3], Gm.line_func + 3 * r1, Gm.line_func + 3 * r2,
                             Gm.line_func + 3 * r3, Gr.entry_median_depth[v.e0 + i], A.line3D + 6 * slot);
}

// One CTA per group: warp 0 walks the slots in slot order against bit sets of taken keylines in shared memory, one per role (kf_cur,
// then each entry's positional keyframe; a role whose keyframe row an earlier role already has shares that role's set).  Per
// 32-slot chunk of a pair: the state at the chunk's start decides which slots are taken; the passed slots that remain commit in
// ascending ikl, one at a time, and after each commit the later slots of the chunk look again.  A gate-evaluated slot that finds a
// slot taken becomes kTaken.
__global__ void __launch_bounds__(kLineCommitThreads) k_line_tri_commit(const __grid_constant__ LineTriArgs A) {
  extern __shared__ unsigned s_bits[];
  __shared__ int s_alias[kRoles];
  const int g = blockIdx.x, tid = threadIdx.x;
  if (A.status[g]) return;
  const PLTriLineGroups& Gr = A.Gr; const PLTriLineKeyframes& K = A.K;
  const int kc = Gr.kf_cur[g], e0 = Gr.entry_start[g], nE = Gr.n_entries[g], ncur = K.n[kc];
  const long long oo = Gr.out_offset[g];
  const int W = (K.cap + 31) / 32;
  const auto row_of = [&](int r) { return r == 0 ? kc : Gr.entry_kf[e0 + r - 1]; };
  if (tid <= nE) {
    int a = tid;
    for (int r = 0; r < tid; r++)
      if (row_of(r) == row_of(tid)) { a = r; break; }
    s_alias[tid] = a;
  }
  for (int w = tid; w < (nE + 1) * W; w += kLineCommitThreads) s_bits[w] = 0u;
  __syncthreads();
  for (int r = 0; r <= nE; r++) {
    if (s_alias[r] != r) continue;
    const int row = row_of(r), n = K.n[row];
    for (int i = tid; i < n; i += kLineCommitThreads)
      if (K.has_ml[(long long)row * K.cap + i]) atomicOr(&s_bits[r * W + (i >> 5)], 1u << (i & 31));
  }
  __syncthreads();
  if (tid >= 32) return;
  const int lane = tid, np = nE * (nE - 1) / 2;
  const auto bit = [&](int role, int i) { return (s_bits[role * W + (i >> 5)] >> (i & 31)) & 1u; };
  int mine = 0;
  for (int pr = 0; pr < np; pr++) {
    int i, j;
    pair_of(pr, nE, i, j);
    const int ra = s_alias[0], rb = s_alias[1 + i], rc = s_alias[1 + j];
    const int* m1 = A.matches + A.Q.out_offset[Gr.entry_problem[e0 + i]];
    const int* m2 = A.matches + A.Q.out_offset[Gr.entry_problem[e0 + j]];
    const long long base = oo + (long long)pr * ncur;
    for (int c0 = 0; c0 < ncur; c0 += 32) {
      const int ikl = c0 + lane;
      const int8_t c = ikl < ncur ? A.code[base + ikl] : kNoTriple;
      const bool ev = c == kCommitted || c >= kEpipolar;     // the gates ran: the slots were free at the snapshot
      const int idx1 = ev ? m1[ikl] : 0, idx2 = ev ? m2[ikl] : 0;
      const auto taken = [&]() { return bit(ra, ikl) | bit(rb, idx1) | bit(rc, idx2); };
      bool t = ev && taken();
      unsigned rem = __ballot_sync(0xffffffffu, ev && !t && c == kCommitted);
      while (rem) {
        const int L = __ffs(rem) - 1;
        if (lane == L) {
          atomicOr(&s_bits[ra * W + (ikl >> 5)], 1u << (ikl & 31));
          atomicOr(&s_bits[rb * W + (idx1 >> 5)], 1u << (idx1 & 31));
          atomicOr(&s_bits[rc * W + (idx2 >> 5)], 1u << (idx2 & 31));
          mine++;
        }
        __syncwarp();
        if (lane > L && ev && !t) t = taken();
        rem = __ballot_sync(0xffffffffu, lane > L && ev && !t && c == kCommitted);
      }
      if (t) A.code[base + ikl] = kTaken;
      __syncwarp();
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if (lane == 0) A.nnew[g] = mine;
}
}  // namespace

}  // namespace pl

using namespace pl;

extern "C" int pl_lsd_triangulate_dev(const PLTriLineKeyframes* kfs, const PLTriLineGeometry* geom, const PLTriProblems* problems,
                                      const int* matches, const int* nmatches, const int* search_status, const PLTriLineGroups* groups,
                                      int8_t* code, float* line3D, int* nnew, int* status, void* stream) {
  PL_TRY(lsd_tri_args_ok(kfs, problems, matches, nmatches, search_status));
  PL_ARG(groups && groups->G >= 0 && groups->n_entry_list >= 0 && groups->n_out >= 0);
  const PLTriLineGroups& Gr = *groups;
  if (Gr.G == 0) return PL_OK;
  PL_TRY(lsd_tri_table_ok(kfs));
  PL_ARG(Gr.kf_cur && Gr.entry_start && Gr.n_entries && Gr.out_offset && Gr.entry_problem && Gr.entry_kf && Gr.entry_median_depth);
  PL_ARG(geom && geom->keylines && geom->line_func && geom->Tcw && geom->Ow && geom->K && geom->level_sigma2_line && geom->nlevels >= 1);
  PL_ARG(geom->n_kf == kfs->n_kf && geom->cap == kfs->cap);
  PL_ARG(nnew && status && (Gr.n_out == 0 || (code && line3D)));
  PL_TRY(require_device());
  const LineTriArgs A{*kfs, *geom, *problems, Gr, matches, nmatches, search_status, code, line3D, nnew, status};
  const dim3 grid(Gr.G, kMaxPairs, (kfs->cap + kLineGateSlots - 1) / kLineGateSlots);
  k_line_tri_gates<<<grid, kLineGateSlots, 0, (cudaStream_t)stream>>>(A);
  PL_LAUNCH_CHECK();
  const int smem = kRoles * ((kfs->cap + 31) / 32) * (int)sizeof(unsigned);
  PL_CUDA(cudaFuncSetAttribute(k_line_tri_commit, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_line_tri_commit<<<Gr.G, kLineCommitThreads, smem, (cudaStream_t)stream>>>(A);
  PL_LAUNCH_CHECK();
  return PL_OK;
}
