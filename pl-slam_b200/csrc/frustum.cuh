// Frame::isInFrustum(MapPoint*) / (MapLine*) (src/Frame.cc:560-702, + PredictScale) and the camera centre of
// Frame::UpdatePoseMatrices (src/Frame.cc:552-558) as device functions of one frame's arguments: k_frustum_points /
// k_frustum_lines (frame.cu) run them on one frame, k_track_frustum_* (track.cu) on every (frame, local-map entry).
#pragma once
#include "libm_glibc.cuh"

namespace pl {
struct FrustumArgs {
  float T[16], Ow[3], K[4], bounds[4];
  float logScaleFactor, viewingCosLimit; int nScaleLevels, n;
};
__device__ __forceinline__ void gemm3(const float* T, const float* X, float* o) {
  for (int i = 0; i < 3; i++)
    o[i] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4 * i], X[0]), __fmul_rn(T[4 * i + 1], X[1])), __fmul_rn(T[4 * i + 2], X[2])), T[4 * i + 3]);
}
// mOw = -mRcw.t() * mtcw: cv::Mat's unary minus (exact in fp32), then the fp32 3x3 * 3x1 product summed left to right
__device__ __forceinline__ void camera_center(const float* T, float* Ow) {
  for (int i = 0; i < 3; i++)
    Ow[i] = __fadd_rn(__fadd_rn(__fmul_rn(-T[i], T[3]), __fmul_rn(-T[4 + i], T[7])), __fmul_rn(-T[8 + i], T[11]));
}
__device__ __forceinline__ bool project(const FrustumArgs& A, const float* Pc, float& u, float& v) {
  if (Pc[2] < 0.0f) return false;
  const float invz = __fdiv_rn(1.0f, Pc[2]);
  u = __fadd_rn(__fmul_rn(__fmul_rn(A.K[0], Pc[0]), invz), A.K[2]);
  v = __fadd_rn(__fmul_rn(__fmul_rn(A.K[1], Pc[1]), invz), A.K[3]);
  if (u < A.bounds[0] || u > A.bounds[2]) return false;
  if (v < A.bounds[1] || v > A.bounds[3]) return false;
  return true;
}
// MapPoint / MapLine::PredictScale before any clamp (MapPoint.cc:413-428, MapLine.cpp:395-404): ceil(log(maxDist / dist) /
// logScaleFactor) with fp32 operands and glibc's logf, so a ratio on a level boundary lands on the reference's side of it
__device__ __forceinline__ int predict_scale_level(float maxDist, float dist, float logScaleFactor) {
  return (int)ceilf(__fdiv_rn(glibc::logf_(__fdiv_rn(maxDist, dist)), logScaleFactor));
}
// true = mbTrackInView; then {u, v} = {mTrackProjX, mTrackProjY}, level = mnTrackScaleLevel, viewCos = mTrackViewCos
__device__ __forceinline__ bool frustum_point(const FrustumArgs& A, const float* pos, const float* normal, float minDist, float maxDist,
                                              float& u, float& v, int& level, float& viewCos) {
  const float P[3] = {pos[0], pos[1], pos[2]};
  float Pc[3];
  gemm3(A.T, P, Pc);
  if (!project(A, Pc, u, v)) return false;
  const float PO[3] = {__fsub_rn(P[0], A.Ow[0]), __fsub_rn(P[1], A.Ow[1]), __fsub_rn(P[2], A.Ow[2])};
  const float dist = (float)sqrt((double)PO[0] * PO[0] + (double)PO[1] * PO[1] + (double)PO[2] * PO[2]);
  if (dist < __fmul_rn(0.8f, minDist) || dist > __fmul_rn(1.2f, maxDist)) return false;   // Get{Min,Max}DistanceInvariance (MapPoint.cc:384-394)
  viewCos = (float)(((double)PO[0] * normal[0] + (double)PO[1] * normal[1] + (double)PO[2] * normal[2]) / dist);
  if (viewCos < A.viewingCosLimit) return false;
  int nScale = predict_scale_level(maxDist, dist, A.logScaleFactor);
  if (nScale < 0) nScale = 0; else if (nScale >= A.nScaleLevels) nScale = A.nScaleLevels - 1;
  level = nScale;
  return true;
}
// pos = MapLine::mWorldPos (start, end), normal = GetNormal; proj = {mTrackProjX1, Y1, X2, Y2}
__device__ __forceinline__ bool frustum_line(const FrustumArgs& A, const double* pos, const double* normal, float minDist, float maxDist,
                                             float* proj, int& level, float& viewCos) {
  const float SP[3] = {(float)pos[0], (float)pos[1], (float)pos[2]};
  const float EP[3] = {(float)pos[3], (float)pos[4], (float)pos[5]};
  float S[3], E[3], u1, v1, u2, v2;
  gemm3(A.T, SP, S); gemm3(A.T, EP, E);
  if (S[2] < 0.0f || E[2] < 0.0f) return false;
  if (!project(A, S, u1, v1)) return false;
  if (!project(A, E, u2, v2)) return false;
  float OM[3];
  for (int k = 0; k < 3; k++) OM[k] = __fsub_rn((float)(0.5 * (double)__fadd_rn(SP[k], EP[k])), A.Ow[k]);
  const float dist = (float)sqrt((double)OM[0] * OM[0] + (double)OM[1] * OM[1] + (double)OM[2] * OM[2]);
  if (dist < __fmul_rn(0.8f, minDist) || dist > __fmul_rn(1.2f, maxDist)) return false;   // MapLine.cpp:383-393
  const float pn[3] = {(float)normal[0], (float)normal[1], (float)normal[2]};
  viewCos = (float)(((double)OM[0] * pn[0] + (double)OM[1] * pn[1] + (double)OM[2] * pn[2]) / dist);
  if (viewCos < A.viewingCosLimit) return false;
  proj[0] = u1; proj[1] = v1; proj[2] = u2; proj[3] = v2;
  level = predict_scale_level(maxDist, dist, A.logScaleFactor);
  return true;
}
}  // namespace pl
