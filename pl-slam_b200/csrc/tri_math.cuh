// The rounding helpers of the triangulation kernels (triangulate.cu, triangulate_lines.cu): each reference expression on
// CV_32F Mats keeps its C++ promotions and its cv::Mat order, with every operation an _rn intrinsic so that nothing is contracted
// whatever -fmad says (DESIGN.md §8f.5, §8f.6).
#pragma once
#include <cuda_runtime.h>

namespace pl {
namespace tri {
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
// Mat::dot of a 3-vector pair in fp64 from 0, in index order
__device__ __forceinline__ double ddot3(const float* a, const float* b) {
  double s = 0;
#pragma unroll
  for (int k = 0; k < 3; k++) s = __dadd_rn(s, __dmul_rn((double)a[k], (double)b[k]));
  return s;
}
// row r of Rcw times x in fp64, plus t[r], rounded to fp32:  Rcw.row(r).dot(x3Dt) + tcw.at<float>(r)
__device__ __forceinline__ float cam(const float* T, int r, const float* x) {
  const float R[3] = {T[4 * r], T[4 * r + 1], T[4 * r + 2]};
  return __double2float_rn(__dadd_rn(ddot3(R, x), (double)T[4 * r + 3]));
}
// (float)(1.0 / v)
__device__ __forceinline__ float inv_d(float v) { return __double2float_rn(__ddiv_rn(1.0, (double)v)); }
}  // namespace tri
}  // namespace pl
