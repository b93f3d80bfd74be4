// SE3Quat arithmetic on the device (fp64): restated from Thirdparty/g2o/g2o/types/se3quat.h and the Eigen quaternion
// routines it calls.  Used by the optimisers: lm.cu, ba.cu and gba.cu, through g2o.cuh.
#pragma once
#include "common.cuh"
namespace pl {
struct Quat { double x, y, z, w; };
struct SE3 { Quat r; double t[3]; };

__device__ __forceinline__ void quat_normalize(Quat& q) {
  if (q.w < 0) { q.x = -q.x; q.y = -q.y; q.z = -q.z; q.w = -q.w; }
  double n = sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  q.x /= n; q.y /= n; q.z /= n; q.w /= n;
}
static __device__ Quat quat_from_matrix(const double m[3][3]) {
  Quat q;
  double t = m[0][0] + m[1][1] + m[2][2];
  if (t > 0) {
    t = sqrt(t + 1.0);
    q.w = 0.5 * t;
    t = 0.5 / t;
    q.x = (m[2][1] - m[1][2]) * t;
    q.y = (m[0][2] - m[2][0]) * t;
    q.z = (m[1][0] - m[0][1]) * t;
  } else {
    int i = 0;
    if (m[1][1] > m[0][0]) i = 1;
    if (m[2][2] > m[i][i]) i = 2;
    int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0);
    double v[3];
    v[i] = 0.5 * t;
    t = 0.5 / t;
    q.w = (m[k][j] - m[j][k]) * t;
    v[j] = (m[j][i] + m[i][j]) * t;
    v[k] = (m[k][i] + m[i][k]) * t;
    q.x = v[0]; q.y = v[1]; q.z = v[2];
  }
  return q;
}
__device__ __forceinline__ Quat quat_mul(const Quat& a, const Quat& b) {
  Quat r;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
  r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
  return r;
}
__device__ __forceinline__ void quat_rotate(const Quat& q, const double v[3], double out[3]) {
  double uv0 = q.y * v[2] - q.z * v[1], uv1 = q.z * v[0] - q.x * v[2], uv2 = q.x * v[1] - q.y * v[0];
  uv0 += uv0; uv1 += uv1; uv2 += uv2;
  out[0] = v[0] + q.w * uv0 + (q.y * uv2 - q.z * uv1);
  out[1] = v[1] + q.w * uv1 + (q.z * uv0 - q.x * uv2);
  out[2] = v[2] + q.w * uv2 + (q.x * uv1 - q.y * uv0);
}
static __device__ void quat_to_matrix(const Quat& q, double R[3][3]) {
  const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz; R[0][2] = txz + twy;
  R[1][0] = txy + twz; R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
  R[2][0] = txz - twy; R[2][1] = tyz + twx; R[2][2] = 1 - (txx + tyy);
}
__device__ __forceinline__ void se3_map(const SE3& T, const double X[3], double out[3]) {
  quat_rotate(T.r, X, out);
  out[0] += T.t[0]; out[1] += T.t[1]; out[2] += T.t[2];
}
static __device__ __noinline__ SE3 se3_exp(const double u[6]) {
  const double* w = u;
  const double* up = u + 3;
  double theta = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  double O[3][3] = {{0, -w[2], w[1]}, {w[2], 0, -w[0]}, {-w[1], w[0], 0}};
  double O2[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) { double s = 0; for (int k = 0; k < 3; k++) s += O[i][k] * O[k][j]; O2[i][j] = s; }
  double R[3][3], V[3][3];
  if (theta < 0.00001) {
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) { R[i][j] = (i == j ? 1.0 : 0.0) + O[i][j] + O2[i][j]; V[i][j] = R[i][j]; }
  } else {
    double a = sin(theta) / theta, b = (1 - cos(theta)) / (theta * theta);
    double c = (theta - sin(theta)) / pow(theta, 3.0);
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) {
        R[i][j] = (i == j ? 1.0 : 0.0) + a * O[i][j] + b * O2[i][j];
        V[i][j] = (i == j ? 1.0 : 0.0) + b * O[i][j] + c * O2[i][j];
      }
  }
  SE3 T;
  T.r = quat_from_matrix(R);
  for (int i = 0; i < 3; i++) T.t[i] = V[i][0] * up[0] + V[i][1] * up[1] + V[i][2] * up[2];
  quat_normalize(T.r);
  return T;
}
static __device__ __noinline__ SE3 se3_mul(const SE3& a, const SE3& b) {
  SE3 r;
  double rt[3];
  quat_rotate(a.r, b.t, rt);
  for (int i = 0; i < 3; i++) r.t[i] = a.t[i] + rt[i];
  r.r = quat_mul(a.r, b.r);
  quat_normalize(r.r);
  return r;
}
static __device__ SE3 se3_from_cv(const float* T) {
  double R[3][3];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) R[i][j] = (double)T[4 * i + j];
  SE3 s;
  s.r = quat_from_matrix(R);
  quat_normalize(s.r);
  for (int i = 0; i < 3; i++) s.t[i] = (double)T[4 * i + 3];
  return s;
}
static __device__ void se3_to_cv(const SE3& s, float* T) {
  double R[3][3];
  quat_to_matrix(s.r, R);
  for (int i = 0; i < 3; i++) { for (int j = 0; j < 3; j++) T[4 * i + j] = (float)R[i][j]; T[4 * i + 3] = (float)s.t[i]; }
  T[12] = 0; T[13] = 0; T[14] = 0; T[15] = 1;
}
}  // namespace pl
