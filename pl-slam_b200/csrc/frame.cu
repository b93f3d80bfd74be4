// Frame glue around the hot path (SURVEY.md §8f.1), batched on sm_90a:
//   initUndistortRectifyMap + remap of every frame     Frame::Frame, src/Frame.cc:220-222  (the map is built ONCE per
//                                                      camera here; the reference rebuilds it for every frame)
//   Frame::UndistortKeyPoints                          src/Frame.cc:915-945 (cv::undistortPoints, 5 iterations, fp64)
//   Frame::ComputeImageBounds                          src/Frame.cc:947-985
//   Frame::isInFrustum(MapPoint*) / (MapLine*)         src/Frame.cc:560-702 (+ PredictScale)
// OpenCV arithmetic restated and pinned in the oracle: 1/32-pixel fixed-point bilinear remap with 15-bit weights,
// BORDER_CONSTANT 0; fp32 3x3 gemm as ((a0*b0 + a1*b1) + a2*b2) + c; cv::norm / dot with fp64 accumulation.
#include "common.cuh"
#include "libm_glibc.cuh"
#include <math.h>
#include <vector>

namespace pl {
struct RemapEntry { short ix, iy; unsigned short tab; unsigned short pad; };   // 8 B per output pixel, shared by all frames

// 4 consecutive output pixels per thread (uchar4 store); the 2x2 source taps are gathered through L1/L2
__global__ void __launch_bounds__(256) k_remap(const uint8_t* __restrict__ src, int sstride, long long sframe, int w, int h,
                                               const RemapEntry* __restrict__ map, const int4* __restrict__ tab,
                                               uint8_t* __restrict__ dst, int dstride, long long dframe) {
  const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4, y = blockIdx.y;
  if (x4 >= w) return;
  const uint8_t* S = src + (long long)blockIdx.z * sframe;
  uint8_t o[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int x = min(x4 + k, w - 1);
    const RemapEntry e = map[(long long)y * w + x];
    const int4 t = __ldg(&tab[e.tab]);     // 16 KB table, L1-resident (per-lane index: not constant memory)
    auto px = [&](int yy, int xx) { return (xx >= 0 && xx < w && yy >= 0 && yy < h) ? (int)S[(long long)yy * sstride + xx] : 0; };
    const int acc = px(e.iy, e.ix) * t.x + px(e.iy, e.ix + 1) * t.y + px(e.iy + 1, e.ix) * t.z + px(e.iy + 1, e.ix + 1) * t.w;
    o[k] = (uint8_t)((acc + (1 << 14)) >> 15);
  }
  uint8_t* D = dst + (long long)blockIdx.z * dframe + (long long)y * dstride;
  if (x4 + 3 < w && ((dstride & 3) == 0)) *reinterpret_cast<uchar4*>(D + x4) = make_uchar4(o[0], o[1], o[2], o[3]);
  else for (int k = 0; k < 4 && x4 + k < w; k++) D[x4 + k] = o[k];
}

struct CamD { double fx, fy, cx, cy, k1, k2, p1, p2, k3; };
__host__ __device__ inline void undistort_point(const CamD& c, float u, float v, float* ou, float* ov) {
  const double ifx = 1. / c.fx, ify = 1. / c.fy;
  double x = ((double)u - c.cx) * ifx, y = ((double)v - c.cy) * ify;
  const double x0 = x, y0 = y;
  for (int j = 0; j < 5; j++) {
    const double r2 = x * x + y * y;
    const double icdist = (1 + ((0 * r2 + 0) * r2 + 0) * r2) / (1 + ((c.k3 * r2 + c.k2) * r2 + c.k1) * r2);
    if (icdist < 0) { x = ((double)u - c.cx) * ifx; y = ((double)v - c.cy) * ify; break; }
    const double dX = 2 * c.p1 * x * y + c.p2 * (r2 + 2 * x * x), dY = c.p1 * (r2 + 2 * y * y) + 2 * c.p2 * x * y;
    x = (x0 - dX) * icdist; y = (y0 - dY) * icdist;
  }
  *ou = (float)(x * c.fx + c.cx); *ov = (float)(y * c.fy + c.cy);
}
__global__ void k_undistort_kps(CamD c, const PLKeyPoint* __restrict__ in, const int* __restrict__ n, int cap, PLKeyPoint* __restrict__ out) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= min(n[b], cap)) return;
  PLKeyPoint kp = in[(long long)b * cap + i];
  undistort_point(c, kp.x, kp.y, &kp.x, &kp.y);
  out[(long long)b * cap + i] = kp;
}

struct FrustumArgs {
  float T[16], Ow[3], K[4], bounds[4];
  float logScaleFactor, viewingCosLimit; int nScaleLevels, n;
};
__device__ __forceinline__ void gemm3(const float* T, const float* X, float* o) {
  for (int i = 0; i < 3; i++)
    o[i] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4 * i], X[0]), __fmul_rn(T[4 * i + 1], X[1])), __fmul_rn(T[4 * i + 2], X[2])), T[4 * i + 3]);
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
__global__ void k_frustum_points(FrustumArgs A, const float* __restrict__ pos, const float* __restrict__ normal,
                                 const float* __restrict__ minDist, const float* __restrict__ maxDist, uint8_t* __restrict__ inview,
                                 float* __restrict__ proj, int* __restrict__ level, float* __restrict__ viewcos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  inview[i] = 0; proj[2 * i] = proj[2 * i + 1] = 0; level[i] = 0; viewcos[i] = 0;
  const float P[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
  float Pc[3], u, v;
  gemm3(A.T, P, Pc);
  if (!project(A, Pc, u, v)) return;
  const float PO[3] = {__fsub_rn(P[0], A.Ow[0]), __fsub_rn(P[1], A.Ow[1]), __fsub_rn(P[2], A.Ow[2])};
  const float dist = (float)sqrt((double)PO[0] * PO[0] + (double)PO[1] * PO[1] + (double)PO[2] * PO[2]);
  if (dist < __fmul_rn(0.8f, minDist[i]) || dist > __fmul_rn(1.2f, maxDist[i])) return;   // Get{Min,Max}DistanceInvariance (MapPoint.cc:384-394)
  const float viewCos = (float)(((double)PO[0] * normal[3 * i] + (double)PO[1] * normal[3 * i + 1] + (double)PO[2] * normal[3 * i + 2]) / dist);
  if (viewCos < A.viewingCosLimit) return;
  const float ratio = __fdiv_rn(maxDist[i], dist);
  int nScale = (int)ceilf(__fdiv_rn(glibc::logf_(ratio), A.logScaleFactor));
  if (nScale < 0) nScale = 0; else if (nScale >= A.nScaleLevels) nScale = A.nScaleLevels - 1;
  inview[i] = 1; proj[2 * i] = u; proj[2 * i + 1] = v; level[i] = nScale; viewcos[i] = viewCos;
}
__global__ void k_frustum_lines(FrustumArgs A, const double* __restrict__ pos, const double* __restrict__ normal,
                                const float* __restrict__ minDist, const float* __restrict__ maxDist, uint8_t* __restrict__ inview,
                                float* __restrict__ proj, int* __restrict__ level, float* __restrict__ viewcos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  inview[i] = 0; for (int k = 0; k < 4; k++) proj[4 * i + k] = 0; level[i] = 0; viewcos[i] = 0;
  const float SP[3] = {(float)pos[6 * i], (float)pos[6 * i + 1], (float)pos[6 * i + 2]};
  const float EP[3] = {(float)pos[6 * i + 3], (float)pos[6 * i + 4], (float)pos[6 * i + 5]};
  float S[3], E[3], u1, v1, u2, v2;
  gemm3(A.T, SP, S); gemm3(A.T, EP, E);
  if (S[2] < 0.0f || E[2] < 0.0f) return;
  if (!project(A, S, u1, v1)) return;
  if (!project(A, E, u2, v2)) return;
  float OM[3];
  for (int k = 0; k < 3; k++) OM[k] = __fsub_rn((float)(0.5 * (double)__fadd_rn(SP[k], EP[k])), A.Ow[k]);
  const float dist = (float)sqrt((double)OM[0] * OM[0] + (double)OM[1] * OM[1] + (double)OM[2] * OM[2]);
  if (dist < __fmul_rn(0.8f, minDist[i]) || dist > __fmul_rn(1.2f, maxDist[i])) return;   // MapLine.cpp:383-393
  const float pn[3] = {(float)normal[3 * i], (float)normal[3 * i + 1], (float)normal[3 * i + 2]};
  const float viewCos = (float)(((double)OM[0] * pn[0] + (double)OM[1] * pn[1] + (double)OM[2] * pn[2]) / dist);
  if (viewCos < A.viewingCosLimit) return;
  const float ratio = __fdiv_rn(maxDist[i], dist);
  inview[i] = 1; proj[4 * i] = u1; proj[4 * i + 1] = v1; proj[4 * i + 2] = u2; proj[4 * i + 3] = v2;
  level[i] = (int)ceilf(__fdiv_rn(glibc::logf_(ratio), A.logScaleFactor)); viewcos[i] = viewCos;
}
}  // namespace pl
using namespace pl;

struct PLUndistort {
  int w, h; CamD cam; float K[4], D[5];
  RemapEntry* d_map = nullptr;
  int4* d_tab = nullptr;
  uint8_t *d_src = nullptr, *d_dst = nullptr; int staged = 0;
  cudaStream_t stream = nullptr;
};
static CamD make_cam(const float* K, const float* D) { return CamD{(double)K[0], (double)K[1], (double)K[2], (double)K[3], (double)D[0], (double)D[1], (double)D[2], (double)D[3], (double)D[4]}; }

extern "C" void pl_undistort_destroy(PLUndistort* h) {
  if (!h) return;
  cudaFree(h->d_map); cudaFree(h->d_tab); cudaFree(h->d_src); cudaFree(h->d_dst);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}
extern "C" int pl_undistort_create(const float* K, const float* dist5, int width, int height, PLUndistort** out) {
  PL_ARG(K && dist5 && out && width > 0 && height > 0 && width < 32000 && height < 32000);
  int rc = require_device(); if (rc) return rc;
  PLUndistort* h = new PLUndistort;
  h->w = width; h->h = height; h->cam = make_cam(K, dist5);
  memcpy(h->K, K, 16); memcpy(h->D, dist5, 20);
  const CamD& c = h->cam;
  // initUndistortRectifyMap(K, D, I, K, size, CV_32F): fp64 model per pixel (row-incremental like OpenCV), fp32 maps,
  // then remap's own conversion to 1/32-pixel fixed point; built once per camera on the host
  std::vector<RemapEntry> map((size_t)width * height);
  const double ir0 = 1.0 / c.fx, ir2 = -c.cx / c.fx, ir4 = 1.0 / c.fy, ir5 = -c.cy / c.fy;
  for (int i = 0; i < height; i++) {
    double _x = i * 0.0 + ir2, _y = i * ir4 + ir5, _w = i * 0.0 + 1.0;
    for (int j = 0; j < width; j++, _x += ir0, _y += 0.0, _w += 0.0) {
      const double ww = 1. / _w, x = _x * ww, y = _y * ww, x2 = x * x, y2 = y * y, r2 = x2 + y2, _2xy = 2 * x * y;
      const double kr = (1 + ((c.k3 * r2 + c.k2) * r2 + c.k1) * r2) / (1 + ((0 * r2 + 0) * r2 + 0) * r2);
      const float mx = (float)((x * kr + c.p1 * _2xy + c.p2 * (r2 + 2 * x2)) * c.fx + c.cx);
      const float my = (float)((y * kr + c.p1 * (r2 + 2 * y2) + c.p2 * _2xy) * c.fy + c.cy);
      const int sx = (int)lrintf(mx * 32.f), sy = (int)lrintf(my * 32.f);
      RemapEntry e;
      e.ix = (short)std::max(-32768, std::min(32767, sx >> 5)); e.iy = (short)std::max(-32768, std::min(32767, sy >> 5));
      e.tab = (unsigned short)(((sy & 31) * 32) + (sx & 31)); e.pad = 0;
      map[(size_t)i * width + j] = e;
    }
  }
  int tab[1024 * 4];
  {
    float t1[32][2];
    for (int i = 0; i < 32; i++) { float x = (float)i * (1.f / 32); t1[i][0] = 1.f - x; t1[i][1] = x; }
    for (int i = 0; i < 32; i++)
      for (int j = 0; j < 32; j++) {
        float wf[4] = {t1[i][0] * t1[j][0], t1[i][0] * t1[j][1], t1[i][1] * t1[j][0], t1[i][1] * t1[j][1]};
        int iw[4], isum = 0;
        for (int k = 0; k < 4; k++) { iw[k] = (int)lrintf(wf[k] * 32768.f); isum += iw[k]; }
        if (isum != 32768) {
          int diff = isum - 32768, mn = 0, mxk = 0;
          for (int k = 1; k < 4; k++) { if (iw[k] < iw[mn]) mn = k; if (iw[k] > iw[mxk]) mxk = k; }
          if (diff < 0) iw[mxk] -= diff; else iw[mn] -= diff;
        }
        for (int k = 0; k < 4; k++) tab[(i * 32 + j) * 4 + k] = iw[k];
      }
  }
  cudaError_t e = cudaMalloc((void**)&h->d_map, map.size() * sizeof(RemapEntry));
  if (e == cudaSuccess) e = cudaMemcpy(h->d_map, map.data(), map.size() * sizeof(RemapEntry), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMalloc((void**)&h->d_tab, sizeof(tab));
  if (e == cudaSuccess) e = cudaMemcpy(h->d_tab, tab, sizeof(tab), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { set_error("pl_undistort_create: %s", cudaGetErrorString(e)); pl_undistort_destroy(h); return PL_ERR_CUDA; }
  *out = h;
  return PL_OK;
}
extern "C" int pl_undistort_remap_batch_dev(PLUndistort* h, const uint8_t* src, int sstride, size_t sframe, int B, uint8_t* dst,
                                            int dstride, size_t dframe, void* stream) {
  PL_ARG(h && src && dst && B >= 1 && sstride >= h->w && dstride >= h->w);
  k_remap<<<dim3((h->w + 1023) / 1024, h->h, B), 256, 0, stream ? (cudaStream_t)stream : h->stream>>>(
      src, sstride, (long long)sframe, h->w, h->h, h->d_map, h->d_tab, dst, dstride, (long long)dframe);
  PL_LAUNCH_CHECK();
  return PL_OK;
}
extern "C" int pl_undistort_remap(PLUndistort* h, const uint8_t* src, int sstride, uint8_t* dst, int dstride) {
  PL_ARG(h && src && dst && sstride >= h->w && dstride >= h->w);
  const size_t n = (size_t)h->w * h->h;
  if (!h->staged) { PL_CUDA(cudaMalloc((void**)&h->d_src, n)); PL_CUDA(cudaMalloc((void**)&h->d_dst, n)); h->staged = 1; }
  PL_CUDA(cudaMemcpy2DAsync(h->d_src, h->w, src, sstride, h->w, h->h, cudaMemcpyHostToDevice, h->stream));
  int rc = pl_undistort_remap_batch_dev(h, h->d_src, h->w, n, 1, h->d_dst, h->w, n, h->stream);
  if (rc) return rc;
  PL_CUDA(cudaMemcpy2DAsync(dst, dstride, h->d_dst, h->w, h->w, h->h, cudaMemcpyDeviceToHost, h->stream));
  PL_CUDA(cudaStreamSynchronize(h->stream));
  return PL_OK;
}
extern "C" int pl_undistort_keypoints_dev(PLUndistort* h, const PLKeyPoint* kps, const int* n, int cap, int B, PLKeyPoint* out, void* stream) {
  PL_ARG(h && kps && n && out && cap > 0 && B > 0);
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  if (h->D[0] == 0.0f) { PL_CUDA(cudaMemcpyAsync(out, kps, (size_t)cap * B * sizeof(PLKeyPoint), cudaMemcpyDeviceToDevice, st)); return PL_OK; }  // Frame.cc:917-921
  k_undistort_kps<<<dim3((cap + 127) / 128, B), 128, 0, st>>>(h->cam, kps, n, cap, out);
  PL_LAUNCH_CHECK();
  return PL_OK;
}
extern "C" int pl_undistort_keypoints(PLUndistort* h, const PLKeyPoint* kps, int n, PLKeyPoint* out) {
  PL_ARG(h && kps && out && n >= 0);
  if (n == 0) return PL_OK;
  PLKeyPoint *di = nullptr, *dout = nullptr; int* dn = nullptr;
  PL_CUDA(cudaMalloc((void**)&di, (size_t)n * 28)); PL_CUDA(cudaMalloc((void**)&dout, (size_t)n * 28)); PL_CUDA(cudaMalloc((void**)&dn, 4));
  cudaMemcpy(di, kps, (size_t)n * 28, cudaMemcpyHostToDevice); cudaMemcpy(dn, &n, 4, cudaMemcpyHostToDevice);
  int rc = pl_undistort_keypoints_dev(h, di, dn, n, 1, dout, h->stream);
  cudaError_t e = cudaStreamSynchronize(h->stream);
  if (rc == PL_OK && e == cudaSuccess) e = cudaMemcpy(out, dout, (size_t)n * 28, cudaMemcpyDeviceToHost);
  cudaFree(di); cudaFree(dout); cudaFree(dn);
  if (rc) return rc;
  if (e != cudaSuccess) { set_error("pl_undistort_keypoints: %s", cudaGetErrorString(e)); return PL_ERR_CUDA; }
  return PL_OK;
}
// Frame::ComputeImageBounds: four corner points, host arithmetic (4 points)
extern "C" int pl_frame_image_bounds(const float* K, const float* dist5, int width, int height, float* bounds) {
  PL_ARG(K && dist5 && bounds);
  if (dist5[0] != 0.0f) {
    CamD c = make_cam(K, dist5);
    float m[4][2];
    const float pts[4][2] = {{0, 0}, {(float)width, 0}, {0, (float)height}, {(float)width, (float)height}};
    for (int i = 0; i < 4; i++) undistort_point(c, pts[i][0], pts[i][1], &m[i][0], &m[i][1]);
    bounds[0] = fminf(m[0][0], m[2][0]); bounds[2] = fmaxf(m[1][0], m[3][0]);
    bounds[1] = fminf(m[0][1], m[1][1]); bounds[3] = fmaxf(m[2][1], m[3][1]);
  } else { bounds[0] = 0; bounds[1] = 0; bounds[2] = (float)width; bounds[3] = (float)height; }
  return PL_OK;
}

static int frustum_common(FrustumArgs& A, const float* Tcw, const float* Ow, const float* K, const float* bounds, float logSF,
                          int nLevels, float cosLimit, int n) {
  PL_ARG(Tcw && Ow && K && bounds && n >= 0);
  memcpy(A.T, Tcw, 64); memcpy(A.Ow, Ow, 12); memcpy(A.K, K, 16); memcpy(A.bounds, bounds, 16);
  A.logScaleFactor = logSF; A.viewingCosLimit = cosLimit; A.nScaleLevels = nLevels; A.n = n;
  return require_device();
}
template <typename T> static T* upd(const T* h, size_t n, std::vector<void*>& fr) {
  T* d = nullptr;
  if (cudaMalloc((void**)&d, std::max<size_t>(n, 1) * sizeof(T)) != cudaSuccess) return nullptr;
  fr.push_back(d);
  if (h && n) cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice);
  return d;
}
extern "C" int pl_frame_is_in_frustum_points(const float* Tcw, const float* Ow, const float* K, const float* bounds,
                                             float log_scale_factor, int n_scale_levels, float viewing_cos_limit, int n,
                                             const float* pos, const float* normal, const float* min_dist, const float* max_dist,
                                             uint8_t* inview, float* proj, int* level, float* viewcos) {
  FrustumArgs A;
  int rc = frustum_common(A, Tcw, Ow, K, bounds, log_scale_factor, n_scale_levels, viewing_cos_limit, n); if (rc) return rc;
  if (n == 0) return PL_OK;
  std::vector<void*> fr;
  float* dp = upd(pos, (size_t)n * 3, fr); float* dn = upd(normal, (size_t)n * 3, fr); float* dmin = upd(min_dist, n, fr); float* dmax = upd(max_dist, n, fr);
  uint8_t* div = upd<uint8_t>(nullptr, n, fr); float* dpr = upd<float>(nullptr, (size_t)n * 2, fr); int* dl = upd<int>(nullptr, n, fr); float* dvc = upd<float>(nullptr, n, fr);
  int ret = PL_ERR_CUDA;
  if (dp && dn && dmin && dmax && div && dpr && dl && dvc) {
    k_frustum_points<<<(n + 127) / 128, 128>>>(A, dp, dn, dmin, dmax, div, dpr, dl, dvc);
    count_launch();
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(inview, div, n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(proj, dpr, (size_t)n * 8, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(level, dl, (size_t)n * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(viewcos, dvc, (size_t)n * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) ret = PL_OK; else set_error("isInFrustum: %s", cudaGetErrorString(e));
  } else set_error("isInFrustum: device allocation failed");
  for (void* p : fr) cudaFree(p);
  return ret;
}
extern "C" int pl_frame_is_in_frustum_lines(const float* Tcw, const float* Ow, const float* K, const float* bounds,
                                            float log_scale_factor, float viewing_cos_limit, int n, const double* pos,
                                            const double* normal, const float* min_dist, const float* max_dist,
                                            uint8_t* inview, float* proj, int* level, float* viewcos) {
  FrustumArgs A;
  int rc = frustum_common(A, Tcw, Ow, K, bounds, log_scale_factor, 0, viewing_cos_limit, n); if (rc) return rc;
  if (n == 0) return PL_OK;
  std::vector<void*> fr;
  double* dp = upd(pos, (size_t)n * 6, fr); double* dn = upd(normal, (size_t)n * 3, fr); float* dmin = upd(min_dist, n, fr); float* dmax = upd(max_dist, n, fr);
  uint8_t* div = upd<uint8_t>(nullptr, n, fr); float* dpr = upd<float>(nullptr, (size_t)n * 4, fr); int* dl = upd<int>(nullptr, n, fr); float* dvc = upd<float>(nullptr, n, fr);
  int ret = PL_ERR_CUDA;
  if (dp && dn && dmin && dmax && div && dpr && dl && dvc) {
    k_frustum_lines<<<(n + 127) / 128, 128>>>(A, dp, dn, dmin, dmax, div, dpr, dl, dvc);
    count_launch();
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(inview, div, n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(proj, dpr, (size_t)n * 16, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(level, dl, (size_t)n * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(viewcos, dvc, (size_t)n * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) ret = PL_OK; else set_error("isInFrustum(lines): %s", cudaGetErrorString(e));
  } else set_error("isInFrustum(lines): device allocation failed");
  for (void* p : fr) cudaFree(p);
  return ret;
}
