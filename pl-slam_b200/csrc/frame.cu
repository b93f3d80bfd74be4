// Frame glue around the hot path (SURVEY.md §8f.1), batched on sm_90a:
//   initUndistortRectifyMap + remap of every frame     Frame::Frame, src/Frame.cc:220-222  (the map is built ONCE per
//                                                      camera here; the reference rebuilds it for every frame)
//   Frame::UndistortKeyPoints                          src/Frame.cc:915-945 (cv::undistortPoints, 5 iterations, fp64)
//   Frame::ComputeImageBounds                          src/Frame.cc:947-985
//   Frame::isInFrustum(MapPoint*) / (MapLine*)         src/Frame.cc:560-702 (+ PredictScale)
// OpenCV arithmetic restated and pinned in the oracle: 1/32-pixel fixed-point bilinear remap with 15-bit weights,
// BORDER_CONSTANT 0; fp32 3x3 gemm as ((a0*b0 + a1*b1) + a2*b2) + c; cv::norm / dot with fp64 accumulation.
#include "common.cuh"
#include "frustum.cuh"
#include "remap.cuh"
#include <math.h>
#include <vector>

namespace pl {
// 4 consecutive output pixels per thread (uchar4 store where the row pointer is 4-byte aligned: a destination ROI may start
// at any column and dframe may be any size); the 2x2 source taps are gathered through L1/L2
__global__ void __launch_bounds__(256) k_remap(const uint8_t* __restrict__ src, int sstride, long long sframe, int w, int h,
                                               const RemapEntry* __restrict__ map, const int4* __restrict__ tab,
                                               uint8_t* __restrict__ dst, int dstride, long long dframe) {
  const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4, y = blockIdx.y;
  if (x4 >= w) return;
  const uint8_t* S = src + (long long)blockIdx.z * sframe;
  uint8_t o[4];
#pragma unroll
  for (int k = 0; k < 4; k++) o[k] = remap_px(S, sstride, w, h, map[(long long)y * w + min(x4 + k, w - 1)], tab);
  uint8_t* D = dst + (long long)blockIdx.z * dframe + (long long)y * dstride;
  if (x4 + 3 < w && (((uintptr_t)D & 3) == 0)) *reinterpret_cast<uchar4*>(D + x4) = make_uchar4(o[0], o[1], o[2], o[3]);
  else for (int k = 0; k < 4 && x4 + k < w; k++) D[x4 + k] = o[k];
}

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

__global__ void k_frustum_points(FrustumArgs A, const float* __restrict__ pos, const float* __restrict__ normal,
                                 const float* __restrict__ minDist, const float* __restrict__ maxDist, uint8_t* __restrict__ inview,
                                 float* __restrict__ proj, int* __restrict__ level, float* __restrict__ viewcos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  inview[i] = 0; proj[2 * i] = proj[2 * i + 1] = 0; level[i] = 0; viewcos[i] = 0;
  float u, v, vc; int l;
  if (!frustum_point(A, pos + 3 * i, normal + 3 * i, minDist[i], maxDist[i], u, v, l, vc)) return;
  inview[i] = 1; proj[2 * i] = u; proj[2 * i + 1] = v; level[i] = l; viewcos[i] = vc;
}
__global__ void k_frustum_lines(FrustumArgs A, const double* __restrict__ pos, const double* __restrict__ normal,
                                const float* __restrict__ minDist, const float* __restrict__ maxDist, uint8_t* __restrict__ inview,
                                float* __restrict__ proj, int* __restrict__ level, float* __restrict__ viewcos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  inview[i] = 0; for (int k = 0; k < 4; k++) proj[4 * i + k] = 0; level[i] = 0; viewcos[i] = 0;
  float pr[4], vc; int l;
  if (!frustum_line(A, pos + 6 * i, normal + 3 * i, minDist[i], maxDist[i], pr, l, vc)) return;
  inview[i] = 1; for (int k = 0; k < 4; k++) proj[4 * i + k] = pr[k];
  level[i] = l; viewcos[i] = vc;
}
}  // namespace pl
using namespace pl;

static CamD make_cam(const float* K, const float* D) { return CamD{(double)K[0], (double)K[1], (double)K[2], (double)K[3], (double)D[0], (double)D[1], (double)D[2], (double)D[3], (double)D[4]}; }

extern "C" void pl_undistort_destroy(PLUndistort* h) {
  if (!h) return;
  delete h;
}
extern "C" int pl_undistort_create(const float* K, const float* dist5, int width, int height, PLUndistort** out) {
  PL_ARG(K && dist5 && out && width > 0 && height > 0 && width < 32000 && height < 32000);
  int rc = require_device(); if (rc) return rc;
  std::unique_ptr<PLUndistort> h(new PLUndistort);
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
  PL_TRY(h->d_map.alloc(map.size()));
  PL_CUDA(cudaMemcpy(h->d_map, map.data(), map.size() * sizeof(RemapEntry), cudaMemcpyHostToDevice));
  PL_TRY(h->d_tab.alloc(sizeof(tab) / sizeof(int4)));
  PL_CUDA(cudaMemcpy(h->d_tab, tab, sizeof(tab), cudaMemcpyHostToDevice));
  PL_TRY(h->stream.create(cudaStreamNonBlocking));
  *out = h.release();
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
  if (!h->io) {
    auto io = std::make_unique<PLUndistort::HostStaging>();
    PL_TRY(io->d_src.alloc(n));
    PL_TRY(io->d_dst.alloc(n));
    h->io = std::move(io);
  }
  PL_CUDA(cudaMemcpy2DAsync(h->io->d_src, h->w, src, sstride, h->w, h->h, cudaMemcpyHostToDevice, h->stream));
  int rc = pl_undistort_remap_batch_dev(h, h->io->d_src, h->w, n, 1, h->io->d_dst, h->w, n, h->stream);
  if (rc) return rc;
  PL_CUDA(cudaMemcpy2DAsync(dst, dstride, h->io->d_dst, h->w, h->w, h->h, cudaMemcpyDeviceToHost, h->stream));
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
  Staging s;
  PLKeyPoint* di = s.in(kps, n); int* dn = s.in(&n, 1); PLKeyPoint* dout = s.out(out, n);
  int rc;
  if ((rc = s.status()) || (rc = s.sync()) || (rc = pl_undistort_keypoints_dev(h, di, dn, n, 1, dout, h->stream))) return rc;
  PL_CUDA(cudaStreamSynchronize(h->stream));
  return s.fetch();
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
extern "C" int pl_frame_is_in_frustum_points(const float* Tcw, const float* Ow, const float* K, const float* bounds,
                                             float log_scale_factor, int n_scale_levels, float viewing_cos_limit, int n,
                                             const float* pos, const float* normal, const float* min_dist, const float* max_dist,
                                             uint8_t* inview, float* proj, int* level, float* viewcos) {
  FrustumArgs A;
  int rc = frustum_common(A, Tcw, Ow, K, bounds, log_scale_factor, n_scale_levels, viewing_cos_limit, n); if (rc) return rc;
  if (n == 0) return PL_OK;
  PL_ARG(inview && proj && level && viewcos);
  Staging s;
  float* dp = s.in(pos, (size_t)n * 3); float* dn = s.in(normal, (size_t)n * 3); float* dmin = s.in(min_dist, n); float* dmax = s.in(max_dist, n);
  uint8_t* div = s.out(inview, n); float* dpr = s.out(proj, (size_t)n * 2); int* dl = s.out(level, n); float* dvc = s.out(viewcos, n);
  if ((rc = s.status())) return rc;
  k_frustum_points<<<(n + 127) / 128, 128>>>(A, dp, dn, dmin, dmax, div, dpr, dl, dvc);
  PL_LAUNCH_CHECK();
  PL_CUDA(cudaDeviceSynchronize());
  return s.fetch();
}
extern "C" int pl_frame_is_in_frustum_lines(const float* Tcw, const float* Ow, const float* K, const float* bounds,
                                            float log_scale_factor, float viewing_cos_limit, int n, const double* pos,
                                            const double* normal, const float* min_dist, const float* max_dist,
                                            uint8_t* inview, float* proj, int* level, float* viewcos) {
  FrustumArgs A;
  int rc = frustum_common(A, Tcw, Ow, K, bounds, log_scale_factor, 0, viewing_cos_limit, n); if (rc) return rc;
  if (n == 0) return PL_OK;
  PL_ARG(inview && proj && level && viewcos);
  Staging s;
  double* dp = s.in(pos, (size_t)n * 6); double* dn = s.in(normal, (size_t)n * 3); float* dmin = s.in(min_dist, n); float* dmax = s.in(max_dist, n);
  uint8_t* div = s.out(inview, n); float* dpr = s.out(proj, (size_t)n * 4); int* dl = s.out(level, n); float* dvc = s.out(viewcos, n);
  if ((rc = s.status())) return rc;
  k_frustum_lines<<<(n + 127) / 128, 128>>>(A, dp, dn, dmin, dmax, div, dpr, dl, dvc);
  PL_LAUNCH_CHECK();
  PL_CUDA(cudaDeviceSynchronize());
  return s.fetch();
}
