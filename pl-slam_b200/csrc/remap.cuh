// The undistortion map of a camera and the pixel arithmetic of cv::remap with it, shared by k_remap (frame.cu), which
// writes the undistorted frame, and k_lsd_front (line.cu), which reads undistorted pixels straight from the raw frame.
// initUndistortRectifyMap + remap(INTER_LINEAR, BORDER_CONSTANT 0): 1/32-pixel fixed point, 15-bit weights.
#pragma once
#include "common.cuh"

namespace pl {
struct RemapEntry { short ix, iy; unsigned short tab; unsigned short pad; };   // 8 B per output pixel, shared by all frames

// undistorted pixel of the frame S (row stride sstride, w x h) for map entry e: the 2x2 taps with the weights tab[e.tab]
// (16 KB int4 table, read through L1: per-lane index, not constant memory), taps outside the frame read 0
__device__ __forceinline__ uint8_t remap_px(const uint8_t* __restrict__ S, int sstride, int w, int h, RemapEntry e,
                                            const int4* __restrict__ tab) {
  const int4 t = __ldg(&tab[e.tab]);
  auto px = [&](int yy, int xx) { return (xx >= 0 && xx < w && yy >= 0 && yy < h) ? (int)S[(long long)yy * sstride + xx] : 0; };
  const int acc = px(e.iy, e.ix) * t.x + px(e.iy, e.ix + 1) * t.y + px(e.iy + 1, e.ix) * t.z + px(e.iy + 1, e.ix + 1) * t.w;
  return (uint8_t)((acc + (1 << 14)) >> 15);
}
struct CamD { double fx, fy, cx, cy, k1, k2, p1, p2, k3; };
}  // namespace pl

// pl_undistort_create: the map of one camera and frame size, on the device
struct PLUndistort {
  int w, h; pl::CamD cam; float K[4], D[5];
  pl::DevBuf<pl::RemapEntry> d_map;
  pl::DevBuf<int4> d_tab;
  struct HostStaging { pl::DevBuf<uint8_t> d_src, d_dst; };   // pl_undistort_remap (made on first use)
  std::unique_ptr<HostStaging> io;
  pl::Stream stream;
};
