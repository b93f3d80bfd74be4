// Line-feature extraction (LSD segments + LBD descriptors) for batches of frames on sm_90a.
//
// Replaces LINEextractor::operator() (reference src/LineExtractor.cpp:26-93) and what it calls:
//   LSDDetector::detect           opencv_contrib line_descriptor; spec copy Thirdparty/line_descriptor/src/LSDDetector_custom.cpp:56-215
//   cv::LineSegmentDetector       OpenCV imgproc lsd.cpp (defaults: REFINE_STD, scale .8, sigma_scale .6, quant 2, 22.5 deg, density .7)
//   BinaryDescriptor::compute     spec copy Thirdparty/line_descriptor/src/binary_descriptor_custom.cpp:350-398,539-687,1026-1372
//
// Kernel map (DESIGN.md §6)
//   k_lsd_front     one tiled pass from the raw frame (undistorted on the fly when a camera map is bound): 7x7 sigma .75
//                   Gaussian + 0.8x INTER_LINEAR_EXACT resize, 2x2 gradient -> one 16-byte record per pixel (angle, cos,
//                   sin), squared magnitude, seed cos/sin, per-frame max; and the LBD Sobel pair (below)
//   k_lsd_seed_order  stable counting sort of the defined pixels into 1024 magnitude bins (descending),
//                   equal bins keep row-major order == OpenCV 4.13's seed order (pinned in the oracle tests); one
//                   8-CTA cluster per frame, the order assembled in distributed shared memory.  k_lsd_hist/scan/scatter:
//                   the same sort through HBM (below 32 frames per SM, and frames too large for the cluster)
//   k_lsd_grow_ordered  region growing + rectangle fit + density refinement (lsd_grow_ordered.cuh); inherently ordered (a
//                   pixel consumed by an earlier seed is unavailable to later ones) -> ONE warp per frame walks the seeds in
//                   order; the 32 lanes test the 3x3 neighbourhood, evaluate angles and reduce the rectangle moments in parallel.
//   k_keylines      KeyLine records, mask filter, response sort (bitonic, ties keep detection order), truncation
//                   quirk of LineExtractor.cpp:44-67, normalised 2-D line equations
//   (k_lsd_front)   5x5 sigma 1 Gaussian (8.8 fixed point) fused with the 3x3 Sobel pair -> int16 dx, dy
//   k_lbd_describe  one CTA per line: 63 support rows in parallel (each row accumulates along the line in the
//                   reference's order, fp32 without FMA), band statistics, 72-float LBD, 32-byte binarisation

#include "common.cuh"
#include "libm_glibc.cuh"
#include "remap.cuh"
#include <cooperative_groups.h>
#include <math.h>
#include <string.h>
#include <stdlib.h>
#include <vector>
#include <algorithm>

namespace pl {

namespace cg = cooperative_groups;
constexpr double kPI = 3.14159265358979323846;
constexpr double kDegToRads = kPI / 180;
constexpr int kBins = 1024;
constexpr int kChunkRows = 8;


struct PLKeyLineRec {  // cv::line_descriptor::KeyLine, 68 bytes
  float angle; int class_id; int octave; float ptx, pty; float response; float size;
  float startPointX, startPointY, endPointX, endPointY;
  float sPointInOctaveX, sPointInOctaveY, ePointInOctaveX, ePointInOctaveY;
  float lineLength; int numOfPixels;
};
static_assert(sizeof(PLKeyLineRec) == 68, "KeyLine layout");

struct LineParams {
  int w, h, sw, sh, npx;        // image, scaled image, sw*sh
  int nchunk;                   // ceil((sh-1)/kChunkRows)
  int s_th;                     // gradient defined  <=>  gx^2+gy^2 > s_th
  int min_reg_size;
  int seg_cap, capL, nfeatures;
  double min_line_length;
  double prec, prec_hi, p, density_th;   // prec_hi: see region_grow (lsd_grow_ordered.cuh)
  float sure_ca2, sure_cn2;              // cos^2(prec -/+ 0.05 deg): lsd_grow_ordered.cuh Sure
};

// ---------------------------------------------------------------------------------------------- shared helpers
// ownership word of a pixel record (REC .x): free, or gradient undefined (never available); region growing marks USED with 0
constexpr int kFree = 0x7fffffff;
constexpr int kNotDef = -1;
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {  // cv::fastAtan2 (degrees), no FMA
  const float k = (float)(180.0 / 3.14159265358979323846);
  const float p1 = 0.9997878412794807f * k, p3 = -0.3258083974640975f * k;
  const float p5 = 0.1555786518463281f * k, p7 = -0.04432655554792128f * k;
  const float eps = 2.220446049250313e-16f;
  // ax >= ay ? ay/(ax+eps) : ax/(ay+eps)  ==  min/(max+eps): one division, no branch (this sits on the serial commit loop)
  const float ax = fabsf(x), ay = fabsf(y);
  const float c = __fdiv_rn(fminf(ax, ay), __fadd_rn(fmaxf(ax, ay), eps)), c2 = __fmul_rn(c, c);
  float a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
  if (ax < ay) a = __fsub_rn(90.f, a);
  if (x < 0) a = __fsub_rn(180.f, a);
  if (y < 0) a = __fsub_rn(360.f, a);
  return a;
}
__device__ __forceinline__ double angle_diff_signed(double a, double b) {
  double diff = a - b;
  while (diff <= -kPI) diff += 2 * kPI;
  while (diff > kPI) diff -= 2 * kPI;
  return diff;
}
__device__ __forceinline__ double dist_d(double x1, double y1, double x2, double y2) { return sqrt((x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1)); }
__device__ __forceinline__ double dist_sq(double x1, double y1, double x2, double y2) { return (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1); }

// ---------------------------------------------------------------------------------------------- gradient records
// Per scaled pixel, what region growing needs:
//   REC = 16-byte record {own, angle, cos, sin}: own = ownership word of the region growing (kFree or kNotDef here),
//         angle = level-line angle in degrees (cv::fastAtan2(gx, -gy)), cos/sin of float(angle_rad) rounded
//         to fp32 (what region_grow adds to sumdx/sumdy) -> ONE 16-byte load per neighbour in the growing step
//   S2  = s = gx^2+gy^2 (a pixel is defined iff s > s_th; modgrad = sqrt(s/4) comes from a table); seedcs: see grad_record
constexpr float kNotDefDeg = -1024.f;
// The level-line record of a pixel depends only on its integer gradient (gx, gy) in [-510, 510]^2: the angle in degrees
// (cv::fastAtan2(gx, -gy)), cos/sin of that angle as region_grow adds them, and the cos/sin a region SEEDED there starts
// from.  The fp64 sincos behind them is the whole cost of the gradient pass, so it is evaluated once per (gx, gy) into a
// 25 MB table at handle creation (L2-resident, the hot entries are the small gradients) and the per-frame kernel is loads.
constexpr int kGradR = 510, kGradN = 2 * kGradR + 1;
struct GradRec { float deg, c, s, pad; };
__device__ __forceinline__ void grad_record(int gx, int gy, GradRec& rec, float2& scs) {
  const float deg = fast_atan2_deg((float)gx, (float)(-gy));
  const double af = (double)(float)((double)deg * kDegToRads);
  double sn, cs;
  sincos(af, &sn, &cs);
  rec.deg = deg; rec.c = (float)cs; rec.s = (float)sn; rec.pad = 0.f;
  // a region SEEDED here starts from cos/sin of the fp64 angle ad = af + dl, |dl| <= half an fp32 ulp (< 4e-7):
  // angle-addition with cos(dl) = 1 - dl^2/2, sin(dl) = dl is exact to ~1e-27, far below fp64 rounding
  const double ad = (double)deg * kDegToRads, dl = ad - af, h2 = 1.0 - 0.5 * dl * dl;
  scs = make_float2((float)(cs * h2 - sn * dl), (float)(sn * h2 + cs * dl));
}
__global__ void __launch_bounds__(256) k_lsd_grad_table(GradRec* __restrict__ T, float2* __restrict__ TS) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= kGradN * kGradN) return;
  GradRec rec; float2 scs;
  grad_record(i / kGradN - kGradR, i % kGradN - kGradR, rec, scs);
  T[i] = rec; TS[i] = scs;
}
// ---------------------------------------------------------------------------------------------- K_A front: image -> LSD + LBD inputs
// One pass per (tile, frame) builds everything the later stages read from the frame, from the raw frame in HBM:
//   source    the undistorted pixel (remap.cuh, when a camera map is bound) or the frame itself, at reflect-101 coordinates
//   LSD       7x7 sigma .75 Gaussian (8.8 fixed point; its taps at +-3 are zero) + 0.8x INTER_LINEAR_EXACT resize -> scaled
//             image; 2x2 gradient -> pixel record, gx^2+gy^2 and seed cos/sin (see grad_record), per-frame max of gx^2+gy^2
//   LBD       5x5 sigma 1 Gaussian (8.8 fixed point) + 3x3 Sobel pair -> int16 dx, dy
// Tile: 64x32 scaled pixels <-> 80x40 undistorted pixels.  Scaled x reads blurred (10x+1)>>3 and the pixel after it, so
// scaled columns [64i, 64i+64) read blurred columns [80i, 80i+80), and the same 80 columns are the tile's Sobel outputs.
// One source tile serves both: undistorted columns 80i-3 .. 80i+83, rows 40j-3 .. 40j+43 (the 5-tap blurs, one more scaled
// column and row for the 2x2 gradient, the blurred ring of the Sobel).  Every source position is loaded at the
// reflect-101 coordinate both kernels it restates used: the LBD blur is symmetric, so the blurred value of the reflected
// image at -1 equals the one at +1, exactly Sobel's own BORDER_REFLECT_101 of the blurred image; no tap reflects again.
// A CTA keeps its tile and walks kFrontFrames frames: the camera map of the tile (32 KB) is read from L2 once per CTA.
// Every output row of a warp is contiguous (one thread per pixel): a warp stores 512 B of records, 256 B of seed cos/sin
// and 128 B of gx^2+gy^2 in whole sectors.
constexpr int kFrontSX = 64, kFrontSY = 32;                          // scaled pixels per tile
constexpr int kFrontUX = 80, kFrontUY = 40;                          // undistorted (Sobel) pixels per tile
constexpr int kFrontSrcW = kFrontUX + 7, kFrontSrcH = kFrontUY + 7;  // source tile: 3 before, 4 after
constexpr int kFrontSrcP = kFrontSrcW + 1;
constexpr int kFrontBW = kFrontUX + 2, kFrontBH = kFrontUY + 2;      // blurred tiles (LSD: +2 after; LBD: 1 before, 1 after)
constexpr int kFrontSegRows = kFrontBH / 3;                          // blur: 3 row segments x 82 columns = 246 threads
constexpr int kFrontFrames = 8;                                      // frames per CTA
constexpr int kFrontThreads = 256;
static_assert(kFrontBH % 3 == 0 && 3 * kFrontBW <= kFrontThreads, "blur thread layout");
constexpr size_t kFrontMapSmem = (size_t)kFrontSrcH * kFrontSrcW * sizeof(RemapEntry);

template <bool kMap>
__global__ void __launch_bounds__(kFrontThreads) k_lsd_front(LineParams P, const uint8_t* __restrict__ imgs, int stride,
                                                             long long frame_stride, int B, const RemapEntry* __restrict__ map,
                                                             const int4* __restrict__ tab, const float4* __restrict__ T,
                                                             const float2* __restrict__ TS, uint8_t* __restrict__ scaled,
                                                             int4* __restrict__ REC, int* __restrict__ S2, float2* __restrict__ seedcs,
                                                             int* __restrict__ maxs, short2* __restrict__ dxy) {
  extern __shared__ __align__(16) unsigned char front_smem[];
  RemapEntry* mp = reinterpret_cast<RemapEntry*>(front_smem);        // [kFrontSrcH * kFrontSrcW] (kMap only)
  __shared__ uint8_t src[kFrontSrcH * kFrontSrcP];                   // undistorted (V0-3+r, U0-3+c)
  __shared__ uint8_t bl[kFrontBH * kFrontBW];                        // LSD blur at (V0+r, U0+c)
  __shared__ uint8_t bs[kFrontBH * kFrontBW];                        // LBD blur at (V0-1+r, U0-1+c)
  __shared__ uint8_t sc[(kFrontSY + 1) * (kFrontSX + 1)];           // scaled (Y0+r, X0+c), 0 outside the image
  __shared__ int smax[kFrontFrames];
  const int tid = threadIdx.x, lane = tid & 31;
  const int X0 = blockIdx.x * kFrontSX, Y0 = blockIdx.y * kFrontSY, U0 = blockIdx.x * kFrontUX, V0 = blockIdx.y * kFrontUY;
  const int f0 = blockIdx.z * kFrontFrames, nf = min(kFrontFrames, B - f0);
  auto srow = [&](int r) { return reflect101(min(V0 - 3 + r, 2 * P.h - 2), P.h); };
  auto scol = [&](int c) { return reflect101(min(U0 - 3 + c, 2 * P.w - 2), P.w); };
  if (tid < kFrontFrames) smax[tid] = 0;
  if (kMap)
    for (int i = tid; i < kFrontSrcH * kFrontSrcW; i += kFrontThreads) {
      const int r = i / kFrontSrcW, c = i - r * kFrontSrcW;
      mp[i] = map[(long long)srow(r) * P.w + scol(c)];
    }
  __syncthreads();
  for (int fi = 0; fi < nf; fi++) {
    const int f = f0 + fi;
    const uint8_t* img = imgs + (long long)f * frame_stride;
    // 1. source tile
    for (int i = tid; i < kFrontSrcH * kFrontSrcW; i += kFrontThreads) {
      const int r = i / kFrontSrcW, c = i - r * kFrontSrcW;
      src[r * kFrontSrcP + c] = kMap ? remap_px(img, stride, P.w, P.h, mp[i], tab) : img[(long long)srow(r) * stride + scol(c)];
    }
    __syncthreads();
    // 2. both blurs: a thread walks down one blurred column of a row segment with the last five row sums of each in registers;
    //    LBD column c reads source columns c..c+4, LSD column c source columns c+1..c+5
    if (tid < 3 * kFrontBW) {
      const int c = tid % kFrontBW, r0 = (tid / kFrontBW) * kFrontSegRows;
      const uint8_t* p = src + r0 * kFrontSrcP + c;
      int hs[5] = {0, 0, 0, 0, 0}, hl[5] = {0, 0, 0, 0, 0};
#pragma unroll
      for (int k = 0; k < kFrontSegRows + 5; k++, p += kFrontSrcP) {
        const int q0 = p[0], q1 = p[1], q2 = p[2], q3 = p[3], q4 = p[4], q5 = p[5];
#pragma unroll
        for (int j = 0; j < 4; j++) { hs[j] = hs[j + 1]; hl[j] = hl[j + 1]; }
        hs[4] = 14 * (q0 + q4) + 62 * (q1 + q3) + 104 * q2;
        hl[4] = 4 * (q1 + q5) + 56 * (q2 + q4) + 136 * q3;
        if (k >= 4 && k - 4 < kFrontSegRows) {       // LBD row r0+k-4 <- source rows r0+k-4 .. r0+k
          const unsigned acc = 14u * (unsigned)(hs[0] + hs[4]) + 62u * (unsigned)(hs[1] + hs[3]) + 104u * (unsigned)hs[2];
          bs[(r0 + k - 4) * kFrontBW + c] = (uint8_t)((acc + 32768u) >> 16);
        }
        if (k >= 5) {                                 // LSD row r0+k-5 <- source rows r0+k-4 .. r0+k
          const unsigned s = 4u * (unsigned)(hl[0] + hl[4]) + 56u * (unsigned)(hl[1] + hl[3]) + 136u * (unsigned)hl[2];
          bl[(r0 + k - 5) * kFrontBW + c] = (uint8_t)((s + 32768u) >> 16);
        }
      }
    }
    __syncthreads();
    // 3. 0.8x resize (INTER_LINEAR_EXACT, clamps at w-1 and h-1) of the tile and one more column and row
    uint8_t* out = scaled + (long long)f * P.npx;
    for (int i = tid; i < (kFrontSY + 1) * (kFrontSX + 1); i += kFrontThreads) {
      const int ty = i / (kFrontSX + 1), tx = i - ty * (kFrontSX + 1);
      const int x = X0 + tx, y = Y0 + ty;
      uint8_t v = 0;
      if (x < P.sw && y < P.sh) {
        int sx = (10 * x + 1) >> 3, xf = ((10 * x + 1) & 7) * 32;
        int sy = (10 * y + 1) >> 3, yf = ((10 * y + 1) & 7) * 32;
        if (sx >= P.w - 1) { sx = P.w - 1; xf = 0; }
        if (sy >= P.h - 1) { sy = P.h - 1; yf = 0; }
        const int sx1 = min(sx + 1, P.w - 1), sy1 = min(sy + 1, P.h - 1);
        const uint8_t* b0 = bl + (sy - V0) * kFrontBW;
        const uint8_t* b1 = bl + (sy1 - V0) * kFrontBW;
        const int h0 = b0[sx - U0] * (256 - xf) + b0[sx1 - U0] * xf;
        const int h1 = b1[sx - U0] * (256 - xf) + b1[sx1 - U0] * xf;
        v = (uint8_t)((h0 * (256 - yf) + h1 * yf + 32768) >> 16);
        if (tx < kFrontSX && ty < kFrontSY) out[(long long)y * P.sw + x] = v;
      }
      sc[i] = v;
    }
    __syncthreads();
    // 4. gradient records: one pixel per thread, a warp on 32 consecutive pixels of a row
    int smx = 0;
    for (int i = tid; i < kFrontSY * kFrontSX; i += kFrontThreads) {
      const int ty = i / kFrontSX, tx = i - ty * kFrontSX;
      const int x = X0 + tx, y = Y0 + ty;
      if (x >= P.sw || y >= P.sh) continue;
      int4 rec = make_int4(kNotDef, __float_as_int(kNotDefDeg), 0, 0);
      float2 se = make_float2(0.f, 0.f);
      int sq = 0;
      if (x < P.sw - 1 && y < P.sh - 1) {
        const uint8_t* q = sc + ty * (kFrontSX + 1) + tx;
        const int DA = q[kFrontSX + 2] - q[0], BC = q[1] - q[kFrontSX + 1];
        const int gx = DA + BC, gy = DA - BC;
        sq = gx * gx + gy * gy;
        if (sq > P.s_th) {
          const int ti = (gx + kGradR) * kGradN + (gy + kGradR);
          const float4 t = __ldg(&T[ti]);
          se = __ldg(&TS[ti]);
          rec = make_int4(kFree, __float_as_int(t.x), __float_as_int(t.y), __float_as_int(t.z));
          smx = max(smx, sq);
        }
      }
      const long long o = (long long)f * P.npx + (long long)y * P.sw + x;
      REC[o] = rec; S2[o] = sq; seedcs[o] = se;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) smx = max(smx, __shfl_xor_sync(0xffffffffu, smx, o));
    if (lane == 0 && smx > 0) atomicMax(&smax[fi], smx);
    // 5. Sobel pair of the tile's undistorted pixels
    short2* D = dxy + (long long)f * P.w * P.h;
    for (int i = tid; i < kFrontUY * kFrontUX; i += kFrontThreads) {
      const int ry = i / kFrontUX, rx = i - ry * kFrontUX;
      const int x = U0 + rx, y = V0 + ry;
      if (x >= P.w || y >= P.h) continue;
      const uint8_t* b = bs + ry * kFrontBW + rx;
      const int a00 = b[0], a01 = b[1], a02 = b[2];
      const int a10 = b[kFrontBW], a12 = b[kFrontBW + 2];
      const int a20 = b[2 * kFrontBW], a21 = b[2 * kFrontBW + 1], a22 = b[2 * kFrontBW + 2];
      D[(long long)y * P.w + x] = make_short2((short)((a02 - a00) + 2 * (a12 - a10) + (a22 - a20)),
                                              (short)((a20 - a00) + 2 * (a21 - a01) + (a22 - a02)));
    }
    // the next frame's stages 1-3 overwrite src, bl/bs and sc only after its first barrier: every read of this frame is done
  }
  __syncthreads();
  if (tid < nf && smax[tid] > 0) atomicMax(&maxs[f0 + tid], smax[tid]);
}
__device__ __forceinline__ double s_norm(int s) { return sqrt((double)s / 4.0); }
__device__ __forceinline__ int s_bin(int s, double bin_coef) { return (int)(s_norm(s) * bin_coef); }

// K_C per-chunk histograms of the defined pixels (chunk = kChunkRows image rows)
__global__ void __launch_bounds__(256) k_lsd_hist(LineParams P, const int* __restrict__ S2, const int* __restrict__ maxs,
                                                  unsigned short* __restrict__ counts /*[B][kBins][nchunk]*/) {
  __shared__ int hist[kBins];
  const int chunk = blockIdx.x, f = blockIdx.y, tid = threadIdx.x;
  for (int i = tid; i < kBins; i += 256) hist[i] = 0;
  __syncthreads();
  const int ms = maxs[f];
  const double max_grad = ms > 0 ? sqrt((double)ms / 4.0) : -1.0;
  const double bin_coef = (max_grad > 0) ? (double)(kBins - 1) / max_grad : 0.0;
  const int y0 = chunk * kChunkRows, y1 = min(y0 + kChunkRows, P.sh - 1);
  const int* SS = S2 + (long long)f * P.npx;
  for (int i = tid; i < (y1 - y0) * P.sw; i += 256) {
    int y = y0 + i / P.sw, x = i % P.sw;
    const int sv = SS[y * P.sw + x];                 // border pixels carry s = 0: never above the threshold
    if (sv > P.s_th) atomicAdd(&hist[s_bin(sv, bin_coef)], 1);
  }
  __syncthreads();
  for (int i = tid; i < kBins; i += 256) counts[((long long)f * kBins + i) * P.nchunk + chunk] = (unsigned short)hist[i];
}

// K_D offsets[bin][chunk] = number of defined pixels that precede (bin desc, chunk asc); ndef = total
__global__ void __launch_bounds__(kBins) k_lsd_scan(LineParams P, const unsigned short* __restrict__ counts,
                                                    int* __restrict__ offsets, int* __restrict__ ndef) {
  __shared__ int wsum[32];
  const int f = blockIdx.x, t = threadIdx.x, bin = kBins - 1 - t, lane = t & 31, wid = t >> 5;
  const unsigned short* c = counts + ((long long)f * kBins + bin) * P.nchunk;
  int tot = 0;
  for (int k = 0; k < P.nchunk; k++) tot += c[k];
  int incl = tot;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  if (lane == 31) wsum[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int v = wsum[lane], in2 = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, in2, o); if (lane >= o) in2 += u; }
    wsum[lane] = in2 - v;
    if (lane == 31) ndef[f] = in2;
  }
  __syncthreads();
  int base = wsum[wid] + incl - tot;
  int* o = offsets + ((long long)f * kBins + bin) * P.nchunk;
  for (int k = 0; k < P.nchunk; k++) { o[k] = base; base += c[k]; }
}

// K_E stable scatter: one warp per chunk walks its pixels in row-major order
__global__ void __launch_bounds__(128) k_lsd_scatter(LineParams P, const int* __restrict__ S2, const int* __restrict__ maxs,
                                                     const int* __restrict__ offsets, unsigned* __restrict__ order) {
  __shared__ unsigned short cnt[4][kBins];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunk = blockIdx.x * 4 + wid, f = blockIdx.y;
  for (int i = lane; i < kBins; i += 32) cnt[wid][i] = 0;
  __syncwarp();
  if (chunk >= P.nchunk) return;
  const int ms = maxs[f];
  const double max_grad = ms > 0 ? sqrt((double)ms / 4.0) : -1.0;
  const double bin_coef = (max_grad > 0) ? (double)(kBins - 1) / max_grad : 0.0;
  const int y0 = chunk * kChunkRows, y1 = min(y0 + kChunkRows, P.sh - 1);
  const int* SS = S2 + (long long)f * P.npx;
  const int* off = offsets + (long long)f * kBins * P.nchunk;
  unsigned* O = order + (long long)f * P.npx;
  const int n = (y1 - y0) * P.sw;
  const unsigned lt = (1u << lane) - 1u;
  for (int i0 = 0; i0 < n; i0 += 32) {
    int i = i0 + lane, bin = -1, pix = 0;
    if (i < n) {
      int y = y0 + i / P.sw, x = i % P.sw;
      pix = x | (y << 16);                       // packed (x, y): the grow kernel never divides
      const int sv = SS[y * P.sw + x];
      if (sv > P.s_th) bin = s_bin(sv, bin_coef);
    }
    unsigned peers = __match_any_sync(0xffffffffu, bin);
    if (bin >= 0) O[off[bin * P.nchunk + chunk] + cnt[wid][bin] + __popc(peers & lt)] = (unsigned)pix;
    __syncwarp();
    if (bin >= 0 && (peers & lt) == 0) cnt[wid][bin] += (unsigned short)__popc(peers);
    __syncwarp();
  }
}

// K_CDE the same stable counting sort in one thread-block cluster per frame, on chip (the default from 32 frames per SM on,
// see pl_line_extract_batch_dev).  The scatter above stores 4 bytes per pixel into ~50k (bin, chunk) runs of
// 2-4 entries spread over the whole order array, so at full batches the order sectors leave L2 partly written.  Here:
//   CTA r of the cluster covers the pixel range [r*Q, (r+1)*Q) of the frame (rows 0..sh-2, row-major), its warp w the
//   w-th piece of U pixels of that range
//   1. histogram   per-(warp, bin) counts in shared memory (16-bit, two per 32-bit word for the atomics)
//   2. scan        counts -> within-CTA exclusive offsets over the warps; the CTA's per-bin totals are exchanged through
//                  distributed shared memory, every CTA derives the (bin desc, CTA asc) bases itself; CTA 0 writes ndef
//   3. scatter     each warp walks its piece in row-major order exactly like k_lsd_scatter and stores every entry into the
//                  shared memory of the CTA that owns its output position (CTA q owns [q*S, (q+1)*S))
//   4. flush       after a cluster barrier each CTA writes its slice of order [0, ndef) with 16-byte stores
// S2 is read twice (the second pass finds it in L2: the cluster has just read it); order is written once, in full sectors.
constexpr int kSeedCta = 8;       // CTAs per cluster (one cluster per frame)
constexpr int kSeedWarps = 32;    // warps per CTA
__device__ __forceinline__ int seed_bin(int sv, int s_th, double bin_coef) { return sv > s_th ? s_bin(sv, bin_coef) : -1; }

__global__ void __cluster_dims__(kSeedCta, 1, 1) __launch_bounds__(kSeedWarps * 32, 1)
k_lsd_seed_order(LineParams P, int Q, int U, int S, const int* __restrict__ S2, const int* __restrict__ maxs,
                 unsigned* __restrict__ order, int* __restrict__ ndef) {
  extern __shared__ __align__(16) unsigned char seed_smem[];
  unsigned* slice = reinterpret_cast<unsigned*>(seed_smem);                     // [S] this CTA's part of the order
  unsigned short* cnt = reinterpret_cast<unsigned short*>(slice + S);           // [kSeedWarps][kBins]
  int* tot = reinterpret_cast<int*>(cnt + kSeedWarps * kBins);                  // [kBins] this CTA's count per bin
  int* base = tot + kBins;                                                      // [kBins] first position of (bin, this CTA)
  __shared__ int wsum[kSeedWarps];
  __shared__ int s_nd;
  cg::cluster_group cluster = cg::this_cluster();
  const int r = (int)cluster.block_rank(), f = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int i = tid; i < kSeedWarps * kBins / 2; i += kSeedWarps * 32) reinterpret_cast<unsigned*>(cnt)[i] = 0u;
  const int ms = maxs[f];
  const double max_grad = ms > 0 ? sqrt((double)ms / 4.0) : -1.0;
  const double bin_coef = (max_grad > 0) ? (double)(kBins - 1) / max_grad : 0.0;
  const int nrow = (P.sh - 1) * P.sw;                 // the last row is never defined
  const int c1 = min((r + 1) * Q, nrow);
  const int u0 = min(r * Q + wid * U, c1), u1 = min(u0 + U, c1);
  const int* SS = S2 + (long long)f * P.npx;
  __syncthreads();
  // 1. histogram of this warp's piece (4 loads in flight per lane)
  unsigned* cw = reinterpret_cast<unsigned*>(cnt + wid * kBins);
  for (int i0 = u0; i0 < u1; i0 += 128) {
    int sv[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { const int i = i0 + 32 * k + lane; sv[k] = i < u1 ? SS[i] : 0; }
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int b = seed_bin(sv[k], P.s_th, bin_coef);
      if (b >= 0) atomicAdd(&cw[b >> 1], 1u << ((b & 1) * 16));
    }
  }
  __syncthreads();
  // 2. thread t <-> bin kBins-1-t: exclusive offsets over the warps, CTA totals, then the cluster-wide bases
  const int bin = kBins - 1 - tid;
  {
    int run = 0;
    for (int w = 0; w < kSeedWarps; w++) { unsigned short& c = cnt[w * kBins + bin]; const int v = c; c = (unsigned short)run; run += v; }
    tot[bin] = run;
  }
  cluster.sync();
  int pre = 0, all = 0;
#pragma unroll
  for (int q = 0; q < kSeedCta; q++) {
    const int v = cluster.map_shared_rank(tot, q)[bin];
    all += v;
    if (q < r) pre += v;
  }
  int incl = all;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  if (lane == 31) wsum[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    const int v = wsum[lane];
    int in2 = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, in2, o); if (lane >= o) in2 += u; }
    wsum[lane] = in2 - v;
    if (lane == 31) { s_nd = in2; if (r == 0) ndef[f] = in2; }
  }
  __syncthreads();
  base[bin] = wsum[wid] + incl - all + pre;
  __syncthreads();
  // 3. stable scatter of this warp's piece into the owners' shared memory
  unsigned short* wc = cnt + wid * kBins;
  const unsigned lt = (1u << lane) - 1u;
  int y = (u0 + lane) / P.sw, x = (u0 + lane) - y * P.sw;      // sw > 32: one wrap at most per 32 pixels
  for (int i0 = u0; i0 < u1; i0 += 128) {
    int sv[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { const int i = i0 + 32 * k + lane; sv[k] = i < u1 ? SS[i] : 0; }
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int b = seed_bin(sv[k], P.s_th, bin_coef);
      const unsigned peers = __match_any_sync(0xffffffffu, b);
      if (b >= 0) {
        const int pos = base[b] + wc[b] + __popc(peers & lt);
        const int q = pos / S;
        cluster.map_shared_rank(slice, q)[pos - q * S] = (unsigned)(x | (y << 16));
      }
      __syncwarp();
      if (b >= 0 && (peers & lt) == 0) wc[b] += (unsigned short)__popc(peers);
      __syncwarp();
      x += 32;
      if (x >= P.sw) { x -= P.sw; y++; }
    }
  }
  cluster.sync();
  // 4. flush [r*S, min((r+1)*S, ndef)) to HBM: scalar head up to 16-byte alignment, 16-byte body, scalar tail
  const int n = min(S, s_nd - r * S);
  if (n <= 0) return;
  unsigned* g = order + (long long)f * P.npx + (long long)r * S;
  const int head = min(n, (int)((4u - (unsigned)((reinterpret_cast<uintptr_t>(g) >> 2) & 3u)) & 3u));
  if (tid < head) g[tid] = slice[tid];
  const int nv = (n - head) >> 2;
  uint4* g4 = reinterpret_cast<uint4*>(g + head);
  if (head == 0) {
    const uint4* s4 = reinterpret_cast<const uint4*>(slice);
    for (int k = tid; k < nv; k += kSeedWarps * 32) g4[k] = s4[k];
  } else {
    for (int k = tid; k < nv; k += kSeedWarps * 32) {
      const unsigned* s = slice + head + 4 * k;
      g4[k] = make_uint4(s[0], s[1], s[2], s[3]);
    }
  }
  for (int k = head + 4 * nv + tid; k < n; k += kSeedWarps * 32) g[k] = slice[k];
}

// ---------------------------------------------------------------------------------------------- K_F region growing
// k_lsd_grow_ordered (lsd_grow_ordered.cuh, included below); here the table of gradient magnitudes it weights the
// rectangle moments with: W[s] = sqrt(s / 4), s = gx^2 + gy^2
__global__ void k_lsd_wtab(double* __restrict__ W, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) W[i] = sqrt((double)i / 4.0);
}

}  // namespace pl
#include "lsd_grow_ordered.cuh"
namespace pl {

// ---------------------------------------------------------------------------------------------- K_G keylines
__global__ void __launch_bounds__(256) k_keylines(LineParams P, const float4* __restrict__ segs, const int* __restrict__ nseg,
                                                  const uint8_t* __restrict__ mask, PLKeyLineRec* __restrict__ kls,
                                                  double* __restrict__ linefunc, int* __restrict__ nl) {
  extern __shared__ unsigned long long keys[];   // seg_cap rounded to a power of two
  __shared__ int s_cnt;
  const int f = blockIdx.x, tid = threadIdx.x;
  const float4* S = segs + (long long)f * P.seg_cap;
  const int n = nseg[f];
  int cap2 = 1;
  while (cap2 < max(n, 1)) cap2 <<= 1;
  auto clampseg = [&](float4 e) {
    if (e.x < 0) e.x = 0; if (e.x >= P.w) e.x = (float)P.w - 1.0f;
    if (e.z < 0) e.z = 0; if (e.z >= P.w) e.z = (float)P.w - 1.0f;
    if (e.y < 0) e.y = 0; if (e.y >= P.h) e.y = (float)P.h - 1.0f;
    if (e.w < 0) e.w = 0; if (e.w >= P.h) e.w = (float)P.h - 1.0f;
    return e;
  };
  auto seglen = [&](float4 e) {
    const double a = (double)__fsub_rn(e.x, e.z), b = (double)__fsub_rn(e.y, e.w);
    return (float)sqrt(a * a + b * b);
  };
  if (tid == 0) s_cnt = 0;
  __syncthreads();
  for (int i = tid; i < cap2; i += 256) {
    unsigned long long key = ~0ull;
    if (i < n) {
      const float4 e = clampseg(S[i]);
      bool drop = false;
      if (mask) drop = mask[(long long)(int)e.y * P.w + (int)e.x] == 0 && mask[(long long)(int)e.w * P.w + (int)e.z] == 0;
      if (!drop) {
        const float resp = __fdiv_rn(seglen(e), (float)max(P.w, P.h));
        key = ((unsigned long long)(~__float_as_uint(resp)) << 32) | (unsigned)i;   // response desc, detection order asc
        atomicAdd(&s_cnt, 1);
      }
    }
    keys[i] = key;
  }
  __syncthreads();
  for (int k = 2; k <= cap2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < cap2; i += 256) {
        int ixj = i ^ j;
        if (ixj > i) {
          unsigned long long a = keys[i], b = keys[ixj];
          bool up = ((i & k) == 0);
          if ((a > b) == up) { keys[i] = b; keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  const int size = s_cnt;
  // LineExtractor.cpp:44-67 truncation (total/index quirk)
  int total = size > P.nfeatures ? P.nfeatures : size, index = total;
  __shared__ int s_index;
  if (tid == 0) {
    if (total > 0) {
      const float lastLen = seglen(clampseg(S[(unsigned)(keys[total - 1] & 0xffffffffu)]));
      if ((double)lastLen < P.min_line_length) {
        for (int i = 0; i < total - 1; i++) {
          const float l0 = seglen(clampseg(S[(unsigned)(keys[i] & 0xffffffffu)]));
          const float l1 = seglen(clampseg(S[(unsigned)(keys[i + 1] & 0xffffffffu)]));
          if ((double)l0 >= P.min_line_length && (double)l1 < P.min_line_length) { index = i; break; }
        }
      }
    }
    s_index = index;
  }
  __syncthreads();
  index = s_index;
  const int nout = index + 1;
  PLKeyLineRec* K = kls + (long long)f * P.capL;
  double* LF = linefunc + (long long)f * P.capL * 3;
  for (int i = tid; i < nout && i < P.capL; i += 256) {
    PLKeyLineRec kl;
    if (i < size) {
      const float4 e = clampseg(S[(unsigned)(keys[i] & 0xffffffffu)]);
      kl.startPointX = e.x; kl.startPointY = e.y; kl.endPointX = e.z; kl.endPointY = e.w;
      kl.sPointInOctaveX = e.x; kl.sPointInOctaveY = e.y; kl.ePointInOctaveX = e.z; kl.ePointInOctaveY = e.w;
      kl.lineLength = seglen(e);
      const int x0 = __float2int_rn(e.x), y0 = __float2int_rn(e.y), x1 = __float2int_rn(e.z), y1 = __float2int_rn(e.w);
      kl.numOfPixels = max(abs(x1 - x0), abs(y1 - y0)) + 1;
      kl.angle = glibc::atan2f_(__fsub_rn(e.w, e.y), __fsub_rn(e.z, e.x));   // libm's atan2f, bit for bit (libm_glibc.cuh)
      kl.octave = 0;
      kl.size = __fmul_rn(__fsub_rn(e.z, e.x), __fsub_rn(e.w, e.y));
      kl.response = __fdiv_rn(kl.lineLength, (float)max(P.w, P.h));
      kl.ptx = __fdiv_rn(__fadd_rn(e.z, e.x), 2.f); kl.pty = __fdiv_rn(__fadd_rn(e.w, e.y), 2.f);
    } else {
      memset(&kl, 0, sizeof(kl));   // the KeyLine appended by resize(index+1)
    }
    kl.class_id = i;
    K[i] = kl;
    const double sx = kl.startPointX, sy = kl.startPointY, ex = kl.endPointX, ey = kl.endPointY;
    const double lx = sy * 1.0 - 1.0 * ey, ly = 1.0 * ex - sx * 1.0, lz = sx * ey - sy * ex;
    const double nn = sqrt(lx * lx + ly * ly);
    LF[3 * i] = lx / nn; LF[3 * i + 1] = ly / nn; LF[3 * i + 2] = lz / nn;
  }
  if (tid == 0) nl[f] = min(nout, P.capL);
}

// ---------------------------------------------------------------------------------------------- K_I LBD describe
__constant__ float c_gaussG[63];
__constant__ float c_gaussL[21];
__constant__ unsigned char c_comb[64];

__global__ void __launch_bounds__(64) k_lbd_describe(LineParams P, const PLKeyLineRec* __restrict__ kls, const int* __restrict__ nl,
                                                     const short2* __restrict__ dxyi, uint8_t* __restrict__ desc) {
  __shared__ float rs[63][8];
  __shared__ float band[8][9];
  __shared__ float des[72];
  const int li = blockIdx.x, f = blockIdx.y, tid = threadIdx.x;
  if (li >= nl[f]) return;
  const PLKeyLineRec kl = kls[(long long)f * P.capL + li];
  const short2* DXY = dxyi + (long long)f * P.w * P.h;
  const short realWidth = (short)P.w, imageWidth = (short)(P.w - 1), imageHeight = (short)(P.h - 1);
  const short lengthOfLSP = (short)kl.numOfPixels;
  const short halfHeight = (63 - 1) / 2, halfWidth = (short)((lengthOfLSP - 1) / 2);
  const float midX = (float)(0.5 * (double)__fadd_rn(kl.sPointInOctaveX, kl.ePointInOctaveX));
  const float midY = (float)(0.5 * (double)__fadd_rn(kl.sPointInOctaveY, kl.ePointInOctaveY));
  __shared__ float s_dL[2], s_gL[21], s_norm2[2];
  if (tid < 21) s_gL[tid] = c_gaussL[tid];
  if (tid == 0) glibc::sincosf_(kl.angle, &s_dL[1], &s_dL[0]);   // libm's sincosf, bit for bit (libm_glibc.cuh); once per line
  __syncthreads();
  const float dL0 = s_dL[0], dL1 = s_dL[1];
  const float dO0 = -dL1, dO1 = dL0;
  if (tid < 63) {
    const short hID = (short)tid;
    // sCorX0/Y0 after hID updates "sCorX0 -= dL[1]; sCorY0 += dL[0]" applied sequentially (fp32, same order)
    float sCorX0 = __fadd_rn(__fadd_rn(__fmul_rn(-dL0, (float)halfWidth), __fmul_rn(dL1, (float)halfHeight)), midX);
    float sCorY0 = __fadd_rn(__fsub_rn(__fmul_rn(-dL1, (float)halfWidth), __fmul_rn(dL0, (float)halfHeight)), midY);
    for (short k = 0; k < hID; k++) { sCorX0 = __fsub_rn(sCorX0, dL1); sCorY0 = __fadd_rn(sCorY0, dL0); }
    float sCorX = sCorX0, sCorY = sCorY0;
    float pgdL = 0, ngdL = 0, pgdO = 0, ngdO = 0;
    for (short wID = 0; wID < lengthOfLSP; wID++) {
      short t = (short)roundf(sCorX);
      const short xCor = (t < 0) ? 0 : (t > imageWidth) ? imageWidth : t;
      t = (short)roundf(sCorY);
      const short yCor = (t < 0) ? 0 : (t > imageHeight) ? imageHeight : t;
      const short2 g2 = __ldg(&DXY[(int)yCor * realWidth + xCor]);
      const short ddx = g2.x, ddy = g2.y;
      const float gDL = __fadd_rn(__fmul_rn((float)ddx, dL0), __fmul_rn((float)ddy, dL1));
      const float gDO = __fadd_rn(__fmul_rn((float)ddx, dO0), __fmul_rn((float)ddy, dO1));
      if (gDL > 0) pgdL = __fadd_rn(pgdL, gDL); else ngdL = __fsub_rn(ngdL, gDL);
      if (gDO > 0) pgdO = __fadd_rn(pgdO, gDO); else ngdO = __fsub_rn(ngdO, gDO);
      sCorX = __fadd_rn(sCorX, dL0); sCorY = __fadd_rn(sCorY, dL1);
    }
    const float c = c_gaussG[hID];
    pgdL = __fmul_rn(c, pgdL); ngdL = __fmul_rn(c, ngdL); pgdO = __fmul_rn(c, pgdO); ngdO = __fmul_rn(c, ngdO);
    rs[hID][0] = pgdL; rs[hID][1] = ngdL; rs[hID][2] = __fmul_rn(pgdL, pgdL); rs[hID][3] = __fmul_rn(ngdL, ngdL);
    rs[hID][4] = pgdO; rs[hID][5] = ngdO; rs[hID][6] = __fmul_rn(pgdO, pgdO); rs[hID][7] = __fmul_rn(ngdO, ngdO);
  }
  __syncthreads();
  // Band sums: band[q][k] is its own accumulator, fed in row order by the 7 rows of band k-1 (Gaussian taps 0..6), of band
  // k (taps 7..13) and of band k+1 (taps 14..20) — the order in which the reference's row loop touches it.  72 accumulators
  // in parallel, <= 21 ordered fp32 adds each.
  for (int a = tid; a < 72; a += 64) {
    const int q = a / 9, k = a - q * 9;
    const bool sq = (q == 2 || q == 3 || q == 6 || q == 7);
    float b = 0.f;
    for (int B = max(k - 1, 0); B <= min(k + 1, 8); B++) {
      const int off = (B - k + 1) * 7;
      for (int j = 0; j < 7; j++) {
        const float cg = s_gL[j + off], v = rs[B * 7 + j][q];
        b = __fadd_rn(b, sq ? __fmul_rn(__fmul_rn(cg, cg), v) : __fmul_rn(cg, v));
      }
    }
    band[q][k] = b;
  }
  __syncthreads();
  if (tid < 36) {       // mean / stddev of the four quantities of band bb
    const int bb = tid >> 2, c = tid & 3;
    const int qm = (c & 1) + ((c & 2) << 1), qs = qm + 2;          // {0,1,4,5} and {2,3,6,7}
    const float invN = (bb == 0 || bb == 8) ? (float)(1.0 / (7 * 2.0)) : (float)(1.0 / (7 * 3.0));
    const float temp = __fmul_rn(band[qm][bb], invN);
    des[8 * bb + c] = temp;
    des[8 * bb + 4 + c] = sqrtf(__fsub_rn(__fmul_rn(band[qs][bb], invN), __fmul_rn(temp, temp)));
  }
  __syncthreads();
  if (tid == 0 || tid == 32) {   // the two ordered norms (means: k = 0..3, stddevs: k = 4..7), one warp each
    const int k0 = tid ? 4 : 0;
    float acc = 0;
    for (int i = 0; i < 72; i += 8)
      for (int k = k0; k < k0 + 4; k++) acc = __fadd_rn(acc, __fmul_rn(des[i + k], des[i + k]));
    s_norm2[tid ? 1 : 0] = __fdiv_rn(1.f, sqrtf(acc));
  }
  __syncthreads();
  for (int i = tid; i < 72; i += 64) {
    float v = __fmul_rn(des[i], s_norm2[(i & 7) >> 2]);
    if ((double)v > 0.4) v = (float)0.4;
    des[i] = v;
  }
  __syncthreads();
  if (tid == 0) {
    float temp = 0;
    for (int i = 0; i < 72; i++) temp = __fadd_rn(temp, __fmul_rn(des[i], des[i]));
    s_norm2[0] = __fdiv_rn(1.f, sqrtf(temp));
  }
  __syncthreads();
  for (int i = tid; i < 72; i += 64) des[i] = __fmul_rn(des[i], s_norm2[0]);
  __syncthreads();
  if (tid < 32) {
    const float* f1 = &des[8 * c_comb[2 * tid]];
    const float* f2 = &des[8 * c_comb[2 * tid + 1]];
    unsigned r = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) if (f1[i] > f2[i]) r += (1u << i);
    desc[((long long)f * P.capL + li) * 32 + tid] = (uint8_t)r;
  }
}

}  // namespace pl

// ================================================================================================ host side
using namespace pl;

struct PLLine {
  PLLineConfig cfg;
  LineParams P;
  Stream stream;
  DevBuf<uint8_t> d_scaled;
  DevBuf<float2> d_seedcs;
  // region growing (lsd_grow_ordered.cuh): pixel records, squared gradients, region lists, far-pixel masks, weight table
  DevBuf<int4> d_rec; DevBuf<int> d_sq;
  DevBuf<unsigned> d_region, d_far; DevBuf<double> d_wtab;
  int region_stride = 0;                // words of d_region per frame
  DevBuf<GradRec> d_gtab; DevBuf<float2> d_gtab_seed;   // (gx, gy) -> level-line record, built once (k_lsd_grad_table)
  // k_lsd_seed_order: pixels per CTA (Q) and per warp (U), order positions per CTA (S), dynamic shared memory, clusters
  // resident on the device (0: the frame does not fit the cluster, k_lsd_hist/scan/scatter sort it)
  int seed_q = 0, seed_u = 0, seed_s = 0, seed_clusters = 0;
  int seed_min_batch = 132 * kSerialFramesPerSM;   // default: the cluster sort from this batch on
  int last_seed_cluster = 0;            // the LAST call sorted with k_lsd_seed_order
  size_t seed_smem = 0;
  DevBuf<unsigned short> d_counts;     // k_lsd_hist/scan/scatter
  DevBuf<int> d_offsets, d_ndef, d_maxs, d_nseg, d_overflow;
  DevBuf<unsigned> d_order;
  DevBuf<float4> d_segs;
  DevBuf<short2> d_dxy;
  // host-pointer API staging (made on first use)
  struct HostStaging { DevBuf<uint8_t> d_img, d_desc, d_mask; DevBuf<PLKeyLineRec> d_kls; DevBuf<double> d_lf; DevBuf<int> d_nl; };
  std::unique_ptr<HostStaging> io;
  const PLUndistort* und = nullptr;     // pl_line_set_undistort: the frames are raw, k_lsd_front undistorts them (owned by the caller)
  DevBuf<uint8_t> d_und;                // undistorted frames of batches below 32 frames per SM (made on first use)
  size_t key_smem = 0;
  int last_B = 0;
  // optional device timing of the dominant kernel (bench.py roofline): events on the launching stream
  int timing = 0;
  Event ev0, ev1;
};

static const unsigned char h_comb[64] = {0, 1, 0, 2, 0, 3, 0, 4, 0, 5, 0, 6, 1, 2, 1, 3, 1, 4, 1, 5, 1, 6, 2, 3, 2, 4, 2, 5, 2, 6, 2, 7,
                                         2, 8, 3, 4, 3, 5, 3, 6, 3, 7, 3, 8, 4, 5, 4, 6, 4, 7, 4, 8, 5, 6, 5, 7, 5, 8, 6, 7, 6, 8, 7, 8};

extern "C" void pl_line_destroy(PLLine* h) {
  if (!h) return;
  delete h;
}

extern "C" int pl_line_create(const PLLineConfig* cfg, PLLine** out) {
  PL_ARG(cfg && out);
  PL_ARG(cfg->width >= 64 && cfg->height >= 64 && cfg->width < 8000 && cfg->height < 8000 && cfg->nfeatures > 0 && cfg->max_batch >= 1);
  PL_ARG(cfg->segment_cap >= 0);
  int rc = require_device();
  if (rc) return rc;
  {  // k_keylines sorts a frame's segments in shared memory: 8 B per key, segment_cap rounded up to a power of two
    int dev = 0, optin = 0;
    cudaFuncAttributes fa;
    PL_CUDA(cudaGetDevice(&dev));
    PL_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    PL_CUDA(cudaFuncGetAttributes(&fa, k_keylines));
    const size_t room = optin > (int)fa.sharedSizeBytes ? (size_t)optin - fa.sharedSizeBytes : 0;
    size_t c2 = 1, fit = 1;
    while (c2 < (size_t)(cfg->segment_cap > 0 ? cfg->segment_cap : 8192)) c2 <<= 1;
    while (fit * 2 * 8 <= room) fit <<= 1;
    if (c2 * 8 > room) {
      set_error("segment_cap=%d: k_keylines sorts %zu keys of 8 B in shared memory, over the %zu B the device gives it per block; "
                "at most segment_cap=%zu fits", cfg->segment_cap, c2, room, fit);
      return PL_ERR_ARG;
    }
  }
  std::unique_ptr<PLLine> h(new PLLine);
  h->cfg = *cfg;
  LineParams& P = h->P;
  P.w = cfg->width; P.h = cfg->height;
  P.sw = (int)lrint(P.w * 0.8); P.sh = (int)lrint(P.h * 0.8);
  P.npx = P.sw * P.sh;
  P.nchunk = (P.sh - 1 + kChunkRows - 1) / kChunkRows;
  const double ANG_TH = 22.5, QUANT = 2.0;
  P.prec = kPI * ANG_TH / 180; P.p = ANG_TH / 180; P.density_th = 0.7;
  {  // smallest double n with (2pi - n) <= prec, the subtraction being exact in that range
    const double twopi = 2 * kPI;
    double c = twopi - P.prec;
    while ((twopi - nextafter(c, 0.0)) <= P.prec) c = nextafter(c, 0.0);
    while (!((twopi - c) <= P.prec)) c = nextafter(c, 10.0);
    P.prec_hi = c;
  }
  {
    const double M = 0.05 * M_PI / 180.0, ca = cos(P.prec - M), cn = cos(P.prec + M);
    P.sure_ca2 = (float)(ca * ca); P.sure_cn2 = (float)(cn * cn);
  }
  const double rho = QUANT / sin(P.prec);
  int s = 0;
  while (sqrt((double)(s + 1) / 4.0) <= rho) s++;   // largest s with sqrt(s/4) <= rho
  P.s_th = s;
  const double LOG_NT = 5 * (log10((double)P.sw) + log10((double)P.sh)) / 2 + log10(11.0);
  P.min_reg_size = (int)(size_t)(-LOG_NT / log10(P.p));
  P.seg_cap = cfg->segment_cap > 0 ? cfg->segment_cap : 8192;
  P.nfeatures = cfg->nfeatures; P.capL = cfg->nfeatures + 1; P.min_line_length = cfg->min_line_length;
  { size_t c2 = 1; while (c2 < (size_t)P.seg_cap) c2 <<= 1; h->key_smem = c2 * 8; }
  const size_t B = cfg->max_batch, npx = P.npx;
  PL_TRY(h->stream.create(cudaStreamNonBlocking));
  PL_TRY(h->d_scaled.alloc(npx * B)); PL_TRY(h->d_seedcs.alloc(npx * B)); PL_TRY(h->d_rec.alloc(npx * B));
  PL_TRY(h->d_sq.alloc(npx * B));
  {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    h->seed_min_batch = sms * kSerialFramesPerSM;
    // a region holds at most npx pixels; reduce_round's swap-remove scratch follows it (fill_off = npx)
    h->region_stride = 2 * P.npx;
    PL_TRY(h->d_region.alloc((size_t)h->region_stride * B)); PL_TRY(h->d_far.alloc(npx * B));
    const int nw = 2 * kGradR * kGradR + 1;
    PL_TRY(h->d_wtab.alloc((size_t)nw));
    k_lsd_wtab<<<(nw + 255) / 256, 256, 0, h->stream>>>(h->d_wtab, nw);
    PL_CUDA(cudaGetLastError());
    count_launch();
  }
  PL_TRY(h->d_counts.alloc((size_t)kBins * P.nchunk * B)); PL_TRY(h->d_offsets.alloc((size_t)kBins * P.nchunk * B));
  PL_TRY(h->d_ndef.alloc(B)); PL_TRY(h->d_maxs.alloc(B)); PL_TRY(h->d_nseg.alloc(B)); PL_TRY(h->d_overflow.alloc(1));
  PL_TRY(h->d_order.alloc(npx * B)); PL_TRY(h->d_segs.alloc((size_t)P.seg_cap * B));
  PL_TRY(h->d_dxy.alloc((size_t)P.w * P.h * B));
  PL_CUDA(cudaMemset(h->d_overflow, 0, sizeof(int)));
  PL_TRY(h->d_gtab.alloc((size_t)kGradN * kGradN)); PL_TRY(h->d_gtab_seed.alloc((size_t)kGradN * kGradN));
  k_lsd_grad_table<<<(kGradN * kGradN + 255) / 256, 256, 0, h->stream>>>(h->d_gtab, h->d_gtab_seed);
  PL_CUDA(cudaGetLastError());
  PL_CUDA(cudaStreamSynchronize(h->stream));
  count_launch();
  {  // LBD weights (binary_descriptor_custom.cpp:217-259), integer divisions as in the reference
    float gG[63], gL[21];
    double u = (7 * 3 - 1) / 2, sigma = (7 * 2 + 1) / 2, inv = -1 / (2 * sigma * sigma);
    for (int i = 0; i < 21; i++) { double d = i - u; gL[i] = (float)exp(d * d * inv); }
    u = (9 * 7 - 1) / 2; sigma = u; inv = -1 / (2 * sigma * sigma);
    for (int i = 0; i < 63; i++) { double d = i - u; gG[i] = (float)exp(d * d * inv); }
    PL_CUDA(cudaMemcpyToSymbol(c_gaussG, gG, sizeof(gG)));
    PL_CUDA(cudaMemcpyToSymbol(c_gaussL, gL, sizeof(gL)));
    PL_CUDA(cudaMemcpyToSymbol(c_comb, h_comb, sizeof(h_comb)));
  }
  PL_CUDA(cudaFuncSetAttribute(k_keylines, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->key_smem));
  {  // seed order on chip: 8 CTAs share the frame's rows 0..sh-2 and its (sw-1)(sh-1) possible order positions
    const int nrow = (P.sh - 1) * P.sw, maxdef = (P.sw - 1) * (P.sh - 1);
    h->seed_q = (nrow + kSeedCta - 1) / kSeedCta;
    h->seed_u = ((h->seed_q + kSeedWarps - 1) / kSeedWarps + 31) & ~31;
    h->seed_s = ((maxdef + kSeedCta - 1) / kSeedCta + 3) & ~3;
    h->seed_smem = (size_t)h->seed_s * sizeof(unsigned) + (size_t)kSeedWarps * kBins * sizeof(unsigned short) + 2 * kBins * sizeof(int);
    int dev = 0, smem_max = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    // 16-bit per-warp counters hold within-CTA offsets: at most 65535 pixels per CTA
    if (h->seed_q <= 65535 && h->seed_smem + 2 * 1024 <= (size_t)smem_max) {
      PL_CUDA(cudaFuncSetAttribute(k_lsd_seed_order, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->seed_smem));
      cudaLaunchConfig_t lc = {};
      lc.gridDim = dim3(kSeedCta, 1, 1); lc.blockDim = dim3(kSeedWarps * 32, 1, 1); lc.dynamicSmemBytes = h->seed_smem;
      PL_CUDA(cudaOccupancyMaxActiveClusters(&h->seed_clusters, (void*)k_lsd_seed_order, &lc));
    }
  }
  // cfg->lsd_used_in_global is accepted for ABI compatibility and ignored: the USED state is the ownership word of the pixel record
  *out = h.release();
  return PL_OK;
}

extern "C" int pl_line_capacity(const PLLine* h) { return h ? h->P.capL : PL_ERR_ARG; }

extern "C" int pl_line_set_undistort(PLLine* h, const PLUndistort* und) {
  PL_ARG(h);
  if (und && (und->w != h->P.w || und->h != h->P.h)) {
    set_error("pl_line_set_undistort: a %dx%d map for %dx%d frames", und->w, und->h, h->P.w, h->P.h);
    return PL_ERR_ARG;
  }
  h->und = und;
  return PL_OK;
}

// Device timing of k_lsd_grow_ordered (the dominant kernel): enable, run, then read the duration of the LAST launch.
extern "C" int pl_line_set_timing(PLLine* h, int on) {
  PL_ARG(h);
  if (on) for (Event* e : {&h->ev0, &h->ev1}) if (!*e) PL_TRY(e->create(cudaEventDefault));
  h->timing = on;
  return PL_OK;
}
extern "C" int pl_line_grow_ms(PLLine* h, float* ms) {
  PL_ARG(h && ms && h->ev1);
  PL_CUDA(cudaEventSynchronize(h->ev1));
  PL_CUDA(cudaEventElapsedTime(ms, h->ev0, h->ev1));
  return PL_OK;
}
/* algorithmic bytes k_lsd_grow_ordered must move for one frame (DESIGN.md §6): per scaled pixel: record (16) + seed cos/sin (8)
 * + seed order entry (4); the USED map lives in shared memory */
extern "C" long long pl_line_grow_bytes_per_frame(const PLLine* h) { return h ? (long long)h->P.npx * 28 : 0; }

extern "C" int pl_line_extract_batch_dev(PLLine* h, const uint8_t* imgs, int stride, size_t frame_stride, int B,
                                         const uint8_t* mask, void* keylines, uint8_t* desc, double* linefunc, int* n,
                                         void* stream_) {
  PL_ARG(h && imgs && keylines && desc && linefunc && n && B >= 1 && B <= h->cfg.max_batch && stride >= h->cfg.width);
  // The cluster sort by default from kSerialFramesPerSM frames per SM on, where the three-kernel scatter is slow and the
  // front-end runs its chains on one stream (frontend.cu, serial_batch).  Below that, kernels of the other chains hold SMs
  // beside it and an 8-SM cluster with up to 217 KB of shared memory per CTA waits for whole SMs to drain (KITTI
  // configuration: 21 % slower, DESIGN.md §7).  PLSLAM_LSD_SEED_ORDER=legacy | cluster forces one of the two; a forced
  // cluster sort the frame shape or the device cannot run is an error.
  const char* so = getenv("PLSLAM_LSD_SEED_ORDER");
  const bool force_cluster = so && strcmp(so, "cluster") == 0, force_legacy = so && strcmp(so, "legacy") == 0;
  if (force_cluster && h->seed_clusters == 0) {
    set_error("PLSLAM_LSD_SEED_ORDER=cluster: a %dx%d scaled frame does not fit k_lsd_seed_order (%zu B of shared memory, %d pixels per CTA)",
              h->P.sw, h->P.sh, h->seed_smem, h->seed_q);
    return PL_ERR_ARG;
  }
  const bool cluster = h->seed_clusters > 0 && !force_legacy && (force_cluster || B >= h->seed_min_batch);
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : h->stream;
  const LineParams& P = h->P;
  h->last_B = B;
  h->last_seed_cluster = cluster;
  PL_CUDA(cudaMemsetAsync(h->d_maxs, 0, sizeof(int) * B, st));
  {  // scaled image, pixel records, gx^2+gy^2, seed cos/sin, per-frame max and the LBD Sobel pair in one pass
    // Below 32 frames per SM the front-end runs its chains on three streams (frontend.cu), and there the fused pass is placed
    // beside the ORB chain's kernels.  Measured there (DESIGN.md §7), the grow that follows on the same SMs ran 10-20 % slower
    // in two cases.  Case 1: the camera map read inside this pass (EuRoC configuration); so such batches undistort the frames
    // first with k_remap, as before.  Case 2: this kernel's default shared-memory carve-out (KITTI configuration), which an SM
    // keeps while other kernels stay resident; so such batches ask for the smallest carve-out, and the grow keeps its L1.
    const bool serial = B >= h->seed_min_batch;
    int rc = PL_OK;
    const uint8_t* src = imgs; int sstride = stride; long long sframe = (long long)frame_stride;
    if (h->und && !serial) {
      const size_t fb = (size_t)P.w * P.h;
      if (!h->d_und && (rc = h->d_und.alloc(fb * h->cfg.max_batch))) return rc;
      // the remap only reads the map: the handle stays the caller's
      if ((rc = pl_undistort_remap_batch_dev(const_cast<PLUndistort*>(h->und), imgs, stride, frame_stride, B, h->d_und, P.w, fb, st))) return rc;
      src = h->d_und; sstride = P.w; sframe = (long long)fb;
    }
    const bool map = h->und && serial;
    const dim3 grd(std::max((P.sw + kFrontSX - 1) / kFrontSX, (P.w + kFrontUX - 1) / kFrontUX),
                   std::max((P.sh + kFrontSY - 1) / kFrontSY, (P.h + kFrontUY - 1) / kFrontUY), (B + kFrontFrames - 1) / kFrontFrames);
    const float4* T = reinterpret_cast<const float4*>(h->d_gtab.get());
    const RemapEntry* mp = map ? h->und->d_map.get() : nullptr;
    const int4* tab = map ? h->und->d_tab.get() : nullptr;
    cudaLaunchConfig_t lc = {};
    lc.gridDim = grd; lc.blockDim = dim3(kFrontThreads); lc.dynamicSmemBytes = map ? kFrontMapSmem : 0; lc.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributePreferredSharedMemoryCarveout; at[0].val.sharedMemCarveout = 0;
    if (!serial) { lc.attrs = at; lc.numAttrs = 1; }
    PL_CUDA(cudaLaunchKernelEx(&lc, map ? k_lsd_front<true> : k_lsd_front<false>, P, src, sstride, sframe, B, mp, tab, T,
                               (const float2*)h->d_gtab_seed, h->d_scaled, h->d_rec, h->d_sq, h->d_seedcs, h->d_maxs, h->d_dxy));
  }
  PL_LAUNCH_CHECK();
  if (cluster) {
    k_lsd_seed_order<<<dim3(kSeedCta, B), kSeedWarps * 32, h->seed_smem, st>>>(P, h->seed_q, h->seed_u, h->seed_s, h->d_sq, h->d_maxs,
                                                                             h->d_order, h->d_ndef);
    PL_LAUNCH_CHECK();
  } else {
    k_lsd_hist<<<dim3(P.nchunk, B), 256, 0, st>>>(P, h->d_sq, h->d_maxs, h->d_counts);
    PL_LAUNCH_CHECK();
    k_lsd_scan<<<B, kBins, 0, st>>>(P, h->d_counts, h->d_offsets, h->d_ndef);
    PL_LAUNCH_CHECK();
    k_lsd_scatter<<<dim3((P.nchunk + 3) / 4, B), 128, 0, st>>>(P, h->d_sq, h->d_maxs, h->d_offsets, h->d_order);
    PL_LAUNCH_CHECK();
  }
  // one warp per frame, the 32 lanes on one region at a time (lsd_grow_ordered.cuh).  Batches up to kPreMaxBatch frames do
  // not fill the GPU with frames: there the kernel examines the neighbourhoods of 32 seeds at a time up front (kPre)
  constexpr int kPreMaxBatch = 256;
  const auto grow = B <= kPreMaxBatch ? k_lsd_grow_ordered<true> : k_lsd_grow_ordered<false>;
  if (h->timing) PL_CUDA(cudaEventRecord(h->ev0, st));
  // the kernel addresses the per-frame arrays with 32-bit element indices (frame * npx + pixel): at most 2^32 / npx frames per grid
  const int chunk = (int)std::min<long long>(B, 0xffffffffLL / P.npx);
  for (int b0 = 0; b0 < B; b0 += chunk) {
    const int nb = std::min(chunk, B - b0);
    const size_t po = (size_t)b0 * P.npx;
    grow<<<nb, 32, 0, st>>>(P, h->d_rec + po, h->d_sq + po, h->d_seedcs + po, h->d_order + po, h->d_ndef + b0,
                            h->d_region + (size_t)b0 * h->region_stride, h->region_stride, h->d_far + po, h->d_wtab,
                            h->d_segs + (size_t)b0 * P.seg_cap, h->d_nseg + b0, h->d_overflow, nb);
  }
  PL_LAUNCH_CHECK();
  if (h->timing) PL_CUDA(cudaEventRecord(h->ev1, st));
  k_keylines<<<B, 256, h->key_smem, st>>>(P, h->d_segs, h->d_nseg, mask, (PLKeyLineRec*)keylines, linefunc, n);
  PL_LAUNCH_CHECK();
  k_lbd_describe<<<dim3(P.capL, B), 64, 0, st>>>(P, (const PLKeyLineRec*)keylines, n, h->d_dxy, desc);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

// capacity flag of the calls since the last check (segment_cap exceeded);
// the *_dev entry points are asynchronous and never look at them: their callers do, after synchronising
extern "C" int pl_line_check_overflow(PLLine* h) {
  PL_ARG(h);
  int ov = 0;
  PL_CUDA(cudaMemcpy(&ov, h->d_overflow, sizeof(int), cudaMemcpyDeviceToHost));
  if (ov) {
    cudaMemset(h->d_overflow, 0, sizeof(int));
    set_error("LSD produced more than segment_cap=%d segments", h->P.seg_cap);
    return PL_ERR_CAPACITY;
  }
  return PL_OK;
}

extern "C" int pl_line_extract_batch(PLLine* h, const uint8_t* imgs, int stride, size_t frame_stride, int B,
                                     const uint8_t* mask, void* keylines, uint8_t* desc, double* linefunc, int* n) {
  PL_ARG(h && imgs && keylines && desc && linefunc && n && B >= 1 && B <= h->cfg.max_batch && stride >= h->cfg.width);
  if (!h->io) {
    const size_t Bm = h->cfg.max_batch, npx = (size_t)h->P.w * h->P.h, cap = h->P.capL;
    auto io = std::make_unique<PLLine::HostStaging>();
    PL_TRY(io->d_img.alloc(npx * Bm)); PL_TRY(io->d_kls.alloc(cap * Bm)); PL_TRY(io->d_desc.alloc(cap * 32 * Bm));
    PL_TRY(io->d_lf.alloc(cap * 3 * Bm)); PL_TRY(io->d_nl.alloc(Bm)); PL_TRY(io->d_mask.alloc(npx));
    h->io = std::move(io);
  }
  const PLLine::HostStaging& io = *h->io;
  const int W = h->P.w, H = h->P.h;
  for (int b = 0; b < B; b++)
    PL_CUDA(cudaMemcpy2DAsync(io.d_img + (size_t)b * W * H, W, imgs + (size_t)b * frame_stride, stride, W, H, cudaMemcpyHostToDevice, h->stream));
  if (mask) PL_CUDA(cudaMemcpyAsync(io.d_mask, mask, (size_t)W * H, cudaMemcpyHostToDevice, h->stream));
  int rc = pl_line_extract_batch_dev(h, io.d_img, W, (size_t)W * H, B, mask ? io.d_mask.get() : nullptr, io.d_kls, io.d_desc, io.d_lf, io.d_nl, h->stream);
  if (rc) return rc;
  const size_t cap = h->P.capL;
  PL_CUDA(cudaMemcpyAsync(keylines, io.d_kls, cap * B * sizeof(PLKeyLineRec), cudaMemcpyDeviceToHost, h->stream));
  PL_CUDA(cudaMemcpyAsync(desc, io.d_desc, cap * B * 32, cudaMemcpyDeviceToHost, h->stream));
  PL_CUDA(cudaMemcpyAsync(linefunc, io.d_lf, cap * B * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  PL_CUDA(cudaMemcpyAsync(n, io.d_nl, (size_t)B * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  PL_CUDA(cudaStreamSynchronize(h->stream));
  return pl_line_check_overflow(h);
}

extern "C" int pl_line_extract(PLLine* h, const uint8_t* img, int stride, const uint8_t* mask, void* keylines,
                               uint8_t* desc, double* linefunc, int* n) {
  return pl_line_extract_batch(h, img, stride, 0, 1, mask, keylines, desc, linefunc, n);
}

// parity taps of the LAST call
extern "C" int pl_line_debug_segments(PLLine* h, int frame, float* out, int cap) {
  PL_ARG(h && frame >= 0 && frame < h->last_B);
  int n = 0;
  PL_CUDA(cudaStreamSynchronize(h->stream));
  PL_CUDA(cudaMemcpy(&n, h->d_nseg + frame, sizeof(int), cudaMemcpyDeviceToHost));
  if (out && n) PL_CUDA(cudaMemcpy(out, h->d_segs + (size_t)frame * h->P.seg_cap, sizeof(float4) * std::min(n, cap), cudaMemcpyDeviceToHost));
  return n;
}
extern "C" int pl_line_debug_scaled(PLLine* h, int frame, uint8_t* out, int* sw, int* sh) {
  PL_ARG(h && frame >= 0 && frame < h->last_B && sw && sh);
  *sw = h->P.sw; *sh = h->P.sh;
  PL_CUDA(cudaStreamSynchronize(h->stream));
  if (out) PL_CUDA(cudaMemcpy(out, h->d_scaled + (size_t)frame * h->P.npx, h->P.npx, cudaMemcpyDeviceToHost));
  return PL_OK;
}
extern "C" int pl_line_debug_sobel(PLLine* h, int frame, short* dx, short* dy) {
  PL_ARG(h && frame >= 0 && frame < h->last_B && dx && dy);
  const size_t n = (size_t)h->P.w * h->P.h;
  PL_CUDA(cudaStreamSynchronize(h->stream));
  std::vector<short2> tmp(n);
  PL_CUDA(cudaMemcpy(tmp.data(), h->d_dxy + frame * n, n * sizeof(short2), cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < n; i++) { dx[i] = tmp[i].x; dy[i] = tmp[i].y; }
  return PL_OK;
}
// which sort built the seed order of the LAST call: 1 k_lsd_seed_order, 0 k_lsd_hist/scan/scatter
extern "C" int pl_line_debug_seed_path(PLLine* h) {
  PL_ARG(h);
  return h->last_seed_cluster;
}
// fill every byte of the seed order and of ndef with `byte` (a test writes 0xff before a call: every position the call does
// not write then reads back as an invalid entry, and an unwritten ndef as -1)
extern "C" int pl_line_debug_fill_order(PLLine* h, int byte) {
  PL_ARG(h);
  PL_CUDA(cudaStreamSynchronize(h->stream));
  PL_CUDA(cudaMemset(h->d_order, byte, sizeof(unsigned) * (size_t)h->P.npx * h->cfg.max_batch));
  PL_CUDA(cudaMemset(h->d_ndef, byte, sizeof(int) * (size_t)h->cfg.max_batch));
  PL_CUDA(cudaDeviceSynchronize());
  return PL_OK;
}
extern "C" int pl_line_debug_order(PLLine* h, int frame, unsigned* out, int cap) {
  PL_ARG(h && frame >= 0 && frame < h->last_B);
  int n = 0;
  PL_CUDA(cudaStreamSynchronize(h->stream));
  PL_CUDA(cudaMemcpy(&n, h->d_ndef + frame, sizeof(int), cudaMemcpyDeviceToHost));
  if (n < 0) { set_error("seed order of frame %d: ndef = %d was not written by the last call", frame, n); return PL_ERR_ARG; }
  if (out && n) {
    PL_CUDA(cudaMemcpy(out, h->d_order + (size_t)frame * h->P.npx, sizeof(unsigned) * std::min(n, cap), cudaMemcpyDeviceToHost));
    for (int i = 0; i < std::min(n, cap); i++) out[i] = (out[i] >> 16) * (unsigned)h->P.sw + (out[i] & 0xffffu);   // packed (x,y) -> y*sw+x
  }
  return n;
}

#ifdef PL_GROW_STATS
extern "C" int pl_line_grow_stats(unsigned long long* out, int reset) {
  cudaDeviceSynchronize();
  if (out) cudaMemcpyFromSymbol(out, pl::ord::g_grow_stats, sizeof(unsigned long long) * 24);
  if (reset) { unsigned long long z[24] = {0}; cudaMemcpyToSymbol(pl::ord::g_grow_stats, z, sizeof(z)); }
  return 0;
}
#endif
