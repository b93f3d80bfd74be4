// Line-feature extraction (LSD segments + LBD descriptors) for batches of frames on sm_90a.
//
// Replaces LINEextractor::operator() (reference src/LineExtractor.cpp:26-93) and what it calls:
//   LSDDetector::detect           opencv_contrib line_descriptor; spec copy Thirdparty/line_descriptor/src/LSDDetector_custom.cpp:56-215
//   cv::LineSegmentDetector       OpenCV imgproc lsd.cpp (defaults: REFINE_STD, scale .8, sigma_scale .6, quant 2, 22.5 deg, density .7)
//   BinaryDescriptor::compute     spec copy Thirdparty/line_descriptor/src/binary_descriptor_custom.cpp:350-398,539-687,1026-1372
//
// Kernel map (DESIGN.md §6)
//   k_lsd_scale     7x7 sigma .75 Gaussian (8.8 fixed point) fused with the 0.8x INTER_LINEAR_EXACT resize, smem tiles
//   k_lsd_grad      2x2 gradient -> one 16-byte record per pixel (angle, cos, sin, squared magnitude), per-frame max
//   k_lsd_hist/scan/scatter   stable counting sort of the defined pixels into 1024 magnitude bins (descending),
//                   equal bins keep row-major order == OpenCV 4.13's seed order (pinned in the oracle tests)
//   k_lsd_grow      region growing + rectangle fit + density refinement; inherently ordered (a pixel consumed by an
//                   earlier seed is unavailable to later ones) -> ONE warp per frame walks the seeds in order; the 32
//                   lanes test the 3x3 neighbourhood, evaluate angles and reduce the rectangle moments in parallel.
//   k_keylines      KeyLine records, mask filter, response sort (bitonic, ties keep detection order), truncation
//                   quirk of LineExtractor.cpp:44-67, normalised 2-D line equations
//   k_lbd_sobel     5x5 sigma 1 Gaussian (8.8 fixed point) fused with the 3x3 Sobel pair -> int16 dx, dy
//   k_lbd_describe  one CTA per line: 63 support rows in parallel (each row accumulates along the line in the
//                   reference's order, fp32 without FMA), band statistics, 72-float LBD, 32-byte binarisation

#include "common.cuh"
#include "lsd_grow_core.cuh"
#include "libm_glibc.cuh"
#include <math.h>
#include <string.h>
#include <stdlib.h>
#include <vector>
#include <algorithm>

namespace pl {

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
  double prec, prec_hi, p, density_th;   // prec_hi: see region_grow_t
  float sure_ca2, sure_cn2;              // cos^2(prec -/+ 0.05 deg): lsd_grow_ordered.cuh Sure
};

// ---------------------------------------------------------------------------------------------- shared helpers
__device__ __forceinline__ float fast_atan2_deg_l(float y, float x) {  // cv::fastAtan2, no FMA
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
__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_min_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---------------------------------------------------------------------------------------------- K_A scale
// Output tile 32x32 of the 0.8x image <- 40x40 blurred pixels <- 44x44 raw pixels (taps at +-3 are zero).
__global__ void __launch_bounds__(256) k_lsd_scale(LineParams P, const uint8_t* __restrict__ imgs, int stride,
                                                   long long frame_stride, uint8_t* __restrict__ scaled) {
  __shared__ uint8_t raw[44][48];
  __shared__ uint16_t hp[44][40];
  __shared__ uint8_t bl[40][40];
  const int tid = threadIdx.x;
  const int X0 = blockIdx.x * 32, Y0 = blockIdx.y * 32;
  const int bx0 = (5 * X0) >> 2, by0 = (5 * Y0) >> 2;
  const uint8_t* img = imgs + (long long)blockIdx.z * frame_stride;
  for (int i = tid; i < 44 * 44; i += 256) {
    int r = i / 44, c = i - r * 44;
    int gy = reflect101(min(by0 - 2 + r, 2 * P.h - 2), P.h), gx = reflect101(min(bx0 - 2 + c, 2 * P.w - 2), P.w);
    raw[r][c] = img[(long long)gy * stride + gx];
  }
  __syncthreads();
  for (int i = tid; i < 44 * 40; i += 256) {
    int r = i / 40, c = i - r * 40;
    const uint8_t* p = &raw[r][c];
    hp[r][c] = (uint16_t)(4 * (p[0] + p[4]) + 56 * (p[1] + p[3]) + 136 * p[2]);
  }
  __syncthreads();
  for (int i = tid; i < 40 * 40; i += 256) {
    int r = i / 40, c = i - r * 40;
    uint32_t s = 4u * (hp[r][c] + hp[r + 4][c]) + 56u * (hp[r + 1][c] + hp[r + 3][c]) + 136u * hp[r + 2][c];
    bl[r][c] = (uint8_t)((s + 32768u) >> 16);
  }
  __syncthreads();
  uint8_t* out = scaled + (long long)blockIdx.z * P.npx;
  for (int i = tid; i < 32 * 32; i += 256) {
    int ty = i >> 5, tx = i & 31;
    int x = X0 + tx, y = Y0 + ty;
    if (x >= P.sw || y >= P.sh) continue;
    int sx = (10 * x + 1) >> 3, xf = ((10 * x + 1) & 7) * 32;
    int sy = (10 * y + 1) >> 3, yf = ((10 * y + 1) & 7) * 32;
    if (sx >= P.w - 1) { sx = P.w - 1; xf = 0; }
    if (sy >= P.h - 1) { sy = P.h - 1; yf = 0; }
    int sx1 = min(sx + 1, P.w - 1), sy1 = min(sy + 1, P.h - 1);
    int lx = sx - bx0, lx1 = sx1 - bx0, ly = sy - by0, ly1 = sy1 - by0;
    int h0 = bl[ly][lx] * (256 - xf) + bl[ly][lx1] * xf;
    int h1 = bl[ly1][lx] * (256 - xf) + bl[ly1][lx1] * xf;
    out[(long long)y * P.sw + x] = (uint8_t)((h0 * (256 - yf) + h1 * yf + 32768) >> 16);
  }
}

// ---------------------------------------------------------------------------------------------- K_B gradient
// Per scaled pixel, what region growing needs:
//   REC = 16-byte record {own, angle, cos, sin}: own = ownership word of the speculative growing (lsd_grow_core.cuh; free or
//         NOTDEF here), angle = level-line angle in degrees (cv::fastAtan2(gx, -gy)), cos/sin of float(angle_rad) rounded
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
  const float deg = fast_atan2_deg_l((float)gx, (float)(-gy));
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
// One thread = 4 consecutive pixels of a row: two 8-byte row reads, four table lookups, 16-byte stores (the pass is bound by
// the number of memory instructions, not by bytes).  kVec needs sw % 4 == 0 (rows of every output array 16-byte aligned).
template <bool kVec>
__global__ void __launch_bounds__(256) k_lsd_grad(LineParams P, const uint8_t* __restrict__ scaled, const float4* __restrict__ T,
                                                  const float2* __restrict__ TS,
                                                  int4* __restrict__ REC, int* __restrict__ S2, float2* __restrict__ seedcs, int* __restrict__ maxs) {
  __shared__ int smax;
  if (threadIdx.x == 0) smax = 0;
  __syncthreads();
  const int x0 = (blockIdx.x * 64 + (threadIdx.x & 63)) * 4, y = blockIdx.y * 4 + (threadIdx.x >> 6);
  const int f = blockIdx.z;
  int smx = 0;
  if (x0 < P.sw && y < P.sh) {
    const uint8_t* S = scaled + (long long)f * P.npx + (long long)y * P.sw + x0;
    const bool lastrow = (y >= P.sh - 1);
    int r0[5], r1[5];
    if (kVec) {       // x0 % 4 == 0 and sw % 4 == 0: one aligned word + one byte per row
      const unsigned w0 = *reinterpret_cast<const unsigned*>(S), w1 = lastrow ? 0u : *reinterpret_cast<const unsigned*>(S + P.sw);
#pragma unroll
      for (int k = 0; k < 4; k++) { r0[k] = (w0 >> (8 * k)) & 0xff; r1[k] = (w1 >> (8 * k)) & 0xff; }
      const bool in4 = (x0 + 4 < P.sw);
      r0[4] = in4 ? S[4] : 0; r1[4] = (in4 && !lastrow) ? S[P.sw + 4] : 0;
    } else {
#pragma unroll
      for (int k = 0; k < 5; k++) {
        const bool in = (x0 + k < P.sw);
        r0[k] = in ? S[k] : 0;
        r1[k] = (in && !lastrow) ? S[P.sw + k] : 0;
      }
    }
    int4 rec[4];
    float se[4][2];
    int sq[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      rec[k] = make_int4(lg::kNotDef, __float_as_int(kNotDefDeg), 0, 0); se[k][0] = se[k][1] = 0.f; sq[k] = 0;
      if (x0 + k < P.sw - 1 && !lastrow) {
        const int DA = r1[k + 1] - r0[k], BC = r0[k + 1] - r1[k];
        const int gx = DA + BC, gy = DA - BC;
        const int s = gx * gx + gy * gy;
        sq[k] = s;
        if (s > P.s_th) {
          const int ti = (gx + kGradR) * kGradN + (gy + kGradR);
          const float4 t = __ldg(&T[ti]);
          const float2 scs = __ldg(&TS[ti]);
          rec[k] = make_int4(lg::kFree, __float_as_int(t.x), __float_as_int(t.y), __float_as_int(t.z));
          se[k][0] = scs.x; se[k][1] = scs.y;
          smx = max(smx, s);
        }
      }
    }
    const long long o = (long long)f * P.npx + (long long)y * P.sw + x0;
    if (kVec) {
#pragma unroll
      for (int k = 0; k < 4; k++) REC[o + k] = rec[k];
      *reinterpret_cast<int4*>(S2 + o) = make_int4(sq[0], sq[1], sq[2], sq[3]);
      float4* e4 = reinterpret_cast<float4*>(seedcs + o);
      e4[0] = make_float4(se[0][0], se[0][1], se[1][0], se[1][1]); e4[1] = make_float4(se[2][0], se[2][1], se[3][0], se[3][1]);
    } else {
      for (int k = 0; k < 4 && x0 + k < P.sw; k++) { REC[o + k] = rec[k]; S2[o + k] = sq[k]; seedcs[o + k] = make_float2(se[k][0], se[k][1]); }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) smx = max(smx, __shfl_xor_sync(0xffffffffu, smx, o));
  if ((threadIdx.x & 31) == 0 && smx > 0) atomicMax(&smax, smx);
  __syncthreads();
  if (threadIdx.x == 0 && smax > 0) atomicMax(&maxs[f], smax);
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

// ---------------------------------------------------------------------------------------------- K_F region growing
// Ordered speculative execution (lsd_grow_core.cuh has the protocol and everything a lane does).  Here: the warp loop.
//   frame f is served by `wpf` consecutive warps (one warp per CTA); every LANE runs one region task at a time, so a
//   warp is 32 regions in flight and the instruction stream is shared by 32 independent serial chains
//   per iteration (converged):   commit   the warp that holds the frame's commit lock validates the next 32 status
//                                         words in order (two passes around a fence), appends the segments of the
//                                         newly final tasks in order, advances the frontier, and hands an invalid
//                                         head task out for re-execution
//                                feed     idle lanes: take the re-execution, else scan the next 32 seeds of the
//                                         order (coalesced), retire the consumed ones, queue the rest for the lanes
//                                step     every busy lane advances its task by one micro-step (lane_step)
// Why it is fast where the previous one-warp-per-region kernel was not: a region is a serial chain (one angle update
// per added pixel), so 32 lanes on ONE region idle; 32 regions on one warp keep all lanes on useful work, and the
// number of regions in flight (32 x warps) no longer depends on the batch: B = 1 fills the GPU as well as a full batch.
constexpr int kGrowQ = 256;
constexpr int kCommitBatches = 4;
constexpr unsigned kGrowWatchdog = 6u * 1000u * 1000u;
__device__ __forceinline__ int first_zero(unsigned m) { return m == 0xffffffffu ? 32 : __ffs(~m) - 1; }

__device__ __forceinline__ void warp_commit(const lg::Params& GP, const lg::Frame& Fm, float4* __restrict__ segs, int lane) {
  using namespace lg;
  const unsigned lt = (1u << lane) - 1u;
  for (int round = 0; round < kCommitBatches; round++) {
    const int F = ld_i(&Fm.ctl[C_FIN]);
    if (F >= Fm.n) return;
    const int i = F + lane;
    const unsigned w1 = (i < Fm.n) ? ld_u(&Fm.st[i]) : 0u;
    const unsigned s1 = w1 & ST_STATE;
    const int pre1 = first_zero(__ballot_sync(0xffffffffu, s1 == ST_NOOP || s1 == ST_EATEN || s1 == ST_DONE));
    if (pre1 == 0) return;
    __threadfence();            // every claim / steal of the tasks seen DONE is visible to the second pass
    unsigned w2 = 0u;
    bool ok = false;
    if (lane < pre1) { w2 = ld_u(&Fm.st[i]); ok = task_valid(GP, Fm, i, w2); }
    const int pre2 = min(pre1, first_zero(__ballot_sync(0xffffffffu, ok)));
    float4 sg;
    const bool has = (lane < pre2) && task_has_segment(Fm, w2, sg);
    const unsigned ms = __ballot_sync(0xffffffffu, has);
    const int ns = ld_i(&Fm.ctl[C_NS]);
    if (has) { const int slot = ns + __popc(ms & lt); if (slot < GP.seg_cap) segs[slot] = sg; }
    __syncwarp();
    if (lane == 0) {
      st_i(&Fm.ctl[C_NS], ns + __popc(ms));
      __threadfence();
      a_max(&Fm.ctl[C_FIN], F + pre2);
    }
    if (pre2 < pre1) {          // the head is finished but not valid: it is executed again, now with nothing earlier in flight
      // (an idle lane may be taking the same task off the redo ring right now: the compare-and-swap decides)
      // only a task that is still finished (DONE / EATEN) in the second pass: between the passes an idle lane may have taken
      // it off the redo ring and be running it already
      const unsigned s2 = w2 & ST_STATE;
      if (lane == pre2 && (s2 == ST_DONE || s2 == ST_EATEN) &&
          (unsigned)a_cas(reinterpret_cast<int*>(&Fm.st[i]), (int)w2, (int)((w2 & ~(ST_STATE | ST_ABORT)) | ST_REDO)) == w2) {
        __threadfence();
        st_i(&Fm.ctl[C_REDO], i);
      }
      __syncwarp();
      return;
    }
    __syncwarp();
    if (pre2 < 32) return;
  }
}

template <int kWPC>
__global__ void __launch_bounds__(32 * kWPC) k_lsd_grow(LineParams P, lg::Params GP, int4* __restrict__ REC, const float2* __restrict__ seedcs,
                                                        const int* __restrict__ SQ, const unsigned* __restrict__ order, const int* __restrict__ ndef,
                                                        unsigned* __restrict__ ST, unsigned* __restrict__ POOL, int* __restrict__ CTL,
                                                        unsigned* __restrict__ LANEBUF, const double* __restrict__ wtab,
                                                        float4* __restrict__ segs, int* __restrict__ nseg, int* __restrict__ overflow,
                                                        int nframes, int wpf) {
  using namespace lg;
  __shared__ int wq_all[kWPC][kGrowQ];
  __shared__ unsigned ring_all[kWPC][32 * lg::kRing];
  const int lane = threadIdx.x & 31, wic = threadIdx.x >> 5;
  const long long gw = (long long)blockIdx.x * kWPC + wic;
  const int f = (int)(gw / wpf), wif = (int)(gw % wpf);      // frame, warp inside the frame's group
  if (f >= nframes) return;
  int* wq = wq_all[wic];
  Frame Fm;
  Fm.rec = REC + (long long)f * P.npx; Fm.seedcs = seedcs + (long long)f * P.npx; Fm.sq = SQ + (long long)f * P.npx;
  Fm.order = order + (long long)f * P.npx; Fm.n = ndef[f];
  Fm.st = ST + (long long)f * P.npx; Fm.pool = POOL + (long long)f * GP.pool_cap; Fm.ctl = CTL + (long long)f * kCtlStride; Fm.wtab = wtab;
  float4* S = segs + (long long)f * P.seg_cap;
  const bool solo = (wpf == 1);
  if (!solo && wif == 0) {
    // ---- the COMMITTER of the frame: nothing but the in-order validation, as fast as the status words arrive
    for (unsigned iter = 0;; iter++) {
      __syncwarp();
      const int F = __shfl_sync(0xffffffffu, ld_i(&Fm.ctl[C_FIN]), 0);
      if (F >= Fm.n) break;
      if (iter > 4u * kGrowWatchdog) {
        if (lane == 0) { a_or(reinterpret_cast<unsigned*>(&Fm.ctl[C_ERR]), (unsigned)ERR_WATCHDOG); a_max(&Fm.ctl[C_FIN], Fm.n); }
        break;
      }
      warp_commit(GP, Fm, S, lane);
      if (__shfl_sync(0xffffffffu, ld_i(&Fm.ctl[C_FIN]), 0) == F) __nanosleep(200);   // the head is still running
    }
    if (lane == 0) {
      __threadfence();
      const int ns = ld_i(&Fm.ctl[C_NS]), err = ld_i(&Fm.ctl[C_ERR]);
      nseg[f] = min(ns, P.seg_cap);
      if (ns > P.seg_cap) atomicOr(overflow, 1);
      if (err) atomicOr(overflow, 2);
    }
    return;
  }
  Lane L;
  L.home = LANEBUF + ((size_t)gw * 32 + lane) * (size_t)GP.lane_cap; L.home_cap = GP.lane_cap;
  L.buf = L.home; L.cap = L.home_cap;
  L.ring = ring_all[wic] + lane * lg::kRing;
  L.phase = P_IDLE; L.task = -1; L.fresh = 1; L.off = 0; L.j = 0; L.m = 0;
  lane_reset(L);
  const unsigned lt = (1u << lane) - 1u;
  int whead = 0, wcount = 0, rsc = 0;
  bool exhausted = false;
  unsigned iter_total = 0; unsigned long long busy_total = 0;
  for (unsigned iter = 0;; iter++) {
    __syncwarp();
    iter_total = iter;
    const int F = __shfl_sync(0xffffffffu, ld_i(&Fm.ctl[C_FIN]), 0);
    if (F >= Fm.n) break;
    if (iter > kGrowWatchdog) {          // cannot happen (the head task always completes); never hang the GPU on a bug
      // post-mortem for pl_line_debug_ctl(): where the frontier stood, what the head looked like, what this warp held
      int first = 0;
      if (lane == 0 && a_cas(&Fm.ctl[C_STAT0 + 7 - 1], 0, F + 1) == 0 && false) {
        first = 1;
        Fm.ctl[C_STAT0 + 6] = (int)ld_u(&Fm.st[F]);
        Fm.ctl[C_WORDS + 0] = 0x7777; Fm.ctl[C_WORDS + 1] = wif; Fm.ctl[C_WORDS + 2] = wcount; Fm.ctl[C_WORDS + 3] = (int)exhausted;
        Fm.ctl[C_WORDS + 4] = ld_i(&Fm.ctl[C_NXT]); Fm.ctl[C_WORDS + 5] = ld_i(&Fm.ctl[C_REDO]); Fm.ctl[C_WORDS + 6] = ld_i(&Fm.ctl[C_LOCK]);
        Fm.ctl[C_WORDS + 7] = Fm.n;
      }
      first = __shfl_sync(0xffffffffu, first, 0);
      if (first) { Fm.ctl[C_WORDS + 8 + 2 * lane] = L.phase; Fm.ctl[C_WORDS + 9 + 2 * lane] = L.task; }
      __syncwarp();
      if (lane == 0) { a_or(reinterpret_cast<unsigned*>(&Fm.ctl[C_ERR]), (unsigned)ERR_WATCHDOG); a_max(&Fm.ctl[C_FIN], Fm.n); }
      break;
    }
    // ---- commit (only when this warp is the whole group)
    if (solo) warp_commit(GP, Fm, S, lane);
    // ---- feed
    unsigned mi = __ballot_sync(0xffffffffu, L.phase == P_IDLE);
    // a warp that carries a long region is on the frame's critical path (the chain of long, refine-heavy regions is what
    // a single frame waits for): it looks for new work only every 8th iteration, the other warps feed the idle lanes
    const bool heavy = __any_sync(0xffffffffu, L.phase != P_IDLE && L.hi >= 64);
    if (mi && (!heavy || (iter & 7u) == 0u)) {
      // lane 0 looks at the three hand-over words at once: the re-execution slot of the committer and the redo ring
      int redo = -1, rqh = 0, rqt = 0;
      if (lane == 0) { redo = ld_i(&Fm.ctl[C_REDO]); rqh = ld_i(&Fm.ctl[C_RQH]); rqt = ld_i(&Fm.ctl[C_RQT]); if (redo >= 0) redo = a_exch(&Fm.ctl[C_REDO], -1); }
      redo = __shfl_sync(0xffffffffu, redo, 0);
      if (redo >= 0) {
        const int k = __ffs(mi) - 1;
        if (lane == k) lane_take_redo(Fm, L, redo);
        mi &= mi - 1u;
      }
      // aborted tasks that are already published: re-execute them now rather than when they reach the head
      int pending = __shfl_sync(0xffffffffu, rqt - rqh, 0);
      for (int tries = 0; tries < 2 && mi && pending > 0; tries++, pending--) {
        int m = -1;
        if (lane == 0) {
          const int hq = a_add(&Fm.ctl[C_RQH], 1);
          m = a_exch(&Fm.ctl[C_WORDS + (hq & (kRedoQ - 1))], 0) - 1;
          if (m >= 0) {
            const unsigned w = ld_u(&Fm.st[m]);
            if ((w & ST_STATE) != ST_DONE || !(w & ST_ABORT) ||
                (unsigned)a_cas(reinterpret_cast<int*>(&Fm.st[m]), (int)w, (int)((w & ~(ST_STATE | ST_ABORT)) | ST_REDO)) != w) m = -1;
          }
        }
        m = __shfl_sync(0xffffffffu, m, 0);
        if (m >= 0) {
          const int k = __ffs(mi) - 1;
          if (lane == k) lane_take_redo(Fm, L, m);
          mi &= mi - 1u;
        }
      }
      // new seeds: 4 x 32 entries of the order per scan (one atomic, the loads of the four batches overlap)
      if (__popc(mi) > wcount && !exhausted) {
        int base = -1;
        if (lane == 0 && !(GP.window > 0 && ld_i(&Fm.ctl[C_NXT]) - F >= GP.window)) base = a_add(&Fm.ctl[C_NXT], 128);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= Fm.n) exhausted = true;
        else if (base >= 0) {
          unsigned pix[4]; int own[4];
#pragma unroll
          for (int q = 0; q < 4; q++) { const int i = base + 32 * q + lane; pix[q] = (i < Fm.n) ? ldg_u(&Fm.order[i]) : 0u; }
#pragma unroll
          for (int q = 0; q < 4; q++) { const int i = base + 32 * q + lane; own[q] = (i < Fm.n) ? ld_i(&Fm.rec[(int)(pix[q] >> 16) * P.sw + (int)(pix[q] & 0xffffu)].x) : 0; }
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const int i = base + 32 * q + lane;
            bool cand = false;
            if (i < Fm.n) {
              if (own_candidate(own[q], 2 * i, F)) cand = true;
              else st_u(&Fm.st[i], (!(own[q] & 1) && (own[q] >> 1) < F) ? ST_NOOP : ST_EATEN);
            }
            const unsigned mc = __ballot_sync(0xffffffffu, cand);
            if (cand) wq[(whead + wcount + __popc(mc & lt)) & (kGrowQ - 1)] = i;
            wcount += __popc(mc);
          }
          __syncwarp();
        }
      }
      // lanes still idle: look again at seeds found consumed by a task that was not final then (it may have let go)
      if (__popc(mi) > wcount && wcount <= kGrowQ - 32) {
        const int hi = min(__shfl_sync(0xffffffffu, ld_i(&Fm.ctl[C_NXT]), 0), Fm.n);
        if (hi > F) {
          if (rsc < F || rsc >= hi) rsc = F;
          const int i = rsc + lane;
          rsc += 32;
          bool cand = false;
          if (i < hi) {
            const unsigned w = ld_u(&Fm.st[i]);
            if ((w & ST_STATE) == ST_EATEN) {
              const unsigned pix = ldg_u(&Fm.order[i]);
              const int o = ld_i(&Fm.rec[(int)(pix >> 16) * P.sw + (int)(pix & 0xffffu)].x);
              if (own_candidate(o, 2 * i, F)) cand = ((unsigned)a_cas(reinterpret_cast<int*>(&Fm.st[i]), (int)w, (int)ST_RUN) == w);
              else if (!(o & 1) && (o >> 1) < F) st_u(&Fm.st[i], ST_NOOP);
            }
          }
          const unsigned mc = __ballot_sync(0xffffffffu, cand);
          if (cand) wq[(whead + wcount + __popc(mc & lt)) & (kGrowQ - 1)] = i;
          wcount += __popc(mc);
          __syncwarp();
        }
      }
      const int r = __popc(mi & lt);
      if (((mi >> lane) & 1u) && r < wcount) lane_take_seed(L, wq[(whead + r) & (kGrowQ - 1)]);
      const int taken = min(__popc(mi), wcount);
      whead += taken; wcount -= taken;
    }
    // ---- step
    busy_total += __popc(__ballot_sync(0xffffffffu, L.phase != P_IDLE));
    if (L.phase != P_IDLE) lane_step<false>(GP, Fm, L);
  }
  if (lane == 0) { a_max(&Fm.ctl[C_STAT0 + 5], (int)iter_total); a_add(&Fm.ctl[C_STAT0 + 6], (int)(busy_total >> 5)); }
  // frame finished (or given up): in a one-warp group the worker reports
  if (solo && lane == 0) {
    __threadfence();
    const int ns = ld_i(&Fm.ctl[C_NS]), err = ld_i(&Fm.ctl[C_ERR]);
    nseg[f] = min(ns, P.seg_cap);
    if (ns > P.seg_cap) atomicOr(overflow, 1);
    if (err) atomicOr(overflow, 2);
  }
}
// per-frame control words of the grow kernel (re-armed before every launch)
__global__ void k_lsd_grow_init(int* __restrict__ CTL, int nframes) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nframes) return;
  int* c = CTL + (long long)f * lg::kCtlStride;
  for (int k = 0; k < lg::kCtlStride; k++) c[k] = 0;
  c[lg::C_REDO] = -1; c[lg::C_POOL] = 1;
}
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

// ---------------------------------------------------------------------------------------------- K_H LBD blur + Sobel
// GaussianBlur 5x5 sigma 1 (8.8 fixed point rows [14 62 104 62 14]) fused with the Sobel pair (dx, dy as int16).
// Tile: 64x64 blurred pixels <- 68x68 raw pixels in shared memory -> 62x62 outputs.  The raw tile is loaded at
// reflect-101 coordinates; because the kernel is symmetric, the blur of the reflected image at column -1 equals the
// blurred value at column +1, i.e. exactly what Sobel's own BORDER_REFLECT_101 of the BLURRED image needs, so no tap
// ever reflects again.  One thread walks down one column: the last five horizontal sums live in registers (blur), then
// a sliding 3x3 window of blurred bytes (Sobel).
constexpr int kSobT = 64, kSobOut = kSobT - 2, kSobRawP = kSobT + 8, kSobSeg = kSobT / 4;
__global__ void __launch_bounds__(256) k_lbd_sobel(LineParams P, const uint8_t* __restrict__ imgs, int stride,
                                                   long long frame_stride, short2* __restrict__ dxy) {
  __shared__ uint8_t raw[(kSobT + 4) * kSobRawP];
  __shared__ uint8_t bl[kSobT * (kSobT + 4)];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int X0 = blockIdx.x * kSobOut, Y0 = blockIdx.y * kSobOut;   // first output pixel of the tile
  const uint8_t* img = imgs + (long long)blockIdx.z * frame_stride;
  auto r101 = [](int p, int n) { if (p < 0) p = -p; if (p >= n) p = 2 * (n - 1) - p; return min(max(p, 0), n - 1); };
  // raw rows Y0-3 .. Y0+64, columns X0-3 .. X0+64
  for (int r = ty; r < kSobT + 4; r += 4) {
    const uint8_t* row = img + (long long)r101(Y0 - 3 + r, P.h) * stride;
    raw[r * kSobRawP + tx] = row[r101(X0 - 3 + tx, P.w)];
    if (tx < 4) raw[r * kSobRawP + kSobT + tx] = row[r101(X0 - 3 + kSobT + tx, P.w)];
  }
  __syncthreads();
  {  // blurred pixel (bx, by) of the tile = image pixel (X0-1+bx, Y0-1+by); thread: column tx, rows ty*16 .. +15
    const uint8_t* p = raw + (ty * kSobSeg) * kSobRawP + tx;
    auto hrow = [&](const uint8_t* q) { return 14 * (q[0] + q[4]) + 62 * (q[1] + q[3]) + 104 * q[2]; };
    int w0 = hrow(p), w1 = hrow(p + kSobRawP), w2 = hrow(p + 2 * kSobRawP), w3 = hrow(p + 3 * kSobRawP);
    p += 4 * kSobRawP;
    uint8_t* o = bl + (ty * kSobSeg) * (kSobT + 4) + tx;
#pragma unroll 4
    for (int r = 0; r < kSobSeg; r++, p += kSobRawP, o += kSobT + 4) {
      const int w4 = hrow(p);
      const unsigned acc = 14u * (unsigned)(w0 + w4) + 62u * (unsigned)(w1 + w3) + 104u * (unsigned)w2;
      *o = (uint8_t)((acc + 32768u) >> 16);
      w0 = w1; w1 = w2; w2 = w3; w3 = w4;
    }
  }
  __syncthreads();
  const int x = X0 + tx - 1;                       // output column of blurred column tx (1..62 produce outputs)
  if (tx < 1 || tx > kSobOut || x >= P.w) return;
  const int rbeg = max(ty * kSobSeg, 1), rend = min(ty * kSobSeg + kSobSeg - 1, kSobOut);   // blurred rows of my outputs
  const uint8_t* b = bl + (rbeg - 1) * (kSobT + 4) + tx;
  int a00 = b[-1], a01 = b[0], a02 = b[1];
  b += kSobT + 4;
  int a10 = b[-1], a11 = b[0], a12 = b[1];
  short2* D = dxy + (long long)blockIdx.z * P.w * P.h;
  for (int r = rbeg; r <= rend; r++) {
    b += kSobT + 4;
    const int a20 = b[-1], a21 = b[0], a22 = b[1];
    const int y = Y0 + r - 1;
    if (y < P.h)
      D[(long long)y * P.w + x] = make_short2((short)((a02 - a00) + 2 * (a12 - a10) + (a22 - a20)),
                                              (short)((a20 - a00) + 2 * (a21 - a01) + (a22 - a02)));
    a00 = a10; a01 = a11; a02 = a12; a10 = a20; a11 = a21; a12 = a22;
  }
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
  cudaStream_t stream = nullptr;
  uint8_t* d_scaled = nullptr;
  float2* d_seedcs = nullptr;
  // region growing (lsd_grow_core.cuh): pixel records, status words, list pool, control words, lane buffers, weight table
  lg::Params GP;
  int grow_warps_target = 132 * 16;   // warps the grow kernel spreads over the GPU when the batch is small (env PLSLAM_LSD_GROW_WARPS)
  int grow_wpf_max = 64;              // at most this many warps on one frame (env PLSLAM_LSD_GROW_WPF)
  // batches up to this size use the speculative kernel, larger ones the ordered one (env PLSLAM_LSD_GROW_SPEC_MAXB).  Default 0:
  // the speculative kernel wins on frames made of many small regions (DESIGN.md §6)
  // and loses on frames whose long, refine-heavy regions form a dependency chain
  int grow_spec_max_batch = 0;
  size_t lane_warps = 0;              // lane buffers are allocated for this many warps
  int4* d_rec = nullptr; int* d_sq = nullptr;
  unsigned *d_st = nullptr, *d_pool = nullptr, *d_lanebuf = nullptr; int* d_ctl = nullptr; double* d_wtab = nullptr;
  GradRec* d_gtab = nullptr; float2* d_gtab_seed = nullptr;   // (gx, gy) -> level-line record, built once (k_lsd_grad_table)
  unsigned short* d_counts = nullptr;
  int *d_offsets = nullptr, *d_ndef = nullptr, *d_maxs = nullptr, *d_nseg = nullptr, *d_overflow = nullptr;
  unsigned* d_order = nullptr;
  float4* d_segs = nullptr;
  short2* d_dxy = nullptr;
  // host-pointer API staging
  uint8_t* d_img = nullptr; PLKeyLineRec* d_kls = nullptr; uint8_t* d_desc = nullptr; double* d_lf = nullptr; int* d_nl = nullptr;
  uint8_t* d_mask = nullptr;
  size_t key_smem = 0;
  int last_B = 0;
  // optional device timing of the dominant kernel (bench.py roofline): events on the launching stream
  int timing = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

static const unsigned char h_comb[64] = {0, 1, 0, 2, 0, 3, 0, 4, 0, 5, 0, 6, 1, 2, 1, 3, 1, 4, 1, 5, 1, 6, 2, 3, 2, 4, 2, 5, 2, 6, 2, 7,
                                         2, 8, 3, 4, 3, 5, 3, 6, 3, 7, 3, 8, 4, 5, 4, 6, 4, 7, 4, 8, 5, 6, 5, 7, 5, 8, 6, 7, 6, 8, 7, 8};

extern "C" void pl_line_destroy(PLLine* h) {
  if (!h) return;
  cudaFree(h->d_gtab); cudaFree(h->d_gtab_seed); cudaFree(h->d_scaled); cudaFree(h->d_seedcs); cudaFree(h->d_rec); cudaFree(h->d_sq); cudaFree(h->d_st); cudaFree(h->d_pool); cudaFree(h->d_lanebuf); cudaFree(h->d_ctl); cudaFree(h->d_wtab); cudaFree(h->d_counts); cudaFree(h->d_offsets);
  cudaFree(h->d_ndef); cudaFree(h->d_maxs); cudaFree(h->d_nseg); cudaFree(h->d_overflow); cudaFree(h->d_order);
  cudaFree(h->d_segs); cudaFree(h->d_dxy); cudaFree(h->d_img); cudaFree(h->d_kls);
  cudaFree(h->d_desc); cudaFree(h->d_lf); cudaFree(h->d_nl); cudaFree(h->d_mask);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

extern "C" int pl_line_create(const PLLineConfig* cfg, PLLine** out) {
  PL_ARG(cfg && out);
  PL_ARG(cfg->width >= 64 && cfg->height >= 64 && cfg->width < 8000 && cfg->height < 8000 && cfg->nfeatures > 0 && cfg->max_batch >= 1);
  int rc = require_device();
  if (rc) return rc;
  PLLine* h = new PLLine;
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
#define LN_TRY(e) do { int _r = (e); if (_r) { pl_line_destroy(h); return _r; } } while (0)
#define LN_CUDA(e) do { cudaError_t _e = (e); if (_e != cudaSuccess) { set_error("%s -> %s", #e, cudaGetErrorString(_e)); pl_line_destroy(h); return PL_ERR_CUDA; } } while (0)
  LN_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  LN_TRY(dev_alloc(&h->d_scaled, npx * B)); LN_TRY(dev_alloc(&h->d_seedcs, npx * B)); LN_TRY(dev_alloc(&h->d_rec, npx * B));
  LN_TRY(dev_alloc(&h->d_sq, npx * B));
  {  // speculative region growing: geometry of the run-time structures
    int dev = 0, sms = 132;
    cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    h->grow_warps_target = sms * 16;
    if (const char* e = getenv("PLSLAM_LSD_GROW_WARPS")) { const int v = atoi(e); if (v > 0) h->grow_warps_target = v; }
    if (const char* e = getenv("PLSLAM_LSD_GROW_WPF")) { const int v = atoi(e); if (v > 0) h->grow_wpf_max = v; }
    if (const char* e = getenv("PLSLAM_LSD_GROW_SPEC_MAXB")) h->grow_spec_max_batch = atoi(e);
    lg::Params& G = h->GP;
    G.sw = P.sw; G.sh = P.sh; G.npx = P.npx; G.min_reg_size = P.min_reg_size; G.seg_cap = P.seg_cap;
    G.lane_cap = 1024; G.pool_cap = 4 * P.npx; G.window = 8192;
    if (const char* e = getenv("PLSLAM_LSD_GROW_WINDOW")) G.window = atoi(e);
    G.prec = P.prec; G.prec_hi = P.prec_hi; G.density_th = P.density_th;
    h->lane_warps = std::max<size_t>(std::min<size_t>(B * (size_t)h->grow_wpf_max, (size_t)h->grow_warps_target), B);
    LN_TRY(dev_alloc(&h->d_st, npx * B)); LN_TRY(dev_alloc(&h->d_pool, (size_t)G.pool_cap * B)); LN_TRY(dev_alloc(&h->d_ctl, (size_t)lg::kCtlStride * B));
    LN_TRY(dev_alloc(&h->d_lanebuf, h->lane_warps * 32 * (size_t)G.lane_cap));
    const int nw = 2 * kGradR * kGradR + 1;
    LN_TRY(dev_alloc(&h->d_wtab, (size_t)nw));
    k_lsd_wtab<<<(nw + 255) / 256, 256, 0, h->stream>>>(h->d_wtab, nw);
    LN_CUDA(cudaGetLastError());
    count_launch();
  }
  LN_TRY(dev_alloc(&h->d_counts, (size_t)kBins * P.nchunk * B)); LN_TRY(dev_alloc(&h->d_offsets, (size_t)kBins * P.nchunk * B));
  LN_TRY(dev_alloc(&h->d_ndef, B)); LN_TRY(dev_alloc(&h->d_maxs, B)); LN_TRY(dev_alloc(&h->d_nseg, B)); LN_TRY(dev_alloc(&h->d_overflow, 1));
  LN_TRY(dev_alloc(&h->d_order, npx * B)); LN_TRY(dev_alloc(&h->d_segs, (size_t)P.seg_cap * B));
  LN_TRY(dev_alloc(&h->d_dxy, (size_t)P.w * P.h * B));
  LN_CUDA(cudaMemset(h->d_overflow, 0, sizeof(int)));
  LN_TRY(dev_alloc(&h->d_gtab, (size_t)kGradN * kGradN)); LN_TRY(dev_alloc(&h->d_gtab_seed, (size_t)kGradN * kGradN));
  k_lsd_grad_table<<<(kGradN * kGradN + 255) / 256, 256, 0, h->stream>>>(h->d_gtab, h->d_gtab_seed);
  LN_CUDA(cudaGetLastError());
  LN_CUDA(cudaStreamSynchronize(h->stream));
  count_launch();
  {  // LBD weights (binary_descriptor_custom.cpp:217-259), integer divisions as in the reference
    float gG[63], gL[21];
    double u = (7 * 3 - 1) / 2, sigma = (7 * 2 + 1) / 2, inv = -1 / (2 * sigma * sigma);
    for (int i = 0; i < 21; i++) { double d = i - u; gL[i] = (float)exp(d * d * inv); }
    u = (9 * 7 - 1) / 2; sigma = u; inv = -1 / (2 * sigma * sigma);
    for (int i = 0; i < 63; i++) { double d = i - u; gG[i] = (float)exp(d * d * inv); }
    LN_CUDA(cudaMemcpyToSymbol(c_gaussG, gG, sizeof(gG)));
    LN_CUDA(cudaMemcpyToSymbol(c_gaussL, gL, sizeof(gL)));
    LN_CUDA(cudaMemcpyToSymbol(c_comb, h_comb, sizeof(h_comb)));
  }
  LN_CUDA(cudaFuncSetAttribute(k_keylines, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->key_smem));
  // cfg->lsd_used_in_global is accepted for ABI compatibility and ignored: the USED state is the ownership word of the pixel record
  *out = h;
  return PL_OK;
}

extern "C" int pl_line_capacity(const PLLine* h) { return h ? h->P.capL : PL_ERR_ARG; }

// Device timing of k_lsd_grow (the dominant kernel): enable, run, then read the duration of the LAST launch.
extern "C" int pl_line_set_timing(PLLine* h, int on) {
  PL_ARG(h);
  if (on && !h->ev0) { PL_CUDA(cudaEventCreate(&h->ev0)); PL_CUDA(cudaEventCreate(&h->ev1)); }
  h->timing = on;
  return PL_OK;
}
extern "C" int pl_line_grow_ms(PLLine* h, float* ms) {
  PL_ARG(h && ms && h->ev0);
  PL_CUDA(cudaEventSynchronize(h->ev1));
  PL_CUDA(cudaEventElapsedTime(ms, h->ev0, h->ev1));
  return PL_OK;
}
/* algorithmic bytes k_lsd_grow must move for one frame (DESIGN.md §6): per scaled pixel: record (16) + seed cos/sin (8)
 * + seed order entry (4); the USED map lives in shared memory */
extern "C" long long pl_line_grow_bytes_per_frame(const PLLine* h) { return h ? (long long)h->P.npx * 28 : 0; }

extern "C" int pl_line_extract_batch_dev(PLLine* h, const uint8_t* imgs, int stride, size_t frame_stride, int B,
                                         const uint8_t* mask, void* keylines, uint8_t* desc, double* linefunc, int* n,
                                         void* stream_) {
  PL_ARG(h && imgs && keylines && desc && linefunc && n && B >= 1 && B <= h->cfg.max_batch && stride >= h->cfg.width);
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : h->stream;
  const LineParams& P = h->P;
  h->last_B = B;
  PL_CUDA(cudaMemsetAsync(h->d_maxs, 0, sizeof(int) * B, st));
  k_lsd_scale<<<dim3((P.sw + 31) / 32, (P.sh + 31) / 32, B), 256, 0, st>>>(P, imgs, stride, (long long)frame_stride, h->d_scaled);
  PL_LAUNCH_CHECK();
  {
    const dim3 grd((P.sw + 255) / 256, (P.sh + 3) / 4, B);
    if (P.sw % 4 == 0)
      k_lsd_grad<true><<<grd, 256, 0, st>>>(P, h->d_scaled, reinterpret_cast<const float4*>(h->d_gtab), h->d_gtab_seed, h->d_rec, h->d_sq, h->d_seedcs, h->d_maxs);
    else
      k_lsd_grad<false><<<grd, 256, 0, st>>>(P, h->d_scaled, reinterpret_cast<const float4*>(h->d_gtab), h->d_gtab_seed, h->d_rec, h->d_sq, h->d_seedcs, h->d_maxs);
  }
  PL_LAUNCH_CHECK();
  k_lsd_hist<<<dim3(P.nchunk, B), 256, 0, st>>>(P, h->d_sq, h->d_maxs, h->d_counts);
  PL_LAUNCH_CHECK();
  k_lsd_scan<<<B, kBins, 0, st>>>(P, h->d_counts, h->d_offsets, h->d_ndef);
  PL_LAUNCH_CHECK();
  k_lsd_scatter<<<dim3((P.nchunk + 3) / 4, B), 128, 0, st>>>(P, h->d_sq, h->d_maxs, h->d_offsets, h->d_order);
  PL_LAUNCH_CHECK();
  if (B <= h->grow_spec_max_batch) {
    // few frames: many regions of each frame in flight (ordered speculative execution, lsd_grow_core.cuh)
    PL_CUDA(cudaMemsetAsync(h->d_st, 0, sizeof(unsigned) * (size_t)P.npx * B, st));
    k_lsd_grow_init<<<(B + 127) / 128, 128, 0, st>>>(h->d_ctl, B);
    PL_LAUNCH_CHECK();
    if (h->timing) PL_CUDA(cudaEventRecord(h->ev0, st));
    // warps per frame (one of them is the frame's committer when there is more than one)
    const int wpf = std::max(1, std::min(h->grow_wpf_max, h->grow_warps_target / B));
    k_lsd_grow<1><<<B * wpf, 32, 0, st>>>(P, h->GP, h->d_rec, h->d_seedcs, h->d_sq, h->d_order, h->d_ndef, h->d_st, h->d_pool, h->d_ctl,
                                          h->d_lanebuf, h->d_wtab, h->d_segs, h->d_nseg, h->d_overflow, B, wpf);
    PL_LAUNCH_CHECK();
  } else {
    // many frames: one warp per frame, the 32 lanes on one region at a time (lsd_grow_ordered.cuh); the list pool and the
    // status words of the speculative kernel serve as region list and far-pixel mask
    if (h->timing) PL_CUDA(cudaEventRecord(h->ev0, st));
    static const int pre_maxb = getenv("PLSLAM_LSD_PRE_MAXB") ? atoi(getenv("PLSLAM_LSD_PRE_MAXB")) : 256;
    // the kernel addresses the per-frame arrays with 32-bit element indices (frame * npx + pixel): at most 2^32 / npx frames per grid
    const int chunk = (int)std::min<long long>(B, 0xffffffffLL / P.npx);
    for (int b0 = 0; b0 < B; b0 += chunk) {
      const int nb = std::min(chunk, B - b0);
      const size_t po = (size_t)b0 * P.npx;
      if (B <= pre_maxb)
        k_lsd_grow_ordered<true><<<nb, 32, 0, st>>>(P, h->d_rec + po, h->d_sq + po, h->d_seedcs + po, h->d_order + po, h->d_ndef + b0,
                                                    h->d_pool + (size_t)b0 * h->GP.pool_cap, h->GP.pool_cap, h->d_st + po, h->d_wtab,
                                                    h->d_segs + (size_t)b0 * P.seg_cap, h->d_nseg + b0, h->d_overflow, nb);
      else
        k_lsd_grow_ordered<false><<<nb, 32, 0, st>>>(P, h->d_rec + po, h->d_sq + po, h->d_seedcs + po, h->d_order + po, h->d_ndef + b0,
                                                     h->d_pool + (size_t)b0 * h->GP.pool_cap, h->GP.pool_cap, h->d_st + po, h->d_wtab,
                                                     h->d_segs + (size_t)b0 * P.seg_cap, h->d_nseg + b0, h->d_overflow, nb);
    }
    PL_LAUNCH_CHECK();
  }
  if (h->timing) PL_CUDA(cudaEventRecord(h->ev1, st));
  k_keylines<<<B, 256, h->key_smem, st>>>(P, h->d_segs, h->d_nseg, mask, (PLKeyLineRec*)keylines, linefunc, n);
  PL_LAUNCH_CHECK();
  k_lbd_sobel<<<dim3((P.w + kSobOut - 1) / kSobOut, (P.h + kSobOut - 1) / kSobOut, B), 256, 0, st>>>(P, imgs, stride, (long long)frame_stride, h->d_dxy);
  PL_LAUNCH_CHECK();
  k_lbd_describe<<<dim3(P.capL, B), 64, 0, st>>>(P, (const PLKeyLineRec*)keylines, n, h->d_dxy, desc);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

// capacity flags of the calls since the last check (segment_cap exceeded, or the region growing gave a frame up);
// the *_dev entry points are asynchronous and never look at them: their callers do, after synchronising
extern "C" int pl_line_check_overflow(PLLine* h) {
  PL_ARG(h);
  int ov = 0;
  PL_CUDA(cudaMemcpy(&ov, h->d_overflow, sizeof(int), cudaMemcpyDeviceToHost));
  if (ov) {
    cudaMemset(h->d_overflow, 0, sizeof(int));
    if (ov & 1) set_error("LSD produced more than segment_cap=%d segments", h->P.seg_cap);
    else set_error("LSD region growing gave a frame up (list pool of %d words exhausted, or watchdog): see pl_line_debug_ctl", h->GP.pool_cap);
    return PL_ERR_CAPACITY;
  }
  return PL_OK;
}

static int line_staging(PLLine* h) {
  if (h->d_img) return PL_OK;
  const size_t B = h->cfg.max_batch;
  int rc;
  if ((rc = dev_alloc(&h->d_img, (size_t)h->P.w * h->P.h * B))) return rc;
  if ((rc = dev_alloc(&h->d_kls, (size_t)h->P.capL * B))) return rc;
  if ((rc = dev_alloc(&h->d_desc, (size_t)h->P.capL * 32 * B))) return rc;
  if ((rc = dev_alloc(&h->d_lf, (size_t)h->P.capL * 3 * B))) return rc;
  if ((rc = dev_alloc(&h->d_nl, B))) return rc;
  if ((rc = dev_alloc(&h->d_mask, (size_t)h->P.w * h->P.h))) return rc;
  return PL_OK;
}

extern "C" int pl_line_extract_batch(PLLine* h, const uint8_t* imgs, int stride, size_t frame_stride, int B,
                                     const uint8_t* mask, void* keylines, uint8_t* desc, double* linefunc, int* n) {
  PL_ARG(h && imgs && keylines && desc && linefunc && n && B >= 1 && B <= h->cfg.max_batch && stride >= h->cfg.width);
  int rc = line_staging(h);
  if (rc) return rc;
  const int W = h->P.w, H = h->P.h;
  for (int b = 0; b < B; b++)
    PL_CUDA(cudaMemcpy2DAsync(h->d_img + (size_t)b * W * H, W, imgs + (size_t)b * frame_stride, stride, W, H, cudaMemcpyHostToDevice, h->stream));
  if (mask) PL_CUDA(cudaMemcpyAsync(h->d_mask, mask, (size_t)W * H, cudaMemcpyHostToDevice, h->stream));
  rc = pl_line_extract_batch_dev(h, h->d_img, W, (size_t)W * H, B, mask ? h->d_mask : nullptr, h->d_kls, h->d_desc, h->d_lf, h->d_nl, h->stream);
  if (rc) return rc;
  const size_t cap = h->P.capL;
  PL_CUDA(cudaMemcpyAsync(keylines, h->d_kls, cap * B * sizeof(PLKeyLineRec), cudaMemcpyDeviceToHost, h->stream));
  PL_CUDA(cudaMemcpyAsync(desc, h->d_desc, cap * B * 32, cudaMemcpyDeviceToHost, h->stream));
  PL_CUDA(cudaMemcpyAsync(linefunc, h->d_lf, cap * B * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  PL_CUDA(cudaMemcpyAsync(n, h->d_nl, (size_t)B * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
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
extern "C" int pl_line_debug_ctl(PLLine* h, int frame, int* out, int nwords) {
  PL_ARG(h && out && frame >= 0 && frame < h->cfg.max_batch && nwords > 0 && nwords <= lg::kCtlStride);
  PL_CUDA(cudaStreamSynchronize(h->stream));
  PL_CUDA(cudaMemcpy(out, h->d_ctl + (size_t)frame * lg::kCtlStride, sizeof(int) * nwords, cudaMemcpyDeviceToHost));
  return PL_OK;
}
extern "C" int pl_line_debug_order(PLLine* h, int frame, unsigned* out, int cap) {
  PL_ARG(h && frame >= 0 && frame < h->last_B);
  int n = 0;
  PL_CUDA(cudaStreamSynchronize(h->stream));
  PL_CUDA(cudaMemcpy(&n, h->d_ndef + frame, sizeof(int), cudaMemcpyDeviceToHost));
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
