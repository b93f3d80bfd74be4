// ORB extraction for batches of frames on sm_90a.
//
// Replaces ORB_SLAM2::ORBextractor (reference src/ORBextractor.cc).  Kernel map (DESIGN.md §3):
//   k_resize_level   ComputePyramid         :1107-1132  (cv::resize INTER_LINEAR, 11-bit fixed point)
//   k_fast_cells     ComputeKeyPointsOctTree:765-829    (cv::FAST 9/16 + NMS per ~30x30 cell, ini/min threshold)
//   k_quadtree       DistributeOctTree      :539-763    (one warp per (frame, level); exact sequential semantics)
//   k_describe       IC_Angle :77-104, GaussianBlur :1086, computeOrbDescriptor :108-147, scaling :1095-1101
//
// Design notes
//  * No blurred level image is ever materialised: k_describe blurs the 43x43 neighbourhood of each
//    selected keypoint in shared memory (same 8.8 fixed-point arithmetic as cv::GaussianBlur), which
//    removes 2 bytes/pixel of HBM traffic per level compared with the reference's clone + blur.
//  * The 19-px pyramid border is never read on this path (all keypoints are >= 19 px inside), so levels are
//    stored border-less; pl_orb_get_level() re-creates the border on request for the mvImagePyramid member.
//  * Level 0 is the caller's image; it is not copied.
//  * Arithmetic that feeds a rounding (fastAtan2, rBRIEF rotation) uses explicit __f*_rn intrinsics: no FMA.

#include "common.cuh"
#include "tma.cuh"
#include "libm_glibc.cuh"
#include <math.h>
#include <vector>
#include <algorithm>
#include <string.h>

namespace pl {

constexpr int kMaxLevels = 12;
constexpr int kEdge = 19;        // EDGE_THRESHOLD
constexpr int kHalfPatch = 15;   // HALF_PATCH_SIZE
constexpr int kMaxWin = 72;      // max FAST cell window side (cell + 6)

__device__ char4 g_pattern[256];      // rBRIEF pairs; global (L1) because every lane reads a different entry
__constant__ int c_umax[16];
static const int8_t h_pattern[256 * 4] = {
#include "../data/orb_pattern_31.inc"
};

struct LevelInfo {
  int w, h, pitch;        // level size; pitch of the stored level (level 0: caller's stride)
  long long off;          // byte offset of the level inside one frame's pyramid block (levels >= 1)
  long long boff;         // byte offset of the BLURRED level inside one frame's blur block (all levels), pitch = bpitch
  int bpitch;
  int cell0, ncells;      // first cell / number of cells in the cell table
  int nfeat;              // mnFeaturesPerLevel
  int nIni;               // DistributeOctTree: number of root nodes
  float hX;               // root node width
  int regW, regH;         // maxBorderX-minBorderX, maxBorderY-minBorderY
  float scale;            // mvScaleFactor[level]
  float size;             // (float)(int)(31*scale)
  long long keyoff;       // offset (in keys) of this level inside one frame's quadtree key scratch
  int keycap;             // ncells*slotcap
  int tab_x, tab_y;       // offsets into the resize tables
};

struct CellInfo {
  short level, x0, y0, x1, y1, sx, sy, pad;  // window [x0,x1)x[y0,y1) in level coords; shift j*wCell,i*hCell
};

struct OrbParams {
  LevelInfo lv[kMaxLevels];
  int nlevels, ncells, slotcap, cap, iniTh, minTh, poolcap, width, height;
  long long pyr_frame;   // bytes of one frame's pyramid block (levels 1..)
  long long blur_frame;  // bytes of one frame's blurred-levels block (levels 0..)
  long long key_frame;   // keys per frame in the quadtree scratch (per buffer)
  int selcap;            // per (frame,level) selected capacity
  int sortcap;           // power of two >= poolcap (bitonic sort region)
};

// ------------------------------------------------------------------------------------------------
// K1  pyramid level l from level l-1 (cv::resize, INTER_LINEAR, 8U).  Tables are computed on the host.
// One thread = 4 consecutive output pixels (uchar4 store).
__global__ void __launch_bounds__(256) k_resize_level(const uint8_t* __restrict__ src, int spitch, long long sframe,
                                                      int sw, int sh, uint8_t* __restrict__ dst, int dpitch,
                                                      long long dframe, int dw, int dh,
                                                      const short4* __restrict__ xtab, const short4* __restrict__ ytab) {
  int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  int y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x4 >= dw || y >= dh) return;
  const uint8_t* S = src + (long long)blockIdx.z * sframe;
  uint8_t* D = dst + (long long)blockIdx.z * dframe + (long long)y * dpitch;
  short4 ty = __ldg(&ytab[y]);
  const uint8_t* S0 = S + (long long)ty.x * spitch;
  const uint8_t* S1 = S + (long long)min(ty.x + 1, sh - 1) * spitch;
  int b0 = ty.y, b1 = ty.z;
  uint8_t o[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    int x = min(x4 + k, dw - 1);
    short4 tx = __ldg(&xtab[x]);
    int sx = tx.x, sx1 = min(sx + 1, sw - 1);
    int r0 = S0[sx] * tx.y + S0[sx1] * tx.z;
    int r1 = S1[sx] * tx.y + S1[sx1] * tx.z;
    o[k] = (uint8_t)((((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2);
  }
  if (x4 + 3 < dw) {
    *reinterpret_cast<uchar4*>(D + x4) = make_uchar4(o[0], o[1], o[2], o[3]);
  } else {
    for (int k = 0; x4 + k < dw; k++) D[x4 + k] = o[k];
  }
}

// ------------------------------------------------------------------------------------------------
// K2  FAST-9/16 score + strict 8-neighbour NMS + ini/min threshold choice, one CTA per cell.
// Score = largest threshold the pixel passes (OpenCV cornerScore).  Scores below minTh are stored as 0,
// which is equivalent for both thresholds (a neighbour that is not a corner counts as 0 in cv::FAST).
__host__ __device__ __forceinline__ int fast_score_px(const uint8_t* p, int pitch, int minTh) {
  int v = p[0];
  // quick reject (any 9-arc contains pixel 0 or 8 of the circle, and 4 or 12)
  int d0 = v - p[3 * pitch], d8 = v - p[-3 * pitch];
  if (abs(d0) <= minTh && abs(d8) <= minTh) return 0;
  int d4 = v - p[3], d12 = v - p[-3];
  if (abs(d4) <= minTh && abs(d12) <= minTh) return 0;
  int d[16];
  d[0] = d0; d[1] = v - p[3 * pitch + 1]; d[2] = v - p[2 * pitch + 2]; d[3] = v - p[pitch + 3];
  d[4] = d4; d[5] = v - p[-pitch + 3]; d[6] = v - p[-2 * pitch + 2]; d[7] = v - p[-3 * pitch + 1];
  d[8] = d8; d[9] = v - p[-3 * pitch - 1]; d[10] = v - p[-2 * pitch - 2]; d[11] = v - p[-pitch - 3];
  d[12] = d12; d[13] = v - p[pitch - 3]; d[14] = v - p[2 * pitch - 2]; d[15] = v - p[3 * pitch - 1];
  // NOTE: the dark side is evaluated on e = -d with min() only.  Writing it as max(mn, -mx) makes ptxas 12.9
  // fuse the negation into VIMNMX3 and drop it on sm_100a (observed: wrong scores on the device, right on host).
  int e[16];
#pragma unroll
  for (int k = 0; k < 16; k++) e[k] = -d[k];
  int a2[16], b2[16], a4[16], b4[16];
#pragma unroll
  for (int k = 0; k < 16; k++) { a2[k] = min(d[k], d[(k + 1) & 15]); b2[k] = min(e[k], e[(k + 1) & 15]); }
#pragma unroll
  for (int k = 0; k < 16; k++) { a4[k] = min(a2[k], a2[(k + 2) & 15]); b4[k] = min(b2[k], b2[(k + 2) & 15]); }
  int bestA = -256, bestB = -256;
#pragma unroll
  for (int k = 0; k < 16; k++) {
    int a9 = min(min(a4[k], a4[(k + 4) & 15]), d[(k + 8) & 15]);
    int b9 = min(min(b4[k], b4[(k + 4) & 15]), e[(k + 8) & 15]);
    bestA = max(bestA, a9);
    bestB = max(bestB, b9);
  }
  int best = bestA > bestB ? bestA : bestB;
  int s = best - 1;
  return s >= minTh ? s : 0;
}

// Two horizontally adjacent pixels per thread in the two 16-bit halves of a register (s16x2).  The 16 circle differences
// d[k] = ring[k] - centre are signed 9-bit values: they fit a half exactly, and sm_90a has single-instruction packed 16-bit
// add and 3-input min / max (VIADD.16x2, VIMNMX3.S16x2 - the DPX family), so
//   m9[k] = min(d[k .. k+8]) = min3(m3[k], m3[k+3], m3[k+6]),  m3[k] = min3(d[k], d[k+1], d[k+2])      (32 instructions)
//   M9[k] = max(d[k .. k+8]) likewise                                                                  (32 instructions)
//   bright arcs: best = max_k m9[k];  dark arcs: max_k min(-d[..]) = -min_k M9[k]                       (16 instructions)
// for BOTH pixels: no negated copy of the ring, no quick-reject pass, no compaction - every pixel of the cell costs the
// same ~85 instructions, against ~215 per surviving pixel for the scalar network (and on textured frames most pixels
// survive the 4-point pre-test).  score = max(best, -worst) - 1, stored as 0 below minTh (see fast_score_px).
__device__ __forceinline__ unsigned fast_score_pair(const uint8_t* p, int pitch, int minTh) {
  auto pair = [&](int off) { return (unsigned)p[off] | ((unsigned)p[off + 1] << 16); };
  const unsigned negv = __vneg2(pair(0));
  unsigned d[16];
  d[0] = pair(3 * pitch); d[1] = pair(3 * pitch + 1); d[2] = pair(2 * pitch + 2); d[3] = pair(pitch + 3);
  d[4] = pair(3); d[5] = pair(-pitch + 3); d[6] = pair(-2 * pitch + 2); d[7] = pair(-3 * pitch + 1);
  d[8] = pair(-3 * pitch); d[9] = pair(-3 * pitch - 1); d[10] = pair(-2 * pitch - 2); d[11] = pair(-pitch - 3);
  d[12] = pair(-3); d[13] = pair(pitch - 3); d[14] = pair(2 * pitch - 2); d[15] = pair(3 * pitch - 1);
#pragma unroll
  for (int k = 0; k < 16; k++) d[k] = __vadd2(d[k], negv);           // ring - centre, per half
  unsigned m3[16], M3[16];
#pragma unroll
  for (int k = 0; k < 16; k++) {
    m3[k] = __vimin3_s16x2(d[k], d[(k + 1) & 15], d[(k + 2) & 15]);
    M3[k] = __vimax3_s16x2(d[k], d[(k + 1) & 15], d[(k + 2) & 15]);
  }
  unsigned best = 0x80008000u, worst = 0x7fff7fffu;
#pragma unroll
  for (int k = 0; k < 16; k += 2) {
    const unsigned a0 = __vimin3_s16x2(m3[k], m3[(k + 3) & 15], m3[(k + 6) & 15]);
    const unsigned a1 = __vimin3_s16x2(m3[k + 1], m3[(k + 4) & 15], m3[(k + 7) & 15]);
    const unsigned b0 = __vimax3_s16x2(M3[k], M3[(k + 3) & 15], M3[(k + 6) & 15]);
    const unsigned b1 = __vimax3_s16x2(M3[k + 1], M3[(k + 4) & 15], M3[(k + 7) & 15]);
    best = __vimax3_s16x2(best, a0, a1);
    worst = __vimin3_s16x2(worst, b0, b1);
  }
  // per half: score = max(best, -worst) - 1 (the negation is a separate scalar subtraction: see the note in fast_score_px)
  unsigned out = 0;
#pragma unroll
  for (int hv = 0; hv < 2; hv++) {
    const int bb = (int)(short)(best >> (16 * hv)), ww = (int)(short)(worst >> (16 * hv));
    const int nw = 0 - ww;
    const int sc = (bb > nw ? bb : nw) - 1;
    out |= (unsigned)(sc >= minTh ? sc : 0) << (16 * hv);
  }
  return out;
}

// One CTA per cell.  The cell window (cell + 3 px on every side) is staged in shared memory by the TMA engine: one bulk
// asynchronous copy per window row (cp.async.bulk -> UBLKCP; 16-byte granular, so a row is fetched from the 16-byte boundary
// below the window's left edge), all rows completing ONE mbarrier; the score plane is cleared while the copies fly.  Used when
// base and pitch of the source are multiples of 16 bytes (always for the pyramid levels, for level 0 when the caller's buffer
// allows: `bulk` bit per level); otherwise a plain strided copy.  (Why rows and not one tensor tile: tma.cuh.)
constexpr int kFastPitchMax = 96;     // kMaxWin + 15 rounded up to a multiple of 16

__global__ void __launch_bounds__(128) k_fast_cells(OrbParams P, unsigned bulk, const CellInfo* __restrict__ cells,
                                                    const uint8_t* __restrict__ img0, int stride0, long long frame0,
                                                    const uint8_t* __restrict__ pyr, uint32_t* __restrict__ slots,
                                                    int* __restrict__ counts, int* __restrict__ overflow) {
  __shared__ __align__(128) uint8_t win_s[kMaxWin * kFastPitchMax];
  __shared__ __align__(16) uint8_t sc[kMaxWin * kFastPitchMax];
  __shared__ __align__(8) unsigned long long mbar;
  __shared__ int wsum[4];
  const int cell = blockIdx.x, frame = blockIdx.y, tid = threadIdx.x;
  CellInfo c = cells[cell];
  const LevelInfo& L = P.lv[c.level];
  const int w = c.x1 - c.x0, h = c.y1 - c.y0;
  const uint8_t* img;
  int pitch;
  if (c.level == 0) { img = img0 + (long long)frame * frame0; pitch = stride0; }
  else { img = pyr + (long long)frame * P.pyr_frame + L.off; pitch = L.pitch; }
  constexpr int WP = kFastPitchMax;     // shared-memory pitch of the window and of the score plane
  const uint8_t* win = win_s;
  if ((bulk >> c.level) & 1u) {
    const int x0a = c.x0 & ~15, rowbytes = ((c.x1 + 15) & ~15) - x0a;     // <= pitch - x0a: x1 <= width <= pitch, both multiples of 16
    win = win_s + (c.x0 - x0a);
    if (tid == 0) {
      tma::mbar_init(&mbar, 1);
      tma::fence_mbar_init();
      tma::mbar_expect_tx(&mbar, (unsigned)(rowbytes * h));
    }
    __syncthreads();
    if (tid < h) tma::bulk_load(win_s + tid * WP, img + (long long)(c.y0 + tid) * pitch + x0a, (unsigned)rowbytes, &mbar);
    for (int i = tid; i < (WP * h + 3) / 4; i += 128) reinterpret_cast<unsigned*>(sc)[i] = 0u;   // overlaps the copies
    tma::mbar_wait(&mbar, 0);
  } else {
    const float inv_w = 1.0f / (float)w;               // i / w for i < 72*72 without an integer division
    for (int i = tid; i < w * h; i += 128) {
      const int y = __float2int_rz(__fmul_rn((float)i + 0.5f, inv_w)), x = i - y * w;
      win_s[y * WP + x] = img[(long long)(c.y0 + y) * pitch + c.x0 + x];
    }
    for (int i = tid; i < (WP * h + 3) / 4; i += 128) reinterpret_cast<unsigned*>(sc)[i] = 0u;
  }
  __syncthreads();
  const int dw = w - 6, dh = h - 6;  // detection area
  const int npx = (dw > 0 && dh > 0) ? dw * dh : 0;
  const float inv_dw = dw > 0 ? 1.0f / (float)dw : 0.f;   // i / dw for i < 4096 without an integer division
  // scores: one thread = two adjacent pixels of a row (the second half of an odd row end is computed and dropped)
  {
    const int pw = (dw + 1) >> 1, npair = (dw > 0 && dh > 0) ? pw * dh : 0;
    const float inv_pw = pw > 0 ? 1.0f / (float)pw : 0.f;
    for (int j = tid; j < npair; j += 128) {
      const int y = __float2int_rz(__fmul_rn((float)j + 0.5f, inv_pw)), x = 2 * (j - y * pw);
      const unsigned s2 = fast_score_pair(&win[(y + 3) * WP + x + 3], WP, P.minTh);
      sc[(y + 3) * WP + x + 3] = (uint8_t)(s2 & 0xffu);
      if (x + 1 < dw) sc[(y + 3) * WP + x + 4] = (uint8_t)(s2 >> 16);
    }
  }
  __syncthreads();
  // NMS flags (0 none, 1 max>=minTh, 2 max>=iniTh)
  int n20 = 0;
  uint8_t fl[ (kMaxWin * kMaxWin + 127) / 128 ];
  int nfl = 0;
  const int ppt = (npx + 127) / 128;   // contiguous chunk per thread, row-major order
  const int beg = tid * ppt, end = min(beg + ppt, npx);
  for (int i = beg; i < end; i++) {
    int y = __float2int_rz(__fmul_rn((float)i + 0.5f, inv_dw)), x = i - y * dw;
    const uint8_t* s = &sc[(y + 3) * WP + x + 3];
    int v = s[0];
    uint8_t f = 0;
    if (v > 0 && v > s[-1] && v > s[1] && v > s[-WP - 1] && v > s[-WP] && v > s[-WP + 1] && v > s[WP - 1] &&
        v > s[WP] && v > s[WP + 1]) {
      f = (v >= P.iniTh) ? 2 : 1;
      n20 += (f == 2);
    }
    fl[nfl++] = f;
  }
  const int tot20 = __syncthreads_count(n20 > 0);
  const uint8_t need = tot20 > 0 ? 2 : 1;
  int mycount = 0;
  for (int k = 0; k < nfl; k++) mycount += (fl[k] >= need);
  // block exclusive scan of mycount
  int lane = tid & 31, wid = tid >> 5;
  int incl = mycount;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
  if (lane == 31) wsum[wid] = incl;
  __syncthreads();
  int base = 0, total = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) { if (k < wid) base += wsum[k]; total += wsum[k]; }
  int pos = base + incl - mycount;
  uint32_t* out = slots + ((long long)frame * P.ncells + cell) * P.slotcap;
  for (int k = 0; k < nfl; k++) {
    if (fl[k] >= need) {
      int i = beg + k;
      int y = __float2int_rz(__fmul_rn((float)i + 0.5f, inv_dw)), x = i - y * dw;
      if (pos < P.slotcap)
        out[pos] = (uint32_t)(x + 3 + c.sx) | ((uint32_t)(y + 3 + c.sy) << 12) | ((uint32_t)sc[(y + 3) * WP + x + 3] << 24);
      pos++;
    }
  }
  if (tid == 0) {
    counts[(long long)frame * P.ncells + cell] = min(total, P.slotcap);
    if (total > P.slotcap) atomicExch(overflow, 1);
  }
}

// ------------------------------------------------------------------------------------------------
// K3  DistributeOctTree, one warp per (frame, level).  Nodes live in shared memory as a doubly linked list
// (std::list semantics: children are pushed to the FRONT, the parent is erased); a node owns a contiguous key
// range in one of two ping-pong global buffers; DivideNode is a stable 4-way warp partition of that range.
// The reference's sort on pair<size, node pointer> is realised as (size, creation sequence) — see DESIGN.md.
struct QNode {
  short x0, y0, x1, y1;
  int beg, cnt;
  short prev, next;
  unsigned seq;
  unsigned char buf, noMore;
  short pad;
};
constexpr short QNIL = -1;

struct QState {  // per-warp bookkeeping (every lane holds identical copies; lane 0 writes shared memory)
  QNode* nodes;
  short* freel;
  int nfree;
  short head, tail;
  int size;
  unsigned seq;
};

__device__ __forceinline__ short q_alloc(QState& s) { return s.freel[--s.nfree]; }
__device__ __forceinline__ void q_free(QState& s, short id, int lane) {
  if (lane == 0) s.freel[s.nfree] = id;
  s.nfree++;
}
__device__ __forceinline__ void q_push_front(QState& s, short id, int lane) {
  if (lane == 0) {
    s.nodes[id].prev = QNIL;
    s.nodes[id].next = s.head;
    if (s.head != QNIL) s.nodes[s.head].prev = id;
  }
  if (s.head == QNIL) s.tail = id;
  s.head = id;
  s.size++;
}
__device__ __forceinline__ void q_push_back(QState& s, short id, int lane) {
  if (lane == 0) {
    s.nodes[id].next = QNIL;
    s.nodes[id].prev = s.tail;
    if (s.tail != QNIL) s.nodes[s.tail].next = id;
  }
  if (s.tail == QNIL) s.head = id;
  s.tail = id;
  s.size++;
}
__device__ __forceinline__ void q_erase(QState& s, short id, int lane) {
  short p = s.nodes[id].prev, n = s.nodes[id].next;
  __syncwarp();
  if (lane == 0) {
    if (p != QNIL) s.nodes[p].next = n;
    if (n != QNIL) s.nodes[n].prev = p;
  }
  if (p == QNIL) s.head = n;
  if (n == QNIL) s.tail = p;
  s.size--;
  q_free(s, id, lane);
  __syncwarp();
}

// Divide node `id` (ExtractorNode::DivideNode, ORBextractor.cc:481-537): children with keys are pushed to
// the list front in the order n1..n4; children with more than one key are appended to vs[] (vSizeAndPointerToNode).
__device__ void q_divide(QState& s, short id, uint32_t* kA, uint32_t* kB, short* vs, int& nv, int& nToExpand,
                         int lane) {
  QNode nd = s.nodes[id];
  const int halfX = (nd.x1 - nd.x0 + 1) >> 1;  // ceil(float(dx)/2)
  const int halfY = (nd.y1 - nd.y0 + 1) >> 1;
  const int sxp = nd.x0 + halfX, syp = nd.y0 + halfY;
  const uint32_t* src = (nd.buf ? kB : kA) + nd.beg;
  uint32_t* dst = (nd.buf ? kA : kB) + nd.beg;
  int c[4] = {0, 0, 0, 0};
  for (int i = lane; i < nd.cnt; i += 32) {
    uint32_t k = src[i];
    int kx = k & 0xfff, ky = (k >> 12) & 0xfff;
    int q = (kx < sxp) ? ((ky < syp) ? 0 : 2) : ((ky < syp) ? 1 : 3);
    c[q]++;
  }
#pragma unroll
  for (int q = 0; q < 4; q++) c[q] = warp_sum(c[q]);
  int b[4];
  b[0] = 0; b[1] = c[0]; b[2] = c[0] + c[1]; b[3] = c[0] + c[1] + c[2];
  int run[4] = {0, 0, 0, 0};
  const unsigned lt = (1u << lane) - 1u;
  for (int i0 = 0; i0 < nd.cnt; i0 += 32) {
    int i = i0 + lane;
    uint32_t k = 0;
    int q = -1;
    if (i < nd.cnt) {
      k = src[i];
      int kx = k & 0xfff, ky = (k >> 12) & 0xfff;
      q = (kx < sxp) ? ((ky < syp) ? 0 : 2) : ((ky < syp) ? 1 : 3);
    }
#pragma unroll
    for (int qq = 0; qq < 4; qq++) {
      unsigned m = __ballot_sync(0xffffffffu, q == qq);
      if (q == qq) dst[b[qq] + run[qq] + __popc(m & lt)] = k;
      run[qq] += __popc(m);
    }
  }
  __syncwarp();
  // child geometry
  short cx0[4] = {nd.x0, (short)sxp, nd.x0, (short)sxp};
  short cy0[4] = {nd.y0, nd.y0, (short)syp, (short)syp};
  short cx1[4] = {(short)sxp, nd.x1, (short)sxp, nd.x1};
  short cy1[4] = {(short)syp, (short)syp, nd.y1, nd.y1};
#pragma unroll
  for (int q = 0; q < 4; q++) {
    if (c[q] > 0) {
      short cid = q_alloc(s);
      unsigned sq = ++s.seq;
      if (lane == 0) {
        QNode& n = s.nodes[cid];
        n.x0 = cx0[q]; n.y0 = cy0[q]; n.x1 = cx1[q]; n.y1 = cy1[q];
        n.beg = nd.beg + b[q]; n.cnt = c[q];
        n.seq = sq; n.buf = nd.buf ^ 1; n.noMore = (c[q] == 1);
      }
      q_push_front(s, cid, lane);
      if (c[q] > 1) {
        nToExpand++;
        if (lane == 0) vs[nv] = cid;
        nv++;
      }
    }
  }
  __syncwarp();
}

__global__ void __launch_bounds__(32) k_quadtree(OrbParams P, const uint32_t* __restrict__ slots,
                                                 const int* __restrict__ counts, uint32_t* __restrict__ keysA,
                                                 uint32_t* __restrict__ keysB, uint32_t* __restrict__ sel,
                                                 int* __restrict__ nsel) {
  extern __shared__ unsigned char smem[];
  const int level = blockIdx.x, frame = blockIdx.y, lane = threadIdx.x;
  const LevelInfo& L = P.lv[level];
  const int pool = P.poolcap;
  QNode* nodes = reinterpret_cast<QNode*>(smem);
  unsigned long long* sortbuf = reinterpret_cast<unsigned long long*>(nodes + pool);
  short* freel = reinterpret_cast<short*>(sortbuf + P.sortcap);
  short* vs = freel + pool;
  short* order = vs + pool;
  uint32_t* kA = keysA + (long long)frame * P.key_frame + L.keyoff;
  uint32_t* kB = keysB + (long long)frame * P.key_frame + L.keyoff;
  const int N = L.nfeat;

  // gather the level's candidates from the per-cell slots in cell order (= reference push_back order)
  int n = 0;
  {
    const int* cnt = counts + (long long)frame * P.ncells + L.cell0;
    const uint32_t* sl = slots + ((long long)frame * P.ncells + L.cell0) * P.slotcap;
    for (int c0 = 0; c0 < L.ncells; c0 += 32) {
      int c = c0 + lane;
      int k = (c < L.ncells) ? cnt[c] : 0;
      int incl = k;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
      int excl = n + incl - k;
      for (int j = 0; j < k; j++) kA[excl + j] = sl[(long long)c * P.slotcap + j];
      n += __shfl_sync(0xffffffffu, incl, 31);
    }
  }
  __syncwarp();
  uint32_t* out = sel + ((long long)frame * P.nlevels + level) * P.selcap;
  if (n == 0) { if (lane == 0) nsel[frame * P.nlevels + level] = 0; return; }

  QState s;
  s.nodes = nodes; s.freel = freel; s.head = QNIL; s.tail = QNIL; s.size = 0; s.seq = 0;
  for (int i = lane; i < pool; i += 32) freel[i] = (short)(pool - 1 - i);
  s.nfree = pool;
  __syncwarp();

  // root nodes (ORBextractor.cc:543-570) and stable distribution of the keys into them
  {
    int begin = 0;
    const bool single = (L.nIni == 1);
    for (int i = 0; i < L.nIni; i++) {
      int cnt_i;
      if (single) {
        cnt_i = n;
      } else {
        // stable compaction of keys whose (int)(x / hX) == i from kA into kB
        int run = 0;
        const unsigned lt = (1u << lane) - 1u;
        for (int j0 = 0; j0 < n; j0 += 32) {
          int j = j0 + lane;
          uint32_t k = 0; bool mine = false;
          if (j < n) { k = kA[j]; mine = (__float2int_rz(__fdiv_rn((float)(k & 0xfff), L.hX)) == i); }
          unsigned m = __ballot_sync(0xffffffffu, mine);
          if (mine) kB[begin + run + __popc(m & lt)] = k;
          run += __popc(m);
        }
        cnt_i = run;
      }
      short id = q_alloc(s);
      unsigned sq = ++s.seq;
      if (lane == 0) {
        QNode& nd = nodes[id];
        nd.x0 = (short)__float2int_rz(__fmul_rn(L.hX, (float)i)); nd.y0 = 0;
        nd.x1 = (short)__float2int_rz(__fmul_rn(L.hX, (float)(i + 1))); nd.y1 = (short)L.regH;
        nd.beg = begin; nd.cnt = cnt_i; nd.seq = sq; nd.buf = single ? 0 : 1; nd.noMore = (cnt_i == 1);
      }
      q_push_back(s, id, lane);
      begin += cnt_i;
    }
    __syncwarp();
    // erase empty roots
    short it = s.head;
    while (it != QNIL) {
      short nx = nodes[it].next;
      if (nodes[it].cnt == 0) q_erase(s, it, lane);
      it = nx;
    }
  }
  __syncwarp();

  bool finish = false;
  int nv = 0;
  while (!finish) {
    int prevSize = s.size;
    int nToExpand = 0;
    nv = 0;
    short it = s.head;
    while (it != QNIL) {
      short nx = nodes[it].next;
      if (!nodes[it].noMore) {
        q_divide(s, it, kA, kB, vs, nv, nToExpand, lane);
        q_erase(s, it, lane);
      }
      it = nx;
    }
    if (s.size >= N || s.size == prevSize) {
      finish = true;
    } else if (s.size + nToExpand * 3 > N) {
      while (!finish) {
        prevSize = s.size;
        const int np = nv;
        // sort (size, seq) ascending; key = size<<48 | seq<<16 | node id
        for (int i = lane; i < np; i += 32) {
          short id = vs[i];
          sortbuf[i] = ((unsigned long long)nodes[id].cnt << 48) | ((unsigned long long)nodes[id].seq << 16) |
                       (unsigned long long)(unsigned short)id;
        }
        int np2 = 1;
        while (np2 < np) np2 <<= 1;
        for (int i = np + lane; i < np2; i += 32) sortbuf[i] = ~0ull;
        __syncwarp();
        for (int k = 2; k <= np2; k <<= 1)
          for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < np2; i += 32) {
              int ixj = i ^ j;
              if (ixj > i) {
                unsigned long long a = sortbuf[i], b2 = sortbuf[ixj];
                bool up = ((i & k) == 0);
                if ((a > b2) == up) { sortbuf[i] = b2; sortbuf[ixj] = a; }
              }
            }
            __syncwarp();
          }
        nv = 0;
        int dummy = 0;
        for (int j = np - 1; j >= 0; j--) {
          short id = (short)(sortbuf[j] & 0xffff);
          q_divide(s, id, kA, kB, vs, nv, dummy, lane);
          q_erase(s, id, lane);
          if (s.size >= N) break;
        }
        if (s.size >= N || s.size == prevSize) finish = true;
      }
    }
  }
  __syncwarp();
  // best key per node (first maximum wins), output in list order
  {
    int r = 0;
    short it = s.head;
    while (it != QNIL) { if (lane == 0) order[r] = it; r++; it = nodes[it].next; }
    __syncwarp();
    for (int i = lane; i < r && i < P.selcap; i += 32) {
      const QNode& nd = nodes[order[i]];
      const uint32_t* src = (nd.buf ? kB : kA) + nd.beg;
      uint32_t best = src[0];
      for (int k = 1; k < nd.cnt; k++) { uint32_t v = src[k]; if ((v >> 24) > (best >> 24)) best = v; }
      out[i] = best;
    }
    if (lane == 0) nsel[frame * P.nlevels + level] = min(r, P.selcap);
  }
}

// ------------------------------------------------------------------------------------------------
// K4  orientation + blur + rBRIEF + output record, one warp per selected keypoint.
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
  const float k = (float)(180.0 / 3.14159265358979323846);
  const float p1 = 0.9997878412794807f * k, p3 = -0.3258083974640975f * k;
  const float p5 = 0.1555786518463281f * k, p7 = -0.04432655554792128f * k;
  const float eps = 2.220446049250313e-16f;  // (float)DBL_EPSILON
  float ax = fabsf(x), ay = fabsf(y), a, c, c2;
  if (ax >= ay) {
    c = __fdiv_rn(ay, __fadd_rn(ax, eps));
    c2 = __fmul_rn(c, c);
    a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
  } else {
    c = __fdiv_rn(ax, __fadd_rn(ay, eps));
    c2 = __fmul_rn(c, c);
    a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
  }
  if (x < 0) a = __fsub_rn(180.f, a);
  if (y < 0) a = __fsub_rn(360.f, a);
  return a;
}

// K4a  GaussianBlur(level, 7x7, sigma 2, BORDER_REFLECT_101) of every pyramid level (ORBextractor.cc:1077-1079), once per
// level instead of once per keypoint patch: the 1000 43x43 patches of a frame cover twice the pixels of its pyramid.
// 8.8 fixed point rows [18 34 48 56 48 34 18] (sum 256), horizontal then vertical, (acc + 2^15) >> 16 — cv's
// FixedPtCast path for CV_8U.  One thread walks DOWN one column of a 64 x kBlurRows tile with the last seven horizontal
// results in registers, so every pixel costs one 7-tap row from shared memory and one 7-tap column from registers.
constexpr int kBlurCols = 64, kBlurRows = 32, kBlurTy = 4;            // block = 64 x 4 threads, tile = 64 x 128 outputs
constexpr int kBlurTileH = kBlurRows * kBlurTy, kBlurSP = kBlurCols + 8;
__global__ void __launch_bounds__(kBlurCols * kBlurTy) k_blur_level(const uint8_t* __restrict__ src, int spitch, long long sframe,
                                                                    int w, int h, uint8_t* __restrict__ dst, int dpitch, long long dframe) {
  __shared__ uint8_t raw[(kBlurTileH + 6) * kBlurSP];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int x0 = blockIdx.x * kBlurCols, y0 = blockIdx.y * kBlurTileH;
  const uint8_t* S = src + (long long)blockIdx.z * sframe;
  const int rows = min(kBlurTileH, h - y0) + 6;
  for (int r = ty; r < rows; r += kBlurTy) {
    const int yy = min(max(reflect101(y0 + r - 3, h), 0), h - 1);
    const uint8_t* row = S + (long long)yy * spitch;
    raw[r * kBlurSP + tx] = row[min(max(reflect101(x0 + tx - 3, w), 0), w - 1)];
    if (tx < 6) raw[r * kBlurSP + kBlurCols + tx] = row[min(max(reflect101(x0 + kBlurCols + tx - 3, w), 0), w - 1)];
  }
  __syncthreads();
  const int x = x0 + tx, ybeg = y0 + ty * kBlurRows;
  if (x >= w || ybeg >= h) return;
  const int nrow = min(kBlurRows, h - ybeg);
  const uint8_t* p = raw + (ty * kBlurRows) * kBlurSP + tx;
  auto hrow = [&](const uint8_t* q) { return 18 * (q[0] + q[6]) + 34 * (q[1] + q[5]) + 48 * (q[2] + q[4]) + 56 * q[3]; };
  int w0 = hrow(p), w1 = hrow(p + kBlurSP), w2 = hrow(p + 2 * kBlurSP), w3 = hrow(p + 3 * kBlurSP), w4 = hrow(p + 4 * kBlurSP),
      w5 = hrow(p + 5 * kBlurSP);
  uint8_t* D = dst + (long long)blockIdx.z * dframe + (long long)ybeg * dpitch + x;
  p += 6 * kBlurSP;
  for (int r = 0; r < nrow; r++, p += kBlurSP, D += dpitch) {
    const int w6 = hrow(p);
    const unsigned acc = 18u * (unsigned)(w0 + w6) + 34u * (unsigned)(w1 + w5) + 48u * (unsigned)(w2 + w4) + 56u * (unsigned)w3;
    *D = (uint8_t)((acc + 32768u) >> 16);
    w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; w5 = w6;
  }
}

// K4b  one warp per selected keypoint: IC_Angle on the level image (lanes = columns of the 31-wide circular patch, rows
// read coalesced), steered BRIEF on the blurred level (512 byte reads inside a 37x37 window, L1-resident).
constexpr int kDescWarps = 4;
__global__ void __launch_bounds__(32 * kDescWarps) k_describe(OrbParams P, const uint8_t* __restrict__ img0,
                                                             int stride0, long long frame0,
                                                             const uint8_t* __restrict__ pyr, const uint8_t* __restrict__ blur,
                                                             const uint32_t* __restrict__ sel,
                                                             const int* __restrict__ nsel, PLKeyPoint* __restrict__ kps,
                                                             uint8_t* __restrict__ desc, int* __restrict__ nout) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int frame = blockIdx.y;
  const int idx = blockIdx.x * kDescWarps + wid;
  // locate (level, rank) from the per-level counts
  int level = -1, rank = 0, total = 0;
  {
    int acc = 0;
    for (int l = 0; l < P.nlevels; l++) {
      int c = nsel[frame * P.nlevels + l];
      if (level < 0 && idx < acc + c) { level = l; rank = idx - acc; }
      acc += c;
    }
    total = acc;
  }
  if (idx == 0 && lane == 0) nout[frame] = total;
  if (level < 0) return;
  const LevelInfo& L = P.lv[level];
  const uint8_t* img;
  int pitch;
  if (level == 0) { img = img0 + (long long)frame * frame0; pitch = stride0; }
  else { img = pyr + (long long)frame * P.pyr_frame + L.off; pitch = L.pitch; }
  const uint32_t key = sel[((long long)frame * P.nlevels + level) * P.selcap + rank];
  const int px = (int)(key & 0xfff) + (kEdge - 3), py = (int)((key >> 12) & 0xfff) + (kEdge - 3);
  const int resp = (int)(key >> 24);
  // IC_Angle (ORBextractor.cc:76-105): m10 = sum u*I, m01 = sum v*I over |u| <= umax[|v|]; keypoints sit >= 19 px inside
  int m10, m01 = 0;
  {
    const int u = lane - kHalfPatch;
    const uint8_t* c0 = img + (long long)py * pitch + px + u;
    int colsum = 0;
#pragma unroll
    for (int v = -kHalfPatch; v <= kHalfPatch; v++) {      // fully unrolled: 31 independent row loads in flight
      if (lane <= 2 * kHalfPatch && abs(u) <= c_umax[abs(v)]) {
        const int p = c0[v * pitch];
        colsum += p; m01 += v * p;
      }
    }
    m10 = warp_sum(u * colsum);
    m01 = warp_sum(m01);
  }
  const float angle = fast_atan2_deg((float)m01, (float)m10);
  // steered BRIEF: lane computes descriptor byte `lane`
  const float factorPI = (float)(3.1415926535897932384626433832795 / 180.f);
  const float ang = __fmul_rn(angle, factorPI);
  float a = 0.f, b = 0.f;
  if (lane == 0) glibc::sincosf_(ang, &b, &a);   // the C library's sincosf, bit for bit (libm_glibc.cuh); once per keypoint
  a = __shfl_sync(0xffffffffu, a, 0); b = __shfl_sync(0xffffffffu, b, 0);
  const int bp = L.bpitch;
  const uint8_t* ctr = blur + (long long)frame * P.blur_frame + L.boff + (long long)py * bp + px;
  int val = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const char4 pt = __ldg(&g_pattern[lane * 8 + k]);
    float x0 = (float)pt.x, y0 = (float)pt.y, x1 = (float)pt.z, y1 = (float)pt.w;
    int r0 = __float2int_rn(__fadd_rn(__fmul_rn(x0, b), __fmul_rn(y0, a)));
    int c0 = __float2int_rn(__fsub_rn(__fmul_rn(x0, a), __fmul_rn(y0, b)));
    int r1 = __float2int_rn(__fadd_rn(__fmul_rn(x1, b), __fmul_rn(y1, a)));
    int c1 = __float2int_rn(__fsub_rn(__fmul_rn(x1, a), __fmul_rn(y1, b)));
    int t0 = ctr[r0 * bp + c0], t1 = ctr[r1 * bp + c1];
    val |= (t0 < t1) << k;
  }
  desc[((long long)frame * P.cap + idx) * 32 + lane] = (uint8_t)val;
  if (lane == 0) {
    PLKeyPoint kp;
    kp.x = (float)px; kp.y = (float)py;
    if (level != 0) { kp.x = __fmul_rn(kp.x, L.scale); kp.y = __fmul_rn(kp.y, L.scale); }
    kp.size = L.size; kp.angle = angle; kp.response = (float)resp; kp.octave = level; kp.class_id = -1;
    kps[(long long)frame * P.cap + idx] = kp;
  }
}

}  // namespace pl

// ================================================================================================ host side
using namespace pl;

struct PLOrb {
  PLOrbConfig cfg;
  OrbParams P;
  std::vector<float> scale, invScale, sigma2, invSigma2;
  std::vector<int> perLevel;
  std::vector<CellInfo> cells;
  cudaStream_t stream = nullptr;
  // device
  CellInfo* d_cells = nullptr;
  short4* d_tabs = nullptr;
  uint8_t* d_pyr = nullptr;
  uint8_t* d_blur = nullptr;   // blurred levels 0.. (K4a output)
  uint32_t *d_slots = nullptr, *d_keysA = nullptr, *d_keysB = nullptr, *d_sel = nullptr;
  int *d_counts = nullptr, *d_nsel = nullptr, *d_overflow = nullptr;
  // staging for the host-pointer API
  uint8_t* d_img = nullptr;
  PLKeyPoint* d_kps = nullptr;
  uint8_t* d_desc = nullptr;
  int* d_n = nullptr;
  uint8_t* h_pin = nullptr;  // pinned staging (images in, results out)
  size_t pin_bytes = 0;
  // last call (for pl_orb_get_level / debug taps)
  const uint8_t* last_img = nullptr;
  int last_stride = 0;
  long long last_frame_stride = 0;
  int last_B = 0;
  size_t quad_smem = 0;
  unsigned fast_bulk = 0;    // levels whose FAST windows are staged by bulk copies (bit 0 = level 0, decided per call)
};

static inline int cvRoundf_h(float v) { return (int)lrintf(v); }

static void build_resize_table(int s, int d, std::vector<short4>& tab) {
  double scale = (double)s / d;
  for (int i = 0; i < d; i++) {
    float f = (float)((i + 0.5) * scale - 0.5);
    int si = (int)floorf(f);
    f -= si;
    if (si < 0) { si = 0; f = 0; }
    if (si >= s - 1) { si = s - 1; f = 0; }
    short4 t;
    t.x = (short)si;
    t.y = (short)cvRoundf_h((1.f - f) * 2048);
    t.z = (short)cvRoundf_h(f * 2048);
    t.w = 0;
    tab.push_back(t);
  }
}

extern "C" int pl_orb_create(const PLOrbConfig* cfg, PLOrb** out) {
  PL_ARG(cfg && out);
  PL_ARG(cfg->width >= 64 && cfg->height >= 64 && cfg->width < 4000 && cfg->height < 4000);
  PL_ARG(cfg->nlevels >= 1 && cfg->nlevels <= kMaxLevels && cfg->nfeatures > 0 && cfg->max_batch >= 1);
  PL_ARG(cfg->scale_factor > 1.0f && cfg->min_th_fast >= 1 && cfg->ini_th_fast >= cfg->min_th_fast);
  int rc = require_device();
  if (rc) return rc;
  PLOrb* h = new PLOrb;
  h->cfg = *cfg;
  const int nl = cfg->nlevels;
  // scale tables, quotas: ORBextractor ctor (ORBextractor.cc:410-446); scaleFactor is held in a double member
  const double sf = (double)cfg->scale_factor;
  h->scale.resize(nl); h->invScale.resize(nl); h->sigma2.resize(nl); h->invSigma2.resize(nl); h->perLevel.resize(nl);
  h->scale[0] = 1.f; h->sigma2[0] = 1.f;
  for (int i = 1; i < nl; i++) { h->scale[i] = (float)(h->scale[i - 1] * sf); h->sigma2[i] = h->scale[i] * h->scale[i]; }
  for (int i = 0; i < nl; i++) { h->invScale[i] = 1.0f / h->scale[i]; h->invSigma2[i] = 1.0f / h->sigma2[i]; }
  {
    float factor = (float)(1.0f / sf);
    float nDes = cfg->nfeatures * (1 - factor) / (1 - (float)pow((double)factor, (double)nl));
    int sum = 0;
    for (int l = 0; l < nl - 1; l++) { h->perLevel[l] = cvRoundf_h(nDes); sum += h->perLevel[l]; nDes *= factor; }
    h->perLevel[nl - 1] = std::max(cfg->nfeatures - sum, 0);
  }
  int umax[16];
  {
    int v, v0, vmax = (int)floor(kHalfPatch * sqrt(2.f) / 2 + 1), vmin = (int)ceil(kHalfPatch * sqrt(2.f) / 2);
    const double hp2 = kHalfPatch * kHalfPatch;
    for (v = 0; v <= vmax; ++v) umax[v] = (int)lrint(sqrt(hp2 - v * v));
    for (v = kHalfPatch, v0 = 0; v >= vmin; --v) { while (umax[v0] == umax[v0 + 1]) ++v0; umax[v] = v0; ++v0; }
  }
  OrbParams& P = h->P;
  memset(&P, 0, sizeof(P));
  P.nlevels = nl; P.iniTh = cfg->ini_th_fast; P.minTh = cfg->min_th_fast;
  P.slotcap = cfg->cell_slot_cap > 0 ? cfg->cell_slot_cap : 128;
  P.width = cfg->width; P.height = cfg->height;
  std::vector<short4> tabs;
  long long off = 0, keyoff = 0, boff = 0;
  int maxN = 0, maxIni = 1;
  for (int l = 0; l < nl; l++) {
    LevelInfo& L = P.lv[l];
    L.w = cvRoundf_h((float)cfg->width * h->invScale[l]);
    L.h = cvRoundf_h((float)cfg->height * h->invScale[l]);
    if (L.w < 2 * kEdge + 8 || L.h < 2 * kEdge + 8) { delete h; set_error("level %d too small", l); return PL_ERR_ARG; }
    L.pitch = (L.w + 63) / 64 * 64;
    L.off = off;
    L.bpitch = L.pitch; L.boff = boff;
    boff += ((long long)L.bpitch * L.h + 255) / 256 * 256;
    if (l > 0) {
      off += (long long)L.pitch * L.h;
      off = (off + 255) / 256 * 256;
      L.tab_x = (int)tabs.size(); build_resize_table(P.lv[l - 1].w, L.w, tabs);
      L.tab_y = (int)tabs.size(); build_resize_table(P.lv[l - 1].h, L.h, tabs);
    }
    L.nfeat = h->perLevel[l];
    L.scale = h->scale[l];
    L.size = (float)(int)(31 * h->scale[l]);
    // cells: ComputeKeyPointsOctTree (ORBextractor.cc:769-806)
    const int minBX = kEdge - 3, minBY = minBX, maxBX = L.w - kEdge + 3, maxBY = L.h - kEdge + 3;
    const float width = (float)(maxBX - minBX), height = (float)(maxBY - minBY);
    const int nCols = (int)(width / 30.f), nRows = (int)(height / 30.f);
    if (nCols < 1 || nRows < 1) { delete h; set_error("level %d has no FAST cells", l); return PL_ERR_ARG; }
    const int wCell = (int)ceilf(width / nCols), hCell = (int)ceilf(height / nRows);
    if (wCell + 6 > kMaxWin || hCell + 6 > kMaxWin) { delete h; set_error("FAST cell larger than %d", kMaxWin); return PL_ERR_ARG; }
    L.cell0 = (int)h->cells.size();
    for (int i = 0; i < nRows; i++) {
      const float iniY = (float)(minBY + i * hCell);
      float maxY = iniY + hCell + 6;
      if (iniY >= maxBY - 3) continue;
      if (maxY > maxBY) maxY = (float)maxBY;
      for (int j = 0; j < nCols; j++) {
        const float iniX = (float)(minBX + j * wCell);
        float maxX = iniX + wCell + 6;
        if (iniX >= maxBX - 6) continue;
        if (maxX > maxBX) maxX = (float)maxBX;
        CellInfo c;
        c.level = (short)l; c.x0 = (short)iniX; c.x1 = (short)maxX; c.y0 = (short)iniY; c.y1 = (short)maxY;
        c.sx = (short)(j * wCell); c.sy = (short)(i * hCell); c.pad = 0;
        h->cells.push_back(c);
      }
    }
    L.ncells = (int)h->cells.size() - L.cell0;
    L.regW = maxBX - minBX; L.regH = maxBY - minBY;
    L.nIni = (int)roundf((float)L.regW / (float)L.regH);
    if (L.nIni < 1) { delete h; set_error("aspect ratio gives 0 quadtree roots (reference divides by zero)"); return PL_ERR_ARG; }
    L.hX = (float)L.regW / L.nIni;
    L.keyoff = keyoff; L.keycap = L.ncells * P.slotcap;
    keyoff += L.keycap;
    maxN = std::max(maxN, L.nfeat); maxIni = std::max(maxIni, L.nIni);
  }
  P.ncells = (int)h->cells.size();
  P.pyr_frame = off; P.key_frame = keyoff; P.blur_frame = boff;
  P.poolcap = (maxN + 4 * maxIni + 24 + 1) & ~1;
  P.selcap = maxN + 4;
  P.cap = cfg->nfeatures + 4 * nl;
  {  // bitonic sort needs a power-of-two region
    int p2 = 1; while (p2 < P.poolcap) p2 <<= 1;
    P.sortcap = p2;
    h->quad_smem = (size_t)P.poolcap * sizeof(QNode) + (size_t)p2 * 8 + (size_t)P.poolcap * 6 + 64;
  }
  const int B = cfg->max_batch;
#define ORB_TRY(e) do { int _r = (e); if (_r) { pl_orb_destroy(h); return _r; } } while (0)
#define ORB_CUDA(e) do { cudaError_t _e = (e); if (_e != cudaSuccess) { set_error("%s -> %s", #e, cudaGetErrorString(_e)); pl_orb_destroy(h); return PL_ERR_CUDA; } } while (0)
  ORB_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  static_assert(sizeof(h_pattern) == sizeof(char4) * 256, "pattern size");
  ORB_CUDA(cudaMemcpyToSymbol(g_pattern, h_pattern, sizeof(h_pattern)));
  ORB_CUDA(cudaMemcpyToSymbol(c_umax, umax, sizeof(umax)));
  ORB_TRY(dev_alloc(&h->d_cells, h->cells.size()));
  ORB_CUDA(cudaMemcpy(h->d_cells, h->cells.data(), h->cells.size() * sizeof(CellInfo), cudaMemcpyHostToDevice));
  ORB_TRY(dev_alloc(&h->d_tabs, std::max<size_t>(tabs.size(), 1)));
  if (!tabs.empty()) ORB_CUDA(cudaMemcpy(h->d_tabs, tabs.data(), tabs.size() * sizeof(short4), cudaMemcpyHostToDevice));
  ORB_TRY(dev_alloc(&h->d_pyr, (size_t)std::max<long long>(off, 256) * B));
  // FAST windows of the pyramid levels are staged by TMA bulk copies (pitch and level offsets are multiples of 64 / 256)
  h->fast_bulk = getenv("PLSLAM_NO_TMA") ? 0u : (((1u << nl) - 1u) & ~1u);
  ORB_TRY(dev_alloc(&h->d_blur, (size_t)boff * B));
  ORB_TRY(dev_alloc(&h->d_slots, (size_t)P.ncells * P.slotcap * B));
  ORB_TRY(dev_alloc(&h->d_counts, (size_t)P.ncells * B));
  ORB_TRY(dev_alloc(&h->d_keysA, (size_t)P.key_frame * B));
  ORB_TRY(dev_alloc(&h->d_keysB, (size_t)P.key_frame * B));
  ORB_TRY(dev_alloc(&h->d_sel, (size_t)P.selcap * nl * B));
  ORB_TRY(dev_alloc(&h->d_nsel, (size_t)nl * B));
  ORB_TRY(dev_alloc(&h->d_overflow, 1));
  ORB_CUDA(cudaMemset(h->d_overflow, 0, sizeof(int)));
  ORB_CUDA(cudaFuncSetAttribute(k_quadtree, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->quad_smem));
  *out = h;
  return PL_OK;
}

extern "C" void pl_orb_destroy(PLOrb* h) {
  if (!h) return;
  cudaFree(h->d_cells); cudaFree(h->d_tabs); cudaFree(h->d_pyr); cudaFree(h->d_blur); cudaFree(h->d_slots); cudaFree(h->d_counts);
  cudaFree(h->d_keysA); cudaFree(h->d_keysB); cudaFree(h->d_sel); cudaFree(h->d_nsel); cudaFree(h->d_overflow);
  cudaFree(h->d_img); cudaFree(h->d_kps); cudaFree(h->d_desc); cudaFree(h->d_n);
  if (h->h_pin) cudaFreeHost(h->h_pin);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

extern "C" int pl_orb_capacity(const PLOrb* h) { return h ? h->P.cap : PL_ERR_ARG; }

extern "C" int pl_orb_tables(const PLOrb* h, float* scale, float* inv_scale, float* sigma2, float* inv_sigma2,
                             int* features_per_level, int* level_w, int* level_h) {
  PL_ARG(h);
  for (int i = 0; i < h->P.nlevels; i++) {
    if (scale) scale[i] = h->scale[i];
    if (inv_scale) inv_scale[i] = h->invScale[i];
    if (sigma2) sigma2[i] = h->sigma2[i];
    if (inv_sigma2) inv_sigma2[i] = h->invSigma2[i];
    if (features_per_level) features_per_level[i] = h->perLevel[i];
    if (level_w) level_w[i] = h->P.lv[i].w;
    if (level_h) level_h[i] = h->P.lv[i].h;
  }
  return PL_OK;
}

extern "C" int pl_orb_extract_batch_dev(PLOrb* h, const uint8_t* imgs, int stride, size_t frame_stride, int B,
                                        PLKeyPoint* kps, uint8_t* desc, int* n, void* stream_) {
  PL_ARG(h && imgs && kps && desc && n);
  PL_ARG(B >= 1 && B <= h->cfg.max_batch && stride >= h->cfg.width);
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : h->stream;
  const OrbParams& P = h->P;
  h->last_img = imgs; h->last_stride = stride; h->last_frame_stride = (long long)frame_stride; h->last_B = B;
  for (int l = 1; l < P.nlevels; l++) {
    const LevelInfo& S = P.lv[l - 1];
    const LevelInfo& D = P.lv[l];
    const uint8_t* src = (l == 1) ? imgs : h->d_pyr + S.off;
    int spitch = (l == 1) ? stride : S.pitch;
    long long sframe = (l == 1) ? (long long)frame_stride : P.pyr_frame;
    dim3 blk(64, 4), grd((D.w + 255) / 256, (D.h + 3) / 4, B);
    k_resize_level<<<grd, blk, 0, st>>>(src, spitch, sframe, S.w, S.h, h->d_pyr + D.off, D.pitch, P.pyr_frame, D.w,
                                        D.h, h->d_tabs + D.tab_x, h->d_tabs + D.tab_y);
    PL_LAUNCH_CHECK();
  }
  // level 0 is the caller's buffer: bulk copies need its base, row pitch and frame pitch to be multiples of 16 bytes
  unsigned bulk = h->fast_bulk & ~1u;
  if (h->fast_bulk && !(((uintptr_t)imgs | (uintptr_t)stride | (uintptr_t)frame_stride) & 15)) bulk |= 1u;
  k_fast_cells<<<dim3(P.ncells, B), 128, 0, st>>>(P, bulk, h->d_cells, imgs, stride, (long long)frame_stride, h->d_pyr,
                                                  h->d_slots, h->d_counts, h->d_overflow);
  PL_LAUNCH_CHECK();
  k_quadtree<<<dim3(P.nlevels, B), 32, h->quad_smem, st>>>(P, h->d_slots, h->d_counts, h->d_keysA, h->d_keysB,
                                                           h->d_sel, h->d_nsel);
  PL_LAUNCH_CHECK();
  for (int l = 0; l < P.nlevels; l++) {
    const LevelInfo& L = P.lv[l];
    const uint8_t* src = (l == 0) ? imgs : h->d_pyr + L.off;
    k_blur_level<<<dim3((L.w + kBlurCols - 1) / kBlurCols, (L.h + kBlurTileH - 1) / kBlurTileH, B), dim3(kBlurCols, kBlurTy), 0, st>>>(
        src, (l == 0) ? stride : L.pitch, (l == 0) ? (long long)frame_stride : P.pyr_frame, L.w, L.h, h->d_blur + L.boff, L.bpitch,
        P.blur_frame);
    PL_LAUNCH_CHECK();
  }
  k_describe<<<dim3((P.cap + kDescWarps - 1) / kDescWarps, B), 32 * kDescWarps, 0, st>>>(
      P, imgs, stride, (long long)frame_stride, h->d_pyr, h->d_blur, h->d_sel, h->d_nsel, kps, desc, n);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

extern "C" int pl_orb_check_overflow(PLOrb* h) {
  PL_ARG(h);
  int ov = 0;
  PL_CUDA(cudaMemcpy(&ov, h->d_overflow, sizeof(int), cudaMemcpyDeviceToHost));
  if (ov) {
    cudaMemset(h->d_overflow, 0, sizeof(int));
    set_error("a FAST cell produced more than cell_slot_cap=%d NMS maxima", h->P.slotcap);
    return PL_ERR_CAPACITY;
  }
  return PL_OK;
}

static int orb_ensure_staging(PLOrb* h) {
  if (h->d_img) return PL_OK;
  const int B = h->cfg.max_batch;
  const size_t img_bytes = (size_t)h->cfg.width * h->cfg.height;
  int rc;
  if ((rc = dev_alloc(&h->d_img, img_bytes * B))) return rc;
  if ((rc = dev_alloc(&h->d_kps, (size_t)h->P.cap * B))) return rc;
  if ((rc = dev_alloc(&h->d_desc, (size_t)h->P.cap * 32 * B))) return rc;
  if ((rc = dev_alloc(&h->d_n, (size_t)B))) return rc;
  return PL_OK;
}

extern "C" int pl_orb_extract_batch(PLOrb* h, const uint8_t* imgs, int stride, size_t frame_stride, int B,
                                    PLKeyPoint* kps, uint8_t* desc, int* n) {
  PL_ARG(h && imgs && kps && desc && n);
  PL_ARG(B >= 1 && B <= h->cfg.max_batch && stride >= h->cfg.width);
  int rc = orb_ensure_staging(h);
  if (rc) return rc;
  const int W = h->cfg.width, H = h->cfg.height;
  for (int b = 0; b < B; b++)
    PL_CUDA(cudaMemcpy2DAsync(h->d_img + (size_t)b * W * H, W, imgs + (size_t)b * frame_stride, stride, W, H,
                              cudaMemcpyHostToDevice, h->stream));
  rc = pl_orb_extract_batch_dev(h, h->d_img, W, (size_t)W * H, B, h->d_kps, h->d_desc, h->d_n, h->stream);
  if (rc) return rc;
  const size_t cap = (size_t)h->P.cap;
  PL_CUDA(cudaMemcpyAsync(kps, h->d_kps, cap * B * sizeof(PLKeyPoint), cudaMemcpyDeviceToHost, h->stream));
  PL_CUDA(cudaMemcpyAsync(desc, h->d_desc, cap * B * 32, cudaMemcpyDeviceToHost, h->stream));
  PL_CUDA(cudaMemcpyAsync(n, h->d_n, (size_t)B * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  PL_CUDA(cudaStreamSynchronize(h->stream));
  return pl_orb_check_overflow(h);
}

extern "C" int pl_orb_extract(PLOrb* h, const uint8_t* img, int stride, PLKeyPoint* kps, uint8_t* desc, int* n) {
  return pl_orb_extract_batch(h, img, stride, 0, 1, kps, desc, n);
}

extern "C" int pl_orb_get_level(PLOrb* h, int frame, int level, uint8_t* out, int with_border) {
  PL_ARG(h && out && h->last_img && frame >= 0 && frame < h->last_B && level >= 0 && level < h->P.nlevels);
  const LevelInfo& L = h->P.lv[level];
  std::vector<uint8_t> tmp((size_t)L.w * L.h);
  PL_CUDA(cudaStreamSynchronize(h->stream));
  if (level == 0)
    PL_CUDA(cudaMemcpy2D(tmp.data(), L.w, h->last_img + (size_t)frame * h->last_frame_stride, h->last_stride, L.w,
                         L.h, cudaMemcpyDeviceToHost));
  else
    PL_CUDA(cudaMemcpy2D(tmp.data(), L.w, h->d_pyr + (size_t)frame * h->P.pyr_frame + L.off, L.pitch, L.w, L.h,
                         cudaMemcpyDeviceToHost));
  if (!with_border) { memcpy(out, tmp.data(), tmp.size()); return PL_OK; }
  const int bw = L.w + 2 * kEdge, bh = L.h + 2 * kEdge;
  auto refl = [](int p, int n) { if (p < 0) p = -p; if (p >= n) p = 2 * (n - 1) - p; return p; };
  for (int y = 0; y < bh; y++)
    for (int x = 0; x < bw; x++)
      out[(size_t)y * bw + x] = tmp[(size_t)refl(y - kEdge, L.h) * L.w + refl(x - kEdge, L.w)];
  return PL_OK;
}

extern "C" int pl_orb_debug_candidates(PLOrb* h, int frame, int level, PLKeyPoint* out, int cap) {
  PL_ARG(h && frame >= 0 && frame < h->last_B && level >= 0 && level < h->P.nlevels);
  const OrbParams& P = h->P;
  const LevelInfo& L = P.lv[level];
  std::vector<int> cnt(L.ncells);
  std::vector<uint32_t> sl((size_t)L.ncells * P.slotcap);
  PL_CUDA(cudaStreamSynchronize(h->stream));
  PL_CUDA(cudaMemcpy(cnt.data(), h->d_counts + (size_t)frame * P.ncells + L.cell0, cnt.size() * sizeof(int),
                     cudaMemcpyDeviceToHost));
  PL_CUDA(cudaMemcpy(sl.data(), h->d_slots + ((size_t)frame * P.ncells + L.cell0) * P.slotcap,
                     sl.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  int n = 0;
  for (int c = 0; c < L.ncells; c++)
    for (int j = 0; j < cnt[c]; j++) {
      uint32_t k = sl[(size_t)c * P.slotcap + j];
      if (out && n < cap) {
        PLKeyPoint kp;
        kp.x = (float)(k & 0xfff); kp.y = (float)((k >> 12) & 0xfff); kp.size = 7.f; kp.angle = -1.f;
        kp.response = (float)(k >> 24); kp.octave = 0; kp.class_id = -1;
        out[n] = kp;
      }
      n++;
    }
  return n;
}
