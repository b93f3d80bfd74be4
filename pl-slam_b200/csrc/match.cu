// Descriptor matching for batches of frames on sm_90a.
//
// Replaces (reference file:line)
//   ORBmatcher::DescriptorDistance / LSDmatcher::DescriptorDistance   ORBmatcher.cc:1764-1780, LSDmatcher.cpp:654-670
//   Frame::AssignFeaturesToGrid, PosInGrid, GetFeaturesInArea         Frame.cc:278-294, :893-903, :713-766
//   Frame::AssignFeaturesToGridForLine, GetFeaturesInAreaForLine      Frame.cc:296-320, :768-842, lineIterator.cpp
//   ORBmatcher::SearchForInitialization                               ORBmatcher.cc:455-572
//   ORBmatcher::SearchByProjection(F, LastFrame, th, mono)            ORBmatcher.cc:1441-1585
//   ORBmatcher::SearchByProjection(F, vpMapPoints, th)                ORBmatcher.cc:56-152
//   LSDmatcher::FrameBFMatch + lineDescriptorMAD + SearchDouble       LSDmatcher.cpp:440-486, :627-652
//   LSDmatcher::SearchByProjection (F,Last) / (F,vpMapLines)          LSDmatcher.cpp:72-176, :221-338
//
// The windowed searches are order dependent in the reference (a keypoint that received a match is skipped by later
// queries), so each frame is walked by ONE warp in the reference's query order; inside a query the 32 lanes scan
// the 64x48 bucket grid window and compute Hamming distances (8 x u32 xor + __popc) in parallel and the winner is
// chosen with a packed (distance, traversal order) key, which reproduces "first best wins" exactly.
// Frames of a batch are independent -> one warp (CTA) per frame, grid = B.

#include "common.cuh"
#include "search.cuh"
#include "frustum.cuh"
#include <climits>
#include <vector>

namespace pl {

constexpr int GC = 64, GR = 48, NCELL = GC * GR, HISTO = 30;

__device__ __forceinline__ int hamming256(const uint8_t* a, const uint8_t* b) {
  const uint4* pa = reinterpret_cast<const uint4*>(a);
  const uint4* pb = reinterpret_cast<const uint4*>(b);
  uint4 a0 = pa[0], a1 = pa[1], b0 = pb[0], b1 = pb[1];
  return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
         __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    unsigned long long t = __shfl_xor_sync(0xffffffffu, v, o);
    v = t < v ? t : v;
  }
  return v;
}

struct GridP { float minX, minY, maxX, maxY, invW, invH; };
__host__ __device__ inline GridP make_grid(const float* b) {
  GridP g;
  g.minX = b[0]; g.minY = b[1]; g.maxX = b[2]; g.maxY = b[3];
  g.invW = (float)GC / (g.maxX - g.minX);
  g.invH = (float)GR / (g.maxY - g.minY);
  return g;
}

// Frame::AssignFeaturesToGrid by one warp: start[NCELL+1], items[n] (stable: ascending key index inside a cell)
__device__ void build_point_grid(const PLKeyPoint* keys, int n, const GridP& g, unsigned short* start,
                                 unsigned short* fill, unsigned short* items, int lane) {
  for (int i = lane; i < NCELL; i += 32) fill[i] = 0;
  __syncwarp();
  for (int i0 = 0; i0 < n; i0 += 32) {  // counts; one chunk at a time so shared-memory updates never race
    int i = i0 + lane, c = -1;
    if (i < n) {
      int px = (int)roundf(__fmul_rn(__fsub_rn(keys[i].x, g.minX), g.invW));
      int py = (int)roundf(__fmul_rn(__fsub_rn(keys[i].y, g.minY), g.invH));
      if (px >= 0 && px < GC && py >= 0 && py < GR) c = px * GR + py;
    }
    unsigned peers = __match_any_sync(0xffffffffu, c);
    if (c >= 0 && (peers & ((1u << lane) - 1u)) == 0) fill[c] += (unsigned short)__popc(peers);
    __syncwarp();
  }
  int run = 0;
  for (int c0 = 0; c0 < NCELL; c0 += 32) {
    int v = fill[c0 + lane], incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    start[c0 + lane] = (unsigned short)(run + incl - v);
    run += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) start[NCELL] = (unsigned short)run;
  __syncwarp();
  for (int i = lane; i < NCELL; i += 32) fill[i] = 0;
  __syncwarp();
  for (int i0 = 0; i0 < n; i0 += 32) {
    int i = i0 + lane, c = -1;
    if (i < n) {
      int px = (int)roundf(__fmul_rn(__fsub_rn(keys[i].x, g.minX), g.invW));
      int py = (int)roundf(__fmul_rn(__fsub_rn(keys[i].y, g.minY), g.invH));
      if (px >= 0 && px < GC && py >= 0 && py < GR) c = px * GR + py;
    }
    unsigned peers = __match_any_sync(0xffffffffu, c);
    unsigned lt = peers & ((1u << lane) - 1u);
    if (c >= 0) items[start[c] + fill[c] + __popc(lt)] = (unsigned short)i;
    __syncwarp();
    if (c >= 0 && lt == 0) fill[c] += (unsigned short)__popc(peers);
    __syncwarp();
  }
}

struct Window { int x0, x1, y0, y1; bool ok; };
__device__ __forceinline__ Window make_window(const GridP& g, float x, float y, float r) {
  Window w;
  w.ok = false;
  w.x0 = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(x, g.minX), r), g.invW)));
  if (w.x0 >= GC) return w;
  w.x1 = min(GC - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(x, g.minX), r), g.invW)));
  if (w.x1 < 0) return w;
  w.y0 = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(y, g.minY), r), g.invH)));
  if (w.y0 >= GR) return w;
  w.y1 = min(GR - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(y, g.minY), r), g.invH)));
  if (w.y1 < 0) return w;
  w.ok = true;
  return w;
}

// key layout: dist(12) | cell rank(12) | position in cell(20) | candidate index(20)
__device__ __forceinline__ unsigned long long mk_key(int dist, int c, int j, int idx) {
  return ((unsigned long long)dist << 52) | ((unsigned long long)c << 40) | ((unsigned long long)j << 20) |
         (unsigned long long)idx;
}
constexpr unsigned long long KEY_NONE = ~0ull;
__device__ __forceinline__ int key_dist(unsigned long long k) { return (int)(k >> 52); }
__device__ __forceinline__ int key_idx(unsigned long long k) { return (int)(k & 0xfffff); }

struct Top2 { unsigned long long best, second; };

// Grids of frames with at most 2048 keypoints keep the octave (< 32) in the five high bits of each 16-bit item.
constexpr int kPackShift = 11, kPackIdMask = (1 << kPackShift) - 1, kPackMaxKeys = 1 << kPackShift;
__device__ __forceinline__ bool pack_octaves(const PLKeyPoint* keys, int n, int nitems, unsigned short* items, int lane) {
  if (n > kPackMaxKeys) return false;
  for (int j = lane; j < nitems; j += 32) {
    const int id = items[j];
    items[j] = (unsigned short)(id | ((keys[id].octave & 31) << kPackShift));
  }
  __syncwarp();
  return true;
}

// Best and second-best candidate of GetFeaturesInArea(x,y,r,minLevel,maxLevel) for query descriptor q, with a
// per-candidate skip predicate; semantics of the reference's sequential "dist<best / else dist<second" scan.
template <typename Skip>
__device__ __forceinline__ Top2 window_top2(const PLKeyPoint* keys, const uint8_t* desc, const unsigned short* start,
                                            const unsigned short* items, const GridP& g, float x, float y, float r,
                                            int minLevel, int maxLevel, const uint8_t* q, Skip skip, int lane,
                                            bool packed = false) {
  Top2 t;
  t.best = KEY_NONE; t.second = KEY_NONE;
  Window w = make_window(g, x, y, r);
  if (!w.ok) return t;
  const bool checkLevels = (minLevel > 0) || (maxLevel >= 0);
  const int ncy = w.y1 - w.y0 + 1, ncell = (w.x1 - w.x0 + 1) * ncy;
  unsigned long long k1 = KEY_NONE, k2 = KEY_NONE;
  // cell c = (c / ncy, c % ncy) of the window, advanced by 32 per trip without dividing again
  const int q32 = 32 / ncy, r32 = 32 - q32 * ncy;
  int cx = lane / ncy, cy = lane - cx * ncy;
  for (int c = lane; c < ncell; c += 32, cx += q32, cy += r32) {
    if (cy >= ncy) { cy -= ncy; cx++; }
    const int ix = w.x0 + cx, iy = w.y0 + cy;
    int cb = start[ix * GR + iy], ce = start[ix * GR + iy + 1];
    for (int j = cb; j < ce; j++) {
      const int it = items[j];
      const int id = packed ? (it & kPackIdMask) : it;
      if (checkLevels) {       // packed grids carry the octave next to the index: the level filter never touches HBM
        const int oct = packed ? (it >> kPackShift) : keys[id].octave;
        if (oct < minLevel) continue;
        if (maxLevel >= 0 && oct > maxLevel) continue;
      }
      const PLKeyPoint& kp = keys[id];
      if (!(fabsf(__fsub_rn(kp.x, x)) < r && fabsf(__fsub_rn(kp.y, y)) < r)) continue;
      int dist = hamming256(q, desc + 32 * id);
      if (skip(id, dist)) continue;
      unsigned long long k = mk_key(dist, c, j - cb, id);
      if (k < k1) { k2 = k1; k1 = k; }
      else if (k < k2) k2 = k;
    }
  }
  t.best = warp_min_u64(k1);
  t.second = warp_min_u64(k1 == t.best ? k2 : k1);
  return t;
}

// ORBmatcher::ComputeThreeMaxima on bin counts
__device__ void three_maxima(const int* cnt, int& ind1, int& ind2, int& ind3) {
  int max1 = 0, max2 = 0, max3 = 0;
  ind1 = ind2 = ind3 = -1;
  for (int i = 0; i < HISTO; i++) {
    const int s = cnt[i];
    if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
    else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
    else if (s > max3) { max3 = s; ind3 = i; }
  }
  if ((float)max2 < __fmul_rn(0.1f, (float)max1)) { ind2 = -1; ind3 = -1; }
  else if ((float)max3 < __fmul_rn(0.1f, (float)max1)) { ind3 = -1; }
}
__device__ __forceinline__ int rot_bin(float a1, float a2) {
  float rot = __fsub_rn(a1, a2);
  if (rot < 0.0f) rot = __fadd_rn(rot, 360.0f);
  int bin = (int)roundf(__fmul_rn(rot, 1.0f / HISTO));
  if (bin == HISTO) bin = 0;
  return bin;
}

struct SmemGrid {
  unsigned short* start; unsigned short* fill; unsigned short* items;
};
__device__ __forceinline__ SmemGrid carve_grid(unsigned char* smem, int cap) {
  SmemGrid s;
  s.start = reinterpret_cast<unsigned short*>(smem);
  s.fill = s.start + NCELL + 2;
  s.items = s.fill + NCELL;
  (void)cap;
  return s;
}
static size_t grid_smem_bytes(int cap) { return (size_t)(NCELL + 2 + NCELL + cap) * 2; }

// ------------------------------------------------------------------------------------------------ a18
__global__ void __launch_bounds__(32) k_assign_grid(const PLKeyPoint* keys, const int* n, int cap, const float* bounds,
                                                    int* out_start, int* out_items) {
  extern __shared__ unsigned char smem[];
  const int b = blockIdx.x, lane = threadIdx.x;
  SmemGrid sg = carve_grid(smem, cap);
  GridP g = make_grid(bounds);
  const int nn = min(n[b], cap);
  build_point_grid(keys + (long long)b * cap, nn, g, sg.start, sg.fill, sg.items, lane);
  __syncwarp();
  for (int i = lane; i <= NCELL; i += 32) out_start[(long long)b * (NCELL + 1) + i] = sg.start[i];
  for (int i = lane; i < sg.start[NCELL]; i += 32) out_items[(long long)b * cap + i] = sg.items[i];
}

// ------------------------------------------------------------------------------------------------ a15
struct SkipInit {
  const int* matchedDist;
  __device__ bool operator()(int id, int dist) const { return matchedDist[id] <= dist; }
};

__global__ void __launch_bounds__(32) k_search_init(const PLKeyPoint* keys1, const uint8_t* desc1, const int* n1,
                                                    const PLKeyPoint* keys2, const uint8_t* desc2, const int* n2,
                                                    int cap, const float* bounds, float* prev_matched, int* matches12,
                                                    int* nmatches_out, int windowSize, float nnratio, int checkOri,
                                                    int* scratch /* [B][2*cap] matchedDist, matches21 */) {
  extern __shared__ unsigned char smem[];
  __shared__ int hist[HISTO];
  const int b = blockIdx.x, lane = threadIdx.x;
  SmemGrid sg = carve_grid(smem, cap);
  GridP g = make_grid(bounds);
  const PLKeyPoint* k1 = keys1 + (long long)b * cap;
  const PLKeyPoint* k2 = keys2 + (long long)b * cap;
  const uint8_t* d1 = desc1 + (long long)b * cap * 32;
  const uint8_t* d2 = desc2 + (long long)b * cap * 32;
  const int N1 = min(n1[b], cap), N2 = min(n2[b], cap);
  float* pm = prev_matched + (long long)b * cap * 2;
  int* m12 = matches12 + (long long)b * cap;
  int* matchedDist = scratch + (long long)b * 2 * cap;
  int* m21 = matchedDist + cap;
  build_point_grid(k2, N2, g, sg.start, sg.fill, sg.items, lane);
  const bool packed = pack_octaves(k2, N2, sg.start[NCELL], sg.items, lane);
  for (int i = lane; i < N1; i += 32) m12[i] = -1;
  for (int i = lane; i < N2; i += 32) { matchedDist[i] = 0x7fffffff; m21[i] = -1; }
  if (lane < HISTO) hist[lane] = 0;
  __syncwarp();
  unsigned char* bins = reinterpret_cast<unsigned char*>(sg.fill);  // rotation bin of query i1 (255 = none); fill is free now
  for (int i = lane; i < N1; i += 32) bins[i] = 255;
  __syncwarp();
  int nmatches = 0;
  SkipInit skip{matchedDist};
  for (int i1 = 0; i1 < N1; i1++) {
    if (k1[i1].octave > 0) continue;
    Top2 t = window_top2(k2, d2, sg.start, sg.items, g, pm[2 * i1], pm[2 * i1 + 1], (float)windowSize, 0, 0,
                         d1 + 32 * i1, skip, lane, packed);
    if (t.best == KEY_NONE) continue;
    const int bestDist = key_dist(t.best), bestIdx2 = key_idx(t.best);
    const float bestDist2 = (t.second == KEY_NONE) ? 2147483648.0f : (float)key_dist(t.second);  // (float)INT_MAX
    if (bestDist <= 50 && (float)bestDist < __fmul_rn(bestDist2, nnratio)) {
      int old = m21[bestIdx2];
      __syncwarp();
      if (old >= 0) nmatches--;
      nmatches++;
      if (lane == 0) {
        if (old >= 0) m12[old] = -1;
        m12[i1] = bestIdx2;
        m21[bestIdx2] = i1;
        matchedDist[bestIdx2] = bestDist;
        if (checkOri) { int bin = rot_bin(k1[i1].angle, k2[bestIdx2].angle); bins[i1] = (unsigned char)bin; hist[bin]++; }
      }
      __syncwarp();
    }
  }
  if (checkOri) {
    int i1m, i2m, i3m;
    three_maxima(hist, i1m, i2m, i3m);
    int removed = 0;
    for (int i = lane; i < N1; i += 32) {
      int bin = bins[i];
      if (bin != 255 && bin != i1m && bin != i2m && bin != i3m && m12[i] >= 0) { m12[i] = -1; removed++; }
    }
    nmatches -= warp_sum(removed);
  }
  __syncwarp();
  for (int i = lane; i < N1; i += 32)
    if (m12[i] >= 0) { pm[2 * i] = k2[m12[i]].x; pm[2 * i + 1] = k2[m12[i]].y; }
  if (lane == 0) nmatches_out[b] = nmatches;
}

// ------------------------------------------------------------------------------------------------ a13 / a14
struct SkipAssigned {
  const int* match;
  __device__ bool operator()(int id, int) const { return match[id] != -1; }
};

struct ProjLastArgs {
  const PLKeyPoint* keys; const uint8_t* desc; const int* n; int cap;   // current frame [B][cap]
  const float* bounds; const float* Tcw; const float* K; const float* scaleFactors; int nlevels;   // Tcw [B][16], K [B][4]
  const int* n_last; int cap_last; const uint8_t* last_valid; const float* last_pos; const uint8_t* last_desc;
  const int* last_octave; const float* last_angle;
  float th; int checkOri; const uint8_t* preassigned; int* match; int* nmatches;
  // keyframe overload (ORBmatcher.cc:1587-1716, relocalisation): level from MapPoint::PredictScale(dist3D, F), no invzc < 0 test
  int kfMode = 0, maxDist = 100; const float *min_dist = nullptr, *max_dist = nullptr; float Ow[3] = {0, 0, 0}; float logSF = 1.f;
  // batched retry (Tracking.cc:1352-1357: "if(nmatches<20) { fill(mvpMapPoints, NULL); SearchByProjection(..., 2*th) }"): frame b runs
  // only if gate[b] < gate_min; the kernel re-initialises its matches, which is the fill
  const int* gate = nullptr; int gate_min = 0;
  // [B][cap_last] row of last_pos / last_desc for each last-frame keypoint (NULL: the keypoint's own [B][cap_last] row)
  const int* last_row = nullptr;
};

__global__ void __launch_bounds__(32) k_search_proj_last(ProjLastArgs A) {
  extern __shared__ unsigned char smem[];
  __shared__ int hist[HISTO];
  const int b = blockIdx.x, lane = threadIdx.x;
  if (A.gate && A.gate[b] >= A.gate_min) return;
  SmemGrid sg = carve_grid(smem, A.cap);
  GridP g = make_grid(A.bounds);
  const PLKeyPoint* kc = A.keys + (long long)b * A.cap;
  const uint8_t* dc = A.desc + (long long)b * A.cap * 32;
  const int N = min(A.n[b], A.cap), NL = min(A.n_last[b], A.cap_last);
  int* match = A.match + (long long)b * A.cap;
  const float* T = A.Tcw + 16 * b;
  const long long lb = (long long)b * A.cap_last;
  build_point_grid(kc, N, g, sg.start, sg.fill, sg.items, lane);
  const bool packed = pack_octaves(kc, N, sg.start[NCELL], sg.items, lane);
  for (int i = lane; i < N; i += 32) match[i] = (A.preassigned && A.preassigned[(long long)b * A.cap + i]) ? -2 : -1;
  if (lane < HISTO) hist[lane] = 0;
  unsigned char* bins = reinterpret_cast<unsigned char*>(sg.fill);
  __syncwarp();
  for (int i = lane; i < N; i += 32) bins[i] = 255;
  __syncwarp();
  int nmatches = 0;
  SkipAssigned skip{match};
  const float* Kb = A.K + 4 * b;      // frame b's camera ([B][4]; the host-pointer entries are B = 1)
  const float fx = Kb[0], fy = Kb[1], cx = Kb[2], cy = Kb[3];
  for (int i = 0; i < NL; i++) {
    if (!A.last_valid[lb + i]) continue;
    const long long row = A.last_row ? (long long)A.last_row[lb + i] : lb + i;
    const float* X = A.last_pos + row * 3;
    float xc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[0], X[0]), __fmul_rn(T[1], X[1])), __fmul_rn(T[2], X[2])), T[3]);
    float yc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4], X[0]), __fmul_rn(T[5], X[1])), __fmul_rn(T[6], X[2])), T[7]);
    float zc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[8], X[0]), __fmul_rn(T[9], X[1])), __fmul_rn(T[10], X[2])), T[11]);
    const float invzc = (float)(1.0 / (double)zc);
    if (!A.kfMode && invzc < 0) continue;
    float u = __fadd_rn(__fmul_rn(__fmul_rn(fx, xc), invzc), cx);
    float v = __fadd_rn(__fmul_rn(__fmul_rn(fy, yc), invzc), cy);
    if (u < g.minX || u > g.maxX) continue;
    if (v < g.minY || v > g.maxY) continue;
    int oct;
    if (A.kfMode) {
      const float p0 = __fsub_rn(X[0], A.Ow[0]), p1 = __fsub_rn(X[1], A.Ow[1]), p2 = __fsub_rn(X[2], A.Ow[2]);
      const float dist3D = (float)sqrt((double)p0 * p0 + (double)p1 * p1 + (double)p2 * p2);
      if (dist3D < __fmul_rn(0.8f, A.min_dist[lb + i]) || dist3D > __fmul_rn(1.2f, A.max_dist[lb + i])) continue;   // invariance range; PredictScale below uses the raw mfMaxDistance
      oct = predict_scale_level(A.max_dist[lb + i], dist3D, A.logSF);
      if (oct < 0) oct = 0; else if (oct >= A.nlevels) oct = A.nlevels - 1;
    } else oct = A.last_octave[lb + i];
    const float radius = __fmul_rn(A.th, A.scaleFactors[oct]);
    Top2 t = window_top2(kc, dc, sg.start, sg.items, g, u, v, radius, oct - 1, oct + 1, A.last_desc + row * 32,
                         skip, lane, packed);
    if (t.best == KEY_NONE) continue;
    const int bestDist = key_dist(t.best), bestIdx2 = key_idx(t.best);
    if (bestDist <= A.maxDist) {
      nmatches++;
      if (lane == 0) {
        match[bestIdx2] = i;
        if (A.checkOri) { int bin = rot_bin(A.last_angle[lb + i], kc[bestIdx2].angle); bins[bestIdx2] = (unsigned char)bin; hist[bin]++; }
      }
      __syncwarp();
    }
  }
  if (A.checkOri) {
    int i1m, i2m, i3m;
    three_maxima(hist, i1m, i2m, i3m);
    int removed = 0;
    for (int i = lane; i < N; i += 32) {
      int bin = bins[i];
      if (bin != 255 && bin != i1m && bin != i2m && bin != i3m) { match[i] = -1; removed++; }
    }
    nmatches -= warp_sum(removed);
  }
  if (lane == 0) A.nmatches[b] = nmatches;
}

struct ProjPointsArgs {
  const PLKeyPoint* keys; const uint8_t* desc; const int* n; int cap;
  const float* bounds; const float* scaleFactors;
  const int* n_mp; int cap_mp; const uint8_t* in_view; const float* proj; const int* level; const float* view_cos;
  const uint8_t* mp_desc; float th; float nnratio; const uint8_t* preassigned; int* match; int* nmatches;
  const float* th_frame;   // [B] per-frame th (NULL: th)
  const int* desc_row;     // [B][cap_mp] row of mp_desc for each entry (NULL: the entry's own [B][cap_mp] row)
};

__global__ void __launch_bounds__(32) k_search_proj_points(ProjPointsArgs A) {
  extern __shared__ unsigned char smem[];
  const int b = blockIdx.x, lane = threadIdx.x;
  SmemGrid sg = carve_grid(smem, A.cap);
  GridP g = make_grid(A.bounds);
  const PLKeyPoint* k = A.keys + (long long)b * A.cap;
  const uint8_t* d = A.desc + (long long)b * A.cap * 32;
  const int N = min(A.n[b], A.cap), NM = min(A.n_mp[b], A.cap_mp);
  int* match = A.match + (long long)b * A.cap;
  const long long mb = (long long)b * A.cap_mp;
  build_point_grid(k, N, g, sg.start, sg.fill, sg.items, lane);
  const bool packed = pack_octaves(k, N, sg.start[NCELL], sg.items, lane);
  for (int i = lane; i < N; i += 32) match[i] = (A.preassigned && A.preassigned[(long long)b * A.cap + i]) ? -2 : -1;
  __syncwarp();
  int nmatches = 0;
  SkipAssigned skip{match};
  const float th = A.th_frame ? A.th_frame[b] : A.th;
  const bool bFactor = th != 1.0f;
  for (int i = 0; i < NM; i++) {
    if (!A.in_view[mb + i]) continue;
    const int lvl = A.level[mb + i];
    float r = ((double)A.view_cos[mb + i] > 0.998) ? 2.5f : 4.0f;  // float vs the double literal 0.998
    if (bFactor) r = __fmul_rn(r, th);
    const long long drow = A.desc_row ? (long long)A.desc_row[mb + i] : mb + i;
    Top2 t = window_top2(k, d, sg.start, sg.items, g, A.proj[(mb + i) * 2], A.proj[(mb + i) * 2 + 1],
                         __fmul_rn(r, A.scaleFactors[lvl]), lvl - 1, lvl, A.mp_desc + drow * 32, skip, lane, packed);
    if (t.best == KEY_NONE) continue;
    const int bestDist = key_dist(t.best), bestIdx = key_idx(t.best);
    if (bestDist <= 100) {
      if (t.second != KEY_NONE) {
        const int bestDist2 = key_dist(t.second);
        if (k[bestIdx].octave == k[key_idx(t.second)].octave && (float)bestDist > __fmul_rn(A.nnratio, (float)bestDist2))
          continue;
      }
      nmatches++;
      if (lane == 0) match[bestIdx] = i;
      __syncwarp();
    }
  }
  if (lane == 0) A.nmatches[b] = nmatches;
}

// ------------------------------------------------------------------------------------------------ a16
// cv::BFMatcher(NORM_HAMMING).knnMatch(k=2): one warp per query row; ties -> lower train index.
__device__ __forceinline__ void knn2_row(const uint8_t* q, const uint8_t* train, int n2, int lane, int& i0, int& d0,
                                         int& i1, int& d1v) {
  unsigned long long k1 = KEY_NONE, k2 = KEY_NONE;
  for (int t = lane; t < n2; t += 32) {
    unsigned long long k = ((unsigned long long)hamming256(q, train + 32 * t) << 32) | (unsigned)t;
    if (k < k1) { k2 = k1; k1 = k; } else if (k < k2) k2 = k;
  }
  unsigned long long b = warp_min_u64(k1);
  unsigned long long s = warp_min_u64(k1 == b ? k2 : k1);
  i0 = b == KEY_NONE ? -1 : (int)(b & 0xffffffffu); d0 = b == KEY_NONE ? -1 : (int)(b >> 32);
  i1 = s == KEY_NONE ? -1 : (int)(s & 0xffffffffu); d1v = s == KEY_NONE ? -1 : (int)(s >> 32);
}

__global__ void __launch_bounds__(128) k_bf_knn2(const uint8_t* d1, const int* n1, const uint8_t* d2, const int* n2,
                                                 int cap1, int cap2, int* idx, int* dist) {
  const int b = blockIdx.y, lane = threadIdx.x & 31, q = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int N1 = min(n1[b], cap1), N2 = min(n2[b], cap2);
  if (q >= N1) return;
  int i0, dd0, i1, dd1;
  knn2_row(d1 + ((long long)b * cap1 + q) * 32, d2 + (long long)b * cap2 * 32, N2, lane, i0, dd0, i1, dd1);
  if (lane == 0) {
    long long o = ((long long)b * cap1 + q) * 2;
    idx[o] = i0; idx[o + 1] = i1; dist[o] = dd0; dist[o + 1] = dd1;
  }
}

// FrameBFMatch (one direction) by one CTA of 128 threads; results in shared memory (m[q] = train idx or -1).
// d12 = d1-d0 is an integer in [0,256] -> the two medians of lineDescriptorMAD come from 257-bin histograms.
__device__ void frame_bf_match_cta(const uint8_t* da, int na, const uint8_t* db, int nb, float TH, float nnratio,
                                   short* m, short* bd0, short* bd1, int* hist /*[257]*/) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int i = tid; i < na; i += 128) m[i] = -1;
  for (int i = tid; i < 257; i += 128) hist[i] = 0;
  __syncthreads();
  if (na < 1 || nb < 2) return;  // uniform
  for (int q = wid; q < na; q += 4) {
    int i0, d0, i1, d1;
    knn2_row(da + 32 * q, db, nb, lane, i0, d0, i1, d1);
    if (lane == 0) { m[q] = (short)i0; bd0[q] = (short)d0; bd1[q] = (short)d1; atomicAdd(&hist[d1 - d0], 1); }
  }
  __syncthreads();
  __shared__ int s_med, s_mad;
  if (tid == 0) {  // element na/2 of the DESCENDING sort of d12
    int need = na / 2, acc = 0, v = 256;
    for (; v >= 0; v--) { acc += hist[v]; if (acc > need) break; }
    s_med = v;
  }
  __syncthreads();
  const int med = s_med;
  for (int i = tid; i < 257; i += 128) hist[i] = 0;
  __syncthreads();
  for (int q = tid; q < na; q += 128) atomicAdd(&hist[abs((int)bd1[q] - (int)bd0[q] - med)], 1);
  __syncthreads();
  if (tid == 0) {  // element na/2 of the ASCENDING sort of |d12 - median|
    int need = na / 2, acc = 0, v = 0;
    for (; v <= 256; v++) { acc += hist[v]; if (acc > need) break; }
    s_mad = v;
  }
  __syncthreads();
  const double nn12_th = 1.4826 * (double)(float)s_mad * 0.5;  // nn12_mad * 0.5, in double as the reference
  for (int q = tid; q < na; q += 128) {
    const float d0 = (float)bd0[q], d1 = (float)bd1[q];
    const double dist_12 = (double)(d1 - d0);
    if (!(dist_12 > nn12_th && d0 < TH && d0 < __fmul_rn(nnratio, d1))) m[q] = -1;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(128) k_search_double(const uint8_t* d1, const int* n1, const uint8_t* d2,
                                                       const int* n2, int cap1, int cap2, float TH, float nnratio,
                                                       int mutual, int* matches, int* nmatches) {
  extern __shared__ unsigned char smem[];
  __shared__ int hist[257];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int N1 = min(n1[b], cap1), N2 = min(n2[b], cap2);
  short* m1 = reinterpret_cast<short*>(smem);
  short* m2 = m1 + cap1;
  short* bd0 = m2 + cap2;
  short* bd1 = bd0 + max(cap1, cap2);
  const uint8_t* a = d1 + (long long)b * cap1 * 32;
  const uint8_t* c = d2 + (long long)b * cap2 * 32;
  int* out = matches + (long long)b * cap1;
  if (N1 == 0 || N2 == 0) {
    for (int i = tid; i < N1; i += 128) out[i] = -1;
    if (tid == 0) nmatches[b] = 0;
    return;
  }
  frame_bf_match_cta(a, N1, c, N2, TH, nnratio, m1, bd0, bd1, hist);
  __syncthreads();
  if (mutual) {
    frame_bf_match_cta(c, N2, a, N1, TH, nnratio, m2, bd0, bd1, hist);
    __syncthreads();
  }
  int cnt = 0;
  for (int i = tid; i < N1; i += 128) {
    int j = m1[i];
    if (j >= 0 && mutual && m2[j] != i) j = -1;
    out[i] = j;
    cnt += (j >= 0);
  }
  __shared__ int total;
  if (tid == 0) total = 0;
  __syncthreads();
  atomicAdd(&total, cnt);
  __syncthreads();
  if (tid == 0) nmatches[b] = total;
}


// ------------------------------------------------------------------------------------------------ a17 lines
struct KeyLine68 {  // cv::line_descriptor::KeyLine (68 B)
  float angle; int class_id; int octave; float ptx, pty; float response; float size;
  float startPointX, startPointY, endPointX, endPointY, sPointInOctaveX, sPointInOctaveY, ePointInOctaveX, ePointInOctaveY;
  float lineLength; int numOfPixels;
};
constexpr int kMaxPath = GC + GR + 2;

// Frame::AssignFeaturesToGridForLine (Frame.cc:296-320 + lineIterator.cpp): CSR of mGridForLine in global scratch.
// start: [NCELL+1] ints, items: [n*kMaxPath] ushort, path scratch: [n][kMaxPath] ushort.
__device__ void build_line_grid(const KeyLine68* kl, int n, const GridP& g, int* start, unsigned short* items,
                                unsigned short* path, unsigned short* plen, int lane) {
  for (int i = lane; i <= NCELL; i += 32) start[i] = 0;
  __syncwarp();
  for (int i = lane; i < n; i += 32) {   // each lane walks its own line (Bresenham in fp64 exactly as the reference)
    double x1 = (double)__fmul_rn(kl[i].startPointX, g.invW), y1 = (double)__fmul_rn(kl[i].startPointY, g.invH);
    double x2 = (double)__fmul_rn(kl[i].endPointX, g.invW), y2 = (double)__fmul_rn(kl[i].endPointY, g.invH);
    const bool steep = fabs(y2 - y1) > fabs(x2 - x1);
    if (steep) { double t = x1; x1 = y1; y1 = t; t = x2; x2 = y2; y2 = t; }
    if (x1 > x2) { double t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
    const double dx = x2 - x1, dy = fabs(y2 - y1);
    double error = dx / 2.0;
    const int ystep = (y1 < y2) ? 1 : -1;
    int x = (int)x1, y = (int)y1;
    const int maxX = (int)x2;
    int len = 0;
    while (x <= maxX) {
      const int px = steep ? y : x, py = steep ? x : y;
      if (px >= 0 && px < GC && py >= 0 && py < GR && len < kMaxPath) { path[i * kMaxPath + len++] = (unsigned short)(px * GR + py); atomicAdd(&start[px * GR + py + 1], 1); }
      error -= dy;
      if (error < 0) { y += ystep; error += dx; }
      x++;
    }
    plen[i] = (unsigned short)len;
  }
  __syncwarp();
  int run = 0;   // inclusive scan over cells (start[c+1] holds count of cell c)
  for (int c0 = 0; c0 < NCELL; c0 += 32) {
    int v = start[c0 + lane + 1], incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    __syncwarp();
    start[c0 + lane + 1] = run + incl;
    run += __shfl_sync(0xffffffffu, incl, 31);
  }
  __syncwarp();
  // fill in ascending line index: per line, its cells are distinct -> lanes never collide; "fill" cursor = items' tail
  // kept in the ushort array `plen`-independent scratch: reuse path of processed lines is not possible, so use a
  // per-cell cursor stored in the items array header region is avoided: cursor lives in shared memory of the caller.
}

struct LineGridS { int* start; unsigned short* items; unsigned short* path; unsigned short* plen; unsigned short* cursor; };

__device__ void fill_line_grid(const LineGridS& L, int n, int lane) {
  for (int i = lane; i < NCELL; i += 32) L.cursor[i] = 0;
  __syncwarp();
  for (int i = 0; i < n; i++) {
    const int len = L.plen[i];
    for (int s = lane; s < len; s += 32) {
      const int c = L.path[i * kMaxPath + s];
      L.items[L.start[c] + L.cursor[c]] = (unsigned short)i;
      L.cursor[c]++;
    }
    __syncwarp();
  }
}

// Frame::GetFeaturesInAreaForLine: marks first[id] = traversal order key of the first accepted occurrence of line id
__device__ void line_candidates(const KeyLine68* kl, const double* lfunc, const LineGridS& L, const GridP& g, float x1, float y1,
                                float x2, float y2, float r, float TH, int* first, int n, int lane) {
  for (int i = lane; i < n; i += 32) first[i] = 0x7fffffff;
  __syncwarp();
  const float xs[3] = {x1, (float)((double)__fadd_rn(x1, x2) / 2.0), x2};
  const float ys[3] = {y1, (float)((double)__fadd_rn(y1, y2) / 2.0), y2};
  float d1x = __fsub_rn(x1, x2), d1y = __fsub_rn(y1, y2);
  const float n1 = sqrtf(__fadd_rn(__fmul_rn(d1x, d1x), __fmul_rn(d1y, d1y)));
  d1x = __fdiv_rn(d1x, n1); d1y = __fdiv_rn(d1y, n1);
  int base = 0;
  for (int i = 0; i < 3; i++) {
    Window w = make_window(g, xs[i], ys[i], r);
    if (!w.ok) continue;
    const int ncy = w.y1 - w.y0 + 1, ncell = (w.x1 - w.x0 + 1) * ncy;
    for (int c = lane; c < ncell; c += 32) {
      const int ix = w.x0 + c / ncy, iy = w.y0 + c % ncy;
      const int cb = L.start[ix * GR + iy], ce = L.start[ix * GR + iy + 1];
      for (int j = cb; j < ce; j++) {
        const int id = L.items[j];
        const KeyLine68& k = kl[id];
        float d2x = __fsub_rn(k.startPointX, k.endPointX), d2y = __fsub_rn(k.startPointY, k.endPointY);
        const float n2 = sqrtf(__fadd_rn(__fmul_rn(d2x, d2x), __fmul_rn(d2y, d2y)));
        d2x = __fdiv_rn(d2x, n2); d2y = __fdiv_rn(d2y, n2);
        const float cosSita = fabsf(__fadd_rn(__fmul_rn(d1x, d2x), __fmul_rn(d1y, d2y)));
        if (cosSita < TH) continue;
        const double* F = lfunc + 3 * id;
        const float dist = (float)(F[0] * (double)xs[i] + F[1] * (double)ys[i] + F[2]);
        // order key: probe, cell rank, slot.  A cell holds up to cap < 65536 lines, so the slot gets 16 bits; with 1024 a cell
        // crossed by more lines would sort its slot 1024 + k like slot k of the next cell
        if (fabsf(dist) < r) atomicMin(&first[id], base + c * 65536 + (j - cb));
      }
    }
    base += NCELL * 65536;   // three probes: < 2^30, clear of the distance bits of k_line_search's key
    __syncwarp();
  }
  __syncwarp();
}

struct LineSearchArgs {
  const KeyLine68* kl; const double* lfunc; const uint8_t* desc; const int* n; int cap;   // current frame [B][cap]
  const float* bounds;
  const int* n_q; int cap_q; const uint8_t* q_valid; const float* q_proj; const uint8_t* q_desc;
  const float* q_length;        // variant 0: LastFrame.mvKeylinesUn[i].lineLength
  const float* q_view_cos;      // variant 1: mTrackViewCos
  float th, nnratio; int variant;
  const uint8_t* preassigned; int* match; int* nmatches;
  int* g_start; unsigned short* g_items; unsigned short* g_path; unsigned short* g_plen; int* g_first;   // scratch per frame
  const float* th_frame;   // [B] per-frame th (NULL: th)
  const int* q_desc_row;   // [B][cap_q] row of q_desc for each query (NULL: the query's own [B][cap_q] row)
};

__global__ void __launch_bounds__(32) k_line_search(LineSearchArgs A) {
  __shared__ unsigned short cursor[NCELL];
  const int b = blockIdx.x, lane = threadIdx.x;
  GridP g = make_grid(A.bounds);
  const KeyLine68* kl = A.kl + (long long)b * A.cap;
  const double* lf = A.lfunc + (long long)b * A.cap * 3;
  const uint8_t* d = A.desc + (long long)b * A.cap * 32;
  const int N = min(A.n[b], A.cap), NQ = min(A.n_q[b], A.cap_q);
  int* match = A.match + (long long)b * A.cap;
  LineGridS L;
  L.start = A.g_start + (long long)b * (NCELL + 1); L.items = A.g_items + (long long)b * A.cap * kMaxPath;
  L.path = A.g_path + (long long)b * A.cap * kMaxPath; L.plen = A.g_plen + (long long)b * A.cap; L.cursor = cursor;
  int* first = A.g_first + (long long)b * A.cap;
  build_line_grid(kl, N, g, L.start, L.items, L.path, L.plen, lane);
  fill_line_grid(L, N, lane);
  for (int i = lane; i < N; i += 32) match[i] = (A.preassigned && A.preassigned[(long long)b * A.cap + i]) ? -2 : -1;
  __syncwarp();
  int nmatches = 0;
  const long long qb = (long long)b * A.cap_q;
  const float th = A.th_frame ? A.th_frame[b] : A.th;
  const bool bFactor = th != 1.0f;
  for (int q = 0; q < NQ; q++) {
    if (!A.q_valid[qb + q]) continue;
    const float* p = A.q_proj + (qb + q) * 4;
    float r, TH;
    if (A.variant == 0) { r = th; TH = 0.96f; }
    else { r = ((double)A.q_view_cos[qb + q] > 0.998) ? 5.0f : 8.0f; if (bFactor) r = __fmul_rn(r, th); TH = 0.998f; }
    const uint8_t* qd = A.q_desc + (A.q_desc_row ? (long long)A.q_desc_row[qb + q] : qb + q) * 32;
    line_candidates(kl, lf, L, g, p[0], p[1], p[2], p[3], r, TH, first, N, lane);
    // candidates in first-occurrence order; top-2 by (distance, order)
    unsigned long long k1 = KEY_NONE, k2 = KEY_NONE;
    for (int id = lane; id < N; id += 32) {
      const int ord = first[id];
      if (ord == 0x7fffffff) continue;
      if (match[id] != -1) continue;
      const int dist = hamming256(qd, d + 32 * id);
      if (A.variant == 0) {
        const float a = A.q_length[qb + q], c = kl[id].lineLength;
        const float mx = fmaxf(a, c), mn = fminf(a, c);
        if ((double)__fdiv_rn(mn, mx) < 0.75) continue;
      }
      const unsigned long long k = ((unsigned long long)dist << 52) | ((unsigned long long)(unsigned)ord << 20) | (unsigned long long)id;
      if (k < k1) { k2 = k1; k1 = k; } else if (k < k2) k2 = k;
    }
    const unsigned long long best = warp_min_u64(k1);
    const unsigned long long second = warp_min_u64(k1 == best ? k2 : k1);
    if (best == KEY_NONE) continue;
    const int bestDist = key_dist(best), bestIdx = key_idx(best);
    if (bestDist <= 80) {
      if (A.variant == 1 && second != KEY_NONE) {
        const int bestDist2 = key_dist(second);
        if (kl[bestIdx].octave == kl[key_idx(second)].octave && (float)bestDist > __fmul_rn(A.nnratio, (float)bestDist2)) continue;
      }
      nmatches++;
      if (lane == 0) match[bestIdx] = q;
      __syncwarp();
    }
  }
  if (lane == 0) A.nmatches[b] = nmatches;
}

// ------------------------------------------------------------------------------------------------ §8f.2 LocalMapping matchers
// Every query is independent here (one thread per KF1 keypoint / one warp per map point):
//   ORBmatcher::SearchForTriangulation   src/ORBmatcher.cc:720-911
//   ORBmatcher::Fuse (search half)       src/ORBmatcher.cc:914-1034
// DBoW2 feature vectors and the map surgery after Fuse's search are outside the path (third-party / sequential map logic).

// Status of problem blockIdx.x of a triangulation batch (PLTriProblems in plslam_b200.h), the same in every thread of the CTA:
// kf_ok(kf) checks a keyframe's counts against its capacities (status 2), items_ok(kf, t, stride) its CSR items (status 3).
template <typename KfOk, typename ItemsOk>
__device__ int tri_status(const PLTriProblems& Q, int n_kf, const int* n, KfOk kf_ok, ItemsOk items_ok) {
  const int p = blockIdx.x, k1 = Q.kf1[p], k2 = Q.kf2[p];
  if (k1 < 0 || k1 >= n_kf || k2 < 0 || k2 >= n_kf) return 1;
  if (!__syncthreads_and(kf_ok(k1, threadIdx.x, blockDim.x) && kf_ok(k2, threadIdx.x, blockDim.x))) return 2;
  const long long oo = Q.out_offset[p];
  if (oo < 0 || oo + n[k1] > Q.n_out) return 1;
  return __syncthreads_and(items_ok(k1, threadIdx.x, blockDim.x) && items_ok(k2, threadIdx.x, blockDim.x)) ? 0 : 3;
}

// Node b of the ascending list nodes[0 .. nn) that holds `node`, or -1: std::map's lower_bound.
__device__ __forceinline__ int find_node(const unsigned* nodes, int nn, unsigned node) {
  int lo = 0, hi = nn;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (nodes[mid] < node) lo = mid + 1; else hi = mid; }
  return lo < nn && nodes[lo] == node ? lo : -1;
}

// ORBmatcher::SearchForTriangulation: one CTA per problem, one thread per KF1 feature-vector item.  The reference walks the two
// node lists together with lower_bound jumps (:760-884); both hold ascending unique keys, so it visits exactly the nodes of KF1
// that KF2 also holds, and a binary search per item finds the same ones.  Every query (idx1, KF2's items of that node) is
// independent: the reference never sets vbMatched2.  The rotation histogram is a CTA-level shared-memory histogram.
struct TriBatch { PLTriKeyframes K; PLTriProblems Q; int checkOri; int *match, *nmatches, *status; };
constexpr int kTriThreads = 256;
__global__ void __launch_bounds__(kTriThreads) k_search_triangulation(const __grid_constant__ TriBatch A) {
  __shared__ int hist[HISTO];
  __shared__ int s_nm, s_keep[3];
  __shared__ float s_F[9], s_e[2];
  const PLTriKeyframes& K = A.K; const PLTriProblems& Q = A.Q;
  const int p = blockIdx.x, tid = threadIdx.x;
  const int st = tri_status(Q, K.n_kf, K.n,
    [&](int kf, int t, int stride) {
      const int n = K.n[kf], nn = K.nn[kf];
      if (n < 0 || n > K.cap || nn < 0 || nn > K.cap_nodes) return false;
      const int* s = K.fv_start + (long long)kf * (K.cap_nodes + 1);
      bool ok = t > 0 || (s[0] >= 0 && s[nn] <= n);
      for (int a = t; a < nn; a += stride) ok = ok && s[a] <= s[a + 1];
      return ok;
    },
    [&](int kf, int t, int stride) {
      const int n = K.n[kf];
      const int* s = K.fv_start + (long long)kf * (K.cap_nodes + 1);
      const int* items = K.fv_items + (long long)kf * K.cap;
      bool ok = true;
      for (int j = s[0] + t; j < s[K.nn[kf]]; j += stride) ok = ok && items[j] >= 0 && items[j] < n;
      return ok;
    });
  if (tid == 0) A.status[p] = st;
  if (st) return;
  const int k1 = Q.kf1[p], k2 = Q.kf2[p], n1 = K.n[k1], nn1 = K.nn[k1], nn2 = K.nn[k2];
  const long long r1 = (long long)k1 * K.cap, r2 = (long long)k2 * K.cap;
  const PLKeyPoint* key1 = K.keys_un + r1; const PLKeyPoint* key2 = K.keys_un + r2;
  const uint8_t* d1 = K.desc + 32 * r1; const uint8_t* d2 = K.desc + 32 * r2;
  const uint8_t* mp1 = K.has_mp + r1; const uint8_t* mp2 = K.has_mp + r2;
  const unsigned* nodes1 = K.fv_nodes + (long long)k1 * K.cap_nodes; const unsigned* nodes2 = K.fv_nodes + (long long)k2 * K.cap_nodes;
  const int* s1 = K.fv_start + (long long)k1 * (K.cap_nodes + 1); const int* s2 = K.fv_start + (long long)k2 * (K.cap_nodes + 1);
  const int* items1 = K.fv_items + r1; const int* items2 = K.fv_items + r2;
  int* match = A.match + Q.out_offset[p];
  if (tid < HISTO) hist[tid] = 0;
  if (tid < 9) s_F[tid] = Q.F12[9LL * p + tid];
  if (tid == 0) {
    s_nm = 0;
    // epipole of camera 1 in image 2 (:729-737): C2 = R2w*Cw + t2w in cv::gemm's fp32 order, every operation rounded on its own
    const float* T = K.Tcw + 16LL * k2; const float* Cw = K.Ow + 3LL * k1; const float* Kc = K.K + 4LL * k2;
    float C2[3];
    for (int i = 0; i < 3; i++)
      C2[i] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4 * i], Cw[0]), __fmul_rn(T[4 * i + 1], Cw[1])), __fmul_rn(T[4 * i + 2], Cw[2])), T[4 * i + 3]);
    const float invz = __fdiv_rn(1.0f, C2[2]);
    s_e[0] = __fadd_rn(__fmul_rn(__fmul_rn(Kc[0], C2[0]), invz), Kc[2]);
    s_e[1] = __fadd_rn(__fmul_rn(__fmul_rn(Kc[1], C2[1]), invz), Kc[3]);
  }
  for (int i = tid; i < n1; i += kTriThreads) match[i] = -1;
  __syncthreads();
  const float* F = s_F; const float ex = s_e[0], ey = s_e[1];
  for (int q = s1[0] + tid; q < s1[nn1]; q += kTriThreads) {
    int lo = 0, hi = nn1 - 1;          // the node of item q: the last a with s1[a] <= q
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (s1[mid] <= q) lo = mid; else hi = mid - 1; }
    const int b = find_node(nodes2, nn2, nodes1[lo]);
    if (b < 0) continue;
    const int idx1 = items1[q];
    if (mp1[idx1]) continue;
    const PLKeyPoint kp1 = key1[idx1];
    // epipolar line of kp1 in image 2 (CheckDistEpipolarLine, :155-172): l = x1' F12
    const float la = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, F[0]), __fmul_rn(kp1.y, F[3])), F[6]);
    const float lb = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, F[1]), __fmul_rn(kp1.y, F[4])), F[7]);
    const float lc = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, F[2]), __fmul_rn(kp1.y, F[5])), F[8]);
    const float den = __fadd_rn(__fmul_rn(la, la), __fmul_rn(lb, lb));
    int bestDist = 50, bestIdx2 = -1;
    for (int i2 = s2[b]; i2 < s2[b + 1]; i2++) {
      const int idx2 = items2[i2];
      if (mp2[idx2]) continue;
      const int dist = hamming256(d1 + 32 * idx1, d2 + 32 * idx2);
      if (dist > 50 || dist > bestDist) continue;
      const PLKeyPoint kp2 = key2[idx2];
      const float dx = __fsub_rn(ex, kp2.x), dy = __fsub_rn(ey, kp2.y);
      if (__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) < __fmul_rn(100.f, K.scale_factors[kp2.octave])) continue;
      const float num = __fadd_rn(__fadd_rn(__fmul_rn(la, kp2.x), __fmul_rn(lb, kp2.y)), lc);
      if (den == 0.f) continue;
      const float dsqr = __fdiv_rn(__fmul_rn(num, num), den);
      if ((double)dsqr < 3.84 * (double)K.level_sigma2[kp2.octave]) { bestIdx2 = idx2; bestDist = dist; }
    }
    if (bestIdx2 >= 0) {
      match[idx1] = bestIdx2;
      atomicAdd(&s_nm, 1);
      if (A.checkOri) atomicAdd(&hist[rot_bin(kp1.angle, key2[bestIdx2].angle)], 1);
    }
  }
  __syncthreads();
  if (A.checkOri) {
    if (tid == 0) { int a, b, c; three_maxima(hist, a, b, c); s_keep[0] = a; s_keep[1] = b; s_keep[2] = c; }
    __syncthreads();
    for (int i = tid; i < n1; i += kTriThreads) {
      const int j = match[i];
      if (j < 0) continue;
      const int bin = rot_bin(key1[i].angle, key2[j].angle);
      if (bin != s_keep[0] && bin != s_keep[1] && bin != s_keep[2]) { match[i] = -1; atomicSub(&s_nm, 1); }
    }
    __syncthreads();
  }
  if (tid == 0) A.nmatches[p] = s_nm;
}

// LSDmatcher::SearchForTriangulation (src/LSDmatcher.cpp:727-776): k_search_double for P (KF1, KF2) problems of a keyframe table,
// then the pairs whose line already has a MapLine on either side are dropped (:756).  Shared memory is laid out on the problem's
// own counts, m1[N1], m2[N2], bd0 and bd1[max(N1, N2)], inside what the launch reserves for its largest problem.
struct LineTriBatch { PLTriLineKeyframes K; PLTriProblems Q; float th, nnratio; int mutual; int *match, *nmatches, *status; };
__global__ void __launch_bounds__(128) k_lsd_search_triangulation(const __grid_constant__ LineTriBatch A) {
  extern __shared__ unsigned char smem[];
  __shared__ int hist[257];
  __shared__ int total;
  const PLTriLineKeyframes& K = A.K; const PLTriProblems& Q = A.Q;
  const int p = blockIdx.x, tid = threadIdx.x;
  const int st = tri_status(Q, K.n_kf, K.n, [&](int kf, int, int) { return K.n[kf] >= 0 && K.n[kf] <= K.cap; },
                            [](int, int, int) { return true; });
  if (tid == 0) A.status[p] = st;
  if (st) return;
  const int k1 = Q.kf1[p], k2 = Q.kf2[p], N1 = K.n[k1], N2 = K.n[k2];
  const uint8_t* a = K.ldesc + 32LL * k1 * K.cap; const uint8_t* c = K.ldesc + 32LL * k2 * K.cap;
  const uint8_t* ml1 = K.has_ml + (long long)k1 * K.cap; const uint8_t* ml2 = K.has_ml + (long long)k2 * K.cap;
  int* out = A.match + Q.out_offset[p];
  if (N1 == 0 || N2 == 0) {     // ldesc.rows == 0 -> return 0 (:738-739)
    for (int i = tid; i < N1; i += 128) out[i] = -1;
    if (tid == 0) A.nmatches[p] = 0;
    return;
  }
  short* m1 = reinterpret_cast<short*>(smem);
  short* m2 = m1 + N1;
  short* bd0 = m2 + N2;
  short* bd1 = bd0 + max(N1, N2);
  frame_bf_match_cta(a, N1, c, N2, A.th, A.nnratio, m1, bd0, bd1, hist);
  __syncthreads();
  if (A.mutual) {
    frame_bf_match_cta(c, N2, a, N1, A.th, A.nnratio, m2, bd0, bd1, hist);
    __syncthreads();
  }
  int cnt = 0;
  for (int i = tid; i < N1; i += 128) {
    int j = m1[i];
    if (j >= 0 && ((A.mutual && m2[j] != i) || ml1[i] || ml2[j])) j = -1;
    out[i] = j;
    cnt += (j >= 0);
  }
  if (tid == 0) total = 0;
  __syncthreads();
  atomicAdd(&total, cnt);
  __syncthreads();
  if (tid == 0) A.nmatches[p] = total;
}

struct SkipChi2 {
  const PLKeyPoint* k; const float* inv; float u, v;
  __device__ bool operator()(int id, int) const {
    const float ex = __fsub_rn(u, k[id].x), ey = __fsub_rn(v, k[id].y);
    const float e2 = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey));
    return (double)__fmul_rn(e2, inv[k[id].octave]) > 5.99;
  }
};

// Status of problem blockIdx.x of a Fuse batch (PLFuseProblems in plslam_b200.h), the same in every thread of the CTA: kf_ok(kf)
// checks the keyframe's counts against its capacities.
template <typename KfOk>
__device__ int fuse_status(const PLFuseProblems& Q, int n_kf, int n_lm, KfOk kf_ok) {
  const int p = blockIdx.x, kf = Q.kf[p];
  const long long o = Q.offset[p], c = Q.count[p], oo = Q.out_offset[p];
  if (kf < 0 || kf >= n_kf || o < 0 || c < 0 || o + c > Q.n_entries || oo < 0 || oo + c > Q.n_out) return 1;
  if (!kf_ok(kf)) return 2;
  bool ok = true;
  for (long long j = threadIdx.x; j < c; j += blockDim.x) { const int m = Q.entry_lm[o + j]; ok = ok && m >= 0 && m < n_lm; }
  return __syncthreads_and(ok) ? 0 : 3;
}
// The camera of problem blockIdx.x's keyframe in shared memory: Tcw, Ow, K, bounds.
struct FuseCam { float T[16], Ow[3], K[4], bounds[4]; };
__device__ void load_fuse_cam(FuseCam& c, const float* Tcw, const float* Ow, const float* K, const float* bounds, int kf) {
  const int t = threadIdx.x;
  if (t < 16) c.T[t] = Tcw[16LL * kf + t];
  else if (t < 19) c.Ow[t - 16] = Ow[3LL * kf + t - 16];
  else if (t < 23) c.K[t - 19] = K[4LL * kf + t - 19];
  else if (t < 27) c.bounds[t - 23] = bounds[4LL * kf + t - 23];
}

// ORBmatcher::Fuse, search half: one CTA per problem.  Warp 0 builds the keyframe's bucket grid in shared memory, then the
// problem's map points run one per warp.
struct FuseBatch { PLFuseKeyframes K; PLFusePoints L; PLFuseProblems Q; int *best_idx, *best_dist, *status; };
constexpr int kFuseWarps = 16;
__global__ void __launch_bounds__(32 * kFuseWarps) k_fuse_search(const __grid_constant__ FuseBatch A) {
  extern __shared__ unsigned char smem[];
  __shared__ FuseCam cam;
  __shared__ int s_packed;
  const PLFuseKeyframes& K = A.K; const PLFusePoints& L = A.L; const PLFuseProblems& Q = A.Q;
  const int p = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int st = fuse_status(Q, K.n_kf, L.n, [&](int kf) { return K.n[kf] >= 0 && K.n[kf] <= K.cap; });
  if (threadIdx.x == 0) A.status[p] = st;
  if (st) return;
  const int kf = Q.kf[p], n = K.n[kf], cnt = Q.count[p];
  const long long o = Q.offset[p], oo = Q.out_offset[p], row = (long long)kf * K.cap;
  const PLKeyPoint* keys = K.keys_un + row;
  const uint8_t* desc = K.desc + 32 * row;
  const float th = Q.th[p];
  load_fuse_cam(cam, K.Tcw, K.Ow, K.K, K.bounds, kf);
  __syncthreads();
  SmemGrid sg = carve_grid(smem, K.cap);
  const GridP g = make_grid(cam.bounds);
  if (wid == 0) {
    build_point_grid(keys, n, g, sg.start, sg.fill, sg.items, lane);
    const bool pk = pack_octaves(keys, n, sg.start[NCELL], sg.items, lane);
    if (lane == 0) s_packed = pk;
  }
  __syncthreads();
  const bool packed = s_packed != 0;
  const float* T = cam.T; const float* Ow = cam.Ow; const float* Kc = cam.K; const float* bounds = cam.bounds;
  for (int j = wid; j < cnt; j += kFuseWarps) {
    const long long i = Q.entry_lm[o + j];
    int bi = -1, bd = 256;
    bool go = !Q.entry_skip[o + j];
    float u = 0.f, v = 0.f; int lvl = 0;
    if (go) {
      const float P[3] = {L.pos[3 * i], L.pos[3 * i + 1], L.pos[3 * i + 2]};
      float Pc[3];
      for (int r = 0; r < 3; r++)
        Pc[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4 * r], P[0]), __fmul_rn(T[4 * r + 1], P[1])), __fmul_rn(T[4 * r + 2], P[2])), T[4 * r + 3]);
      go = !(Pc[2] < 0.0f);
      if (go) {
        const float invz = __fdiv_rn(1.0f, Pc[2]);
        u = __fadd_rn(__fmul_rn(Kc[0], __fmul_rn(Pc[0], invz)), Kc[2]);
        v = __fadd_rn(__fmul_rn(Kc[1], __fmul_rn(Pc[1], invz)), Kc[3]);
        go = (u >= bounds[0] && u < bounds[2] && v >= bounds[1] && v < bounds[3]);     // KeyFrame::IsInImage
      }
      if (go) {
        const float PO[3] = {__fsub_rn(P[0], Ow[0]), __fsub_rn(P[1], Ow[1]), __fsub_rn(P[2], Ow[2])};
        const float dist3D = (float)sqrt((double)PO[0] * PO[0] + (double)PO[1] * PO[1] + (double)PO[2] * PO[2]);
        go = !(dist3D < __fmul_rn(0.8f, L.min_dist[i]) || dist3D > __fmul_rn(1.2f, L.max_dist[i]));
        if (go) {
          const double dot = (double)PO[0] * L.normal[3 * i] + (double)PO[1] * L.normal[3 * i + 1] + (double)PO[2] * L.normal[3 * i + 2];
          go = !(dot < 0.5 * (double)dist3D);
          lvl = predict_scale_level(L.max_dist[i], dist3D, K.log_scale_factor);
          if (lvl < 0) lvl = 0; else if (lvl >= K.nlevels) lvl = K.nlevels - 1;
        }
      }
    }
    if (go) {     // warp-uniform: every lane computed the same scalars
      SkipChi2 skip{keys, K.inv_level_sigma2, u, v};
      const Top2 t = window_top2(keys, desc, sg.start, sg.items, g, u, v, __fmul_rn(th, K.scale_factors[lvl]), lvl - 1, lvl,
                                 L.desc + 32 * i, skip, lane, packed);
      if (t.best != KEY_NONE) { bi = key_idx(t.best); bd = key_dist(t.best); }
    }
    if (lane == 0) { A.best_idx[oo + j] = bi; A.best_dist[oo + j] = bd; }
  }
}

// ORBmatcher::SearchByBoW(pKF, F, vpMapPointMatches) (src/ORBmatcher.cc:187-327).  A frame feature lives in exactly one
// vocabulary node, so the "already matched" state couples only the keyframe features of the same node: one warp walks one
// common node in the reference's order (keyframe features sequentially, the node's frame features across the lanes, packed
// (distance, position) key for "first best wins", second = minimum over the rest), the nodes run in parallel.
struct BowArgs {
  const PLKeyPoint *kK, *kF; const uint8_t *dK, *dF, *mpK;
  const int *pairK_s, *pairK_e, *pairF_s, *pairF_e, *itK, *itF; int npairs, nF;
  float nnratio; int checkOri;
  int* matchesF; unsigned char* bins; int* nmatches;
  const uint8_t* mpF = nullptr;    // KeyFrame-KeyFrame overload (:574-709): candidates need a MapPoint too ...
  int strict = 0;                  // ... and the gate is bestDist1 < TH_LOW instead of <=
};
constexpr int kBowWarps = 16;
__global__ void __launch_bounds__(32 * kBowWarps) k_search_by_bow(BowArgs A) {
  __shared__ int hist[HISTO];
  __shared__ int s_nm, s_keep[3];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid < HISTO) hist[tid] = 0;
  if (tid == 0) s_nm = 0;
  for (int j = tid; j < A.nF; j += blockDim.x) { A.matchesF[j] = -1; A.bins[j] = 255; }
  __syncthreads();
  for (int p = wid; p < A.npairs; p += kBowWarps) {
    const int fs = A.pairF_s[p], fe = A.pairF_e[p];
    for (int iK = A.pairK_s[p]; iK < A.pairK_e[p]; iK++) {
      const int idxK = A.itK[iK];
      if (!A.mpK[idxK]) continue;
      unsigned long long k1 = KEY_NONE, k2 = KEY_NONE;
      for (int c = fs + lane; c < fe; c += 32) {
        const int idxF = A.itF[c];
        if (A.matchesF[idxF] >= 0) continue;
        if (A.mpF && !A.mpF[idxF]) continue;
        const int dist = hamming256(A.dK + 32 * idxK, A.dF + 32 * idxF);
        const unsigned long long k = mk_key(dist, 0, c - fs, idxF);
        if (k < k1) { k2 = k1; k1 = k; } else if (k < k2) k2 = k;
      }
      const unsigned long long best = warp_min_u64(k1);
      const unsigned long long second = warp_min_u64(k1 == best ? k2 : k1);
      if (best == KEY_NONE) continue;
      const int bestDist1 = key_dist(best), bestIdxF = key_idx(best);
      const int bestDist2 = (second == KEY_NONE) ? 256 : key_dist(second);
      if ((A.strict ? bestDist1 < 50 : bestDist1 <= 50) && (float)bestDist1 < __fmul_rn(A.nnratio, (float)bestDist2)) {
        if (lane == 0) {
          A.matchesF[bestIdxF] = idxK;
          atomicAdd(&s_nm, 1);
          if (A.checkOri) { const int bin = rot_bin(A.kK[idxK].angle, A.kF[bestIdxF].angle); A.bins[bestIdxF] = (unsigned char)bin; atomicAdd(&hist[bin], 1); }
        }
        __syncwarp();
      }
    }
  }
  __syncthreads();
  if (A.checkOri) {
    if (tid == 0) { int a, b, c; three_maxima(hist, a, b, c); s_keep[0] = a; s_keep[1] = b; s_keep[2] = c; }
    __syncthreads();
    for (int j = tid; j < A.nF; j += blockDim.x) {
      const int bin = A.bins[j];
      if (bin != 255 && bin != s_keep[0] && bin != s_keep[1] && bin != s_keep[2]) { A.matchesF[j] = -1; atomicSub(&s_nm, 1); }
    }
    __syncthreads();
  }
  if (tid == 0) *A.nmatches = s_nm;
}
}  // namespace pl

// ================================================================================================ C ABI
using namespace pl;

// ------------------------------------------------------------------------------------------------ MapPoint descriptor choice
// MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:249-314): one warp per map point.  For every descriptor i of the
// point the lanes compute the distances to all N descriptors into a 257-bin histogram in shared memory; the median
// sorted[int(0.5 * (N - 1))] is the bin where the running count passes that rank (distances are integers in [0, 256]).
constexpr int kDistWarps = 4;
__global__ void __launch_bounds__(32 * kDistWarps) k_distinctive(const uint8_t* __restrict__ desc, const int* __restrict__ offsets, int n_mp,
                                                                 int* __restrict__ best, uint8_t* __restrict__ out_desc) {
  __shared__ int hist[kDistWarps][264];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, m = blockIdx.x * kDistWarps + wid;
  if (m >= n_mp) return;
  const int o0 = offsets[m], N = offsets[m + 1] - o0;
  if (N <= 0) { if (lane == 0) best[m] = -1; return; }
  const uint8_t* d = desc + (long long)o0 * 32;
  int* h = hist[wid];
  const int rank = (int)(0.5 * (double)(N - 1));
  int bestMedian = 0x7fffffff, bestIdx = 0;
  for (int i = 0; i < N; i++) {
    for (int k = lane; k < 257; k += 32) h[k] = 0;
    __syncwarp();
    for (int j = lane; j < N; j += 32) atomicAdd(&h[(i == j) ? 0 : hamming256(d + 32 * i, d + 32 * j)], 1);
    __syncwarp();
    // first bin whose inclusive prefix count exceeds `rank`
    int median = 256, run = 0;
    for (int k0 = 0; k0 < 257 + 31; k0 += 32) {
      const int k = k0 + lane;
      const int c = (k < 257) ? h[k] : 0;
      int incl = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
      const unsigned hit = __ballot_sync(0xffffffffu, run + incl > rank);
      if (hit) { median = k0 + __ffs(hit) - 1; break; }
      run += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (median < bestMedian) { bestMedian = median; bestIdx = i; }
    __syncwarp();
  }
  if (lane == 0) best[m] = bestIdx;
  if (out_desc) out_desc[(long long)m * 32 + lane] = d[32 * bestIdx + lane];
}

// ------------------------------------------------------------------------------------------------ LSDmatcher::Fuse, search half
// End points of a map line (pos: start, end as doubles) in the world, as the reference's floats, and in the camera.
__device__ __forceinline__ void line_ends(const float* T, const double* pos, float SP[3], float EP[3], float S[3], float E[3]) {
#pragma unroll
  for (int k = 0; k < 3; k++) { SP[k] = (float)pos[k]; EP[k] = (float)pos[3 + k]; }
#pragma unroll
  for (int r = 0; r < 3; r++) {
    S[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4 * r], SP[0]), __fmul_rn(T[4 * r + 1], SP[1])), __fmul_rn(T[4 * r + 2], SP[2])), T[4 * r + 3]);
    E[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4 * r], EP[0]), __fmul_rn(T[4 * r + 1], EP[1])), __fmul_rn(T[4 * r + 2], EP[2])), T[4 * r + 3]);
  }
}
// Best keyline of the keyframe for map line i (in front of the camera); bestIdx / bestDist keep -1 / 256 when nothing qualifies.
__device__ void line_fuse_one(const FuseCam& cam, const KeyLine68* kls, int nl, const uint8_t* pdesc, int n_pdesc, float scale_line,
                              float logScaleFactorLine, const PLFuseLines& L, long long i, float th, int& bestIdx, int& bestDist) {
  const float* Kc = cam.K; const float* bounds = cam.bounds;
  float SP[3], EP[3], S[3], E[3];
  line_ends(cam.T, L.pos + 6 * i, SP, EP, S, E);
  const float invz1 = __fdiv_rn(1.0f, S[2]);
  const float u1 = __fadd_rn(__fmul_rn(__fmul_rn(Kc[0], S[0]), invz1), Kc[2]), v1 = __fadd_rn(__fmul_rn(__fmul_rn(Kc[1], S[1]), invz1), Kc[3]);
  if (!(u1 >= bounds[0] && u1 < bounds[2] && v1 >= bounds[1] && v1 < bounds[3])) return;
  const float invz2 = __fdiv_rn(1.0f, E[2]);
  const float u2 = __fadd_rn(__fmul_rn(__fmul_rn(Kc[0], E[0]), invz2), Kc[2]), v2 = __fadd_rn(__fmul_rn(__fmul_rn(Kc[1], E[1]), invz2), Kc[3]);
  if (!(u2 >= bounds[0] && u2 < bounds[2] && v2 >= bounds[1] && v2 < bounds[3])) return;
  float OM[3];
#pragma unroll
  for (int k = 0; k < 3; k++) OM[k] = __fsub_rn((float)(0.5 * (double)__fadd_rn(SP[k], EP[k])), cam.Ow[k]);
  const float dist = (float)sqrt((double)OM[0] * OM[0] + (double)OM[1] * OM[1] + (double)OM[2] * OM[2]);
  if (dist < __fmul_rn(0.8f, L.min_dist[i]) || dist > __fmul_rn(1.2f, L.max_dist[i])) return;
  const float pn[3] = {(float)L.normal[3 * i], (float)L.normal[3 * i + 1], (float)L.normal[3 * i + 2]};
  const double dot = (double)OM[0] * pn[0] + (double)OM[1] * pn[1] + (double)OM[2] * pn[2];
  if (dot < 0.5 * (double)dist) return;
  const int lvl = predict_scale_level(L.max_dist[i], dist, logScaleFactorLine);
  float sf = 1.0f;
  if (lvl >= 0) { for (int k = 0; k < lvl; k++) sf = __fmul_rn(sf, scale_line); }
  else { for (int k = 0; k < -lvl; k++) sf = __fmul_rn(sf, scale_line); sf = __fdiv_rn(1.0f, sf); }
  const float radius = __fmul_rn(th, sf), r2 = __fmul_rn(radius, radius);
  float d1x = __fsub_rn(u1, u2), d1y = __fsub_rn(v1, v2);
  const float n1 = __fsqrt_rn(__fadd_rn(__fmul_rn(d1x, d1x), __fmul_rn(d1y, d1y)));
  d1x = __fdiv_rn(d1x, n1); d1y = __fdiv_rn(d1y, n1);
  const double mxd = 0.5 * (double)__fadd_rn(u1, u2), myd = 0.5 * (double)__fadd_rn(v1, v2);
  const uint8_t* q = L.desc + 32 * i;
  for (int j = 0; j < nl; j++) {
    const KeyLine68& kl = kls[j];
    const double ax = mxd - (double)kl.ptx, ay = myd - (double)kl.pty;
    const float distance = (float)(ax * ax + ay * ay);
    if (distance > r2) continue;
    float d2x = __fsub_rn(kl.startPointX, kl.endPointX), d2y = __fsub_rn(kl.startPointY, kl.endPointY);
    const float n2 = __fsqrt_rn(__fadd_rn(__fmul_rn(d2x, d2x), __fmul_rn(d2y, d2y)));
    d2x = __fdiv_rn(d2x, n2); d2y = __fdiv_rn(d2y, n2);
    const float cs = fabsf(__fadd_rn(__fmul_rn(d1x, d2x), __fmul_rn(d1y, d2y)));
    if (cs < 0.998f) continue;
    if (kl.octave < lvl - 1 || kl.octave > lvl) continue;
    if (j >= n_pdesc) continue;
    const int d = hamming256(q, pdesc + 32 * (long long)j);
    if (d < bestDist) { bestDist = d; bestIdx = j; }
  }
}
struct LineFuseBatch { PLFuseLineKeyframes K; PLFuseLines L; PLFuseProblems Q; int *best_idx, *best_dist, *stop_at, *status; };
// One CTA per problem, one thread per map line (a keyframe has at most a few hundred lines; every candidate test is a handful of
// flops).  Quirks of the reference are listed at pl_lsd_fuse_search (plslam_b200.h) and restated in oracle_lsd_fuse_search.
constexpr int kLineFuseThreads = 128;
__global__ void __launch_bounds__(kLineFuseThreads) k_lsd_fuse_search(const __grid_constant__ LineFuseBatch A) {
  __shared__ FuseCam cam;
  __shared__ int s_stop;
  const PLFuseLineKeyframes& K = A.K; const PLFuseLines& L = A.L; const PLFuseProblems& Q = A.Q;
  const int p = blockIdx.x, tid = threadIdx.x;
  const int st = fuse_status(Q, K.n_kf, L.n, [&](int kf) {
    return K.n[kf] >= 0 && K.n[kf] <= K.cap && K.n_pdesc[kf] >= 0 && K.n_pdesc[kf] <= K.cap_pdesc;
  });
  if (tid == 0) A.status[p] = st;
  if (st) return;
  const int kf = Q.kf[p], nl = K.n[kf], n_pdesc = K.n_pdesc[kf], cnt = Q.count[p];
  const long long o = Q.offset[p], oo = Q.out_offset[p];
  const KeyLine68* kls = reinterpret_cast<const KeyLine68*>(K.keylines) + (long long)kf * K.cap;
  const uint8_t* pdesc = K.pdesc + 32LL * kf * K.cap_pdesc;
  const float th = Q.th[p];
  load_fuse_cam(cam, K.Tcw, K.Ow, K.K, K.bounds, kf);
  if (tid == 0) s_stop = cnt;
  __syncthreads();
  // the first map line with an end point behind the camera ends the reference's loop (`return false`, :907)
  for (int j = tid; j < cnt; j += kLineFuseThreads) {
    if (Q.entry_skip[o + j]) continue;
    float SP[3], EP[3], S[3], E[3];
    line_ends(cam.T, L.pos + 6LL * Q.entry_lm[o + j], SP, EP, S, E);
    if (S[2] < 0.0f || E[2] < 0.0f) atomicMin(&s_stop, j);
  }
  __syncthreads();
  const int stop = s_stop;
  if (tid == 0) A.stop_at[p] = stop;
  for (int j = tid; j < cnt; j += kLineFuseThreads) {
    int bestIdx = -1, bestDist = 256;
    if (j < stop && !Q.entry_skip[o + j])
      line_fuse_one(cam, kls, nl, pdesc, n_pdesc, K.scale_line, K.log_scale_factor_line, L, Q.entry_lm[o + j], th, bestIdx, bestDist);
    A.best_idx[oo + j] = bestIdx; A.best_dist[oo + j] = bestDist;
  }
}

extern "C" int pl_descriptor_distance_batch(const uint8_t* a, const uint8_t* b, int n, int* out) {
  // convenience for tests: n independent 32-byte pairs, host pointers
  PL_ARG(a && b && out && n >= 0);
  int rc = require_device(); if (rc) return rc;
  Staging s;
  uint8_t* da = s.in(a, (size_t)n * 32); uint8_t* db = s.in(b, (size_t)n * 32);
  // reuse k_bf_knn2 with cap2 = 1 per pair would be wasteful; do pairs as n batches of 1x1
  std::vector<int> ones(n, 1), hd((size_t)n * 2);
  int* dn = s.in(ones.data(), (size_t)n);
  int* idx = s.out<int>((size_t)n * 2); int* dist = s.out(hd.data(), (size_t)n * 2);
  if ((rc = s.status())) return rc;
  if (n) { k_bf_knn2<<<dim3(1, n), 128>>>(da, dn, db, dn, 1, 1, idx, dist); PL_LAUNCH_CHECK(); }
  if ((rc = s.fetch())) return rc;
  for (int i = 0; i < n; i++) out[i] = hd[2 * i];
  return PL_OK;
}

extern "C" int pl_frame_assign_grid_dev(const PLKeyPoint* keys, const int* n, int cap, int B, const float* bounds,
                                        int* cell_start, int* cell_items, void* stream) {
  PL_ARG(keys && n && bounds && cell_start && cell_items && cap > 0 && cap < 65535 && B > 0);
  k_assign_grid<<<B, 32, grid_smem_bytes(cap), (cudaStream_t)stream>>>(keys, n, cap, bounds, cell_start, cell_items);
  PL_LAUNCH_CHECK();
  return PL_OK;
}
extern "C" int pl_frame_assign_grid(const PLKeyPoint* keys, int n, const float* bounds, int* cell_start,
                                    int* cell_items) {
  PL_ARG(keys && bounds && cell_start && cell_items && n >= 0 && n < 65535);
  int rc = require_device(); if (rc) return rc;
  Staging s;
  int cap = std::max(n, 1);
  PLKeyPoint* dk = s.in(keys, (size_t)n); int* dn = s.in(&n, 1); float* db = s.in(bounds, 4);
  int* ds = s.out(cell_start, NCELL + 1); int* di = s.out(cell_items, (size_t)n, cap);
  if ((rc = s.status()) || (rc = pl_frame_assign_grid_dev(dk, dn, cap, 1, db, ds, di, nullptr))) return rc;
  return s.fetch();
}

extern "C" int pl_orb_search_for_initialization_dev(const PLKeyPoint* keys1, const uint8_t* desc1, const int* n1,
                                                    const PLKeyPoint* keys2, const uint8_t* desc2, const int* n2,
                                                    int cap, int B, const float* bounds, float* prev_matched,
                                                    int* matches12, int* nmatches, int window_size, float nnratio,
                                                    int check_orientation, int* scratch, void* stream) {
  PL_ARG(keys1 && desc1 && n1 && keys2 && desc2 && n2 && bounds && prev_matched && matches12 && nmatches && scratch);
  PL_ARG(cap > 0 && cap <= kMatchMaxKeys && B > 0);
  size_t sm = grid_smem_bytes(cap);
  PL_CUDA(cudaFuncSetAttribute(k_search_init, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  k_search_init<<<B, 32, sm, (cudaStream_t)stream>>>(keys1, desc1, n1, keys2, desc2, n2, cap, bounds, prev_matched,
                                                     matches12, nmatches, window_size, nnratio, check_orientation,
                                                     scratch);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

extern "C" int pl_orb_search_for_initialization(const PLKeyPoint* keys1, const uint8_t* desc1, int n1,
                                                const PLKeyPoint* keys2, const uint8_t* desc2, int n2,
                                                const float* bounds, float* prev_matched, int* matches12,
                                                int window_size, float nnratio, int check_orientation) {
  PL_ARG(keys1 && desc1 && keys2 && desc2 && bounds && prev_matched && matches12 && n1 >= 0 && n2 >= 0);
  int rc = require_device(); if (rc) return rc;
  Staging s;
  const size_t cap = std::max(std::max(n1, n2), 1);
  PLKeyPoint* dk1 = s.in(keys1, n1, cap); PLKeyPoint* dk2 = s.in(keys2, n2, cap);
  uint8_t* dd1 = s.in(desc1, (size_t)n1 * 32, cap * 32); uint8_t* dd2 = s.in(desc2, (size_t)n2 * 32, cap * 32);
  int* dn1 = s.in(&n1, 1); int* dn2 = s.in(&n2, 1); float* db = s.in(bounds, 4);
  float* dpm = s.in(prev_matched, (size_t)n1 * 2, cap * 2);
  int nm = 0;
  int* dm = s.out(matches12, n1, cap); int* dnm = s.out(&nm, 1); int* scr = s.out<int>(2 * cap);
  if ((rc = s.status()) ||
      (rc = pl_orb_search_for_initialization_dev(dk1, dd1, dn1, dk2, dd2, dn2, (int)cap, 1, db, dpm, dm, dnm, window_size, nnratio,
                                                 check_orientation, scr, nullptr)) ||
      (rc = s.fetch()) || (rc = s.down(prev_matched, dpm, (size_t)n1 * 2)))
    return rc;
  return nm;
}

extern "C" int pl_orb_search_by_projection_last(const PLKeyPoint* keys_cur, const uint8_t* desc_cur, int n_cur,
                                                const float* bounds, const float* Tcw, const float* K,
                                                const float* scale_factors, int nlevels, int n_last,
                                                const uint8_t* last_valid, const float* last_pos,
                                                const uint8_t* last_desc, const int* last_octave,
                                                const float* last_angle, float th, int check_orientation,
                                                const uint8_t* cur_preassigned, int* cur_match) {
  PL_ARG(keys_cur && desc_cur && bounds && Tcw && K && scale_factors && cur_match && n_cur >= 0 && n_cur <= kMatchMaxKeys && n_last >= 0);
  int rc = require_device(); if (rc) return rc;
  Staging s;
  const int cap = std::max(n_cur, 1), capl = std::max(n_last, 1);
  PLKeyPoint* dk = s.in(keys_cur, n_cur); uint8_t* dd = s.in(desc_cur, (size_t)n_cur * 32); int* dn = s.in(&n_cur, 1);
  float* db = s.in(bounds, 4); float* dT = s.in(Tcw, 16); float* dK = s.in(K, 4); float* dsf = s.in(scale_factors, nlevels);
  int* dnl = s.in(&n_last, 1); uint8_t* dv = s.in(last_valid, n_last); float* dp = s.in(last_pos, (size_t)n_last * 3);
  uint8_t* dld = s.in(last_desc, (size_t)n_last * 32); int* dlo = s.in(last_octave, n_last); float* dla = s.in(last_angle, n_last);
  uint8_t* dpre = cur_preassigned ? s.in(cur_preassigned, n_cur) : nullptr;
  int nm = 0;
  int* dm = s.out(cur_match, n_cur, cap); int* dnm = s.out(&nm, 1);
  if ((rc = s.status()) ||
      (rc = search_by_projection_last_launch(dk, dd, dn, cap, 1, db, dT, dK, dsf, nlevels, dnl, capl, dv, dp, dld, nullptr, dlo, dla, th,
                                             check_orientation, dpre, nullptr, 0, dm, dnm, nullptr)) ||
      (rc = s.fetch()))
    return rc;
  return nm;
}

extern "C" int pl_orb_search_by_projection_points(const PLKeyPoint* keys, const uint8_t* desc, int n,
                                                  const float* bounds, const float* scale_factors, int nlevels,
                                                  int n_mp, const uint8_t* in_view, const float* proj,
                                                  const int* level, const float* view_cos, const uint8_t* mp_desc,
                                                  float th, float nnratio, const uint8_t* preassigned, int* match) {
  PL_ARG(keys && desc && bounds && scale_factors && match && n >= 0 && n_mp >= 0);
  int rc = require_device(); if (rc) return rc;
  Staging s;
  const int cap = std::max(n, 1), capm = std::max(n_mp, 1);
  PLKeyPoint* dk = s.in(keys, n); uint8_t* dd = s.in(desc, (size_t)n * 32); int* dn = s.in(&n, 1);
  float* db = s.in(bounds, 4); float* dsf = s.in(scale_factors, nlevels);
  int* dnm_in = s.in(&n_mp, 1); uint8_t* dv = s.in(in_view, n_mp); float* dp = s.in(proj, (size_t)n_mp * 2);
  int* dl = s.in(level, n_mp); float* dvc = s.in(view_cos, n_mp); uint8_t* dmd = s.in(mp_desc, (size_t)n_mp * 32);
  uint8_t* dpre = preassigned ? s.in(preassigned, n) : nullptr;
  int nm = 0;
  int* dm = s.out(match, n, cap); int* dnm = s.out(&nm, 1);
  if ((rc = s.status()) ||
      (rc = search_by_projection_points_launch(dk, dd, dn, cap, 1, db, dsf, dnm_in, capm, dv, dp, dl, dvc, dmd, th, nullptr, nullptr,
                                               nnratio, dpre, dm, dnm, nullptr)) ||
      (rc = s.fetch()))
    return rc;
  return nm;
}

// ---- batched, device-resident forms of the three projection searches of the steady-state tracking step (one warp per frame,
// [B][cap] arrays, asynchronous on `stream`): what pl_frontend_run_dev launches; the host-pointer forms above are the B = 1 case.
extern "C" int pl_orb_search_by_projection_last_dev(const PLKeyPoint* keys_cur, const uint8_t* desc_cur, const int* n_cur, int cap, int B,
                                                    const float* bounds, const float* Tcw, const float* K, const float* scale_factors,
                                                    int nlevels, const int* n_last, int cap_last, const uint8_t* last_valid,
                                                    const float* last_pos, const uint8_t* last_desc, const int* last_octave,
                                                    const float* last_angle, float th, int check_orientation,
                                                    const uint8_t* cur_preassigned, const int* gate_nmatches, int gate_min,
                                                    int* cur_match, int* nmatches, void* stream) {
  return search_by_projection_last_launch(keys_cur, desc_cur, n_cur, cap, B, bounds, Tcw, K, scale_factors, nlevels, n_last, cap_last,
                                          last_valid, last_pos, last_desc, nullptr, last_octave, last_angle, th, check_orientation,
                                          cur_preassigned, gate_nmatches, gate_min, cur_match, nmatches, stream);
}
int pl::search_by_projection_last_launch(const PLKeyPoint* keys_cur, const uint8_t* desc_cur, const int* n_cur, int cap, int B,
                                         const float* bounds, const float* Tcw, const float* K, const float* scale_factors, int nlevels,
                                         const int* n_last, int cap_last, const uint8_t* last_valid, const float* last_pos,
                                         const uint8_t* last_desc, const int* last_row, const int* last_octave, const float* last_angle,
                                         float th, int check_orientation, const uint8_t* cur_preassigned, const int* gate_nmatches,
                                         int gate_min, int* cur_match, int* nmatches, void* stream) {
  PL_ARG(keys_cur && desc_cur && n_cur && bounds && Tcw && K && scale_factors && n_last && last_valid && last_pos && last_desc &&
         last_octave && last_angle && cur_match && nmatches && B >= 1 && cap >= 1 && cap <= kMatchMaxKeys && cap_last >= 1);
  ProjLastArgs A;
  A.last_row = last_row;
  A.keys = keys_cur; A.desc = desc_cur; A.n = n_cur; A.cap = cap; A.bounds = bounds; A.Tcw = Tcw; A.K = K; A.scaleFactors = scale_factors;
  A.nlevels = nlevels; A.n_last = n_last; A.cap_last = cap_last; A.last_valid = last_valid; A.last_pos = last_pos; A.last_desc = last_desc;
  A.last_octave = last_octave; A.last_angle = last_angle; A.th = th; A.checkOri = check_orientation; A.preassigned = cur_preassigned;
  A.match = cur_match; A.nmatches = nmatches; A.gate = gate_nmatches; A.gate_min = gate_min;
  const size_t sm = grid_smem_bytes(cap);
  PL_CUDA(cudaFuncSetAttribute(k_search_proj_last, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  k_search_proj_last<<<B, 32, sm, (cudaStream_t)stream>>>(A);
  PL_LAUNCH_CHECK();
  return PL_OK;
}
int pl::search_by_projection_points_launch(const PLKeyPoint* keys, const uint8_t* desc, const int* n, int cap, int B,
                                           const float* bounds, const float* scale_factors, const int* n_mp, int cap_mp,
                                           const uint8_t* in_view, const float* proj, const int* level, const float* view_cos,
                                           const uint8_t* mp_desc, float th, const float* th_frame, const int* desc_row, float nnratio,
                                           const uint8_t* preassigned, int* match, int* nmatches, void* stream) {
  PL_ARG(keys && desc && n && bounds && scale_factors && n_mp && in_view && proj && level && view_cos && mp_desc && match && nmatches &&
         B >= 1 && cap >= 1 && cap <= kMatchMaxKeys && cap_mp >= 1);
  ProjPointsArgs A{};
  A.th_frame = th_frame; A.desc_row = desc_row;
  A.keys = keys; A.desc = desc; A.n = n; A.cap = cap; A.bounds = bounds; A.scaleFactors = scale_factors; A.n_mp = n_mp; A.cap_mp = cap_mp;
  A.in_view = in_view; A.proj = proj; A.level = level; A.view_cos = view_cos; A.mp_desc = mp_desc; A.th = th; A.nnratio = nnratio;
  A.preassigned = preassigned; A.match = match; A.nmatches = nmatches;
  const size_t sm = grid_smem_bytes(cap);
  PL_CUDA(cudaFuncSetAttribute(k_search_proj_points, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  k_search_proj_points<<<B, 32, sm, (cudaStream_t)stream>>>(A);
  PL_LAUNCH_CHECK();
  return PL_OK;
}
extern "C" int pl_orb_search_by_projection_points_dev(const PLKeyPoint* keys, const uint8_t* desc, const int* n, int cap, int B,
                                                      const float* bounds, const float* scale_factors, const int* n_mp, int cap_mp,
                                                      const uint8_t* in_view, const float* proj, const int* level, const float* view_cos,
                                                      const uint8_t* mp_desc, float th, float nnratio, const uint8_t* preassigned,
                                                      int* match, int* nmatches, void* stream) {
  return search_by_projection_points_launch(keys, desc, n, cap, B, bounds, scale_factors, n_mp, cap_mp, in_view, proj, level, view_cos,
                                            mp_desc, th, nullptr, nullptr, nnratio, preassigned, match, nmatches, stream);
}

extern "C" int pl_match_bf_knn2(const uint8_t* d1, int n1, const uint8_t* d2, int n2, int* idx, int* dist) {
  PL_ARG(d1 && d2 && idx && dist && n1 >= 0 && n2 >= 0);
  int rc = require_device(); if (rc) return rc;
  if (n1 == 0) return PL_OK;
  Staging s;
  uint8_t* a = s.in(d1, (size_t)n1 * 32); uint8_t* b = s.in(d2, (size_t)n2 * 32, 32);
  int* dn1 = s.in(&n1, 1); int* dn2 = s.in(&n2, 1);
  int* di = s.out(idx, (size_t)n1 * 2); int* dd = s.out(dist, (size_t)n1 * 2);
  if ((rc = s.status())) return rc;
  k_bf_knn2<<<dim3((n1 + 3) / 4, 1), 128>>>(a, dn1, b, dn2, n1, std::max(n2, 1), di, dd);
  PL_LAUNCH_CHECK();
  return s.fetch();
}

// m1[cap1], m2[cap2], bd0 and bd1[max(cap1, cap2)] of k_search_double
static size_t search_double_smem(int cap1, int cap2) { return (size_t)(cap1 + cap2 + 2 * std::max(cap1, cap2)) * sizeof(short); }
// PL_OK if search_double_smem(cap1, cap2) fits beside `kernel`'s static shared memory
static int search_double_fits_for(const void* kernel, const char* name, int cap1, int cap2) {
  int dev = 0, optin = 0;
  cudaFuncAttributes fa;
  PL_CUDA(cudaGetDevice(&dev));
  PL_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  PL_CUDA(cudaFuncGetAttributes(&fa, kernel));
  const size_t room = optin > (int)fa.sharedSizeBytes ? (size_t)optin - fa.sharedSizeBytes : 0;
  if (search_double_smem(cap1, cap2) > room) {
    set_error("line matching of %d against %d lines needs %zu B of shared memory beside %s's %zu static B, over the "
              "device's %d B per block; at most %zu lines per side fit", cap1, cap2, search_double_smem(cap1, cap2), name,
              (size_t)fa.sharedSizeBytes, optin, room / (4 * sizeof(short)));
    return PL_ERR_ARG;
  }
  return PL_OK;
}
int pl::search_double_fits(int cap1, int cap2) { return search_double_fits_for((const void*)k_search_double, "k_search_double", cap1, cap2); }

extern "C" int pl_lsd_search_double_dev(const uint8_t* d1, const int* n1, const uint8_t* d2, const int* n2, int cap1,
                                        int cap2, int B, float th, float nnratio, int mutual, int* matches,
                                        int* nmatches, void* stream) {
  PL_ARG(d1 && n1 && d2 && n2 && matches && nmatches && cap1 > 0 && cap2 > 0 && cap1 < 32000 && cap2 < 32000 && B > 0);
  PL_TRY(search_double_fits(cap1, cap2));
  const size_t sm = search_double_smem(cap1, cap2);
  PL_CUDA(cudaFuncSetAttribute(k_search_double, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  k_search_double<<<B, 128, sm, (cudaStream_t)stream>>>(d1, n1, d2, n2, cap1, cap2, th, nnratio, mutual, matches,
                                                        nmatches);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

static int search_double_host(const uint8_t* d1, int n1, const uint8_t* d2, int n2, float th, float nnratio, int mutual,
                              int* matches) {
  PL_ARG(d1 && d2 && matches && n1 >= 0 && n2 >= 0);
  int rc = require_device(); if (rc) return rc;
  Staging s;
  const int c1 = std::max(n1, 1), c2 = std::max(n2, 1);
  uint8_t* a = s.in(d1, (size_t)n1 * 32, 32); uint8_t* b = s.in(d2, (size_t)n2 * 32, 32);
  int* dn1 = s.in(&n1, 1); int* dn2 = s.in(&n2, 1);
  int nm = 0;
  int* dm = s.out(matches, n1, c1); int* dnm = s.out(&nm, 1);
  if ((rc = s.status()) || (rc = pl_lsd_search_double_dev(a, dn1, b, dn2, c1, c2, 1, th, nnratio, mutual, dm, dnm, nullptr)) ||
      (rc = s.fetch()))
    return rc;
  return nm;
}
extern "C" int pl_lsd_frame_bf_match(const uint8_t* d1, int n1, const uint8_t* d2, int n2, float th, float nnratio,
                                     int* matches) {
  return search_double_host(d1, n1, d2, n2, th, nnratio, 0, matches);
}
extern "C" int pl_lsd_search_double(const uint8_t* d1, int n1, const uint8_t* d2, int n2, float nnratio, int* matches) {
  return search_double_host(d1, n1, d2, n2, 50.f, nnratio, 1, matches);
}
// PL_OK if a triangulation batch's problem table can be read as plslam_b200.h states (PLTriProblems); the rest is checked on the
// device.  The line call does not read F12.
static int tri_problems_ok(const PLTriProblems* Q, bool points, const void* match, const void* nmatches, const void* status) {
  PL_ARG(Q && Q->P >= 0 && Q->n_out >= 0);
  if (Q->P == 0) return PL_OK;
  PL_ARG(Q->kf1 && Q->kf2 && Q->out_offset && (Q->F12 || !points) && nmatches && status);
  PL_ARG(Q->n_out == 0 || match);
  return PL_OK;
}

// sm: the dynamic shared memory of the largest problem, search_double_smem(N1, N2)
static int lsd_tri_launch(const PLTriLineKeyframes& K, const PLTriProblems& Q, float th, float nnratio, int mutual, size_t sm, int* match,
                          int* nmatches, int* status, void* stream) {
  PL_CUDA(cudaFuncSetAttribute(k_lsd_search_triangulation, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  const LineTriBatch A{K, Q, th, nnratio, mutual, match, nmatches, status};
  k_lsd_search_triangulation<<<Q.P, 128, sm, (cudaStream_t)stream>>>(A);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

int pl::lsd_tri_table_ok(const PLTriLineKeyframes* kfs) {
  PL_ARG(kfs);
  const PLTriLineKeyframes& K = *kfs;
  PL_ARG(K.n_kf >= 1 && K.cap >= 1 && K.cap < 32000 && (long long)K.n_kf * K.cap <= INT_MAX && K.ldesc && K.has_ml && K.n);
  return PL_OK;
}

int pl::lsd_tri_args_ok(const PLTriLineKeyframes* kfs, const PLTriProblems* problems, const void* match, const void* nmatches,
                        const void* status) {
  PL_TRY(tri_problems_ok(problems, false, match, nmatches, status));
  if (problems->P == 0) return PL_OK;
  return lsd_tri_table_ok(kfs);
}

extern "C" int pl_lsd_search_for_triangulation_dev(const PLTriLineKeyframes* kfs, const PLTriProblems* problems, float th, float nnratio,
                                                   int is_double, int* matched_pairs, int* nmatches, int* status, void* stream) {
  PL_TRY(lsd_tri_args_ok(kfs, problems, matched_pairs, nmatches, status));
  if (problems->P == 0) return PL_OK;
  const PLTriLineKeyframes& K = *kfs;
  PL_TRY(require_device());
  PL_TRY(search_double_fits_for((const void*)k_lsd_search_triangulation, "k_lsd_search_triangulation", K.cap, K.cap));
  return lsd_tri_launch(K, *problems, th, nnratio, is_double ? 1 : 0, search_double_smem(K.cap, K.cap), matched_pairs, nmatches,
                        status, stream);
}

// LSDmatcher::SearchForTriangulation(pKF1, pKF2, vMatchedPairs, isDouble) (src/LSDmatcher.cpp:727-776, the variant
// LocalMapping calls at LocalMapping.cc:961, th = TH_HIGH = 80) and its pair<> twin (:672-725, LocalMapping.cc:679, th = TH_LOW = 50,
// always mutual): the P = 1 case of pl_lsd_search_for_triangulation_dev, a table of the two keyframes.
extern "C" int pl_lsd_search_for_triangulation(const uint8_t* ldesc1, const uint8_t* has_ml1, int n1, const uint8_t* ldesc2,
                                               const uint8_t* has_ml2, int n2, float th, float nnratio, int is_double, int* matched_pairs) {
  PL_ARG(matched_pairs && n1 >= 0 && n2 >= 0 && (n1 == 0 || (ldesc1 && has_ml1)) && (n2 == 0 || (ldesc2 && has_ml2)));
  for (int i = 0; i < n1; i++) matched_pairs[i] = -1;
  if (n1 == 0 || n2 == 0) { int rc = require_device(); return rc ? rc : 0; }     // ldesc.rows == 0 -> return 0 (:738-739)
  int rc = require_device(); if (rc) return rc;
  PL_ARG(n1 < 32000 && n2 < 32000);
  PL_TRY(search_double_fits_for((const void*)k_lsd_search_triangulation, "k_lsd_search_triangulation", n1, n2));
  const int cap = std::max(n1, n2);
  std::vector<uint8_t> desc((size_t)2 * cap * 32, 0), ml((size_t)2 * cap, 0);
  memcpy(desc.data(), ldesc1, (size_t)n1 * 32); memcpy(desc.data() + (size_t)cap * 32, ldesc2, (size_t)n2 * 32);
  memcpy(ml.data(), has_ml1, n1); memcpy(ml.data() + cap, has_ml2, n2);
  const int ints[5] = {n1, n2, 0, 1, 0};     // the keyframes' counts; kf1, kf2, out_offset of the one problem
  Staging s;
  const int* di = s.in(ints, 5);
  const PLTriLineKeyframes K{2, cap, s.in(desc.data(), desc.size()), s.in(ml.data(), ml.size()), di};
  const PLTriProblems Q{1, di + 2, di + 3, nullptr, di + 4, n1};
  int nm = 0, st = 0;
  int* dm = s.out(matched_pairs, n1); int* dnm = s.out(&nm, 1); int* dst = s.out(&st, 1);
  if ((rc = s.status())) return rc;
  PL_TRY(lsd_tri_launch(K, Q, th, nnratio, is_double ? 1 : 0, search_double_smem(n1, n2), dm, dnm, dst, nullptr));
  if ((rc = s.fetch())) return rc;
  return nm;
}


// Frame::AssignFeaturesToGridForLine -> CSR (cell = ix*48+iy), for parity tests of the line grid itself
namespace pl {
__global__ void __launch_bounds__(32) k_line_grid(const KeyLine68* kl, int n, const float* bounds, int* start, unsigned short* items,
                                                  unsigned short* path, unsigned short* plen) {
  __shared__ unsigned short cursor[NCELL];
  GridP g = make_grid(bounds);
  build_line_grid(kl, n, g, start, items, path, plen, threadIdx.x);
  LineGridS L; L.start = start; L.items = items; L.path = path; L.plen = plen; L.cursor = cursor;
  fill_line_grid(L, n, threadIdx.x);
}
}  // namespace pl

extern "C" int pl_frame_assign_grid_lines(const void* keylines_un, int n, const float* bounds, int* cell_start, int* cell_items, int cap_items) {
  PL_ARG(keylines_un && bounds && cell_start && cell_items && n >= 0 && n < 60000);
  int rc = require_device(); if (rc) return rc;
  Staging s;
  const int cap = std::max(n, 1);
  KeyLine68* dk = (KeyLine68*)s.in((const uint8_t*)keylines_un, (size_t)n * 68);
  float* db = s.in(bounds, 4);
  int* ds = s.out(cell_start, NCELL + 1); unsigned short* di = s.out<unsigned short>((size_t)cap * kMaxPath);
  unsigned short* dp = s.out<unsigned short>((size_t)cap * kMaxPath); unsigned short* dl = s.out<unsigned short>(cap);
  if ((rc = s.status())) return rc;
  k_line_grid<<<1, 32>>>(dk, n, db, ds, di, dp, dl);
  PL_LAUNCH_CHECK();
  if ((rc = s.fetch())) return rc;
  const int tot = cell_start[NCELL];
  std::vector<unsigned short> tmp(std::max(tot, 1));
  if ((rc = s.down(tmp.data(), di, (size_t)tot))) return rc;
  for (int i = 0; i < tot && i < cap_items; i++) cell_items[i] = tmp[i];
  return tot;
}

static int line_search_host(int variant, const void* kls, const double* lfunc, const uint8_t* desc, int n, const float* bounds,
                            int n_q, const uint8_t* q_valid, const float* q_proj, const uint8_t* q_desc,
                            const float* q_length_or_view_cos, float th, float nnratio, const uint8_t* preassigned, int* match) {
  PL_ARG(kls && lfunc && desc && bounds && match && n >= 0 && n < 60000 && n_q >= 0);
  int rc = require_device(); if (rc) return rc;
  Staging s;
  const int cap = std::max(n, 1), capq = std::max(n_q, 1);
  uint8_t* dk = s.in((const uint8_t*)kls, (size_t)n * 68); double* dlf = s.in(lfunc, (size_t)n * 3);
  uint8_t* dd = s.in(desc, (size_t)n * 32); int* dn = s.in(&n, 1); float* db = s.in(bounds, 4);
  int* dnq = s.in(&n_q, 1); uint8_t* dv = s.in(q_valid, n_q); float* dp = s.in(q_proj, (size_t)n_q * 4);
  uint8_t* dqd = s.in(q_desc, (size_t)n_q * 32); float* dlv = s.in(q_length_or_view_cos, n_q);
  uint8_t* dpre = preassigned ? s.in(preassigned, n) : nullptr;
  int nm = 0;
  int* dm = s.out(match, n, cap); int* dnm = s.out(&nm, 1);
  uint8_t* scratch = s.out<uint8_t>(pl_lsd_search_scratch_bytes(cap, 1));
  if ((rc = s.status()) ||
      (rc = lsd_search_by_projection_launch(variant, dk, dlf, dd, dn, cap, 1, db, dnq, capq, dv, dp, dqd, dlv, th, nullptr, nullptr,
                                            nnratio, dpre, dm, dnm, scratch, nullptr)) ||
      (rc = s.fetch()))
    return rc;
  return nm;
}

extern "C" int pl_lsd_search_by_projection_last(const void* keylines_cur, const double* linefunc_cur, const uint8_t* desc_cur,
                                                int n_cur, const float* bounds, int n_last, const uint8_t* last_valid,
                                                const float* last_proj, const uint8_t* last_desc, const float* last_length,
                                                float th, const uint8_t* cur_preassigned, int* cur_match) {
  return line_search_host(0, keylines_cur, linefunc_cur, desc_cur, n_cur, bounds, n_last, last_valid, last_proj, last_desc,
                          last_length, th, 0.f, cur_preassigned, cur_match);
}
extern "C" int pl_lsd_search_by_projection_lines(const void* keylines, const double* linefunc, const uint8_t* desc, int n,
                                                 const float* bounds, int n_ml, const uint8_t* in_view, const float* proj,
                                                 const float* view_cos, const uint8_t* ml_desc, float th, float nnratio,
                                                 const uint8_t* preassigned, int* match) {
  return line_search_host(1, keylines, linefunc, desc, n, bounds, n_ml, in_view, proj, ml_desc, view_cos, th, nnratio, preassigned,
                          match);
}

extern "C" size_t pl_lsd_search_scratch_bytes(int cap, int B) {
  const size_t per = (size_t)(NCELL + 1) * 4 + (size_t)cap * kMaxPath * 2 * 2 + (size_t)cap * 2 + (size_t)cap * 4;
  return per * (size_t)B + 256;
}
/* variant 0 = SearchByProjection(CurrentFrame, LastFrame, th) (q_length = last lineLength), 1 = (F, vpMapLines, th) (q_view_cos) */
int pl::lsd_search_by_projection_launch(int variant, const void* keylines, const double* linefunc, const uint8_t* desc, const int* n,
                                       int cap, int B, const float* bounds, const int* n_q, int cap_q, const uint8_t* q_valid,
                                       const float* q_proj, const uint8_t* q_desc, const float* q_length_or_view_cos, float th,
                                       const float* th_frame, const int* q_desc_row, float nnratio, const uint8_t* preassigned, int* match,
                                       int* nmatches, void* scratch, void* stream) {
  PL_ARG(keylines && linefunc && desc && n && bounds && n_q && q_valid && q_proj && q_desc && q_length_or_view_cos && match && nmatches &&
         scratch && B >= 1 && cap >= 1 && cap < 60000 && cap_q >= 1 && (variant == 0 || variant == 1));
  LineSearchArgs A{};
  A.th_frame = th_frame; A.q_desc_row = q_desc_row;
  A.kl = (const KeyLine68*)keylines; A.lfunc = linefunc; A.desc = desc; A.n = n; A.cap = cap; A.bounds = bounds;
  A.n_q = n_q; A.cap_q = cap_q; A.q_valid = q_valid; A.q_proj = q_proj; A.q_desc = q_desc;
  A.q_length = variant == 0 ? q_length_or_view_cos : nullptr; A.q_view_cos = variant == 1 ? q_length_or_view_cos : nullptr;
  A.th = th; A.nnratio = nnratio; A.variant = variant; A.preassigned = preassigned; A.match = match; A.nmatches = nmatches;
  unsigned char* p = (unsigned char*)scratch;
  auto take = [&](size_t bytes) { unsigned char* r = p; p += (bytes + 15) / 16 * 16; return r; };
  A.g_start = (int*)take((size_t)(NCELL + 1) * 4 * B); A.g_first = (int*)take((size_t)cap * 4 * B);
  A.g_items = (unsigned short*)take((size_t)cap * kMaxPath * 2 * B); A.g_path = (unsigned short*)take((size_t)cap * kMaxPath * 2 * B);
  A.g_plen = (unsigned short*)take((size_t)cap * 2 * B);
  k_line_search<<<B, 32, 0, (cudaStream_t)stream>>>(A);
  PL_LAUNCH_CHECK();
  return PL_OK;
}
extern "C" int pl_lsd_search_by_projection_dev(int variant, const void* keylines, const double* linefunc, const uint8_t* desc, const int* n,
                                               int cap, int B, const float* bounds, const int* n_q, int cap_q, const uint8_t* q_valid,
                                               const float* q_proj, const uint8_t* q_desc, const float* q_length_or_view_cos, float th,
                                               float nnratio, const uint8_t* preassigned, int* match, int* nmatches, void* scratch,
                                               void* stream) {
  return lsd_search_by_projection_launch(variant, keylines, linefunc, desc, n, cap, B, bounds, n_q, cap_q, q_valid, q_proj, q_desc,
                                         q_length_or_view_cos, th, nullptr, nullptr, nnratio, preassigned, match, nmatches, scratch, stream);
}

// ------------------------------------------------------------------------------------------------ §8f.2 wrappers

static int orb_tri_launch(const PLTriKeyframes& K, const PLTriProblems& Q, int check_orientation, int* match, int* nmatches, int* status,
                          void* stream) {
  const TriBatch A{K, Q, check_orientation ? 1 : 0, match, nmatches, status};
  k_search_triangulation<<<Q.P, kTriThreads, 0, (cudaStream_t)stream>>>(A);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

int pl::orb_tri_args_ok(const PLTriKeyframes* kfs, const PLTriProblems* problems, const void* match, const void* nmatches,
                        const void* status) {
  PL_TRY(tri_problems_ok(problems, true, match, nmatches, status));
  if (problems->P == 0) return PL_OK;
  PL_ARG(kfs);
  const PLTriKeyframes& K = *kfs;
  PL_ARG(K.n_kf >= 1 && K.cap >= 1 && K.cap <= kMatchMaxKeys && K.cap_nodes >= 1 && K.nlevels >= 1);
  PL_ARG((long long)K.n_kf * K.cap <= INT_MAX && (long long)K.n_kf * (K.cap_nodes + 1) <= INT_MAX);
  PL_ARG(K.keys_un && K.desc && K.has_mp && K.n && K.fv_nodes && K.fv_start && K.fv_items && K.nn && K.Tcw && K.Ow && K.K &&
         K.scale_factors && K.level_sigma2);
  return PL_OK;
}

extern "C" int pl_orb_search_for_triangulation_dev(const PLTriKeyframes* kfs, const PLTriProblems* problems, int check_orientation,
                                                   int* matches12, int* nmatches, int* status, void* stream) {
  PL_TRY(orb_tri_args_ok(kfs, problems, matches12, nmatches, status));
  if (problems->P == 0) return PL_OK;
  const PLTriKeyframes& K = *kfs;
  PL_TRY(require_device());
  return orb_tri_launch(K, *problems, check_orientation, matches12, nmatches, status, stream);
}

// The P = 1 case of pl_orb_search_for_triangulation_dev: a table of the two keyframes, KF1 in row 0 (Ow = Cw1) and KF2 in row 1
// (Tcw from R2w / t2w, K = K2).
extern "C" int pl_orb_search_for_triangulation(const PLKeyPoint* keys1_un, const uint8_t* desc1, const uint8_t* has_mp1, int n1,
                                               const PLKeyPoint* keys2_un, const uint8_t* desc2, const uint8_t* has_mp2, int n2,
                                               const unsigned* fv1_nodes, const int* fv1_start, const int* fv1_items, int nn1,
                                               const unsigned* fv2_nodes, const int* fv2_start, const int* fv2_items, int nn2,
                                               const float* F12, const float* Cw1, const float* R2w, const float* t2w, const float* K2,
                                               const float* scale_factors2, const float* level_sigma2_2, int nlevels,
                                               int check_orientation, int* matches12) {
  PL_ARG(keys1_un && desc1 && has_mp1 && keys2_un && desc2 && has_mp2 && F12 && Cw1 && R2w && t2w && K2 && scale_factors2 &&
         level_sigma2_2 && matches12 && n1 >= 0 && n2 >= 0 && nn1 >= 0 && nn2 >= 0 && nlevels > 0);
  PL_ARG((nn1 == 0 || (fv1_nodes && fv1_start && fv1_items)) && (nn2 == 0 || (fv2_nodes && fv2_start && fv2_items)));
  int rc = require_device(); if (rc) return rc;
  for (int i = 0; i < n1; i++) matches12[i] = -1;
  const int cap = std::max(std::max(n1, n2), 1), capn = std::max(std::max(nn1, nn2), 1);
  std::vector<PLKeyPoint> keys((size_t)2 * cap);
  std::vector<uint8_t> desc((size_t)2 * cap * 32, 0), mp((size_t)2 * cap, 0);
  std::vector<unsigned> nodes((size_t)2 * capn, 0);
  std::vector<int> start((size_t)2 * (capn + 1), 0), items((size_t)2 * cap, 0);
  auto put = [&](int r, const PLKeyPoint* k, const uint8_t* d, const uint8_t* m, int n, const unsigned* fn, const int* fs, const int* fi, int nn) {
    std::copy(k, k + n, keys.begin() + (size_t)r * cap);
    memcpy(desc.data() + (size_t)r * cap * 32, d, (size_t)n * 32); memcpy(mp.data() + (size_t)r * cap, m, n);
    if (nn == 0) return;
    std::copy(fn, fn + nn, nodes.begin() + (size_t)r * capn); std::copy(fs, fs + nn + 1, start.begin() + (size_t)r * (capn + 1));
    const int ni = std::min(std::max(fs[nn], 0), cap);     // a count past n is reported by the kernel (status 2), not read
    std::copy(fi, fi + ni, items.begin() + (size_t)r * cap);
  };
  put(0, keys1_un, desc1, has_mp1, n1, fv1_nodes, fv1_start, fv1_items, nn1);
  put(1, keys2_un, desc2, has_mp2, n2, fv2_nodes, fv2_start, fv2_items, nn2);
  float cam[46] = {0};     // Tcw [2][16], Ow [2][3], K [2][4]: one upload
  for (int r = 0; r < 3; r++) { memcpy(cam + 16 + 4 * r, R2w + 3 * r, 12); cam[16 + 4 * r + 3] = t2w[r]; }
  cam[31] = 1.f;
  memcpy(cam + 32, Cw1, 12); memcpy(cam + 42, K2, 16);
  float fz[9]; memcpy(fz, F12, 36);
  const int ints[7] = {n1, n2, nn1, nn2, 0, 1, 0};     // n [2], nn [2]; kf1, kf2, out_offset of the one problem
  Staging s;
  const float* dc = s.in(cam, 46); const int* di = s.in(ints, 7);
  const PLTriKeyframes K{2, cap, capn, s.in(keys.data(), keys.size()), s.in(desc.data(), desc.size()), s.in(mp.data(), mp.size()), di,
                         s.in(nodes.data(), nodes.size()), s.in(start.data(), start.size()), s.in(items.data(), items.size()), di + 2,
                         dc, dc + 32, dc + 38, s.in(scale_factors2, nlevels), s.in(level_sigma2_2, nlevels), nlevels};
  const PLTriProblems Q{1, di + 4, di + 5, s.in(fz, 9), di + 6, n1};
  int nm = 0, st = 0;
  int* dm = s.out(matches12, n1); int* dnm = s.out(&nm, 1); int* dst = s.out(&st, 1);
  if ((rc = s.status())) return rc;
  PL_TRY(orb_tri_launch(K, Q, check_orientation, dm, dnm, dst, nullptr));
  if ((rc = s.fetch())) return rc;
  if (st) {
    set_error("pl_orb_search_for_triangulation: a feature vector is malformed (%s)",
              st == 2 ? "fv_start not monotone, or past the keypoint count" : "an fv_items entry outside 0 .. n - 1");
    return PL_ERR_ARG;
  }
  return nm;
}

// PL_OK if a Fuse batch's problem table can be read as plslam_b200.h states (PLFuseProblems); the rest is checked on the device.
static int fuse_problems_ok(const PLFuseProblems* Q, int* best_idx, int* best_dist, int* status) {
  PL_ARG(Q && Q->P >= 0 && Q->n_entries >= 0 && Q->n_out >= 0);
  if (Q->P == 0) return PL_OK;
  PL_ARG(Q->kf && Q->th && Q->offset && Q->count && Q->out_offset && status);
  PL_ARG(Q->n_entries == 0 || (Q->entry_lm && Q->entry_skip));
  PL_ARG(Q->n_out == 0 || (best_idx && best_dist));
  return PL_OK;
}

static int orb_fuse_launch(const PLFuseKeyframes& K, const PLFusePoints& L, const PLFuseProblems& Q, int* best_idx, int* best_dist,
                           int* status, void* stream) {
  const size_t sm = grid_smem_bytes(K.cap);
  PL_CUDA(cudaFuncSetAttribute(k_fuse_search, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  const FuseBatch A{K, L, Q, best_idx, best_dist, status};
  k_fuse_search<<<Q.P, 32 * kFuseWarps, sm, (cudaStream_t)stream>>>(A);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

extern "C" int pl_orb_fuse_search_dev(const PLFuseKeyframes* kfs, const PLFusePoints* points, const PLFuseProblems* problems, int* best_idx,
                                      int* best_dist, int* status, void* stream) {
  PL_TRY(fuse_problems_ok(problems, best_idx, best_dist, status));
  PL_ARG(points && points->n >= 0);
  if (problems->P == 0) return PL_OK;
  PL_ARG(kfs);
  const PLFuseKeyframes& K = *kfs;
  const PLFusePoints& L = *points;
  PL_ARG(K.n_kf >= 1 && K.cap >= 1 && K.cap <= kMatchMaxKeys && (long long)K.n_kf * K.cap <= INT_MAX && K.nlevels >= 1);
  PL_ARG(K.keys_un && K.desc && K.n && K.Tcw && K.Ow && K.K && K.bounds && K.scale_factors && K.inv_level_sigma2);
  PL_ARG(L.n == 0 || (L.pos && L.normal && L.min_dist && L.max_dist && L.desc));
  PL_TRY(require_device());
  return orb_fuse_launch(K, L, *problems, best_idx, best_dist, status, stream);
}

// The P = 1 case of pl_orb_fuse_search_dev: one keyframe of capacity n, entry i = map point i.
extern "C" int pl_orb_fuse_search(const PLKeyPoint* keys_un, const uint8_t* desc, int n, const float* bounds, const float* Tcw,
                                  const float* Ow, const float* K, const float* scale_factors, const float* inv_level_sigma2,
                                  int nlevels, float log_scale_factor, int n_mp, const uint8_t* skip, const float* pos,
                                  const float* normal, const float* min_dist, const float* max_dist, const uint8_t* mp_desc,
                                  float th, int* best_idx, int* best_dist) {
  PL_ARG(keys_un && desc && bounds && Tcw && Ow && K && scale_factors && inv_level_sigma2 && best_idx && best_dist && n >= 0 &&
         n_mp >= 0 && nlevels > 0 && n < 65000);
  PL_ARG(n_mp == 0 || (pos && normal && min_dist && max_dist && mp_desc));
  int rc = require_device(); if (rc) return rc;
  if (n_mp == 0) return PL_OK;
  float cam[28];        // Tcw, Ow, K, bounds, th: one upload
  memcpy(cam, Tcw, 64); memcpy(cam + 16, Ow, 12); memcpy(cam + 19, K, 16); memcpy(cam + 23, bounds, 16); cam[27] = th;
  const int ints[5] = {n, 0, 0, n_mp, 0};     // keypoint count; kf, offset, count, out_offset of the one problem
  std::vector<int> lm(n_mp);
  for (int i = 0; i < n_mp; i++) lm[i] = i;
  Staging s;
  const float* dc = s.in(cam, 28); const int* di = s.in(ints, 5);
  const PLFuseKeyframes Kt{1, std::max(n, 1), s.in(keys_un, n), s.in(desc, (size_t)n * 32), di, dc, dc + 16, dc + 19, dc + 23,
                           s.in(scale_factors, nlevels), s.in(inv_level_sigma2, nlevels), nlevels, log_scale_factor};
  const PLFusePoints L{n_mp, s.in(pos, (size_t)n_mp * 3), s.in(normal, (size_t)n_mp * 3), s.in(min_dist, n_mp), s.in(max_dist, n_mp),
                       s.in(mp_desc, (size_t)n_mp * 32)};
  const PLFuseProblems Q{1, di + 1, dc + 27, di + 2, di + 3, di + 4, n_mp, s.in(lm.data(), n_mp), skip ? s.in(skip, n_mp) : s.out<uint8_t>(n_mp), n_mp};
  int* dbi = s.out(best_idx, n_mp); int* dbd = s.out(best_dist, n_mp); int* dst = s.out<int>(1);
  if ((rc = s.status())) return rc;
  PL_TRY(orb_fuse_launch(Kt, L, Q, dbi, dbd, dst, nullptr));
  return s.fetch();
}

static int search_by_bow_host(const PLKeyPoint* keysKF_un, const uint8_t* descKF, const uint8_t* has_mp_kf, int nKF,
                              const PLKeyPoint* keysF, const uint8_t* descF, const uint8_t* has_mp_f, int strict, int nF,
                              const unsigned* fvK_nodes, const int* fvK_start, const int* fvK_items, int nnK,
                              const unsigned* fvF_nodes, const int* fvF_start, const int* fvF_items, int nnF, float nnratio,
                              int check_orientation, int* matchesF) {
  PL_ARG(keysKF_un && descKF && has_mp_kf && keysF && descF && matchesF && nKF >= 0 && nF >= 0 && nnK >= 0 && nnF >= 0);
  PL_ARG((nnK == 0 || (fvK_nodes && fvK_start && fvK_items)) && (nnF == 0 || (fvF_nodes && fvF_start && fvF_items)));
  int rc = require_device(); if (rc) return rc;
  for (int j = 0; j < nF; j++) matchesF[j] = -1;
  std::vector<int> ks, ke, fs, fe;     // the node merge of :203-296 on the host: one entry per common node
  for (int a = 0, b = 0; a < nnK && b < nnF;) {
    if (fvK_nodes[a] == fvF_nodes[b]) { ks.push_back(fvK_start[a]); ke.push_back(fvK_start[a + 1]); fs.push_back(fvF_start[b]); fe.push_back(fvF_start[b + 1]); a++; b++; }
    else if (fvK_nodes[a] < fvF_nodes[b]) a++;
    else b++;
  }
  if (ks.empty() || nKF == 0 || nF == 0) return 0;
  const int nitK = fvK_start[nnK], nitF = fvF_start[nnF];
  for (int i = 0; i < nitK; i++) PL_ARG(fvK_items[i] >= 0 && fvK_items[i] < nKF);
  for (int i = 0; i < nitF; i++) PL_ARG(fvF_items[i] >= 0 && fvF_items[i] < nF);
  PL_ARG(nF < (1 << 20));
  Staging s;
  BowArgs A;
  A.kK = s.in(keysKF_un, nKF); A.kF = s.in(keysF, nF); A.dK = s.in(descKF, (size_t)nKF * 32); A.dF = s.in(descF, (size_t)nF * 32);
  A.mpK = s.in(has_mp_kf, nKF);
  A.pairK_s = s.in(ks.data(), ks.size()); A.pairK_e = s.in(ke.data(), ke.size()); A.pairF_s = s.in(fs.data(), fs.size()); A.pairF_e = s.in(fe.data(), fe.size());
  A.itK = s.in(fvK_items, nitK); A.itF = s.in(fvF_items, nitF); A.npairs = (int)ks.size(); A.nF = nF;
  A.nnratio = nnratio; A.checkOri = check_orientation;
  A.mpF = has_mp_f ? s.in(has_mp_f, nF) : nullptr; A.strict = strict;
  int nm = 0;
  A.matchesF = s.out(matchesF, nF); A.bins = s.out<unsigned char>(nF); A.nmatches = s.out(&nm, 1);
  if ((rc = s.status())) return rc;
  k_search_by_bow<<<1, 32 * kBowWarps>>>(A);
  PL_LAUNCH_CHECK();
  if ((rc = s.fetch())) return rc;
  return nm;
}

extern "C" int pl_orb_search_by_bow(const PLKeyPoint* keysKF_un, const uint8_t* descKF, const uint8_t* has_mp_kf, int nKF,
                                    const PLKeyPoint* keysF, const uint8_t* descF, int nF, const unsigned* fvK_nodes,
                                    const int* fvK_start, const int* fvK_items, int nnK, const unsigned* fvF_nodes,
                                    const int* fvF_start, const int* fvF_items, int nnF, float nnratio, int check_orientation,
                                    int* matchesF) {
  return search_by_bow_host(keysKF_un, descKF, has_mp_kf, nKF, keysF, descF, nullptr, 0, nF, fvK_nodes, fvK_start, fvK_items, nnK, fvF_nodes,
                            fvF_start, fvF_items, nnF, nnratio, check_orientation, matchesF);
}
// ORBmatcher::SearchByBoW(pKF1, pKF2, vpMatches12) (src/ORBmatcher.cc:574-709, loop closing): the same node walk with
// MapPoints required on both sides, vbMatched2 as the taken-state and a strict < TH_LOW gate; reported per feature of KF1.
extern "C" int pl_orb_search_by_bow_keyframes(const PLKeyPoint* keys1_un, const uint8_t* desc1, const uint8_t* has_mp1, int n1,
                                              const PLKeyPoint* keys2_un, const uint8_t* desc2, const uint8_t* has_mp2, int n2,
                                              const unsigned* fv1_nodes, const int* fv1_start, const int* fv1_items, int nn1,
                                              const unsigned* fv2_nodes, const int* fv2_start, const int* fv2_items, int nn2,
                                              float nnratio, int check_orientation, int* matches12) {
  PL_ARG(matches12 && has_mp2 && n1 >= 0 && n2 >= 0);
  std::vector<int> m2(std::max(n2, 1), -1);
  const int nm = search_by_bow_host(keys1_un, desc1, has_mp1, n1, keys2_un, desc2, has_mp2, 1, n2, fv1_nodes, fv1_start, fv1_items, nn1,
                                    fv2_nodes, fv2_start, fv2_items, nn2, nnratio, check_orientation, m2.data());
  if (nm < 0) return nm;
  for (int i = 0; i < n1; i++) matches12[i] = -1;
  for (int j = 0; j < n2; j++) if (m2[j] >= 0) matches12[m2[j]] = j;
  return nm;
}
extern "C" int pl_orb_search_by_projection_keyframe(const PLKeyPoint* keys_cur, const uint8_t* desc_cur, int n_cur, const float* bounds,
                                                    const float* Tcw, const float* Ow, const float* K, const float* scale_factors,
                                                    int nlevels, float log_scale_factor, int n_kf, const uint8_t* kf_valid,
                                                    const float* pos, const uint8_t* mp_desc, const float* min_dist,
                                                    const float* max_dist, const float* kf_angle, float th, int orb_dist,
                                                    int check_orientation, const uint8_t* cur_preassigned, int* cur_match) {
  PL_ARG(keys_cur && desc_cur && bounds && Tcw && Ow && K && scale_factors && cur_match && n_cur >= 0 && n_cur <= kMatchMaxKeys && n_kf >= 0 && nlevels > 0);
  PL_ARG(n_kf == 0 || (kf_valid && pos && mp_desc && min_dist && max_dist && kf_angle));
  int rc = require_device(); if (rc) return rc;
  Staging s;
  const int cap = std::max(n_cur, 1), capl = std::max(n_kf, 1);
  ProjLastArgs A;
  A.keys = s.in(keys_cur, n_cur); A.desc = s.in(desc_cur, (size_t)n_cur * 32); A.n = s.in(&n_cur, 1); A.cap = cap;
  A.bounds = s.in(bounds, 4); A.Tcw = s.in(Tcw, 16); A.K = s.in(K, 4); A.scaleFactors = s.in(scale_factors, nlevels);
  A.nlevels = nlevels; A.n_last = s.in(&n_kf, 1); A.cap_last = capl;
  A.last_valid = s.in(kf_valid, n_kf); A.last_pos = s.in(pos, (size_t)n_kf * 3); A.last_desc = s.in(mp_desc, (size_t)n_kf * 32);
  A.last_octave = nullptr; A.last_angle = s.in(kf_angle, n_kf);
  A.th = th; A.checkOri = check_orientation;
  A.preassigned = cur_preassigned ? s.in(cur_preassigned, n_cur) : nullptr;
  int nm = 0;
  A.match = s.out(cur_match, n_cur, cap); A.nmatches = s.out(&nm, 1);
  A.kfMode = 1; A.maxDist = orb_dist; A.min_dist = s.in(min_dist, n_kf); A.max_dist = s.in(max_dist, n_kf);
  memcpy(A.Ow, Ow, 12); A.logSF = log_scale_factor;
  if ((rc = s.status())) return rc;
  size_t sm = grid_smem_bytes(cap);
  PL_CUDA(cudaFuncSetAttribute(k_search_proj_last, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  k_search_proj_last<<<1, 32, sm>>>(A);
  PL_LAUNCH_CHECK();
  if ((rc = s.fetch())) return rc;
  return nm;
}

extern "C" int pl_mappoint_distinctive_descriptors(const uint8_t* desc, const int* offsets, int n_mp, int* best_idx, uint8_t* out_desc) {
  PL_ARG(offsets && best_idx && n_mp >= 0 && (desc || n_mp == 0));
  int rc = require_device(); if (rc) return rc;
  if (n_mp == 0) return PL_OK;
  const int total = offsets[n_mp];
  PL_ARG(total >= 0);
  Staging s;
  const uint8_t* dd = s.in(desc, (size_t)total * 32); const int* doff = s.in(offsets, (size_t)n_mp + 1);
  int* db = s.out(best_idx, n_mp); uint8_t* dout = s.out(out_desc, (size_t)n_mp * 32);
  if ((rc = s.status())) return rc;
  k_distinctive<<<(n_mp + kDistWarps - 1) / kDistWarps, 32 * kDistWarps>>>(dd, doff, n_mp, db, dout);
  PL_LAUNCH_CHECK();
  return s.fetch();
}

static int lsd_fuse_launch(const PLFuseLineKeyframes& K, const PLFuseLines& L, const PLFuseProblems& Q, int* best_idx, int* best_dist,
                           int* stop_at, int* status, void* stream) {
  const LineFuseBatch A{K, L, Q, best_idx, best_dist, stop_at, status};
  k_lsd_fuse_search<<<Q.P, kLineFuseThreads, 0, (cudaStream_t)stream>>>(A);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

extern "C" int pl_lsd_fuse_search_dev(const PLFuseLineKeyframes* kfs, const PLFuseLines* lines, const PLFuseProblems* problems, int* best_idx,
                                      int* best_dist, int* stop_at, int* status, void* stream) {
  PL_TRY(fuse_problems_ok(problems, best_idx, best_dist, status));
  PL_ARG(lines && lines->n >= 0);
  if (problems->P == 0) return PL_OK;
  PL_ARG(kfs);
  const PLFuseLineKeyframes& K = *kfs;
  const PLFuseLines& L = *lines;
  PL_ARG(stop_at && K.n_kf >= 1 && K.cap >= 1 && K.cap <= 32768 && K.cap_pdesc >= 1 && K.cap_pdesc <= 32768);
  PL_ARG((long long)K.n_kf * K.cap <= INT_MAX && (long long)K.n_kf * K.cap_pdesc <= INT_MAX);
  PL_ARG(K.keylines && K.n && K.pdesc && K.n_pdesc && K.Tcw && K.Ow && K.K && K.bounds);
  PL_ARG(L.n == 0 || (L.pos && L.normal && L.min_dist && L.max_dist && L.desc));
  PL_TRY(require_device());
  return lsd_fuse_launch(K, L, *problems, best_idx, best_dist, stop_at, status, stream);
}

// The P = 1 case of pl_lsd_fuse_search_dev: one keyframe, entry i = map line i.
extern "C" int pl_lsd_fuse_search(const void* keylines, int nl, const uint8_t* kf_point_desc, int n_pdesc, const float* bounds, const float* Tcw,
                                  const float* Ow, const float* K, float scale_line, float log_scale_factor_line, int n_ml,
                                  const uint8_t* skip, const double* pos, const double* normal, const float* min_dist, const float* max_dist,
                                  const uint8_t* ml_desc, float th, int* best_idx, int* best_dist, int* stop_at) {
  PL_ARG(bounds && Tcw && Ow && K && best_idx && best_dist && stop_at && nl >= 0 && n_ml >= 0 && n_pdesc >= 0);
  PL_ARG(n_ml == 0 || (skip && pos && normal && min_dist && max_dist && ml_desc));
  int rc = require_device(); if (rc) return rc;
  *stop_at = n_ml;
  if (n_ml == 0) return PL_OK;
  float cam[28];        // Tcw, Ow, K, bounds, th: one upload
  memcpy(cam, Tcw, 64); memcpy(cam + 16, Ow, 12); memcpy(cam + 19, K, 16); memcpy(cam + 23, bounds, 16); cam[27] = th;
  const int ints[6] = {nl, n_pdesc, 0, 0, n_ml, 0};     // line and descriptor counts; kf, offset, count, out_offset of the one problem
  std::vector<int> lm(n_ml);
  for (int i = 0; i < n_ml; i++) lm[i] = i;
  Staging s;
  const float* dc = s.in(cam, 28); const int* di = s.in(ints, 6);
  const PLFuseLineKeyframes Kt{1, std::max(nl, 1), std::max(n_pdesc, 1), s.in(static_cast<const uint8_t*>(keylines), (size_t)nl * 68), di,
                               s.in(kf_point_desc, (size_t)n_pdesc * 32), di + 1, dc, dc + 16, dc + 19, dc + 23, scale_line, log_scale_factor_line};
  const PLFuseLines L{n_ml, s.in(pos, (size_t)n_ml * 6), s.in(normal, (size_t)n_ml * 3), s.in(min_dist, n_ml), s.in(max_dist, n_ml),
                      s.in(ml_desc, (size_t)n_ml * 32)};
  const PLFuseProblems Q{1, di + 2, dc + 27, di + 3, di + 4, di + 5, n_ml, s.in(lm.data(), n_ml), s.in(skip, n_ml), n_ml};
  int* dbi = s.out(best_idx, n_ml); int* dbd = s.out(best_dist, n_ml); int* dstop = s.out(stop_at, 1); int* dst = s.out<int>(1);
  if ((rc = s.status())) return rc;
  PL_TRY(lsd_fuse_launch(Kt, L, Q, dbi, dbd, dstop, dst, nullptr));
  return s.fetch();
}
