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
#include "libm_glibc.cuh"
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
    const float* X = A.last_pos + (lb + i) * 3;
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
      const float ratio = __fdiv_rn(A.max_dist[lb + i], dist3D);
      oct = (int)ceilf(__fdiv_rn(glibc::logf_(ratio), A.logSF));
      if (oct < 0) oct = 0; else if (oct >= A.nlevels) oct = A.nlevels - 1;
    } else oct = A.last_octave[lb + i];
    const float radius = __fmul_rn(A.th, A.scaleFactors[oct]);
    Top2 t = window_top2(kc, dc, sg.start, sg.items, g, u, v, radius, oct - 1, oct + 1, A.last_desc + (lb + i) * 32,
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
  const bool bFactor = A.th != 1.0f;
  for (int i = 0; i < NM; i++) {
    if (!A.in_view[mb + i]) continue;
    const int lvl = A.level[mb + i];
    float r = ((double)A.view_cos[mb + i] > 0.998) ? 2.5f : 4.0f;  // float vs the double literal 0.998
    if (bFactor) r = __fmul_rn(r, A.th);
    Top2 t = window_top2(k, d, sg.start, sg.items, g, A.proj[(mb + i) * 2], A.proj[(mb + i) * 2 + 1],
                         __fmul_rn(r, A.scaleFactors[lvl]), lvl - 1, lvl, A.mp_desc + (mb + i) * 32, skip, lane, packed);
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
        if (fabsf(dist) < r) atomicMin(&first[id], base + c * 1024 + (j - cb));   // order key: probe, cell rank, slot
      }
    }
    base += 4000000;   // > 3072 cells * 1024
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
  const bool bFactor = A.th != 1.0f;
  for (int q = 0; q < NQ; q++) {
    if (!A.q_valid[qb + q]) continue;
    const float* p = A.q_proj + (qb + q) * 4;
    float r, TH;
    if (A.variant == 0) { r = A.th; TH = 0.96f; }
    else { r = ((double)A.q_view_cos[qb + q] > 0.998) ? 5.0f : 8.0f; if (bFactor) r = __fmul_rn(r, A.th); TH = 0.998f; }
    line_candidates(kl, lf, L, g, p[0], p[1], p[2], p[3], r, TH, first, N, lane);
    // candidates in first-occurrence order; top-2 by (distance, order)
    unsigned long long k1 = KEY_NONE, k2 = KEY_NONE;
    for (int id = lane; id < N; id += 32) {
      const int ord = first[id];
      if (ord == 0x7fffffff) continue;
      if (match[id] != -1) continue;
      const int dist = hamming256(A.q_desc + (qb + q) * 32, d + 32 * id);
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
struct TriArgs {
  const PLKeyPoint *k1, *k2; const uint8_t *d1, *d2, *mp1, *mp2;
  const int *q_idx1, *q_s, *q_e, *fv2_items; int nq, n1;
  float F[9], ex, ey; const float *scale2, *sigma2_2; int checkOri;
  int* matches12; int* nmatches; unsigned char* bins;
};
// One block.  Every query (idx1, candidate range in KF2's node) is independent: the reference never sets vbMatched2.
__global__ void __launch_bounds__(256) k_search_triangulation(TriArgs A) {
  __shared__ int hist[HISTO];
  __shared__ int s_nm, s_keep[3];
  const int tid = threadIdx.x;
  if (tid < HISTO) hist[tid] = 0;
  if (tid == 0) s_nm = 0;
  for (int i = tid; i < A.n1; i += blockDim.x) { A.matches12[i] = -1; A.bins[i] = 255; }
  __syncthreads();
  for (int q = tid; q < A.nq; q += blockDim.x) {
    const int idx1 = A.q_idx1[q];
    if (A.mp1[idx1]) continue;
    const PLKeyPoint kp1 = A.k1[idx1];
    // epipolar line of kp1 in image 2 (CheckDistEpipolarLine, :155-172): l = x1' F12
    const float la = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, A.F[0]), __fmul_rn(kp1.y, A.F[3])), A.F[6]);
    const float lb = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, A.F[1]), __fmul_rn(kp1.y, A.F[4])), A.F[7]);
    const float lc = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, A.F[2]), __fmul_rn(kp1.y, A.F[5])), A.F[8]);
    const float den = __fadd_rn(__fmul_rn(la, la), __fmul_rn(lb, lb));
    int bestDist = 50, bestIdx2 = -1;
    for (int i2 = A.q_s[q]; i2 < A.q_e[q]; i2++) {
      const int idx2 = A.fv2_items[i2];
      if (A.mp2[idx2]) continue;
      const int dist = hamming256(A.d1 + 32 * idx1, A.d2 + 32 * idx2);
      if (dist > 50 || dist > bestDist) continue;
      const PLKeyPoint kp2 = A.k2[idx2];
      const float dx = __fsub_rn(A.ex, kp2.x), dy = __fsub_rn(A.ey, kp2.y);
      if (__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) < __fmul_rn(100.f, A.scale2[kp2.octave])) continue;
      const float num = __fadd_rn(__fadd_rn(__fmul_rn(la, kp2.x), __fmul_rn(lb, kp2.y)), lc);
      if (den == 0.f) continue;
      const float dsqr = __fdiv_rn(__fmul_rn(num, num), den);
      if ((double)dsqr < 3.84 * (double)A.sigma2_2[kp2.octave]) { bestIdx2 = idx2; bestDist = dist; }
    }
    if (bestIdx2 >= 0) {
      A.matches12[idx1] = bestIdx2;
      atomicAdd(&s_nm, 1);
      if (A.checkOri) { const int bin = rot_bin(kp1.angle, A.k2[bestIdx2].angle); A.bins[idx1] = (unsigned char)bin; atomicAdd(&hist[bin], 1); }
    }
  }
  __syncthreads();
  if (A.checkOri) {
    if (tid == 0) { int a, b, c; three_maxima(hist, a, b, c); s_keep[0] = a; s_keep[1] = b; s_keep[2] = c; }
    __syncthreads();
    for (int i = tid; i < A.n1; i += blockDim.x) {
      const int bin = A.bins[i];
      if (bin != 255 && bin != s_keep[0] && bin != s_keep[1] && bin != s_keep[2]) { A.matches12[i] = -1; atomicSub(&s_nm, 1); }
    }
    __syncthreads();
  }
  if (tid == 0) *A.nmatches = s_nm;
}

struct FuseArgs {
  const PLKeyPoint* keys; const uint8_t* desc; int n; float bounds[4]; float T[16], Ow[3], K[4];
  const float *scaleFactors, *invSigma2; float logScaleFactor; int nLevels;
  int n_mp; const uint8_t* skip; const float *pos, *normal, *minDist, *maxDist; const uint8_t* mp_desc; float th;
  int *best_idx, *best_dist;
};
struct SkipChi2 {
  const PLKeyPoint* k; const float* inv; float u, v;
  __device__ bool operator()(int id, int) const {
    const float ex = __fsub_rn(u, k[id].x), ey = __fsub_rn(v, k[id].y);
    const float e2 = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey));
    return (double)__fmul_rn(e2, inv[k[id].octave]) > 5.99;
  }
};
constexpr int kFuseWarps = 16;
__global__ void __launch_bounds__(32 * kFuseWarps) k_fuse_search(FuseArgs A) {
  extern __shared__ unsigned char smem[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  SmemGrid sg = carve_grid(smem, A.n);
  const GridP g = make_grid(A.bounds);
  __shared__ int s_packed;
  if (wid == 0) {
    build_point_grid(A.keys, A.n, g, sg.start, sg.fill, sg.items, lane);
    const bool pk = pack_octaves(A.keys, A.n, sg.start[NCELL], sg.items, lane);
    if (lane == 0) s_packed = pk;
  }
  __syncthreads();
  const bool packed = s_packed != 0;
  for (int i = wid; i < A.n_mp; i += kFuseWarps) {
    int bi = -1, bd = 256;
    bool go = !(A.skip && A.skip[i]);
    float u = 0.f, v = 0.f; int lvl = 0;
    if (go) {
      const float P[3] = {A.pos[3 * i], A.pos[3 * i + 1], A.pos[3 * i + 2]};
      float Pc[3];
      for (int r = 0; r < 3; r++)
        Pc[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(A.T[4 * r], P[0]), __fmul_rn(A.T[4 * r + 1], P[1])), __fmul_rn(A.T[4 * r + 2], P[2])), A.T[4 * r + 3]);
      go = !(Pc[2] < 0.0f);
      if (go) {
        const float invz = __fdiv_rn(1.0f, Pc[2]);
        u = __fadd_rn(__fmul_rn(A.K[0], __fmul_rn(Pc[0], invz)), A.K[2]);
        v = __fadd_rn(__fmul_rn(A.K[1], __fmul_rn(Pc[1], invz)), A.K[3]);
        go = (u >= A.bounds[0] && u < A.bounds[2] && v >= A.bounds[1] && v < A.bounds[3]);     // KeyFrame::IsInImage
      }
      if (go) {
        const float PO[3] = {__fsub_rn(P[0], A.Ow[0]), __fsub_rn(P[1], A.Ow[1]), __fsub_rn(P[2], A.Ow[2])};
        const float dist3D = (float)sqrt((double)PO[0] * PO[0] + (double)PO[1] * PO[1] + (double)PO[2] * PO[2]);
        go = !(dist3D < __fmul_rn(0.8f, A.minDist[i]) || dist3D > __fmul_rn(1.2f, A.maxDist[i]));
        if (go) {
          const double dot = (double)PO[0] * A.normal[3 * i] + (double)PO[1] * A.normal[3 * i + 1] + (double)PO[2] * A.normal[3 * i + 2];
          go = !(dot < 0.5 * (double)dist3D);
          const float ratio = __fdiv_rn(A.maxDist[i], dist3D);
          lvl = (int)ceilf(__fdiv_rn(glibc::logf_(ratio), A.logScaleFactor));
          if (lvl < 0) lvl = 0; else if (lvl >= A.nLevels) lvl = A.nLevels - 1;
        }
      }
    }
    if (go) {     // warp-uniform: every lane computed the same scalars
      SkipChi2 skip{A.keys, A.invSigma2, u, v};
      const Top2 t = window_top2(A.keys, A.desc, sg.start, sg.items, g, u, v, __fmul_rn(A.th, A.scaleFactors[lvl]), lvl - 1, lvl,
                                 A.mp_desc + 32 * (long long)i, skip, lane, packed);
      if (t.best != KEY_NONE) { bi = key_idx(t.best); bd = key_dist(t.best); }
    }
    if (lane == 0) { A.best_idx[i] = bi; A.best_dist[i] = bd; }
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
struct LineFuseArgs {
  const KeyLine68* kl; int nl; const uint8_t* pdesc; int n_pdesc; float bounds[4]; float T[16], Ow[3], K[4];
  float scale_line, logScaleFactorLine; int n_ml; const uint8_t* skip; const double *pos, *normal; const float *minDist, *maxDist;
  const uint8_t* ml_desc; float th; int *best_idx, *best_dist, *stop_at;
};
// One thread per map line (the keyframe has <= a few hundred lines; every candidate test is a handful of flops).
// Quirks of the reference are listed at pl_lsd_fuse_search (plslam_b200.h) and restated in oracle_lsd_fuse_search.
__global__ void __launch_bounds__(128) k_lsd_fuse_search(LineFuseArgs A) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n_ml) return;
  A.best_idx[i] = -1; A.best_dist[i] = 256;
  if (A.skip[i]) return;
  const float SP[3] = {(float)A.pos[6 * i], (float)A.pos[6 * i + 1], (float)A.pos[6 * i + 2]};
  const float EP[3] = {(float)A.pos[6 * i + 3], (float)A.pos[6 * i + 4], (float)A.pos[6 * i + 5]};
  float S[3], E[3];
#pragma unroll
  for (int r = 0; r < 3; r++) {
    S[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(A.T[4 * r], SP[0]), __fmul_rn(A.T[4 * r + 1], SP[1])), __fmul_rn(A.T[4 * r + 2], SP[2])), A.T[4 * r + 3]);
    E[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(A.T[4 * r], EP[0]), __fmul_rn(A.T[4 * r + 1], EP[1])), __fmul_rn(A.T[4 * r + 2], EP[2])), A.T[4 * r + 3]);
  }
  if (S[2] < 0.0f || E[2] < 0.0f) { atomicMin(A.stop_at, i); return; }      // `return false` of the whole call (:907)
  const float invz1 = __fdiv_rn(1.0f, S[2]);
  const float u1 = __fadd_rn(__fmul_rn(__fmul_rn(A.K[0], S[0]), invz1), A.K[2]), v1 = __fadd_rn(__fmul_rn(__fmul_rn(A.K[1], S[1]), invz1), A.K[3]);
  if (!(u1 >= A.bounds[0] && u1 < A.bounds[2] && v1 >= A.bounds[1] && v1 < A.bounds[3])) return;
  const float invz2 = __fdiv_rn(1.0f, E[2]);
  const float u2 = __fadd_rn(__fmul_rn(__fmul_rn(A.K[0], E[0]), invz2), A.K[2]), v2 = __fadd_rn(__fmul_rn(__fmul_rn(A.K[1], E[1]), invz2), A.K[3]);
  if (!(u2 >= A.bounds[0] && u2 < A.bounds[2] && v2 >= A.bounds[1] && v2 < A.bounds[3])) return;
  float OM[3];
#pragma unroll
  for (int k = 0; k < 3; k++) OM[k] = __fsub_rn((float)(0.5 * (double)__fadd_rn(SP[k], EP[k])), A.Ow[k]);
  const float dist = (float)sqrt((double)OM[0] * OM[0] + (double)OM[1] * OM[1] + (double)OM[2] * OM[2]);
  if (dist < __fmul_rn(0.8f, A.minDist[i]) || dist > __fmul_rn(1.2f, A.maxDist[i])) return;
  const float pn[3] = {(float)A.normal[3 * i], (float)A.normal[3 * i + 1], (float)A.normal[3 * i + 2]};
  const double dot = (double)OM[0] * pn[0] + (double)OM[1] * pn[1] + (double)OM[2] * pn[2];
  if (dot < 0.5 * (double)dist) return;
  const float ratio = __fdiv_rn(A.maxDist[i], dist);
  const int lvl = (int)ceilf(__fdiv_rn(glibc::logf_(ratio), A.logScaleFactorLine));
  float sf = 1.0f;
  if (lvl >= 0) { for (int k = 0; k < lvl; k++) sf = __fmul_rn(sf, A.scale_line); }
  else { for (int k = 0; k < -lvl; k++) sf = __fmul_rn(sf, A.scale_line); sf = __fdiv_rn(1.0f, sf); }
  const float radius = __fmul_rn(A.th, sf), r2 = __fmul_rn(radius, radius);
  float d1x = __fsub_rn(u1, u2), d1y = __fsub_rn(v1, v2);
  const float n1 = __fsqrt_rn(__fadd_rn(__fmul_rn(d1x, d1x), __fmul_rn(d1y, d1y)));
  d1x = __fdiv_rn(d1x, n1); d1y = __fdiv_rn(d1y, n1);
  const double mxd = 0.5 * (double)__fadd_rn(u1, u2), myd = 0.5 * (double)__fadd_rn(v1, v2);
  int bestDist = 256, bestIdx = -1;
  const uint8_t* q = A.ml_desc + 32 * (long long)i;
  for (int j = 0; j < A.nl; j++) {
    const KeyLine68& kl = A.kl[j];
    const double ax = mxd - (double)kl.ptx, ay = myd - (double)kl.pty;
    const float distance = (float)(ax * ax + ay * ay);
    if (distance > r2) continue;
    float d2x = __fsub_rn(kl.startPointX, kl.endPointX), d2y = __fsub_rn(kl.startPointY, kl.endPointY);
    const float n2 = __fsqrt_rn(__fadd_rn(__fmul_rn(d2x, d2x), __fmul_rn(d2y, d2y)));
    d2x = __fdiv_rn(d2x, n2); d2y = __fdiv_rn(d2y, n2);
    const float cs = fabsf(__fadd_rn(__fmul_rn(d1x, d2x), __fmul_rn(d1y, d2y)));
    if (cs < 0.998f) continue;
    if (kl.octave < lvl - 1 || kl.octave > lvl) continue;
    if (j >= A.n_pdesc) continue;
    const int d = hamming256(q, A.pdesc + 32 * (long long)j);
    if (d < bestDist) { bestDist = d; bestIdx = j; }
  }
  A.best_idx[i] = bestIdx; A.best_dist[i] = bestDist;
}

namespace {
struct Stage {  // tiny RAII helper for the host-pointer wrappers
  std::vector<void*> ptrs;
  ~Stage() { for (void* p : ptrs) cudaFree(p); }
  template <typename T> T* up(const T* h, size_t n) {
    T* d = nullptr;
    if (cudaMalloc((void**)&d, std::max<size_t>(n, 1) * sizeof(T)) != cudaSuccess) return nullptr;
    ptrs.push_back(d);
    if (h && n) cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice);
    return d;
  }
  template <typename T> T* alloc(size_t n) { return up<T>(nullptr, n); }
};
template <typename T> int down(T* h, const T* d, size_t n) {
  PL_CUDA(cudaMemcpy(h, d, n * sizeof(T), cudaMemcpyDeviceToHost));
  return PL_OK;
}
}  // namespace

extern "C" int pl_descriptor_distance_batch(const uint8_t* a, const uint8_t* b, int n, int* out) {
  // convenience for tests: n independent 32-byte pairs, host pointers
  PL_ARG(a && b && out && n >= 0);
  int rc = require_device(); if (rc) return rc;
  Stage s;
  uint8_t* da = s.up(a, (size_t)n * 32); uint8_t* db = s.up(b, (size_t)n * 32);
  int one = 1; (void)one;
  std::vector<int> n1(1, n);
  // reuse k_bf_knn2 with cap2 = 1 per pair would be wasteful; do pairs as n batches of 1x1
  std::vector<int> ones(n, 1);
  int* dn = s.up(ones.data(), (size_t)n);
  int* idx = s.alloc<int>((size_t)n * 2); int* dist = s.alloc<int>((size_t)n * 2);
  PL_ARG(da && db && dn && idx && dist);
  if (n) { k_bf_knn2<<<dim3(1, n), 128>>>(da, dn, db, dn, 1, 1, idx, dist); PL_LAUNCH_CHECK(); }
  std::vector<int> hd((size_t)n * 2);
  rc = down(hd.data(), dist, (size_t)n * 2); if (rc) return rc;
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
  Stage s;
  int cap = std::max(n, 1);
  PLKeyPoint* dk = s.up(keys, (size_t)n); int* dn = s.up(&n, 1); float* db = s.up(bounds, 4);
  int* ds = s.alloc<int>(NCELL + 1); int* di = s.alloc<int>(cap);
  PL_ARG(dk && dn && db && ds && di);
  rc = pl_frame_assign_grid_dev(dk, dn, cap, 1, db, ds, di, nullptr); if (rc) return rc;
  rc = down(cell_start, ds, NCELL + 1); if (rc) return rc;
  return down(cell_items, di, (size_t)n);
}

extern "C" int pl_orb_search_for_initialization_dev(const PLKeyPoint* keys1, const uint8_t* desc1, const int* n1,
                                                    const PLKeyPoint* keys2, const uint8_t* desc2, const int* n2,
                                                    int cap, int B, const float* bounds, float* prev_matched,
                                                    int* matches12, int* nmatches, int window_size, float nnratio,
                                                    int check_orientation, int* scratch, void* stream) {
  PL_ARG(keys1 && desc1 && n1 && keys2 && desc2 && n2 && bounds && prev_matched && matches12 && nmatches && scratch);
  PL_ARG(cap > 0 && cap <= 6144 && B > 0);
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
  Stage s;
  int cap = std::max(std::max(n1, n2), 1);
  std::vector<PLKeyPoint> k1(cap), k2(cap);
  std::vector<uint8_t> d1((size_t)cap * 32), d2((size_t)cap * 32);
  std::vector<float> pm((size_t)cap * 2, 0.f);
  if (n1) { memcpy(k1.data(), keys1, n1 * sizeof(PLKeyPoint)); memcpy(d1.data(), desc1, (size_t)n1 * 32); memcpy(pm.data(), prev_matched, (size_t)n1 * 8); }
  if (n2) { memcpy(k2.data(), keys2, n2 * sizeof(PLKeyPoint)); memcpy(d2.data(), desc2, (size_t)n2 * 32); }
  PLKeyPoint* dk1 = s.up(k1.data(), cap); PLKeyPoint* dk2 = s.up(k2.data(), cap);
  uint8_t* dd1 = s.up(d1.data(), d1.size()); uint8_t* dd2 = s.up(d2.data(), d2.size());
  int* dn1 = s.up(&n1, 1); int* dn2 = s.up(&n2, 1); float* db = s.up(bounds, 4); float* dpm = s.up(pm.data(), pm.size());
  int* dm = s.alloc<int>(cap); int* dnm = s.alloc<int>(1); int* scr = s.alloc<int>((size_t)2 * cap);
  PL_ARG(dk1 && dk2 && dd1 && dd2 && dn1 && dn2 && db && dpm && dm && dnm && scr);
  rc = pl_orb_search_for_initialization_dev(dk1, dd1, dn1, dk2, dd2, dn2, cap, 1, db, dpm, dm, dnm, window_size, nnratio,
                                            check_orientation, scr, nullptr);
  if (rc) return rc;
  int nm = 0;
  rc = down(&nm, dnm, 1); if (rc) return rc;
  if (n1) { rc = down(matches12, dm, (size_t)n1); if (rc) return rc; rc = down(prev_matched, dpm, (size_t)n1 * 2); if (rc) return rc; }
  return nm;
}

extern "C" int pl_orb_search_by_projection_last(const PLKeyPoint* keys_cur, const uint8_t* desc_cur, int n_cur,
                                                const float* bounds, const float* Tcw, const float* K,
                                                const float* scale_factors, int nlevels, int n_last,
                                                const uint8_t* last_valid, const float* last_pos,
                                                const uint8_t* last_desc, const int* last_octave,
                                                const float* last_angle, float th, int check_orientation,
                                                const uint8_t* cur_preassigned, int* cur_match) {
  PL_ARG(keys_cur && desc_cur && bounds && Tcw && K && scale_factors && cur_match && n_cur >= 0 && n_cur <= 6144 && n_last >= 0);
  int rc = require_device(); if (rc) return rc;
  Stage s;
  const int cap = std::max(n_cur, 1), capl = std::max(n_last, 1);
  ProjLastArgs A;
  A.keys = s.up(keys_cur, n_cur); A.desc = s.up(desc_cur, (size_t)n_cur * 32); A.n = s.up(&n_cur, 1); A.cap = cap;
  A.bounds = s.up(bounds, 4); A.Tcw = s.up(Tcw, 16); A.K = s.up(K, 4); A.scaleFactors = s.up(scale_factors, nlevels);
  A.nlevels = nlevels; A.n_last = s.up(&n_last, 1); A.cap_last = capl;
  A.last_valid = s.up(last_valid, n_last); A.last_pos = s.up(last_pos, (size_t)n_last * 3);
  A.last_desc = s.up(last_desc, (size_t)n_last * 32); A.last_octave = s.up(last_octave, n_last);
  A.last_angle = s.up(last_angle, n_last);
  A.th = th; A.checkOri = check_orientation;
  A.preassigned = cur_preassigned ? s.up(cur_preassigned, n_cur) : nullptr;
  A.match = s.alloc<int>(cap); A.nmatches = s.alloc<int>(1);
  PL_ARG(A.keys && A.desc && A.match && A.nmatches && A.last_pos && A.last_desc);
  size_t sm = grid_smem_bytes(cap);
  PL_CUDA(cudaFuncSetAttribute(k_search_proj_last, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  k_search_proj_last<<<1, 32, sm>>>(A);
  PL_LAUNCH_CHECK();
  int nm = 0;
  rc = down(&nm, A.nmatches, 1); if (rc) return rc;
  if (n_cur) { rc = down(cur_match, A.match, (size_t)n_cur); if (rc) return rc; }
  return nm;
}

extern "C" int pl_orb_search_by_projection_points(const PLKeyPoint* keys, const uint8_t* desc, int n,
                                                  const float* bounds, const float* scale_factors, int nlevels,
                                                  int n_mp, const uint8_t* in_view, const float* proj,
                                                  const int* level, const float* view_cos, const uint8_t* mp_desc,
                                                  float th, float nnratio, const uint8_t* preassigned, int* match) {
  PL_ARG(keys && desc && bounds && scale_factors && match && n >= 0 && n_mp >= 0);
  int rc = require_device(); if (rc) return rc;
  Stage s;
  const int cap = std::max(n, 1), capm = std::max(n_mp, 1);
  ProjPointsArgs A;
  A.keys = s.up(keys, n); A.desc = s.up(desc, (size_t)n * 32); A.n = s.up(&n, 1); A.cap = cap;
  A.bounds = s.up(bounds, 4); A.scaleFactors = s.up(scale_factors, nlevels);
  A.n_mp = s.up(&n_mp, 1); A.cap_mp = capm; A.in_view = s.up(in_view, n_mp); A.proj = s.up(proj, (size_t)n_mp * 2);
  A.level = s.up(level, n_mp); A.view_cos = s.up(view_cos, n_mp); A.mp_desc = s.up(mp_desc, (size_t)n_mp * 32);
  A.th = th; A.nnratio = nnratio; A.preassigned = preassigned ? s.up(preassigned, n) : nullptr;
  A.match = s.alloc<int>(cap); A.nmatches = s.alloc<int>(1);
  PL_ARG(A.keys && A.desc && A.match && A.nmatches);
  size_t sm = grid_smem_bytes(cap);
  PL_CUDA(cudaFuncSetAttribute(k_search_proj_points, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  k_search_proj_points<<<1, 32, sm>>>(A);
  PL_LAUNCH_CHECK();
  int nm = 0;
  rc = down(&nm, A.nmatches, 1); if (rc) return rc;
  if (n) { rc = down(match, A.match, (size_t)n); if (rc) return rc; }
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
  PL_ARG(keys_cur && desc_cur && n_cur && bounds && Tcw && K && scale_factors && n_last && last_valid && last_pos && last_desc &&
         last_octave && last_angle && cur_match && nmatches && B >= 1 && cap >= 1 && cap <= 6144 && cap_last >= 1);
  ProjLastArgs A;
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
extern "C" int pl_orb_search_by_projection_points_dev(const PLKeyPoint* keys, const uint8_t* desc, const int* n, int cap, int B,
                                                      const float* bounds, const float* scale_factors, const int* n_mp, int cap_mp,
                                                      const uint8_t* in_view, const float* proj, const int* level, const float* view_cos,
                                                      const uint8_t* mp_desc, float th, float nnratio, const uint8_t* preassigned,
                                                      int* match, int* nmatches, void* stream) {
  PL_ARG(keys && desc && n && bounds && scale_factors && n_mp && in_view && proj && level && view_cos && mp_desc && match && nmatches &&
         B >= 1 && cap >= 1 && cap <= 6144 && cap_mp >= 1);
  ProjPointsArgs A;
  A.keys = keys; A.desc = desc; A.n = n; A.cap = cap; A.bounds = bounds; A.scaleFactors = scale_factors; A.n_mp = n_mp; A.cap_mp = cap_mp;
  A.in_view = in_view; A.proj = proj; A.level = level; A.view_cos = view_cos; A.mp_desc = mp_desc; A.th = th; A.nnratio = nnratio;
  A.preassigned = preassigned; A.match = match; A.nmatches = nmatches;
  const size_t sm = grid_smem_bytes(cap);
  PL_CUDA(cudaFuncSetAttribute(k_search_proj_points, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  k_search_proj_points<<<B, 32, sm, (cudaStream_t)stream>>>(A);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

extern "C" int pl_match_bf_knn2(const uint8_t* d1, int n1, const uint8_t* d2, int n2, int* idx, int* dist) {
  PL_ARG(d1 && d2 && idx && dist && n1 >= 0 && n2 >= 0);
  int rc = require_device(); if (rc) return rc;
  if (n1 == 0) return PL_OK;
  Stage s;
  uint8_t* a = s.up(d1, (size_t)n1 * 32); uint8_t* b = s.up(d2, (size_t)std::max(n2, 1) * 32);
  int* dn1 = s.up(&n1, 1); int* dn2 = s.up(&n2, 1);
  int* di = s.alloc<int>((size_t)n1 * 2); int* dd = s.alloc<int>((size_t)n1 * 2);
  PL_ARG(a && b && dn1 && dn2 && di && dd);
  k_bf_knn2<<<dim3((n1 + 3) / 4, 1), 128>>>(a, dn1, b, dn2, n1, std::max(n2, 1), di, dd);
  PL_LAUNCH_CHECK();
  rc = down(idx, di, (size_t)n1 * 2); if (rc) return rc;
  return down(dist, dd, (size_t)n1 * 2);
}

extern "C" int pl_lsd_search_double_dev(const uint8_t* d1, const int* n1, const uint8_t* d2, const int* n2, int cap1,
                                        int cap2, int B, float th, float nnratio, int mutual, int* matches,
                                        int* nmatches, void* stream) {
  PL_ARG(d1 && n1 && d2 && n2 && matches && nmatches && cap1 > 0 && cap2 > 0 && cap1 < 32000 && cap2 < 32000 && B > 0);
  size_t sm = (size_t)(cap1 + cap2 + 2 * std::max(cap1, cap2)) * sizeof(short);
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
  Stage s;
  const int c1 = std::max(n1, 1), c2 = std::max(n2, 1);
  uint8_t* a = s.up(d1, (size_t)n1 * 32); uint8_t* b = s.up(d2, (size_t)n2 * 32);
  if (n1 == 0) a = s.alloc<uint8_t>(32);
  if (n2 == 0) b = s.alloc<uint8_t>(32);
  int* dn1 = s.up(&n1, 1); int* dn2 = s.up(&n2, 1);
  int* dm = s.alloc<int>(c1); int* dnm = s.alloc<int>(1);
  PL_ARG(a && b && dn1 && dn2 && dm && dnm);
  rc = pl_lsd_search_double_dev(a, dn1, b, dn2, c1, c2, 1, th, nnratio, mutual, dm, dnm, nullptr); if (rc) return rc;
  int nm = 0;
  rc = down(&nm, dnm, 1); if (rc) return rc;
  if (n1) { rc = down(matches, dm, (size_t)n1); if (rc) return rc; }
  return nm;
}
extern "C" int pl_lsd_frame_bf_match(const uint8_t* d1, int n1, const uint8_t* d2, int n2, float th, float nnratio,
                                     int* matches) {
  return search_double_host(d1, n1, d2, n2, th, nnratio, 0, matches);
}
extern "C" int pl_lsd_search_double(const uint8_t* d1, int n1, const uint8_t* d2, int n2, float nnratio, int* matches) {
  return search_double_host(d1, n1, d2, n2, 50.f, nnratio, 1, matches);
}
// LSDmatcher::SearchForTriangulation(pKF1, pKF2, vMatchedPairs, isDouble) (src/LSDmatcher.cpp:727-776, the variant
// LocalMapping calls at LocalMapping.cc:961, th = TH_HIGH = 80) and its pair<> twin (:672-725, LocalMapping.cc:679, th = TH_LOW = 50,
// always mutual): FrameBFMatch both ways at th, optional mutual check, then pairs
// whose line already has a MapLine on either side are dropped (a few hundred flags: applied on the host).
extern "C" int pl_lsd_search_for_triangulation(const uint8_t* ldesc1, const uint8_t* has_ml1, int n1, const uint8_t* ldesc2,
                                               const uint8_t* has_ml2, int n2, float th, float nnratio, int is_double, int* matched_pairs) {
  PL_ARG(matched_pairs && n1 >= 0 && n2 >= 0 && (n1 == 0 || (ldesc1 && has_ml1)) && (n2 == 0 || (ldesc2 && has_ml2)));
  for (int i = 0; i < n1; i++) matched_pairs[i] = -1;
  if (n1 == 0 || n2 == 0) { int rc = require_device(); return rc ? rc : 0; }     // ldesc.rows == 0 -> return 0 (:738-739)
  int rc = search_double_host(ldesc1, n1, ldesc2, n2, th, nnratio, is_double ? 1 : 0, matched_pairs);
  if (rc < 0) return rc;
  int nm = 0;
  for (int i = 0; i < n1; i++) {
    const int j = matched_pairs[i];
    if (j < 0) continue;
    if (has_ml1[i] || has_ml2[j]) matched_pairs[i] = -1; else nm++;
  }
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
  Stage s;
  const int cap = std::max(n, 1);
  KeyLine68* dk = (KeyLine68*)s.up((const uint8_t*)keylines_un, (size_t)n * 68);
  float* db = s.up(bounds, 4);
  int* ds = s.alloc<int>(NCELL + 1); unsigned short* di = s.alloc<unsigned short>((size_t)cap * kMaxPath);
  unsigned short* dp = s.alloc<unsigned short>((size_t)cap * kMaxPath); unsigned short* dl = s.alloc<unsigned short>(cap);
  PL_ARG(dk && db && ds && di && dp && dl);
  k_line_grid<<<1, 32>>>(dk, n, db, ds, di, dp, dl);
  PL_LAUNCH_CHECK();
  rc = down(cell_start, ds, NCELL + 1); if (rc) return rc;
  const int tot = cell_start[NCELL];
  std::vector<unsigned short> tmp(std::max(tot, 1));
  rc = down(tmp.data(), di, (size_t)tot); if (rc) return rc;
  for (int i = 0; i < tot && i < cap_items; i++) cell_items[i] = tmp[i];
  return tot;
}

static int line_search_host(int variant, const void* kls, const double* lfunc, const uint8_t* desc, int n, const float* bounds,
                            int n_q, const uint8_t* q_valid, const float* q_proj, const uint8_t* q_desc, const float* q_length,
                            const float* q_view_cos, float th, float nnratio, const uint8_t* preassigned, int* match) {
  PL_ARG(kls && lfunc && desc && bounds && match && n >= 0 && n < 60000 && n_q >= 0);
  int rc = require_device(); if (rc) return rc;
  Stage s;
  const int cap = std::max(n, 1), capq = std::max(n_q, 1);
  LineSearchArgs A;
  A.kl = (const KeyLine68*)s.up((const uint8_t*)kls, (size_t)n * 68); A.lfunc = s.up(lfunc, (size_t)n * 3); A.desc = s.up(desc, (size_t)n * 32);
  A.n = s.up(&n, 1); A.cap = cap; A.bounds = s.up(bounds, 4);
  A.n_q = s.up(&n_q, 1); A.cap_q = capq; A.q_valid = s.up(q_valid, n_q); A.q_proj = s.up(q_proj, (size_t)n_q * 4);
  A.q_desc = s.up(q_desc, (size_t)n_q * 32);
  A.q_length = q_length ? s.up(q_length, n_q) : nullptr; A.q_view_cos = q_view_cos ? s.up(q_view_cos, n_q) : nullptr;
  A.th = th; A.nnratio = nnratio; A.variant = variant;
  A.preassigned = preassigned ? s.up(preassigned, n) : nullptr;
  A.match = s.alloc<int>(cap); A.nmatches = s.alloc<int>(1);
  A.g_start = s.alloc<int>(NCELL + 1); A.g_items = s.alloc<unsigned short>((size_t)cap * kMaxPath);
  A.g_path = s.alloc<unsigned short>((size_t)cap * kMaxPath); A.g_plen = s.alloc<unsigned short>(cap); A.g_first = s.alloc<int>(cap);
  PL_ARG(A.kl && A.lfunc && A.desc && A.match && A.nmatches && A.g_start && A.g_items && A.g_path && A.g_plen && A.g_first);
  k_line_search<<<1, 32>>>(A);
  PL_LAUNCH_CHECK();
  int nm = 0;
  rc = down(&nm, A.nmatches, 1); if (rc) return rc;
  if (n) { rc = down(match, A.match, (size_t)n); if (rc) return rc; }
  return nm;
}

extern "C" int pl_lsd_search_by_projection_last(const void* keylines_cur, const double* linefunc_cur, const uint8_t* desc_cur,
                                                int n_cur, const float* bounds, int n_last, const uint8_t* last_valid,
                                                const float* last_proj, const uint8_t* last_desc, const float* last_length,
                                                float th, const uint8_t* cur_preassigned, int* cur_match) {
  return line_search_host(0, keylines_cur, linefunc_cur, desc_cur, n_cur, bounds, n_last, last_valid, last_proj, last_desc,
                          last_length, nullptr, th, 0.f, cur_preassigned, cur_match);
}
extern "C" int pl_lsd_search_by_projection_lines(const void* keylines, const double* linefunc, const uint8_t* desc, int n,
                                                 const float* bounds, int n_ml, const uint8_t* in_view, const float* proj,
                                                 const float* view_cos, const uint8_t* ml_desc, float th, float nnratio,
                                                 const uint8_t* preassigned, int* match) {
  return line_search_host(1, keylines, linefunc, desc, n, bounds, n_ml, in_view, proj, ml_desc, nullptr, view_cos, th, nnratio,
                          preassigned, match);
}

extern "C" size_t pl_lsd_search_scratch_bytes(int cap, int B) {
  const size_t per = (size_t)(NCELL + 1) * 4 + (size_t)cap * kMaxPath * 2 * 2 + (size_t)cap * 2 + (size_t)cap * 4;
  return per * (size_t)B + 256;
}
/* variant 0 = SearchByProjection(CurrentFrame, LastFrame, th) (q_length = last lineLength), 1 = (F, vpMapLines, th) (q_view_cos) */
extern "C" int pl_lsd_search_by_projection_dev(int variant, const void* keylines, const double* linefunc, const uint8_t* desc, const int* n,
                                               int cap, int B, const float* bounds, const int* n_q, int cap_q, const uint8_t* q_valid,
                                               const float* q_proj, const uint8_t* q_desc, const float* q_length_or_view_cos, float th,
                                               float nnratio, const uint8_t* preassigned, int* match, int* nmatches, void* scratch,
                                               void* stream) {
  PL_ARG(keylines && linefunc && desc && n && bounds && n_q && q_valid && q_proj && q_desc && q_length_or_view_cos && match && nmatches &&
         scratch && B >= 1 && cap >= 1 && cap < 60000 && cap_q >= 1 && (variant == 0 || variant == 1));
  LineSearchArgs A;
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

// ------------------------------------------------------------------------------------------------ §8f.2 wrappers

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
  // the node merge of :760-884 (std::map order, lower_bound jumps) on the host: one query per keypoint of a shared node
  std::vector<int> q_idx1, q_s, q_e;
  for (int a = 0, b = 0; a < nn1 && b < nn2;) {
    if (fv1_nodes[a] == fv2_nodes[b]) {
      for (int i1 = fv1_start[a]; i1 < fv1_start[a + 1]; i1++) {
        PL_ARG(fv1_items[i1] >= 0 && fv1_items[i1] < n1);
        q_idx1.push_back(fv1_items[i1]); q_s.push_back(fv2_start[b]); q_e.push_back(fv2_start[b + 1]);
      }
      a++; b++;
    } else if (fv1_nodes[a] < fv2_nodes[b]) a++;
    else b++;
  }
  if (q_idx1.empty() || n1 == 0 || n2 == 0) return 0;
  const int nitems2 = fv2_start[nn2];
  for (int i = 0; i < nitems2; i++) PL_ARG(fv2_items[i] >= 0 && fv2_items[i] < n2);
  Stage s;
  TriArgs A;
  A.k1 = s.up(keys1_un, n1); A.k2 = s.up(keys2_un, n2); A.d1 = s.up(desc1, (size_t)n1 * 32); A.d2 = s.up(desc2, (size_t)n2 * 32);
  A.mp1 = s.up(has_mp1, n1); A.mp2 = s.up(has_mp2, n2);
  A.q_idx1 = s.up(q_idx1.data(), q_idx1.size()); A.q_s = s.up(q_s.data(), q_s.size()); A.q_e = s.up(q_e.data(), q_e.size());
  A.fv2_items = s.up(fv2_items, nitems2); A.nq = (int)q_idx1.size(); A.n1 = n1;
  memcpy(A.F, F12, sizeof(A.F));
  {  // epipole of camera 1 in image 2 (:729-737): C2 = R2w*Cw + t2w in cv::gemm's fp32 order
    float C2[3];
    for (int i = 0; i < 3; i++) C2[i] = ((R2w[3 * i] * Cw1[0] + R2w[3 * i + 1] * Cw1[1]) + R2w[3 * i + 2] * Cw1[2]) + t2w[i];
    const float invz = 1.0f / C2[2];
    A.ex = K2[0] * C2[0] * invz + K2[2]; A.ey = K2[1] * C2[1] * invz + K2[3];
  }
  A.scale2 = s.up(scale_factors2, nlevels); A.sigma2_2 = s.up(level_sigma2_2, nlevels); A.checkOri = check_orientation;
  A.matches12 = s.alloc<int>(n1); A.nmatches = s.alloc<int>(1); A.bins = s.alloc<unsigned char>(n1);
  PL_ARG(A.k1 && A.k2 && A.d1 && A.d2 && A.mp1 && A.mp2 && A.q_idx1 && A.q_s && A.q_e && A.fv2_items && A.scale2 && A.sigma2_2 &&
         A.matches12 && A.nmatches && A.bins);
  k_search_triangulation<<<1, 256>>>(A);
  PL_LAUNCH_CHECK();
  int nm = 0;
  rc = down(&nm, A.nmatches, 1); if (rc) return rc;
  rc = down(matches12, A.matches12, (size_t)n1); if (rc) return rc;
  return nm;
}

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
  Stage s;
  FuseArgs A;
  A.keys = s.up(keys_un, n); A.desc = s.up(desc, (size_t)n * 32); A.n = n;
  memcpy(A.bounds, bounds, 16); memcpy(A.T, Tcw, 64); memcpy(A.Ow, Ow, 12); memcpy(A.K, K, 16);
  A.scaleFactors = s.up(scale_factors, nlevels); A.invSigma2 = s.up(inv_level_sigma2, nlevels);
  A.logScaleFactor = log_scale_factor; A.nLevels = nlevels; A.n_mp = n_mp;
  A.skip = skip ? s.up(skip, n_mp) : nullptr; A.pos = s.up(pos, (size_t)n_mp * 3); A.normal = s.up(normal, (size_t)n_mp * 3);
  A.minDist = s.up(min_dist, n_mp); A.maxDist = s.up(max_dist, n_mp); A.mp_desc = s.up(mp_desc, (size_t)n_mp * 32); A.th = th;
  A.best_idx = s.alloc<int>(n_mp); A.best_dist = s.alloc<int>(n_mp);
  PL_ARG(A.keys && A.desc && A.scaleFactors && A.invSigma2 && A.pos && A.normal && A.minDist && A.maxDist && A.mp_desc && A.best_idx &&
         A.best_dist);
  const size_t sm = grid_smem_bytes(std::max(n, 1));
  PL_CUDA(cudaFuncSetAttribute(k_fuse_search, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  k_fuse_search<<<1, 32 * kFuseWarps, sm>>>(A);
  PL_LAUNCH_CHECK();
  rc = down(best_idx, A.best_idx, (size_t)n_mp); if (rc) return rc;
  return down(best_dist, A.best_dist, (size_t)n_mp);
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
  Stage s;
  BowArgs A;
  A.kK = s.up(keysKF_un, nKF); A.kF = s.up(keysF, nF); A.dK = s.up(descKF, (size_t)nKF * 32); A.dF = s.up(descF, (size_t)nF * 32);
  A.mpK = s.up(has_mp_kf, nKF);
  A.pairK_s = s.up(ks.data(), ks.size()); A.pairK_e = s.up(ke.data(), ke.size()); A.pairF_s = s.up(fs.data(), fs.size()); A.pairF_e = s.up(fe.data(), fe.size());
  A.itK = s.up(fvK_items, nitK); A.itF = s.up(fvF_items, nitF); A.npairs = (int)ks.size(); A.nF = nF;
  A.nnratio = nnratio; A.checkOri = check_orientation;
  A.mpF = has_mp_f ? s.up(has_mp_f, nF) : nullptr; A.strict = strict;
  A.matchesF = s.alloc<int>(nF); A.bins = s.alloc<unsigned char>(nF); A.nmatches = s.alloc<int>(1);
  PL_ARG(A.kK && A.kF && A.dK && A.dF && A.mpK && A.pairK_s && A.pairK_e && A.pairF_s && A.pairF_e && A.itK && A.itF && A.matchesF && A.bins && A.nmatches);
  k_search_by_bow<<<1, 32 * kBowWarps>>>(A);
  PL_LAUNCH_CHECK();
  int nm = 0;
  rc = down(&nm, A.nmatches, 1); if (rc) return rc;
  rc = down(matchesF, A.matchesF, (size_t)nF); if (rc) return rc;
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
  PL_ARG(keys_cur && desc_cur && bounds && Tcw && Ow && K && scale_factors && cur_match && n_cur >= 0 && n_cur <= 6144 && n_kf >= 0 && nlevels > 0);
  PL_ARG(n_kf == 0 || (kf_valid && pos && mp_desc && min_dist && max_dist && kf_angle));
  int rc = require_device(); if (rc) return rc;
  Stage s;
  const int cap = std::max(n_cur, 1), capl = std::max(n_kf, 1);
  ProjLastArgs A;
  A.keys = s.up(keys_cur, n_cur); A.desc = s.up(desc_cur, (size_t)n_cur * 32); A.n = s.up(&n_cur, 1); A.cap = cap;
  A.bounds = s.up(bounds, 4); A.Tcw = s.up(Tcw, 16); A.K = s.up(K, 4); A.scaleFactors = s.up(scale_factors, nlevels);
  A.nlevels = nlevels; A.n_last = s.up(&n_kf, 1); A.cap_last = capl;
  A.last_valid = s.up(kf_valid, n_kf); A.last_pos = s.up(pos, (size_t)n_kf * 3); A.last_desc = s.up(mp_desc, (size_t)n_kf * 32);
  A.last_octave = nullptr; A.last_angle = s.up(kf_angle, n_kf);
  A.th = th; A.checkOri = check_orientation;
  A.preassigned = cur_preassigned ? s.up(cur_preassigned, n_cur) : nullptr;
  A.match = s.alloc<int>(cap); A.nmatches = s.alloc<int>(1);
  A.kfMode = 1; A.maxDist = orb_dist; A.min_dist = s.up(min_dist, n_kf); A.max_dist = s.up(max_dist, n_kf);
  memcpy(A.Ow, Ow, 12); A.logSF = log_scale_factor;
  PL_ARG(A.keys && A.desc && A.match && A.nmatches && A.last_pos && A.last_desc && A.min_dist && A.max_dist && A.last_angle);
  size_t sm = grid_smem_bytes(cap);
  PL_CUDA(cudaFuncSetAttribute(k_search_proj_last, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  k_search_proj_last<<<1, 32, sm>>>(A);
  PL_LAUNCH_CHECK();
  int nm = 0;
  rc = down(&nm, A.nmatches, 1); if (rc) return rc;
  if (n_cur) { rc = down(cur_match, A.match, (size_t)n_cur); if (rc) return rc; }
  return nm;
}

extern "C" int pl_mappoint_distinctive_descriptors(const uint8_t* desc, const int* offsets, int n_mp, int* best_idx, uint8_t* out_desc) {
  PL_ARG(offsets && best_idx && n_mp >= 0 && (desc || n_mp == 0));
  int rc = require_device(); if (rc) return rc;
  if (n_mp == 0) return PL_OK;
  const int total = offsets[n_mp];
  PL_ARG(total >= 0);
  Stage s;
  const uint8_t* dd = s.up(desc, (size_t)total * 32); const int* doff = s.up(offsets, (size_t)n_mp + 1);
  int* db = s.alloc<int>(n_mp); uint8_t* dout = out_desc ? s.alloc<uint8_t>((size_t)n_mp * 32) : nullptr;
  PL_ARG(dd && doff && db);
  k_distinctive<<<(n_mp + kDistWarps - 1) / kDistWarps, 32 * kDistWarps>>>(dd, doff, n_mp, db, dout);
  PL_LAUNCH_CHECK();
  rc = down(best_idx, db, (size_t)n_mp); if (rc) return rc;
  if (out_desc) { rc = down(out_desc, dout, (size_t)n_mp * 32); if (rc) return rc; }
  return PL_OK;
}

extern "C" int pl_lsd_fuse_search(const void* keylines, int nl, const uint8_t* kf_point_desc, int n_pdesc, const float* bounds, const float* Tcw,
                                  const float* Ow, const float* K, float scale_line, float log_scale_factor_line, int n_ml,
                                  const uint8_t* skip, const double* pos, const double* normal, const float* min_dist, const float* max_dist,
                                  const uint8_t* ml_desc, float th, int* best_idx, int* best_dist, int* stop_at) {
  PL_ARG(bounds && Tcw && Ow && K && best_idx && best_dist && stop_at && nl >= 0 && n_ml >= 0 && n_pdesc >= 0);
  PL_ARG(n_ml == 0 || (skip && pos && normal && min_dist && max_dist && ml_desc));
  int rc = require_device(); if (rc) return rc;
  *stop_at = n_ml;
  if (n_ml == 0) return PL_OK;
  Stage s;
  LineFuseArgs A;
  A.kl = reinterpret_cast<const KeyLine68*>(s.up(static_cast<const uint8_t*>(keylines), (size_t)nl * 68)); A.nl = nl;
  A.pdesc = s.up(kf_point_desc, (size_t)n_pdesc * 32); A.n_pdesc = n_pdesc;
  memcpy(A.bounds, bounds, 16); memcpy(A.T, Tcw, 64); memcpy(A.Ow, Ow, 12); memcpy(A.K, K, 16);
  A.scale_line = scale_line; A.logScaleFactorLine = log_scale_factor_line; A.n_ml = n_ml;
  A.skip = s.up(skip, n_ml); A.pos = s.up(pos, (size_t)n_ml * 6); A.normal = s.up(normal, (size_t)n_ml * 3);
  A.minDist = s.up(min_dist, n_ml); A.maxDist = s.up(max_dist, n_ml); A.ml_desc = s.up(ml_desc, (size_t)n_ml * 32); A.th = th;
  A.best_idx = s.alloc<int>(n_ml); A.best_dist = s.alloc<int>(n_ml); A.stop_at = s.up(stop_at, 1);
  PL_ARG(A.kl && A.pdesc && A.skip && A.pos && A.normal && A.minDist && A.maxDist && A.ml_desc && A.best_idx && A.best_dist && A.stop_at);
  k_lsd_fuse_search<<<(n_ml + 127) / 128, 128>>>(A);
  PL_LAUNCH_CHECK();
  rc = down(best_idx, A.best_idx, (size_t)n_ml); if (rc) return rc;
  rc = down(best_dist, A.best_dist, (size_t)n_ml); if (rc) return rc;
  rc = down(stop_at, A.stop_at, 1); if (rc) return rc;
  for (int i = *stop_at; i < n_ml; i++) { best_idx[i] = -1; best_dist[i] = 256; }     // never reached by the reference's loop
  return PL_OK;
}
