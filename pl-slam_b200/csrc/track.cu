// Tracking::TrackLocalMapWithLines (src/Tracking.cc:1491-1562) for a batch of frames against a map that stays on the device:
//   k_track_held             the map indices each frame already holds, sorted (SearchLocalPoints / Lines step 1, :1754-1766)
//   k_track_frustum_points   Frame::isInFrustum(pMP, 0.5) per (frame, local-list entry) unless the frame holds the point (:1769-1786)
//   k_track_frustum_lines    Frame::isInFrustum(pML, 0.5) likewise (:1825-1842)
//   k_search_proj_points     ORBmatcher(0.8).SearchByProjection(F, mvpLocalMapPoints, th)   (match.cu, per-frame th)
//   k_line_search            LSDmatcher().SearchByProjection(F, mvpLocalMapLines, th)       (match.cu, variant 1)
//   k_track_build            the PoseOptimization problem in feature order (Optimizer.cc:640-841)
//   k_pose_opt               Optimizer::PoseOptimization (lm.cu, mode 0, unchanged)
//   k_track_writeback        masks per feature, mnMatchesInliers / mnLineMatchesInliers and the return value (:1504-1561)
// The searches read the map's descriptors through the per-entry map index (desc_row) rather than a [B][cap_local][32] gather.
#include "common.cuh"
#include "frustum.cuh"
#include "search.cuh"
#include <limits.h>
#include <algorithm>
#include <vector>

struct PLMap {
  int n_points = 0, n_lines = 0;
  pl::DevBuf<float> pt_pos, pt_normal, pt_min, pt_max;
  pl::DevBuf<uint8_t> pt_desc;
  pl::DevBuf<double> ln_pos, ln_normal;
  pl::DevBuf<float> ln_min, ln_max;
  pl::DevBuf<uint8_t> ln_desc;
  pl::DevBuf<int> flag;           // sticky: [0] an index outside the map was met, [1] a local list outgrew its capacity
  pl::Stream stream;
  // the keyframe graph (pl_map_set_keyframes; NULL before the first); CSR rows per keyframe, obs per map point
  struct KeyframeGraph {
    int n_kf = 0;
    pl::DevBuf<float> Tcw, Twc;
    pl::DevBuf<uint8_t> bad;
    pl::DevBuf<int> parent, pt_off, pt, ln_off, ln, cov_off, cov, child_off, child, obs_off, obs;
  };
  std::unique_ptr<KeyframeGraph> kf;
};

namespace pl {
constexpr int kTrackThreads = 256;

// Sorted map indices of the matches frame b holds (INT_MAX padded) and the pre-assigned flags the searches take.  seen (may be
// NULL): the entries TrackWithMotionModel discarded as outliers of feature i (-1 none); a feature without a held match contributes
// its seen entry to the sorted list (skipped by the frustum test) but is not pre-assigned.
__global__ void __launch_bounds__(kTrackThreads) k_track_held(const int* __restrict__ map_in, const int* __restrict__ seen,
                                                              const int* __restrict__ n, int cap, int n_map, int pow2,
                                                              int* __restrict__ held, int* __restrict__ n_held,
                                                              uint8_t* __restrict__ pre, int* __restrict__ flag) {
  extern __shared__ int s[];
  __shared__ int cnt;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int N = min(n[b], cap);
  const long long o = (long long)b * cap;
  if (tid == 0) cnt = 0;
  __syncthreads();
  for (int i = tid; i < pow2; i += kTrackThreads) {
    int v = INT_MAX;
    uint8_t p = 0;
    if (i < N) {
      const int m = map_in ? map_in[o + i] : -1;
      if (m >= n_map) atomicOr(flag, 1);
      else if (m >= 0) { v = m; p = 1; }
      else if (seen) {
        const int q = seen[o + i];
        if (q >= n_map) atomicOr(flag, 1);
        else if (q >= 0) v = q;
      }
      if (v != INT_MAX) atomicAdd(&cnt, 1);
    }
    s[i] = v;
    if (i < cap) pre[o + i] = p;
  }
  __syncthreads();
  for (int k = 2; k <= pow2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < pow2; i += kTrackThreads) {
        const int p = i ^ j;
        if (p > i) {
          const int a = s[i], c = s[p];
          if ((a > c) == ((i & k) == 0)) { s[i] = c; s[p] = a; }
        }
      }
      __syncthreads();
    }
  for (int i = tid; i < cap; i += kTrackThreads) held[o + i] = s[i];
  if (tid == 0) n_held[b] = cnt;
}

__device__ __forceinline__ bool held_by(const int* held, int nh, int m) {
  int lo = 0, hi = nh;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (held[mid] < m) lo = mid + 1; else hi = mid; }
  return lo < nh && held[lo] == m;
}

struct TrackFrustumArgs {
  const float* Tcw0; const float* K; const float* bounds; float logScaleFactor; int nlevels;
  const int* off; const int* cnt; const int* index; int n_map; int cap_local;
  const int* held; const int* n_held; int cap;            // held matches, [B][cap] rows
  uint8_t* in_view; float* proj; int* level; float* view_cos; int* row; int* flag;
};
__device__ __forceinline__ int frustum_entry(const TrackFrustumArgs& A, int b, int i, FrustumArgs& F) {
  const int m = A.index[A.off[b] + i];
  if (m < 0 || m >= A.n_map) { atomicOr(A.flag, 1); return -1; }
  A.row[(long long)b * A.cap_local + i] = m;
  if (held_by(A.held + (long long)b * A.cap, A.n_held[b], m)) return -1;   // mnLastFrameSeen == mnId: mbTrackInView stays false
  for (int k = 0; k < 16; k++) F.T[k] = A.Tcw0[16 * b + k];
  camera_center(F.T, F.Ow);
  for (int k = 0; k < 4; k++) { F.K[k] = A.K[4 * b + k]; F.bounds[k] = A.bounds[k]; }
  F.logScaleFactor = A.logScaleFactor; F.viewingCosLimit = 0.5f; F.nScaleLevels = A.nlevels; F.n = 0;
  return m;
}
__global__ void __launch_bounds__(128) k_track_frustum_points(TrackFrustumArgs A, const float* __restrict__ pos, const float* __restrict__ normal,
                                                              const float* __restrict__ minD, const float* __restrict__ maxD) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.cap_local) return;
  const long long o = (long long)b * A.cap_local + i;
  A.in_view[o] = 0; A.proj[2 * o] = A.proj[2 * o + 1] = 0; A.level[o] = 0; A.view_cos[o] = 0; A.row[o] = 0;
  if (i >= A.cnt[b]) return;
  FrustumArgs F;
  const int m = frustum_entry(A, b, i, F);
  if (m < 0) return;
  float u, v, vc; int l;
  if (!frustum_point(F, pos + 3 * (long long)m, normal + 3 * (long long)m, minD[m], maxD[m], u, v, l, vc)) return;
  A.in_view[o] = 1; A.proj[2 * o] = u; A.proj[2 * o + 1] = v; A.level[o] = l; A.view_cos[o] = vc;
}
__global__ void __launch_bounds__(128) k_track_frustum_lines(TrackFrustumArgs A, const double* __restrict__ pos, const double* __restrict__ normal,
                                                             const float* __restrict__ minD, const float* __restrict__ maxD) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.cap_local) return;
  const long long o = (long long)b * A.cap_local + i;
  A.in_view[o] = 0; for (int k = 0; k < 4; k++) A.proj[4 * o + k] = 0; A.level[o] = 0; A.view_cos[o] = 0; A.row[o] = 0;
  if (i >= A.cnt[b]) return;
  FrustumArgs F;
  const int m = frustum_entry(A, b, i, F);
  if (m < 0) return;
  float pr[4], vc; int l;
  if (!frustum_line(F, pos + 6 * (long long)m, normal + 3 * (long long)m, minD[m], maxD[m], pr, l, vc)) return;
  A.in_view[o] = 1; for (int k = 0; k < 4; k++) A.proj[4 * o + k] = pr[k];
  A.level[o] = l; A.view_cos[o] = vc;
}

// Exclusive block scan of one flag per thread; returns the flag's slot, adds the block's total to *base (all threads).
__device__ __forceinline__ int block_slot(bool f, int* warp_tot, int& base) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, f);
  if (lane == 0) warp_tot[w] = __popc(bal);
  __syncthreads();
  int before = base, total = 0;
  for (int k = 0; k < kTrackThreads / 32; k++) { if (k < w) before += warp_tot[k]; total += warp_tot[k]; }
  __syncthreads();
  base += total;
  return before + __popc(bal & ((1u << lane) - 1u));
}

struct TrackBuildArgs {
  const PLKeyPoint* keys; const int* n; int cap; const float* inv_sigma2;
  const double* lfunc; const int* nl; int capL;
  const int* pmap_in; const int* lmap_in;               // may be NULL
  const int* pmatch; const int* lmatch;                 // search results (-2 held, -1, local position)
  const int* prow; int cap_lp; const int* lrow; int cap_ll;
  const float* map_pt; const double* map_ln;
  int* point_map; int* line_map; int* pslot; int* lslot;
  int* np; float* obs; float* w; float* X; int* nlp; double* lf; double* lX;
  // TrackWithMotionModel (NULL for the local-map step): frames with use_alt[b] take their point matches from pmatch_alt (the
  // retry at 2 th), and frames with solve[b] == 0 (the early return) build an empty problem; point_map / line_map are written
  const uint8_t* use_alt = nullptr; const int* pmatch_alt = nullptr; const uint8_t* solve = nullptr;
};
// mvpMapPoints / mvpMapLines after the searches, and the problem in feature order: points then lines
__global__ void __launch_bounds__(kTrackThreads) k_track_build(TrackBuildArgs A) {
  __shared__ int warp_tot[kTrackThreads / 32];
  const int b = blockIdx.x;
  const bool solve = !A.solve || A.solve[b];
  {
    const int N = min(A.n[b], A.cap);
    const long long o = (long long)b * A.cap;
    const int* pmatch = A.use_alt && A.use_alt[b] ? A.pmatch_alt : A.pmatch;
    int base = 0;
    for (int c = 0; c < A.cap; c += kTrackThreads) {
      const int i = c + threadIdx.x;
      int fm = -1;
      if (i < N) {
        const int mm = pmatch[o + i];
        fm = mm == -2 ? A.pmap_in[o + i] : mm >= 0 ? A.prow[(long long)b * A.cap_lp + mm] : -1;
      }
      const bool use = solve && fm >= 0;
      const int slot = block_slot(use, warp_tot, base);
      if (i < A.cap) { A.point_map[o + i] = fm; A.pslot[o + i] = use ? slot : -1; }
      if (use) {
        const PLKeyPoint k = A.keys[o + i];
        const long long s = o + slot;
        A.obs[2 * s] = k.x; A.obs[2 * s + 1] = k.y; A.w[s] = A.inv_sigma2[k.octave];
        for (int d = 0; d < 3; d++) A.X[3 * s + d] = A.map_pt[3 * (long long)fm + d];
      }
    }
    if (threadIdx.x == 0) A.np[b] = base;
  }
  {
    const int N = min(A.nl[b], A.capL);
    const long long o = (long long)b * A.capL;
    int base = 0;
    for (int c = 0; c < A.capL; c += kTrackThreads) {
      const int i = c + threadIdx.x;
      int fm = -1;
      if (i < N) {
        const int mm = A.lmatch[o + i];
        fm = mm == -2 ? A.lmap_in[o + i] : mm >= 0 ? A.lrow[(long long)b * A.cap_ll + mm] : -1;
      }
      const bool use = solve && fm >= 0;
      const int slot = block_slot(use, warp_tot, base);
      if (i < A.capL) { A.line_map[o + i] = fm; A.lslot[o + i] = use ? slot : -1; }
      if (use) {
        const long long s = o + slot;
        for (int d = 0; d < 3; d++) A.lf[3 * s + d] = A.lfunc[3 * (o + i) + d];
        for (int d = 0; d < 6; d++) A.lX[6 * s + d] = A.map_ln[6 * (long long)fm + d];
      }
    }
    if (threadIdx.x == 0) A.nlp[b] = base;
  }
}

// mvbOutlier / mvbLineOutlier per feature, the inlier counts (mbOnlyTracking: every non-outlier match) and the return value
__global__ void __launch_bounds__(kTrackThreads) k_track_writeback(const int* __restrict__ pslot, const uint8_t* __restrict__ pout, int cap,
                                                                   const int* __restrict__ lslot, const uint8_t* __restrict__ lout, int capL,
                                                                   const int* __restrict__ min_inliers, uint8_t* __restrict__ point_outlier,
                                                                   uint8_t* __restrict__ line_outlier, int* __restrict__ inliers,
                                                                   const uint8_t* solve, const int* ok_in, int* ok) {
  __shared__ int cnt[2];
  const int b = blockIdx.x;
  if (threadIdx.x < 2) cnt[threadIdx.x] = 0;
  __syncthreads();
  int np = 0, nl = 0;
  for (int i = threadIdx.x; i < cap; i += kTrackThreads) {
    const long long o = (long long)b * cap + i;
    const int s = pslot[o];
    const uint8_t f = s >= 0 ? pout[(long long)b * cap + s] : 0;
    point_outlier[o] = f;
    np += s >= 0 && !f;
  }
  for (int i = threadIdx.x; i < capL; i += kTrackThreads) {
    const long long o = (long long)b * capL + i;
    const int s = lslot[o];
    const uint8_t f = s >= 0 ? lout[(long long)b * capL + s] : 0;
    line_outlier[o] = f;
    nl += s >= 0 && !f;
  }
  np = warp_sum(np); nl = warp_sum(nl);
  if ((threadIdx.x & 31) == 0) { atomicAdd(&cnt[0], np); atomicAdd(&cnt[1], nl); }
  __syncthreads();
  if (threadIdx.x == 0) {
    inliers[2 * b] = cnt[0]; inliers[2 * b + 1] = cnt[1];
    // < 50 shortly after a relocalisation, < 30 otherwise: false (:1555-1561); a frame gated off keeps bOK (:476)
    if (!solve || solve[b]) ok[b] = cnt[0] >= min_inliers[b];
    else ok[b] = ok_in ? ok_in[b] : 1;
  }
}

// ---- scratch layout (one carve for the size query and the call)
struct TrackScratch {
  int *tab;                 // [5][B]: pt_off, pt_cnt, ln_off, ln_cnt, min_inliers
  float* th;                // [B]
  int *pheld, *nph, *lheld, *nlh;
  uint8_t *ppre, *lpre;
  uint8_t* piv; float* pproj; int* plev; float* pvc; int* prow;
  uint8_t* liv; float* lproj; int* llev; float* lvc; int* lrow;
  int *pmatch, *pnm, *lmatch, *lnm; void* lsd;
  int *np, *nl; float *obs, *w, *X; double *lf, *lX;
  int *pslot, *lslot; uint8_t *pout, *lout; int *inl, *its; double* lm;
};
static size_t carve(void* base, int B, int cap, int capL, int cLP, int cLL, TrackScratch* t) {
  size_t off = 0;
  auto take = [&](size_t bytes) { void* p = base ? (char*)base + off : nullptr; off += (bytes + 15) / 16 * 16; return p; };
  const size_t b = B, k = cap, l = capL, lp = cLP, ll = cLL;
  TrackScratch s;
  s.tab = (int*)take(5 * b * 4); s.th = (float*)take(b * 4);
  s.pheld = (int*)take(b * k * 4); s.nph = (int*)take(b * 4); s.lheld = (int*)take(b * l * 4); s.nlh = (int*)take(b * 4);
  s.ppre = (uint8_t*)take(b * k); s.lpre = (uint8_t*)take(b * l);
  s.piv = (uint8_t*)take(b * lp); s.pproj = (float*)take(b * lp * 8); s.plev = (int*)take(b * lp * 4); s.pvc = (float*)take(b * lp * 4);
  s.prow = (int*)take(b * lp * 4);
  s.liv = (uint8_t*)take(b * ll); s.lproj = (float*)take(b * ll * 16); s.llev = (int*)take(b * ll * 4); s.lvc = (float*)take(b * ll * 4);
  s.lrow = (int*)take(b * ll * 4);
  s.pmatch = (int*)take(b * k * 4); s.pnm = (int*)take(b * 4); s.lmatch = (int*)take(b * l * 4); s.lnm = (int*)take(b * 4);
  s.lsd = take(pl_lsd_search_scratch_bytes(capL, B));
  s.np = (int*)take(b * 4); s.nl = (int*)take(b * 4);
  s.obs = (float*)take(b * k * 8); s.w = (float*)take(b * k * 4); s.X = (float*)take(b * k * 12);
  s.lf = (double*)take(b * l * 24); s.lX = (double*)take(b * l * 48);
  s.pslot = (int*)take(b * k * 4); s.lslot = (int*)take(b * l * 4); s.pout = (uint8_t*)take(b * k); s.lout = (uint8_t*)take(b * l);
  s.inl = (int*)take(b * 4); s.its = (int*)take(b * 4);
  s.lm = (double*)take(pl_pose_optimization_scratch_doubles(B, cap, capL) * 8);
  if (t) *t = s;
  return off;
}
static int pow2_at_least(int n) { int p = 1; while (p < n) p <<= 1; return p; }
static int track_local_map_run(PLMap* map, const PLTrackFrames* F, const int* point_seen, const int* line_seen, const int* pt_index,
                               int cLP, const int* ln_index, int cLL, const uint8_t* solve, const int* ok_in, const PLTrackOut* O,
                               const TrackScratch& s, cudaStream_t st);
}  // namespace pl
using namespace pl;

// n elements of src in a new buffer of max(n, room) elements
template <typename T> static int upload(DevBuf<T>& d, const void* src, size_t n, size_t room) {
  PL_TRY(d.alloc(std::max(n, room)));
  if (n) PL_CUDA(cudaMemcpy(d, src, n * sizeof(T), cudaMemcpyHostToDevice));
  return PL_OK;
}
extern "C" void pl_map_destroy(PLMap* m) {
  if (!m) return;
  delete m;
}
extern "C" int pl_map_create(const PLMapDesc* d, PLMap** out) {
  PL_ARG(d && out && d->n_points >= 0 && d->n_lines >= 0);
  PL_ARG(d->n_points == 0 || (d->pt_pos && d->pt_normal && d->pt_min_dist && d->pt_max_dist && d->pt_desc));
  PL_ARG(d->n_lines == 0 || (d->ln_pos && d->ln_normal && d->ln_min_dist && d->ln_max_dist && d->ln_desc));
  int rc = require_device(); if (rc) return rc;
  std::unique_ptr<PLMap> m(new PLMap);
  m->n_points = d->n_points; m->n_lines = d->n_lines;
  // a map without points or lines still gets one entry of each array
  const size_t P = d->n_points, L = d->n_lines;
  PL_TRY(upload(m->pt_pos, d->pt_pos, P * 3, 3)); PL_TRY(upload(m->pt_normal, d->pt_normal, P * 3, 3));
  PL_TRY(upload(m->pt_min, d->pt_min_dist, P, 1)); PL_TRY(upload(m->pt_max, d->pt_max_dist, P, 1)); PL_TRY(upload(m->pt_desc, d->pt_desc, P * 32, 32));
  PL_TRY(upload(m->ln_pos, d->ln_pos, L * 6, 6)); PL_TRY(upload(m->ln_normal, d->ln_normal, L * 3, 3));
  PL_TRY(upload(m->ln_min, d->ln_min_dist, L, 1)); PL_TRY(upload(m->ln_max, d->ln_max_dist, L, 1)); PL_TRY(upload(m->ln_desc, d->ln_desc, L * 32, 32));
  PL_TRY(m->flag.alloc(2));
  PL_CUDA(cudaMemset(m->flag, 0, 8));
  PL_TRY(m->stream.create(cudaStreamNonBlocking));
  *out = m.release();
  return PL_OK;
}
extern "C" int pl_map_check_indices(PLMap* m) {
  PL_ARG(m);
  int f = 0;
  PL_CUDA(cudaDeviceSynchronize());
  PL_CUDA(cudaMemcpy(&f, m->flag, 4, cudaMemcpyDeviceToHost));
  if (!f) return PL_OK;
  PL_CUDA(cudaMemset(m->flag, 0, 4));
  set_error("track: a local-map entry, a held or discarded match or a last-frame match named an index outside the map");
  return PL_ERR_ARG;
}

extern "C" size_t pl_track_local_map_scratch_bytes(int B, int cap_points, int cap_lines, int cap_local_points, int cap_local_lines) {
  if (B < 1 || cap_points < 1 || cap_lines < 1) return 0;
  return carve(nullptr, B, cap_points, cap_lines, std::max(cap_local_points, 1), std::max(cap_local_lines, 1), nullptr);
}

extern "C" int pl_track_local_map_dev(PLMap* map, const PLTrackFrames* F, const PLTrackLocal* L, const PLTrackOut* O, void* scratch,
                                      void* stream_) {
  return pl_track_local_map_seen_dev(map, F, nullptr, nullptr, L, O, scratch, stream_);
}
extern "C" int pl_track_local_map_seen_dev(PLMap* map, const PLTrackFrames* F, const int* point_seen, const int* line_seen,
                                           const PLTrackLocal* L, const PLTrackOut* O, void* scratch, void* stream_) {
  PL_ARG(map && F && L && O && scratch);
  const int B = F->B, cap = F->cap_points, capL = F->cap_lines;
  // cap_points: the point search's limit; cap_lines: k_track_held sorts a frame's held lines in shared memory (4 B per
  // next_pow2(cap_lines) entries), which fits an SM's 227 KB up to 32768
  PL_ARG(B >= 1 && cap >= 1 && cap <= 6144 && capL >= 1 && capL <= 32768 && F->nlevels >= 1);
  PL_ARG(F->keys_un && F->desc && F->n && F->keylines && F->line_func && F->line_desc && F->nl && F->bounds && F->scale_factors &&
         F->inv_level_sigma2 && F->Tcw0 && F->K);
  PL_ARG(L->pt_offset && L->pt_count && L->ln_offset && L->ln_count && L->frames_since_reloc && L->cap_local_points >= 0 &&
         L->cap_local_lines >= 0 && L->n_pt_index >= 0 && L->n_ln_index >= 0);
  PL_ARG(O->Tcw && O->point_map && O->point_outlier && O->line_map && O->line_outlier && O->inliers && O->ok);
  const int cLP = std::max(L->cap_local_points, 1), cLL = std::max(L->cap_local_lines, 1);
  // host-side checks before anything is enqueued
  std::vector<int> tab((size_t)5 * B);
  std::vector<float> th(B);
  bool any_pt = false, any_ln = false;
  for (int b = 0; b < B; b++) {
    if (L->pt_count[b] < 0 || L->pt_count[b] > L->cap_local_points || L->ln_count[b] < 0 || L->ln_count[b] > L->cap_local_lines) {
      set_error("frame %d has %d local points and %d local lines; the capacities are %d and %d", b, L->pt_count[b], L->ln_count[b],
                L->cap_local_points, L->cap_local_lines);
      return PL_ERR_ARG;
    }
    if (L->pt_offset[b] < 0 || (long long)L->pt_offset[b] + L->pt_count[b] > L->n_pt_index || L->ln_offset[b] < 0 ||
        (long long)L->ln_offset[b] + L->ln_count[b] > L->n_ln_index) {
      set_error("frame %d's local lists [%d, +%d) / [%d, +%d) leave the index arrays of %d points / %d lines", b, L->pt_offset[b],
                L->pt_count[b], L->ln_offset[b], L->ln_count[b], L->n_pt_index, L->n_ln_index);
      return PL_ERR_ARG;
    }
    any_pt |= L->pt_count[b] > 0; any_ln |= L->ln_count[b] > 0;
    tab[b] = L->pt_offset[b]; tab[B + b] = L->pt_count[b]; tab[2 * B + b] = L->ln_offset[b]; tab[3 * B + b] = L->ln_count[b];
    tab[4 * B + b] = L->frames_since_reloc[b] < L->max_frames ? 50 : 30;
    th[b] = L->frames_since_reloc[b] < 2 ? 5.0f : 1.0f;   // if(mCurrentFrame.mnId < mnLastRelocFrameId + 2) th = 5
  }
  PL_ARG(!any_pt || L->pt_index);
  PL_ARG(!any_ln || L->ln_index);
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : map->stream;
  TrackScratch s;
  carve(scratch, B, cap, capL, cLP, cLL, &s);
  // pageable sources: the copies are staged before cudaMemcpyAsync returns, so the vectors may go
  PL_CUDA(cudaMemcpyAsync(s.tab, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(s.th, th.data(), th.size() * 4, cudaMemcpyHostToDevice, st));
  return track_local_map_run(map, F, point_seen, line_seen, L->pt_index, cLP, L->ln_index, cLL, nullptr, nullptr, O, s, st);
}

namespace pl {
// The body of the local-map step once the per-frame table is on the device: s.tab = [5][B] {pt_off, pt_cnt, ln_off, ln_cnt,
// min_inliers} and s.th [B].  solve (may be NULL): frames with solve[b] == 0 build an empty problem, keep their pose and matches,
// and get ok = ok_in[b] (1 if ok_in is NULL).
static int track_local_map_run(PLMap* map, const PLTrackFrames* F, const int* point_seen, const int* line_seen, const int* pt_index,
                               int cLP, const int* ln_index, int cLL, const uint8_t* solve, const int* ok_in, const PLTrackOut* O,
                               const TrackScratch& s, cudaStream_t st) {
  const int B = F->B, cap = F->cap_points, capL = F->cap_lines;
  const int* d_poff = s.tab; const int* d_pcnt = s.tab + B; const int* d_loff = s.tab + 2 * B; const int* d_lcnt = s.tab + 3 * B;
  const int* d_min_inl = s.tab + 4 * B;
  // outputs the caller asked for are the working arrays themselves
  uint8_t* piv = O->pt_in_view ? O->pt_in_view : s.piv; float* pproj = O->pt_proj ? O->pt_proj : s.pproj;
  int* plev = O->pt_level ? O->pt_level : s.plev; float* pvc = O->pt_view_cos ? O->pt_view_cos : s.pvc;
  uint8_t* liv = O->ln_in_view ? O->ln_in_view : s.liv; float* lproj = O->ln_proj ? O->ln_proj : s.lproj;
  int* llev = O->ln_level ? O->ln_level : s.llev; float* lvc = O->ln_view_cos ? O->ln_view_cos : s.lvc;
  int* pmatch = O->pt_match ? O->pt_match : s.pmatch; int* lmatch = O->ln_match ? O->ln_match : s.lmatch;
  int* np = O->prob_n_points ? O->prob_n_points : s.np; int* nl = O->prob_n_lines ? O->prob_n_lines : s.nl;
  float* obs = O->prob_pt_obs ? O->prob_pt_obs : s.obs; float* w = O->prob_pt_inv_sigma2 ? O->prob_pt_inv_sigma2 : s.w;
  float* X = O->prob_pt_Xw ? O->prob_pt_Xw : s.X;
  double* lf = O->prob_line_func ? O->prob_line_func : s.lf; double* lX = O->prob_line_Xw ? O->prob_line_Xw : s.lX;

  // 1. matches already held
  const int p2 = pow2_at_least(cap), l2 = pow2_at_least(capL);
  PL_CUDA(cudaFuncSetAttribute(k_track_held, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(std::max(p2, l2) * 4)));
  k_track_held<<<B, kTrackThreads, p2 * 4, st>>>(F->point_map_in, point_seen, F->n, cap, map->n_points, p2, s.pheld, s.nph, s.ppre,
                                                  map->flag);
  PL_LAUNCH_CHECK();
  k_track_held<<<B, kTrackThreads, l2 * 4, st>>>(F->line_map_in, line_seen, F->nl, capL, map->n_lines, l2, s.lheld, s.nlh, s.lpre,
                                                  map->flag);
  PL_LAUNCH_CHECK();
  // 2. isInFrustum(., 0.5) per (frame, local entry)
  TrackFrustumArgs A;
  A.Tcw0 = F->Tcw0; A.K = F->K; A.bounds = F->bounds; A.logScaleFactor = F->log_scale_factor; A.nlevels = F->nlevels; A.flag = map->flag;
  A.off = d_poff; A.cnt = d_pcnt; A.index = pt_index; A.n_map = map->n_points; A.cap_local = cLP; A.held = s.pheld; A.n_held = s.nph;
  A.cap = cap; A.in_view = piv; A.proj = pproj; A.level = plev; A.view_cos = pvc; A.row = s.prow;
  k_track_frustum_points<<<dim3((cLP + 127) / 128, B), 128, 0, st>>>(A, map->pt_pos, map->pt_normal, map->pt_min, map->pt_max);
  PL_LAUNCH_CHECK();
  A.off = d_loff; A.cnt = d_lcnt; A.index = ln_index; A.n_map = map->n_lines; A.cap_local = cLL; A.held = s.lheld; A.n_held = s.nlh;
  A.cap = capL; A.in_view = liv; A.proj = lproj; A.level = llev; A.view_cos = lvc; A.row = s.lrow;
  k_track_frustum_lines<<<dim3((cLL + 127) / 128, B), 128, 0, st>>>(A, map->ln_pos, map->ln_normal, map->ln_min, map->ln_max);
  PL_LAUNCH_CHECK();
  // 3. the two projection searches, every frame with its own th, descriptors read through the entry's map index
  int rc;
  if ((rc = search_by_projection_points_launch(F->keys_un, F->desc, F->n, cap, B, F->bounds, F->scale_factors, d_pcnt, cLP, piv, pproj, plev,
                                               pvc, map->pt_desc, 1.0f, s.th, s.prow, 0.8f, s.ppre, pmatch, s.pnm, st))) return rc;
  if ((rc = lsd_search_by_projection_launch(1, F->keylines, F->line_func, F->line_desc, F->nl, capL, B, F->bounds, d_lcnt, cLL, liv, lproj,
                                            map->ln_desc, lvc, 1.0f, s.th, s.lrow, 0.7f, s.lpre, lmatch, s.lnm, s.lsd, st))) return rc;
  // 4. the pose problem in feature order, then PoseOptimization
  TrackBuildArgs Bd;
  Bd.keys = F->keys_un; Bd.n = F->n; Bd.cap = cap; Bd.inv_sigma2 = F->inv_level_sigma2; Bd.lfunc = F->line_func; Bd.nl = F->nl; Bd.capL = capL;
  Bd.pmap_in = F->point_map_in; Bd.lmap_in = F->line_map_in; Bd.pmatch = pmatch; Bd.lmatch = lmatch;
  Bd.prow = s.prow; Bd.cap_lp = cLP; Bd.lrow = s.lrow; Bd.cap_ll = cLL; Bd.map_pt = map->pt_pos; Bd.map_ln = map->ln_pos;
  Bd.point_map = O->point_map; Bd.line_map = O->line_map; Bd.pslot = s.pslot; Bd.lslot = s.lslot;
  Bd.np = np; Bd.obs = obs; Bd.w = w; Bd.X = X; Bd.nlp = nl; Bd.lf = lf; Bd.lX = lX;
  Bd.solve = solve;
  k_track_build<<<B, kTrackThreads, 0, st>>>(Bd);
  PL_LAUNCH_CHECK();
  if ((rc = pl_pose_optimization_dev(0, B, F->Tcw0, F->K, np, cap, obs, w, X, nl, capL, lf, lX, O->Tcw, s.pout, s.lout, s.inl, s.its, s.lm,
                                     st))) return rc;
  // 5. write back per feature
  k_track_writeback<<<B, kTrackThreads, 0, st>>>(s.pslot, s.pout, cap, s.lslot, s.lout, capL, d_min_inl, O->point_outlier, O->line_outlier,
                                                  O->inliers, solve, ok_in, O->ok);
  PL_LAUNCH_CHECK();
  return PL_OK;
}
}  // namespace pl

// B = 1 on host pointers: stage, run, copy back, check the index flag.  The device arrays are sized by the counts.
extern "C" int pl_track_local_map(PLMap* map, const PLTrackFrames* F, const PLTrackLocal* L, const PLTrackOut* O) {
  PL_ARG(map && F && L && O && F->B == 1 && F->n && F->nl && L->pt_count && L->ln_count && L->pt_offset && L->ln_offset);
  PL_ARG(O->Tcw && O->point_map && O->point_outlier && O->line_map && O->line_outlier && O->inliers);
  const int n = *F->n, nl = *F->nl;
  PL_ARG(n >= 0 && nl >= 0 && n <= F->cap_points && nl <= F->cap_lines && F->nlevels >= 1);
  PL_ARG(L->pt_count[0] >= 0 && L->ln_count[0] >= 0 && L->pt_offset[0] >= 0 && L->ln_offset[0] >= 0);
  PL_ARG(L->pt_count[0] <= L->cap_local_points && L->ln_count[0] <= L->cap_local_lines);
  PL_ARG((long long)L->pt_offset[0] + L->pt_count[0] <= L->n_pt_index && (long long)L->ln_offset[0] + L->ln_count[0] <= L->n_ln_index);
  int rc = require_device(); if (rc) return rc;
  const int cap = std::max(n, 1), capL = std::max(nl, 1);
  const size_t lp = (size_t)L->pt_count[0], ll = (size_t)L->ln_count[0];
  const int cLP = std::max((int)lp, 1), cLL = std::max((int)ll, 1);
  Staging s;
  PLTrackFrames D = *F;
  D.cap_points = cap; D.cap_lines = capL;
  D.keys_un = s.in(F->keys_un, n); D.desc = s.in(F->desc, (size_t)n * 32); D.n = s.in(&n, 1);
  D.keylines = s.in((const uint8_t*)F->keylines, (size_t)nl * 68); D.line_func = s.in(F->line_func, (size_t)nl * 3);
  D.line_desc = s.in(F->line_desc, (size_t)nl * 32); D.nl = s.in(&nl, 1);
  D.bounds = s.in(F->bounds, 4); D.scale_factors = s.in(F->scale_factors, F->nlevels);
  D.inv_level_sigma2 = s.in(F->inv_level_sigma2, F->nlevels); D.Tcw0 = s.in(F->Tcw0, 16); D.K = s.in(F->K, 4);
  D.point_map_in = F->point_map_in ? s.in(F->point_map_in, n) : nullptr;
  D.line_map_in = F->line_map_in ? s.in(F->line_map_in, nl) : nullptr;
  const int zero = 0;
  PLTrackLocal DL = *L;
  DL.pt_offset = &zero; DL.ln_offset = &zero; DL.cap_local_points = cLP; DL.cap_local_lines = cLL;
  DL.n_pt_index = (int)lp; DL.n_ln_index = (int)ll;
  DL.pt_index = lp ? s.in(L->pt_index + L->pt_offset[0], lp) : nullptr;
  DL.ln_index = ll ? s.in(L->ln_index + L->ln_offset[0], ll) : nullptr;
  // required outputs always get a device array; optional ones only when asked for
  int ok_h = 0;
  PLTrackOut DO;
  DO.Tcw = s.out(O->Tcw, 16); DO.ok = s.out(&ok_h, 1); DO.inliers = s.out(O->inliers, 2);
  DO.point_map = s.out(O->point_map, n, cap); DO.point_outlier = s.out(O->point_outlier, n, cap);
  DO.line_map = s.out(O->line_map, nl, capL); DO.line_outlier = s.out(O->line_outlier, nl, capL);
  DO.pt_in_view = s.out(O->pt_in_view, lp, cLP); DO.pt_proj = s.out(O->pt_proj, lp * 2, (size_t)cLP * 2);
  DO.pt_level = s.out(O->pt_level, lp, cLP); DO.pt_view_cos = s.out(O->pt_view_cos, lp, cLP);
  DO.ln_in_view = s.out(O->ln_in_view, ll, cLL); DO.ln_proj = s.out(O->ln_proj, ll * 4, (size_t)cLL * 4);
  DO.ln_level = s.out(O->ln_level, ll, cLL); DO.ln_view_cos = s.out(O->ln_view_cos, ll, cLL);
  DO.pt_match = s.out(O->pt_match, n, cap); DO.ln_match = s.out(O->ln_match, nl, capL);
  DO.prob_n_points = s.out(O->prob_n_points, 1); DO.prob_n_lines = s.out(O->prob_n_lines, 1);
  DO.prob_pt_obs = s.out(O->prob_pt_obs, (size_t)n * 2, (size_t)cap * 2); DO.prob_pt_inv_sigma2 = s.out(O->prob_pt_inv_sigma2, n, cap);
  DO.prob_pt_Xw = s.out(O->prob_pt_Xw, (size_t)n * 3, (size_t)cap * 3);
  DO.prob_line_func = s.out(O->prob_line_func, (size_t)nl * 3, (size_t)capL * 3);
  DO.prob_line_Xw = s.out(O->prob_line_Xw, (size_t)nl * 6, (size_t)capL * 6);
  void* scr = s.out<uint8_t>(pl_track_local_map_scratch_bytes(1, cap, capL, cLP, cLL));
  if ((rc = s.status()) || (rc = s.sync()) || (rc = pl_track_local_map_dev(map, &D, &DL, &DO, scr, map->stream))) return rc;
  PL_CUDA(cudaStreamSynchronize(map->stream));
  if ((rc = s.fetch()) || (rc = pl_map_check_indices(map))) return rc;
  return ok_h;
}

// ---- Tracking::TrackWithMotionModel (src/Tracking.cc:1316-1431) for a batch of frames, monocular, localisation mode:
//   k_mm_prep                mVelocity * mLastFrame.mTcw (:1332); the last frame's valid keypoints (mvpMapPoints[i] && !mvbOutlier[i],
//                            ORBmatcher.cc:1441-1585) and the LSDmatcher candidates: mvpMapLines[i] && !mvbLineOutlier[i] &&
//                            CurrentFrame.isInFrustum(pML, 0.5) at the guess (LSDmatcher.cpp:95-107)
//   k_search_proj_last       ORBmatcher(0.9, true).SearchByProjection(Current, Last, 15, mono), position and descriptor read
//                            through the last frame's map index; then again at 30 for frames under 20 matches (:1354-1358)
//   k_line_search            LSDmatcher().SearchByProjection(Current, Last, 15)                          (variant 0)
//   k_mm_gate                the retried flag, the counts and the early return (nmatches < 20 && lmatches < 5, :1360-1361)
//   k_track_build            the PoseOptimization problem in feature order (empty for early-return frames)
//   k_pose_opt               Optimizer::PoseOptimization (lm.cu, mode 0, unchanged)
//   k_mm_discard             the outliers dropped (:1376-1419), mbVO and the return value (:1424-1428)
namespace pl {
// cv::Mat's fp32 4x4 product, element (i, j): ((a0 b0 + a1 b1) + a2 b2) + a3 b3 with every operation rounded (cv::gemm's order for
// small matrices, as in the oracle's Mat::operator*; tests/golden/mat4_cv2.npz pins it against cv2)
__device__ __forceinline__ float mat4_elem(const float* A, const float* Bm, int i, int j) {
  float s = __fmul_rn(A[4 * i], Bm[j]);
  for (int k = 1; k < 4; k++) s = __fadd_rn(s, __fmul_rn(A[4 * i + k], Bm[4 * k + j]));
  return s;
}

struct MMPrepArgs {
  const float* Tlast; const float* V; const float* K; const float* bounds; float logScaleFactor;
  const PLKeyPoint* keys; const int* n; int cap; const int* pmap; const uint8_t* pout; int n_pts;
  const void* keylines; const int* nl; int capL; const int* lmap; const uint8_t* lout; int n_lns;
  const double* ln_pos; const double* ln_normal; const float* ln_min; const float* ln_max;
  float* guess; uint8_t* pvalid; int* poct; float* pang;
  uint8_t* liv; float* lproj; int* llev; float* lvc; float* llen; int* flag;
};
// A -1 or outlier entry is skipped without a look at the map; a non-negative index outside the map sets the flag and is skipped.
__global__ void __launch_bounds__(kTrackThreads) k_mm_prep(MMPrepArgs A) {
  __shared__ float G[16];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (tid < 16) {
    const float g = mat4_elem(A.V + 16 * b, A.Tlast + 16 * b, tid >> 2, tid & 3);
    G[tid] = g; A.guess[16 * b + tid] = g;
  }
  __syncthreads();
  {
    const int N = min(A.n[b], A.cap);
    const long long o = (long long)b * A.cap;
    for (int i = tid; i < A.cap; i += kTrackThreads) {
      uint8_t v = 0; int oct = 0; float ang = 0.f;
      if (i < N) {
        const int m = A.pmap[o + i];
        if (m >= 0 && !A.pout[o + i]) { if (m >= A.n_pts) atomicOr(A.flag, 1); else v = 1; }
        oct = A.keys[o + i].octave; ang = A.keys[o + i].angle;
      }
      A.pvalid[o + i] = v; A.poct[o + i] = oct; A.pang[o + i] = ang;
    }
  }
  const int N = min(A.nl[b], A.capL);
  const long long o = (long long)b * A.capL;
  FrustumArgs F;
  for (int k = 0; k < 16; k++) F.T[k] = G[k];
  camera_center(F.T, F.Ow);
  for (int k = 0; k < 4; k++) { F.K[k] = A.K[4 * b + k]; F.bounds[k] = A.bounds[k]; }
  F.logScaleFactor = A.logScaleFactor; F.viewingCosLimit = 0.5f; F.nScaleLevels = 1; F.n = 0;
  for (int i = tid; i < A.capL; i += kTrackThreads) {
    const long long q = o + i;
    A.liv[q] = 0; for (int k = 0; k < 4; k++) A.lproj[4 * q + k] = 0; A.llev[q] = 0; A.lvc[q] = 0; A.llen[q] = 0;
    if (i >= N) continue;
    const int m = A.lmap[q];
    if (m < 0 || A.lout[q]) continue;
    if (m >= A.n_lns) { atomicOr(A.flag, 1); continue; }
    A.llen[q] = *(const float*)((const char*)A.keylines + 68 * q + 60);   // mvKeylinesUn[i].lineLength
    float pr[4], vc; int l;
    if (!frustum_line(F, A.ln_pos + 6 * (long long)m, A.ln_normal + 3 * (long long)m, A.ln_min[m], A.ln_max[m], pr, l, vc)) continue;
    A.liv[q] = 1; for (int k = 0; k < 4; k++) A.lproj[4 * q + k] = pr[k];
    A.llev[q] = l; A.lvc[q] = vc;
  }
}

// nmatches after the retry, the retried flag, and solve = !(nmatches < 20 && lmatches < 5)
__global__ void __launch_bounds__(128) k_mm_gate(int B, const int* __restrict__ pnm, const int* __restrict__ pnm_retry,
                                                 const int* __restrict__ lnm, uint8_t* __restrict__ retried, int* __restrict__ counts,
                                                 uint8_t* __restrict__ solve) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const bool r = pnm[b] < 20;
  const int nm = r ? pnm_retry[b] : pnm[b], lm = lnm[b];
  retried[b] = r; counts[2 * b] = nm; counts[2 * b + 1] = lm; solve[b] = !(nm < 20 && lm < 5);
}

// Discard outliers (:1376-1419): a matched outlier loses its match (its map index goes to point_seen / line_seen, else -1) and
// is taken off nmatches / lmatches; nmatchesMap counts the matches left (every entry of a fixed map has Observations() > 0).
// Frames that returned early have an empty problem, so nothing is discarded and ok = 0 with vo as passed.
__global__ void __launch_bounds__(kTrackThreads) k_mm_discard(const int* __restrict__ pslot, const uint8_t* __restrict__ pout, int cap,
                                                              const int* __restrict__ lslot, const uint8_t* __restrict__ lout, int capL,
                                                              const uint8_t* __restrict__ solve, const int* __restrict__ counts,
                                                              int* __restrict__ point_map, int* __restrict__ line_map,
                                                              int* __restrict__ point_seen, int* __restrict__ line_seen,
                                                              int* __restrict__ nmatches, int* __restrict__ ok, int* __restrict__ vo) {
  __shared__ int cnt[3];
  const int b = blockIdx.x;
  if (threadIdx.x < 3) cnt[threadIdx.x] = 0;
  __syncthreads();
  int dp = 0, dl = 0, kept = 0;
  for (int i = threadIdx.x; i < cap; i += kTrackThreads) {
    const long long o = (long long)b * cap + i;
    const int s = pslot[o], m = point_map[o];
    int seen = -1;
    if (s >= 0 && pout[(long long)b * cap + s]) { seen = m; point_map[o] = -1; dp++; }
    else kept += m >= 0;
    point_seen[o] = seen;
  }
  for (int i = threadIdx.x; i < capL; i += kTrackThreads) {
    const long long o = (long long)b * capL + i;
    const int s = lslot[o], m = line_map[o];
    int seen = -1;
    if (s >= 0 && lout[(long long)b * capL + s]) { seen = m; line_map[o] = -1; dl++; }
    line_seen[o] = seen;
  }
  dp = warp_sum(dp); dl = warp_sum(dl); kept = warp_sum(kept);
  if ((threadIdx.x & 31) == 0) { atomicAdd(&cnt[0], dp); atomicAdd(&cnt[1], dl); atomicAdd(&cnt[2], kept); }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int nm = counts[2 * b] - cnt[0];
    nmatches[2 * b] = nm; nmatches[2 * b + 1] = counts[2 * b + 1] - cnt[1];
    if (solve[b]) { vo[b] = cnt[2] < 10; ok[b] = nm > 20; }
    else ok[b] = 0;
  }
}

// mVelocity = mCurrentFrame.mTcw * LastTwc, LastTwc = [Rcw^T | Ow] of the last frame (Tracking.cc:492-501), where ok[b]
__global__ void __launch_bounds__(128) k_track_velocity(int B, const float* __restrict__ T, const float* __restrict__ Tl,
                                                        const int* __restrict__ ok, float* __restrict__ V) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || !ok[b]) return;
  float L[16], W[16], C[16], Ow[3];
  for (int k = 0; k < 16; k++) { L[k] = Tl[16 * b + k]; C[k] = T[16 * b + k]; }
  camera_center(L, Ow);
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) W[4 * i + j] = L[4 * j + i];
    W[4 * i + 3] = Ow[i];
  }
  W[12] = W[13] = W[14] = 0.f; W[15] = 1.f;
  for (int k = 0; k < 16; k++) V[16 * b + k] = mat4_elem(C, W, k >> 2, k & 3);
}

struct MMScratch {
  float* guess; uint8_t* pvalid; int* poct; float* pang;
  uint8_t* liv; float* lproj; int* llev; float* lvc; float* llen;
  int *pm, *pnm, *pm2, *pnm2, *lmatch, *lnm; void* lsd;
  uint8_t *retried, *solve; int* counts;
  int *np, *nl; float *obs, *w, *X; double *lf, *lX;
  int *pslot, *lslot; uint8_t *pout, *lout; int *inl, *its; double* lm;
};
static size_t carve_mm(void* base, int B, int cap, int capL, MMScratch* t) {
  size_t off = 0;
  auto take = [&](size_t bytes) { void* p = base ? (char*)base + off : nullptr; off += (bytes + 15) / 16 * 16; return p; };
  const size_t b = B, k = cap, l = capL;
  MMScratch s;
  s.guess = (float*)take(b * 64); s.pvalid = (uint8_t*)take(b * k); s.poct = (int*)take(b * k * 4); s.pang = (float*)take(b * k * 4);
  s.liv = (uint8_t*)take(b * l); s.lproj = (float*)take(b * l * 16); s.llev = (int*)take(b * l * 4); s.lvc = (float*)take(b * l * 4);
  s.llen = (float*)take(b * l * 4);
  s.pm = (int*)take(b * k * 4); s.pnm = (int*)take(b * 4); s.pm2 = (int*)take(b * k * 4); s.pnm2 = (int*)take(b * 4);
  s.lmatch = (int*)take(b * l * 4); s.lnm = (int*)take(b * 4);
  s.lsd = take(pl_lsd_search_scratch_bytes(capL, B));
  s.retried = (uint8_t*)take(b); s.solve = (uint8_t*)take(b); s.counts = (int*)take(b * 8);
  s.np = (int*)take(b * 4); s.nl = (int*)take(b * 4);
  s.obs = (float*)take(b * k * 8); s.w = (float*)take(b * k * 4); s.X = (float*)take(b * k * 12);
  s.lf = (double*)take(b * l * 24); s.lX = (double*)take(b * l * 48);
  s.pslot = (int*)take(b * k * 4); s.lslot = (int*)take(b * l * 4); s.pout = (uint8_t*)take(b * k); s.lout = (uint8_t*)take(b * l);
  s.inl = (int*)take(b * 4); s.its = (int*)take(b * 4);
  s.lm = (double*)take(pl_pose_optimization_scratch_doubles(B, cap, capL) * 8);
  if (t) *t = s;
  return off;
}
}  // namespace pl

extern "C" size_t pl_track_motion_model_scratch_bytes(int B, int cap_points, int cap_lines) {
  if (B < 1 || cap_points < 1 || cap_lines < 1) return 0;
  return carve_mm(nullptr, B, cap_points, cap_lines, nullptr);
}

extern "C" int pl_track_motion_model_dev(PLMap* map, const PLTrackFrames* F, const PLTrackLast* Ls, const PLTrackMotionOut* O,
                                         void* scratch, void* stream_) {
  PL_ARG(map && F && Ls && O && scratch);
  const int B = F->B, cap = F->cap_points, capL = F->cap_lines;
  PL_ARG(B >= 1 && cap >= 1 && cap <= 6144 && capL >= 1 && capL <= 32768 && F->nlevels >= 1);
  PL_ARG(F->keys_un && F->desc && F->n && F->keylines && F->line_func && F->line_desc && F->nl && F->bounds && F->scale_factors &&
         F->inv_level_sigma2 && F->K);
  // the guess is computed and the current frame's matches start empty (:1332-1335)
  PL_ARG(!F->Tcw0 && !F->point_map_in && !F->line_map_in);
  PL_ARG(Ls->keys_un && Ls->n && Ls->keylines && Ls->nl && Ls->point_map && Ls->point_outlier && Ls->line_map && Ls->line_outlier &&
         Ls->Tcw && Ls->velocity);
  PL_ARG(O->Tcw && O->point_map && O->line_map && O->point_seen && O->line_seen && O->nmatches && O->ok && O->vo);
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : map->stream;
  MMScratch s;
  carve_mm(scratch, B, cap, capL, &s);
  float* guess = O->guess ? O->guess : s.guess;
  uint8_t* liv = O->ln_in_view ? O->ln_in_view : s.liv; float* lproj = O->ln_proj ? O->ln_proj : s.lproj;
  int* llev = O->ln_level ? O->ln_level : s.llev; float* lvc = O->ln_view_cos ? O->ln_view_cos : s.lvc;
  int* pm = O->pt_match ? O->pt_match : s.pm; int* pm2 = O->pt_match_retry ? O->pt_match_retry : s.pm2;
  int* lmatch = O->ln_match ? O->ln_match : s.lmatch; uint8_t* retried = O->retried ? O->retried : s.retried;
  int* np = O->prob_n_points ? O->prob_n_points : s.np; int* nl = O->prob_n_lines ? O->prob_n_lines : s.nl;
  float* obs = O->prob_pt_obs ? O->prob_pt_obs : s.obs; float* w = O->prob_pt_inv_sigma2 ? O->prob_pt_inv_sigma2 : s.w;
  float* X = O->prob_pt_Xw ? O->prob_pt_Xw : s.X;
  double* lf = O->prob_line_func ? O->prob_line_func : s.lf; double* lX = O->prob_line_Xw ? O->prob_line_Xw : s.lX;

  // 1. the guess, the last frame's valid keypoints and its line candidates at the guess
  MMPrepArgs P;
  P.Tlast = Ls->Tcw; P.V = Ls->velocity; P.K = F->K; P.bounds = F->bounds; P.logScaleFactor = F->log_scale_factor;
  P.keys = Ls->keys_un; P.n = Ls->n; P.cap = cap; P.pmap = Ls->point_map; P.pout = Ls->point_outlier; P.n_pts = map->n_points;
  P.keylines = Ls->keylines; P.nl = Ls->nl; P.capL = capL; P.lmap = Ls->line_map; P.lout = Ls->line_outlier; P.n_lns = map->n_lines;
  P.ln_pos = map->ln_pos; P.ln_normal = map->ln_normal; P.ln_min = map->ln_min; P.ln_max = map->ln_max;
  P.guess = guess; P.pvalid = s.pvalid; P.poct = s.poct; P.pang = s.pang;
  P.liv = liv; P.lproj = lproj; P.llev = llev; P.lvc = lvc; P.llen = s.llen; P.flag = map->flag;
  k_mm_prep<<<B, kTrackThreads, 0, st>>>(P);
  PL_LAUNCH_CHECK();
  // 2. the searches: points at th = 15, lines at 15, points again at 30 for frames under 20 point matches
  int rc;
  if ((rc = search_by_projection_last_launch(F->keys_un, F->desc, F->n, cap, B, F->bounds, guess, F->K, F->scale_factors, F->nlevels,
                                             Ls->n, cap, s.pvalid, map->pt_pos, map->pt_desc, Ls->point_map, s.poct, s.pang, 15.0f, 1,
                                             nullptr, nullptr, 0, pm, s.pnm, st))) return rc;
  if ((rc = lsd_search_by_projection_launch(0, F->keylines, F->line_func, F->line_desc, F->nl, capL, B, F->bounds, Ls->nl, capL, liv,
                                            lproj, map->ln_desc, s.llen, 15.0f, nullptr, Ls->line_map, 0.f, nullptr, lmatch, s.lnm, s.lsd,
                                            st))) return rc;
  if ((rc = search_by_projection_last_launch(F->keys_un, F->desc, F->n, cap, B, F->bounds, guess, F->K, F->scale_factors, F->nlevels,
                                             Ls->n, cap, s.pvalid, map->pt_pos, map->pt_desc, Ls->point_map, s.poct, s.pang, 30.0f, 1,
                                             nullptr, s.pnm, 20, pm2, s.pnm2, st))) return rc;
  k_mm_gate<<<(B + 127) / 128, 128, 0, st>>>(B, s.pnm, s.pnm2, s.lnm, retried, s.counts, s.solve);
  PL_LAUNCH_CHECK();
  // 3. the pose problem (rows: the last frame's matches, since a search result is a last-frame index), then PoseOptimization
  TrackBuildArgs Bd;
  Bd.keys = F->keys_un; Bd.n = F->n; Bd.cap = cap; Bd.inv_sigma2 = F->inv_level_sigma2; Bd.lfunc = F->line_func; Bd.nl = F->nl; Bd.capL = capL;
  Bd.pmap_in = nullptr; Bd.lmap_in = nullptr; Bd.pmatch = pm; Bd.lmatch = lmatch;
  Bd.prow = Ls->point_map; Bd.cap_lp = cap; Bd.lrow = Ls->line_map; Bd.cap_ll = capL; Bd.map_pt = map->pt_pos; Bd.map_ln = map->ln_pos;
  Bd.point_map = O->point_map; Bd.line_map = O->line_map; Bd.pslot = s.pslot; Bd.lslot = s.lslot;
  Bd.np = np; Bd.obs = obs; Bd.w = w; Bd.X = X; Bd.nlp = nl; Bd.lf = lf; Bd.lX = lX;
  Bd.use_alt = retried; Bd.pmatch_alt = pm2; Bd.solve = s.solve;
  k_track_build<<<B, kTrackThreads, 0, st>>>(Bd);
  PL_LAUNCH_CHECK();
  if ((rc = pl_pose_optimization_dev(0, B, guess, F->K, np, cap, obs, w, X, nl, capL, lf, lX, O->Tcw, s.pout, s.lout, s.inl, s.its, s.lm,
                                     st))) return rc;
  // 4. discard the outliers
  k_mm_discard<<<B, kTrackThreads, 0, st>>>(s.pslot, s.pout, cap, s.lslot, s.lout, capL, s.solve, s.counts, O->point_map, O->line_map,
                                            O->point_seen, O->line_seen, O->nmatches, O->ok, O->vo);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

// B = 1 on host pointers: stage, run, copy back, check the index flag.  Both frames' device arrays are sized by the largest count.
extern "C" int pl_track_motion_model(PLMap* map, const PLTrackFrames* F, const PLTrackLast* Ls, const PLTrackMotionOut* O) {
  PL_ARG(map && F && Ls && O && F->B == 1 && F->n && F->nl && Ls->n && Ls->nl && F->nlevels >= 1);
  PL_ARG(!F->Tcw0 && !F->point_map_in && !F->line_map_in);
  PL_ARG(O->Tcw && O->point_map && O->line_map && O->point_seen && O->line_seen && O->nmatches && O->vo);
  const int n = *F->n, nl = *F->nl, n0 = *Ls->n, nl0 = *Ls->nl;
  PL_ARG(n >= 0 && nl >= 0 && n0 >= 0 && nl0 >= 0 && n <= F->cap_points && nl <= F->cap_lines && n0 <= F->cap_points &&
         nl0 <= F->cap_lines);
  int rc = require_device(); if (rc) return rc;
  const int cap = std::max(std::max(n, n0), 1), capL = std::max(std::max(nl, nl0), 1);
  Staging s;
  PLTrackFrames D = *F;
  D.cap_points = cap; D.cap_lines = capL;
  D.keys_un = s.in(F->keys_un, n); D.desc = s.in(F->desc, (size_t)n * 32); D.n = s.in(&n, 1);
  D.keylines = s.in((const uint8_t*)F->keylines, (size_t)nl * 68); D.line_func = s.in(F->line_func, (size_t)nl * 3);
  D.line_desc = s.in(F->line_desc, (size_t)nl * 32); D.nl = s.in(&nl, 1);
  D.bounds = s.in(F->bounds, 4); D.scale_factors = s.in(F->scale_factors, F->nlevels);
  D.inv_level_sigma2 = s.in(F->inv_level_sigma2, F->nlevels); D.K = s.in(F->K, 4);
  PLTrackLast DL;
  DL.keys_un = s.in(Ls->keys_un, n0); DL.n = s.in(&n0, 1);
  DL.keylines = s.in((const uint8_t*)Ls->keylines, (size_t)nl0 * 68); DL.nl = s.in(&nl0, 1);
  DL.point_map = s.in(Ls->point_map, n0); DL.point_outlier = s.in(Ls->point_outlier, n0);
  DL.line_map = s.in(Ls->line_map, nl0); DL.line_outlier = s.in(Ls->line_outlier, nl0);
  DL.Tcw = s.in(Ls->Tcw, 16); DL.velocity = s.in(Ls->velocity, 16);
  int ok_h = 0;
  PLTrackMotionOut DO;
  DO.Tcw = s.out(O->Tcw, 16); DO.ok = s.out(&ok_h, 1); DO.nmatches = s.out(O->nmatches, 2);
  DO.vo = s.in(O->vo, 1);   // in / out
  DO.point_map = s.out(O->point_map, n, cap); DO.line_map = s.out(O->line_map, nl, capL);
  DO.point_seen = s.out(O->point_seen, n, cap); DO.line_seen = s.out(O->line_seen, nl, capL);
  DO.guess = s.out(O->guess, 16);
  DO.pt_match = s.out(O->pt_match, n, cap); DO.pt_match_retry = s.out(O->pt_match_retry, n, cap);
  DO.retried = s.out(O->retried, 1); DO.ln_match = s.out(O->ln_match, nl, capL);
  DO.ln_in_view = s.out(O->ln_in_view, nl0, capL); DO.ln_proj = s.out(O->ln_proj, (size_t)nl0 * 4, (size_t)capL * 4);
  DO.ln_level = s.out(O->ln_level, nl0, capL); DO.ln_view_cos = s.out(O->ln_view_cos, nl0, capL);
  DO.prob_n_points = s.out(O->prob_n_points, 1); DO.prob_n_lines = s.out(O->prob_n_lines, 1);
  DO.prob_pt_obs = s.out(O->prob_pt_obs, (size_t)n * 2, (size_t)cap * 2); DO.prob_pt_inv_sigma2 = s.out(O->prob_pt_inv_sigma2, n, cap);
  DO.prob_pt_Xw = s.out(O->prob_pt_Xw, (size_t)n * 3, (size_t)cap * 3);
  DO.prob_line_func = s.out(O->prob_line_func, (size_t)nl * 3, (size_t)capL * 3);
  DO.prob_line_Xw = s.out(O->prob_line_Xw, (size_t)nl * 6, (size_t)capL * 6);
  void* scr = s.out<uint8_t>(pl_track_motion_model_scratch_bytes(1, cap, capL));
  if ((rc = s.status()) || (rc = s.sync()) || (rc = pl_track_motion_model_dev(map, &D, &DL, &DO, scr, map->stream))) return rc;
  PL_CUDA(cudaStreamSynchronize(map->stream));
  if ((rc = s.fetch()) || (rc = s.down(O->vo, DO.vo, 1)) || (rc = pl_map_check_indices(map))) return rc;
  return ok_h;
}

extern "C" int pl_track_velocity_dev(int B, const float* Tcw, const float* Tcw_last, const int* ok, float* velocity, void* stream) {
  PL_ARG(B >= 1 && Tcw && Tcw_last && ok && velocity);
  k_track_velocity<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(B, Tcw, Tcw_last, ok, velocity);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

// ---- Tracking::UpdateLocalMap (src/Tracking.cc:1899-2081) for a batch of frames against the map's keyframe graph:
//   k_update_local_map       one CTA per frame: UpdateLocalKeyFrames (votes, first maximum, the bounded expansion), then
//                            UpdateLocalPoints / UpdateLocalLines (first occurrences in list order, then slot order)
//   k_ref_pose               Tcr = Tcw * Twc[ref] (:582) and the monocular UpdateLastFrame, Tcr * Tcw[ref] (:1242-1245)
// Shared memory per CTA: 4 B per keyframe (the votes, then the local keyframe list), 1 bit per keyframe (mnTrackReferenceForFrame
// of the keyframes) and 1 bit per map point or map line (mnTrackReferenceForFrame of the entries, points and lines in turn).
namespace pl {
constexpr int kMaxGraphKF = 16384;           // 64 KB of votes + 2 KB of keyframe bits
constexpr int kMaxGraphEntries = 1 << 20;    // map points and map lines each: 128 KB of bits
constexpr int kLocalKFLimit = 80;            // if(mvpLocalKeyFrames.size()>80) break (:2027)

struct ULMArgs {
  int n_kf, n_points, n_lines, bit_words;
  const uint8_t* bad; const int* parent;
  const int *pt_off, *pt, *ln_off, *ln, *cov_off, *cov, *child_off, *child, *obs_off, *obs;
  const int* point_map; int cap; const int* ok; const int* vo;
  int* kf; int* n_kf_out; int cap_kf; int* ref_kf;
  int* lp; int* n_lp; int cap_lp; int* ll; int* n_ll; int cap_ll;
  int* flag;                                  // [0] index, [1] capacity
};

__device__ __forceinline__ bool bit_test(const unsigned* bits, int i) { return (bits[i >> 5] >> (i & 31)) & 1u; }

// First occurrences over the local keyframes list[0..nlist) in list order, then in slot order (mnTrackReferenceForFrame,
// :1916-1971), into out[b][cap_out]; the true count goes to n_out[b].  A chunk of slots claims its entries with atomicOr; when an
// entry occurs twice in one chunk the claim may go to the later slot, so such a chunk decides by slot order instead.
__device__ void local_entries(const ULMArgs& A, const int* list, int nlist, const int* off, const int* slot, unsigned* bits,
                              int* s_val, int* warp_tot, int* out, int* n_out, int cap_out) {
  const int b = blockIdx.x, tid = threadIdx.x;
  __syncthreads();
  for (int w = tid; w < A.bit_words; w += kTrackThreads) bits[w] = 0u;
  __syncthreads();
  int base = 0;
  for (int j = 0; j < nlist; j++) {
    const int k = list[j];
    const int s1 = off[k + 1];
    for (int c = off[k]; c < s1; c += kTrackThreads) {
      const int i = c + tid;
      const int m = i < s1 ? slot[i] : -1;          // in range: pl_map_set_keyframes checked every slot
      const bool fresh = m >= 0 && !bit_test(bits, m);
      __syncthreads();                                  // every test of this chunk before its claims
      bool first = false;
      if (fresh) first = !(atomicOr(&bits[m >> 5], 1u << (m & 31)) & (1u << (m & 31)));
      if (__syncthreads_or(fresh && !first)) {
        s_val[tid] = fresh ? m : -1;
        __syncthreads();
        first = fresh;
        for (int t = 0; t < tid && first; t++) first = s_val[t] != m;
        __syncthreads();
      }
      const int pos = block_slot(first, warp_tot, base);
      if (first && pos < cap_out) out[(long long)b * cap_out + pos] = m;
    }
  }
  if (tid == 0) {
    n_out[b] = base;
    if (base > cap_out) atomicOr(A.flag + 1, 1);
  }
}

__global__ void __launch_bounds__(kTrackThreads) k_update_local_map(ULMArgs A) {
  extern __shared__ int smem[];
  int* list = smem;                                               // [n_kf]: the votes, then mvpLocalKeyFrames
  unsigned* kfbits = (unsigned*)(smem + A.n_kf);                  // [(n_kf + 31) / 32]
  unsigned* bits = kfbits + (A.n_kf + 31) / 32;                   // [bit_words]
  __shared__ int warp_tot[kTrackThreads / 32], s_val[kTrackThreads], red_v[kTrackThreads / 32], red_k[kTrackThreads / 32];
  __shared__ int s_size;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if ((A.ok && !A.ok[b]) || (A.vo && A.vo[b])) {                 // if(bOK && !mbVO) TrackLocalMapWithLines() (:476)
    if (tid == 0) { A.n_lp[b] = 0; A.n_ll[b] = 0; }
    return;
  }
  // 1. keyframeCounter: one vote per observation of every matched point (:1977-1993); lines do not vote
  for (int k = tid; k < A.n_kf; k += kTrackThreads) list[k] = 0;
  for (int w = tid; w < (A.n_kf + 31) / 32; w += kTrackThreads) kfbits[w] = 0u;
  __syncthreads();
  for (int i = tid; i < A.cap; i += kTrackThreads) {
    const int m = A.point_map[(long long)b * A.cap + i];
    if (m < 0) continue;
    if (m >= A.n_points) { atomicOr(A.flag, 1); continue; }
    for (int o = A.obs_off[m]; o < A.obs_off[m + 1]; o++) atomicAdd(&list[A.obs[o]], 1);
  }
  __syncthreads();
  bool any = false;
  for (int k = tid; k < A.n_kf; k += kTrackThreads) any |= list[k] > 0;
  int nlist;
  if (__syncthreads_or(any)) {
    // 2. the good voters in index order (map<KeyFrame*,int> order), and pKFmax = the first strict maximum among them (:2005-2020)
    int bv = 0, bk = -1;
    for (int k = tid; k < A.n_kf; k += kTrackThreads) {
      const int v = list[k];
      if (v > bv && !(A.bad && A.bad[k])) { bv = v; bk = k; }
    }
    for (int d = 16; d; d >>= 1) {
      const int ov = __shfl_down_sync(0xffffffffu, bv, d), ok_ = __shfl_down_sync(0xffffffffu, bk, d);
      if (ov > bv || (ov == bv && ok_ >= 0 && (bk < 0 || ok_ < bk))) { bv = ov; bk = ok_; }
    }
    if (lane == 0) { red_v[warp] = bv; red_k[warp] = bk; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < kTrackThreads / 32; w++)
        if (red_v[w] > bv || (red_v[w] == bv && red_k[w] >= 0 && (bk < 0 || red_k[w] < bk))) { bv = red_v[w]; bk = red_k[w]; }
      if (bk >= 0) A.ref_kf[b] = bk;                               // if(pKFmax) mpReferenceKF = pKFmax (:2076-2080)
    }
    // compact the good voters in place: a voter's position is at most its index, and a chunk reads before it writes
    int base = 0;
    for (int c = 0; c < A.n_kf; c += kTrackThreads) {
      const int k = c + tid;
      const bool f = k < A.n_kf && list[k] > 0 && !(A.bad && A.bad[k]);
      const int pos = block_slot(f, warp_tot, base);
      if (f) { list[pos] = k; atomicOr(&kfbits[k >> 5], 1u << (k & 31)); }
    }
    __syncthreads();
    const int nvot = base;
    // 3. neighbours of the ORIGINAL voters only: itEndKF is fixed before the push_backs (:2024-2074)
    if (warp == 0) {
      int size = nvot;
      for (int i = 0; i < nvot; i++) {
        if (size > kLocalKFLimit) break;
        const int k = list[i];
        // the first of GetBestCovisibilityKeyFrames(10) that is good and not yet in
        const int c0 = A.cov_off[k], nc = min(A.cov_off[k + 1] - c0, 10);
        int c = lane < nc ? A.cov[c0 + lane] : -1;
        unsigned bal = __ballot_sync(0xffffffffu, c >= 0 && !(A.bad && A.bad[c]) && !bit_test(kfbits, c));
        if (bal) {
          c = __shfl_sync(0xffffffffu, c, __ffs(bal) - 1);
          if (lane == 0) { list[size] = c; kfbits[c >> 5] |= 1u << (c & 31); }
          size++;
        }
        __syncwarp();
        // the first child in set order that is good and not yet in
        const int h1 = A.child_off[k + 1];
        for (int j = A.child_off[k]; j < h1; j += 32) {
          int h = j + lane < h1 ? A.child[j + lane] : -1;
          bal = __ballot_sync(0xffffffffu, h >= 0 && !(A.bad && A.bad[h]) && !bit_test(kfbits, h));
          if (bal) {
            h = __shfl_sync(0xffffffffu, h, __ffs(bal) - 1);
            if (lane == 0) { list[size] = h; kfbits[h >> 5] |= 1u << (h & 31); }
            size++;
            break;
          }
        }
        __syncwarp();
        // the parent, not checked for isBad; its break ends the whole expansion
        const int p = A.parent[k];
        if (p >= 0 && !bit_test(kfbits, p)) {
          if (lane == 0) list[size] = p;
          size++;
          break;
        }
      }
      if (lane == 0) s_size = size;
    }
    __syncthreads();
    nlist = s_size;
    for (int j = tid; j < min(nlist, A.cap_kf); j += kTrackThreads) A.kf[(long long)b * A.cap_kf + j] = list[j];
    if (tid == 0) {
      A.n_kf_out[b] = nlist;
      if (nlist > A.cap_kf) atomicOr(A.flag + 1, 1);
    }
  } else {
    // keyframeCounter.empty(): return early; mvpLocalKeyFrames and mpReferenceKF keep their values and the points and lines are
    // rebuilt from that list (:1995-1996)
    nlist = min(min(A.n_kf_out[b], A.cap_kf), A.n_kf);
    __syncthreads();
    for (int j = tid; j < nlist; j += kTrackThreads) {
      int k = A.kf[(long long)b * A.cap_kf + j];
      if (k < 0 || k >= A.n_kf) { atomicOr(A.flag, 1); k = -1; }
      list[j] = k;
    }
    __syncthreads();
    // an index outside the graph is dropped from the walk, keeping the order of the others
    if (tid == 0) {
      int w = 0;
      for (int j = 0; j < nlist; j++) if (list[j] >= 0) list[w++] = list[j];
      s_size = w;
    }
    __syncthreads();
    nlist = s_size;
  }
  // 4. mvpLocalMapPoints and mvpLocalMapLines
  local_entries(A, list, nlist, A.pt_off, A.pt, bits, s_val, warp_tot, A.lp, A.n_lp, A.cap_lp);
  local_entries(A, list, nlist, A.ln_off, A.ln, bits, s_val, warp_tot, A.ll, A.n_ll, A.cap_ll);
}

// out[b] = P[b] * Q[ref[b]] with cv::Mat's fp32 product; a ref outside the graph sets the index flag and leaves out[b]
__global__ void __launch_bounds__(128) k_ref_pose(int B, const float* __restrict__ P, const int* __restrict__ ref, const float* __restrict__ Q,
                                                  int n_kf, float* __restrict__ out, int* __restrict__ flag) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int r = ref[b];
  if (r < 0 || r >= n_kf) { atomicOr(flag, 1); return; }
  float L[16], R[16];
  for (int k = 0; k < 16; k++) { L[k] = P[16 * b + k]; R[k] = Q[16 * (long long)r + k]; }
  for (int k = 0; k < 16; k++) out[16 * b + k] = mat4_elem(L, R, k >> 2, k & 3);
}

// the per-frame table of the local-map step from device lists: offsets b * cap, counts clamped to the capacity (0 for a frame
// gated off), min inliers and th from frames_since_reloc, and the gate itself
__global__ void __launch_bounds__(128) k_lists_prep(int B, const int* __restrict__ pcnt, int cLP, const int* __restrict__ lcnt, int cLL,
                                                    const int* __restrict__ since, int max_frames, const int* __restrict__ ok,
                                                    const int* __restrict__ vo, int* __restrict__ tab, float* __restrict__ th,
                                                    uint8_t* __restrict__ solve) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const bool run = (!ok || ok[b]) && (!vo || !vo[b]);
  tab[b] = b * cLP; tab[B + b] = run ? min(max(pcnt[b], 0), cLP) : 0;
  tab[2 * B + b] = b * cLL; tab[3 * B + b] = run ? min(max(lcnt[b], 0), cLL) : 0;
  tab[4 * B + b] = since[b] < max_frames ? 50 : 30;
  th[b] = since[b] < 2 ? 5.0f : 1.0f;
  solve[b] = run;
}

static size_t up_bytes(size_t n) { return (n + 15) / 16 * 16; }
}  // namespace pl

extern "C" int pl_map_set_keyframes(PLMap* m, const PLKeyFrameGraphDesc* g) {
  PL_ARG(m && g && g->n_kf >= 1 && g->n_kf <= kMaxGraphKF);
  PL_ARG(m->n_points <= kMaxGraphEntries && m->n_lines <= kMaxGraphEntries);
  PL_ARG(g->Tcw && g->Twc && g->parent && g->pt_slot_offset && g->ln_slot_offset && g->cov_offset && g->child_offset && g->obs_offset);
  const int K = g->n_kf;
  // every CSR starts at 0 and is monotone; every index is in range
  auto csr = [](const int* off, int rows, const int* idx, int lo, int hi, const char* what) -> bool {
    if (off[0] != 0) { set_error("keyframe graph: %s offsets must start at 0", what); return false; }
    for (int r = 0; r < rows; r++)
      if (off[r + 1] < off[r]) { set_error("keyframe graph: %s offsets are not monotone at row %d", what, r); return false; }
    if (off[rows] > 0 && !idx) { set_error("keyframe graph: %s has entries but no index array", what); return false; }
    for (int i = 0; i < off[rows]; i++)
      if (idx[i] < lo || idx[i] >= hi) { set_error("keyframe graph: %s entry %d = %d is outside [%d, %d)", what, i, idx[i], lo, hi); return false; }
    return true;
  };
  if (!csr(g->pt_slot_offset, K, g->pt_slot, -1, m->n_points, "point slots") ||
      !csr(g->ln_slot_offset, K, g->ln_slot, -1, m->n_lines, "line slots") || !csr(g->cov_offset, K, g->cov, 0, K, "covisibles") ||
      !csr(g->child_offset, K, g->child, 0, K, "children") || !csr(g->obs_offset, m->n_points, g->obs, 0, K, "observations"))
    return PL_ERR_ARG;
  for (int k = 0; k < K; k++)
    if (g->parent[k] < -1 || g->parent[k] >= K) { set_error("keyframe graph: parent of %d = %d is outside the graph", k, g->parent[k]); return PL_ERR_ARG; }
  int rc = require_device(); if (rc) return rc;
  // mspChildrens iterates in KeyFrame* order, which is index order
  std::vector<int> child(g->child, g->child + g->child_offset[K]);
  for (int k = 0; k < K; k++) std::sort(child.begin() + g->child_offset[k], child.begin() + g->child_offset[k + 1]);
  std::vector<uint8_t> bad(K, 0);
  if (g->bad) for (int k = 0; k < K; k++) bad[k] = g->bad[k] != 0;
  // the new graph replaces the old one only once all of it is on the device; every array takes at least 16 bytes
  auto G = std::make_unique<PLMap::KeyframeGraph>();
  const size_t k = K, np = m->n_points;
  PL_TRY(upload(G->Tcw, g->Tcw, k * 16, 4)); PL_TRY(upload(G->Twc, g->Twc, k * 16, 4));
  PL_TRY(upload(G->bad, bad.data(), k, 16)); PL_TRY(upload(G->parent, g->parent, k, 4));
  PL_TRY(upload(G->pt_off, g->pt_slot_offset, k + 1, 4)); PL_TRY(upload(G->pt, g->pt_slot, (size_t)g->pt_slot_offset[K], 4));
  PL_TRY(upload(G->ln_off, g->ln_slot_offset, k + 1, 4)); PL_TRY(upload(G->ln, g->ln_slot, (size_t)g->ln_slot_offset[K], 4));
  PL_TRY(upload(G->cov_off, g->cov_offset, k + 1, 4)); PL_TRY(upload(G->cov, g->cov, (size_t)g->cov_offset[K], 4));
  PL_TRY(upload(G->child_off, g->child_offset, k + 1, 4)); PL_TRY(upload(G->child, child.data(), child.size(), 4));
  PL_TRY(upload(G->obs_off, g->obs_offset, np + 1, 4)); PL_TRY(upload(G->obs, g->obs, (size_t)g->obs_offset[np], 4));
  G->n_kf = K;
  m->kf = std::move(G);
  return PL_OK;
}

extern "C" int pl_map_check_capacity(PLMap* m) {
  PL_ARG(m);
  int f = 0;
  PL_CUDA(cudaDeviceSynchronize());
  PL_CUDA(cudaMemcpy(&f, m->flag + 1, 4, cudaMemcpyDeviceToHost));
  if (!f) return PL_OK;
  PL_CUDA(cudaMemset(m->flag + 1, 0, 4));
  set_error("track: a local keyframe, map point or map line list outgrew its capacity (the counts hold the true sizes)");
  return PL_ERR_ARG;
}

extern "C" int pl_track_update_local_map_dev(PLMap* map, int B, const int* point_map, int cap_points, const int* ok, const int* vo,
                                             const PLLocalMap* L, void* stream) {
  PL_ARG(map && L && point_map && B >= 1 && cap_points >= 1);
  if (!map->kf) { set_error("pl_track_update_local_map_dev: the map has no keyframe graph (pl_map_set_keyframes)"); return PL_ERR_ARG; }
  PL_ARG(L->kf && L->n_kf && L->ref_kf && L->pt_index && L->pt_count && L->ln_index && L->ln_count);
  PL_ARG(L->cap_kf >= 1 && L->cap_local_points >= 1 && L->cap_local_lines >= 1);
  ULMArgs A;
  const PLMap::KeyframeGraph& G = *map->kf;
  A.n_kf = G.n_kf; A.n_points = map->n_points; A.n_lines = map->n_lines;
  A.bit_words = (std::max(std::max(map->n_points, map->n_lines), 1) + 31) / 32;
  A.bad = G.bad; A.parent = G.parent; A.pt_off = G.pt_off; A.pt = G.pt; A.ln_off = G.ln_off; A.ln = G.ln;
  A.cov_off = G.cov_off; A.cov = G.cov; A.child_off = G.child_off; A.child = G.child;
  A.obs_off = G.obs_off; A.obs = G.obs;
  A.point_map = point_map; A.cap = cap_points; A.ok = ok; A.vo = vo;
  A.kf = L->kf; A.n_kf_out = L->n_kf; A.cap_kf = L->cap_kf; A.ref_kf = L->ref_kf;
  A.lp = L->pt_index; A.n_lp = L->pt_count; A.cap_lp = L->cap_local_points; A.ll = L->ln_index; A.n_ll = L->ln_count;
  A.cap_ll = L->cap_local_lines; A.flag = map->flag;
  const int smem = (A.n_kf + (A.n_kf + 31) / 32 + A.bit_words) * 4;
  PL_CUDA(cudaFuncSetAttribute(k_update_local_map, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_update_local_map<<<B, kTrackThreads, smem, stream ? (cudaStream_t)stream : map->stream>>>(A);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

extern "C" size_t pl_track_local_map_lists_scratch_bytes(int B, int cap_points, int cap_lines, int cap_local_points, int cap_local_lines) {
  const size_t s = pl_track_local_map_scratch_bytes(B, cap_points, cap_lines, cap_local_points, cap_local_lines);
  return s ? s + up_bytes(B) : 0;
}

extern "C" int pl_track_local_map_lists_dev(PLMap* map, const PLTrackFrames* F, const int* point_seen, const int* line_seen,
                                            const PLLocalMap* L, const int* frames_since_reloc, int max_frames, const int* ok,
                                            const int* vo, const PLTrackOut* O, void* scratch, void* stream_) {
  PL_ARG(map && F && L && O && scratch && frames_since_reloc);
  const int B = F->B, cap = F->cap_points, capL = F->cap_lines;
  PL_ARG(B >= 1 && cap >= 1 && cap <= 6144 && capL >= 1 && capL <= 32768 && F->nlevels >= 1);
  PL_ARG(F->keys_un && F->desc && F->n && F->keylines && F->line_func && F->line_desc && F->nl && F->bounds && F->scale_factors &&
         F->inv_level_sigma2 && F->Tcw0 && F->K);
  PL_ARG(L->pt_index && L->pt_count && L->ln_index && L->ln_count && L->cap_local_points >= 1 && L->cap_local_lines >= 1);
  PL_ARG(O->Tcw && O->point_map && O->point_outlier && O->line_map && O->line_outlier && O->inliers && O->ok);
  const int cLP = L->cap_local_points, cLL = L->cap_local_lines;
  PL_ARG((long long)B * cLP <= INT_MAX && (long long)B * cLL <= INT_MAX);   // the frustum kernels index the lists with int offsets
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : map->stream;
  TrackScratch s;
  const size_t off = carve(scratch, B, cap, capL, cLP, cLL, &s);
  uint8_t* solve = (uint8_t*)scratch + off;
  k_lists_prep<<<(B + 127) / 128, 128, 0, st>>>(B, L->pt_count, cLP, L->ln_count, cLL, frames_since_reloc, max_frames, ok, vo, s.tab, s.th,
                                                solve);
  PL_LAUNCH_CHECK();
  return track_local_map_run(map, F, point_seen, line_seen, L->pt_index, cLP, L->ln_index, cLL, solve, ok, O, s, st);
}

extern "C" int pl_track_relative_pose_dev(PLMap* map, int B, const float* Tcw, const int* ref_kf, float* Tcr, void* stream) {
  PL_ARG(map && B >= 1 && Tcw && ref_kf && Tcr);
  if (!map->kf) { set_error("pl_track_relative_pose_dev: the map has no keyframe graph (pl_map_set_keyframes)"); return PL_ERR_ARG; }
  k_ref_pose<<<(B + 127) / 128, 128, 0, stream ? (cudaStream_t)stream : map->stream>>>(B, Tcw, ref_kf, map->kf->Twc, map->kf->n_kf, Tcr, map->flag);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

extern "C" int pl_track_last_pose_dev(PLMap* map, int B, const float* Tcr, const int* ref_kf, float* Tcw_last, void* stream) {
  PL_ARG(map && B >= 1 && Tcr && ref_kf && Tcw_last);
  if (!map->kf) { set_error("pl_track_last_pose_dev: the map has no keyframe graph (pl_map_set_keyframes)"); return PL_ERR_ARG; }
  k_ref_pose<<<(B + 127) / 128, 128, 0, stream ? (cudaStream_t)stream : map->stream>>>(B, Tcr, ref_kf, map->kf->Tcw, map->kf->n_kf, Tcw_last,
                                                                                      map->flag);
  PL_LAUNCH_CHECK();
  return PL_OK;
}
