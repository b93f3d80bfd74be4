// The loop of LocalMapping::KeyFrameCulling (src/LocalMapping.cc:1835-1899, monocular) for many current keyframes, on the device
// (DESIGN.md §8f.7).
//
//   k_keyframe_cull  one CTA per group.  First the group's status, every check a block-wide pass over the list or over the
//                    listed keyframes' slots.  Then the list in order: the threads stride over the entry's slots, each slot scans
//                    its point's observations once against the bit set of the rows culled so far (shared memory), two block sums
//                    give nMPs and nRedundantObservations, and thread 0 decides and sets the entry's bit before the next entry.
//
// Culling a keyframe erases its observations (KeyFrame::SetBadFlag, src/KeyFrame.cc:494-508 -> MapPoint::EraseObservation,
// src/MapPoint.cc:111-137), so each entry sees the state the entries before it left; the walk is serial by construction.  A
// point's live state needs only culled(p), the number of its observers culled so far: Observations() = obs - culled(p), and it is
// bad iff it was bad on input or culled(p) >= 1 and obs - culled(p) <= 2.  Everything is integer but the one double comparison.
#include "common.cuh"

namespace pl {

namespace {
constexpr int kCullThreads = 1024;
constexpr int kCullWarps = kCullThreads / 32;
constexpr int kMaxRows = 65536;          // n_kf: two bit sets of kMaxRows bits in shared memory
constexpr int kMaxCap = 6144;

enum : int8_t { kSkipped = -1, kKept = 0, kCulled = 1, kToBeErased = 2 };

struct CullArgs {
  PLCullKeyframes K; PLCullPoints M; PLCullGroups Gr;
  int8_t* code; int* n_mps; int* n_redundant; int* status;
};

__device__ __forceinline__ bool has_bit(const unsigned* s, int k) { return (s[k >> 5] >> (k & 31)) & 1u; }

// Status 4, 5, 6 of one slot's point (0 when it passes).
__device__ int point_status(const CullArgs& A, int p) {
  const PLCullKeyframes& K = A.K; const PLCullPoints& M = A.M;
  if (p < -1 || p >= M.n_mp) return 4;
  if (p < 0) return 0;
  const int a = M.obs_offset[p], b = M.obs_offset[p + 1];
  if (a < 0 || b < a || b > M.n_obs) return 5;
#pragma unroll 4
  for (int e = a; e < b; e++) {
    const int k = M.obs_kf[e], idx = M.obs_idx[e];
    if (k < 0 || k >= K.n_kf) return 6;
    if (idx < 0 || idx >= K.n[k] || idx >= K.cap || K.mp[(long long)k * K.cap + idx] != p) return 6;
  }
  return 0;
}

// The group's status (plslam_b200.h, pl_keyframe_culling_dev), the same in every thread; s_listed is scratch.
__device__ int group_status(const CullArgs& A, int off, int cnt, unsigned* s_listed) {
  const PLCullKeyframes& K = A.K; const PLCullGroups& Gr = A.Gr;
  const int tid = threadIdx.x;
  if (off < 0 || cnt < 0 || (long long)off + cnt > Gr.n_list) return 1;
  bool f = false;
  for (int t = tid; t < cnt; t += kCullThreads) { const int k = Gr.list[off + t]; f = f || k < 0 || k >= K.n_kf; }
  if (__syncthreads_or(f)) return 1;
  for (int t = tid; t < cnt; t += kCullThreads) { const int n = K.n[Gr.list[off + t]]; f = f || n < 0 || n > K.cap; }
  if (__syncthreads_or(f)) return 2;
  for (int w = tid; w < (K.n_kf + 31) / 32; w += kCullThreads) s_listed[w] = 0u;
  __syncthreads();
  for (int t = tid; t < cnt; t += kCullThreads) {
    const int k = Gr.list[off + t];
    f = f || (atomicOr(&s_listed[k >> 5], 1u << (k & 31)) >> (k & 31)) & 1u;
  }
  if (__syncthreads_or(f)) return 3;
  int worst = 0;                         // 4 before 5 before 6 over the whole group: the least nonzero code of any slot
  for (int t = 0; t < cnt; t++) {
    const int k = Gr.list[off + t], n = K.n[k];
    const int* row = K.mp + (long long)k * K.cap;
    for (int i = tid; i < n; i += kCullThreads) {
      const int s = point_status(A, row[i]);
      if (s && (!worst || s < worst)) worst = s;
    }
  }
  if (__syncthreads_or(worst == 4)) return 4;
  if (__syncthreads_or(worst == 5)) return 5;
  if (__syncthreads_or(worst == 6)) return 6;
  return 0;
}

__global__ void __launch_bounds__(kCullThreads) k_keyframe_cull(const __grid_constant__ CullArgs A) {
  extern __shared__ unsigned s_bits[];   // [W] listed rows (status 3), then [W] rows culled so far
  __shared__ int s_sum[2][kCullWarps];
  const PLCullKeyframes& K = A.K; const PLCullPoints& M = A.M; const PLCullGroups& Gr = A.Gr;
  const int g = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int W = (K.n_kf + 31) / 32;
  unsigned* s_culled = s_bits + W;
  const int off = Gr.offset[g], cnt = Gr.count[g];
  const int st = group_status(A, off, cnt, s_bits);
  if (tid == 0) A.status[g] = st;
  if (st) return;
  for (int w = tid; w < W; w += kCullThreads) s_culled[w] = 0u;
  __syncthreads();
  for (int t = 0; t < cnt; t++) {
    const int k = Gr.list[off + t], j = off + t;
    if (K.origin[k]) {                   // :1846
      if (tid == 0) { A.code[j] = kSkipped; A.n_mps[j] = 0; A.n_redundant[j] = 0; }
      continue;
    }
    const long long row = (long long)k * K.cap;
    int mps = 0, red = 0;
    for (int i = tid; i < K.n[k]; i += kCullThreads) {
      const int p = K.mp[row + i];
      if (p < 0 || M.bad[p]) continue;
      const long long oct = K.keys_un[row + i].octave;
      const int a = M.obs_offset[p], b = M.obs_offset[p + 1];
      int culled = 0, finer = 0;
#pragma unroll 4                         // independent observations: lets their loads overlap
      for (int e = a; e < b; e++) {
        const int ki = M.obs_kf[e];
        if (has_bit(s_culled, ki)) { culled++; continue; }
        if (ki != k && K.keys_un[(long long)ki * K.cap + M.obs_idx[e]].octave <= oct + 1) finer++;   // :1876-1881
      }
      const int nobs = (b - a) - culled;
      if (culled && nobs <= 2) continue;  // erased into badness by an earlier cull
      mps++;                              // :1867
      if (nobs > 3 && finer >= 3) red++;  // :1868, :1886-1889
    }
    mps = warp_sum(mps); red = warp_sum(red);
    if (lane == 0) { s_sum[0][warp] = mps; s_sum[1][warp] = red; }
    __syncthreads();
    if (tid == 0) {
      int nm = 0, nr = 0;
      for (int w = 0; w < kCullWarps; w++) { nm += s_sum[0][w]; nr += s_sum[1][w]; }
      int8_t c = kKept;
      if (nr > 0.9 * nm) c = K.not_erase[k] ? kToBeErased : kCulled;   // :1895-1896
      if (c == kCulled) s_culled[k >> 5] |= 1u << (k & 31);
      A.code[j] = c; A.n_mps[j] = nm; A.n_redundant[j] = nr;
    }
    __syncthreads();
  }
}
}  // namespace

}  // namespace pl

using namespace pl;

extern "C" int pl_keyframe_culling_dev(const PLCullKeyframes* kfs, const PLCullPoints* points, const PLCullGroups* groups, int8_t* code,
                                       int* n_mps, int* n_redundant, int* status, void* stream) {
  PL_ARG(groups && groups->G >= 0 && groups->n_list >= 0);
  const PLCullGroups& Gr = *groups;
  if (Gr.G == 0) return PL_OK;
  PL_ARG(Gr.offset && Gr.count && Gr.list);
  PL_ARG(kfs && kfs->keys_un && kfs->n && kfs->mp && kfs->origin && kfs->not_erase);
  PL_ARG(kfs->n_kf >= 1 && kfs->n_kf <= kMaxRows && kfs->cap >= 1 && kfs->cap <= kMaxCap);
  PL_ARG((long long)kfs->n_kf * kfs->cap <= 0x7fffffffLL);
  PL_ARG(points && points->n_mp >= 0 && points->n_obs >= 0 && points->bad && points->obs_offset && points->obs_kf && points->obs_idx);
  PL_ARG(code && n_mps && n_redundant && status);
  PL_TRY(require_device());
  const CullArgs A{*kfs, *points, Gr, code, n_mps, n_redundant, status};
  const int smem = 2 * ((kfs->n_kf + 31) / 32) * (int)sizeof(unsigned);
  k_keyframe_cull<<<Gr.G, kCullThreads, smem, (cudaStream_t)stream>>>(A);
  PL_LAUNCH_CHECK();
  return PL_OK;
}
