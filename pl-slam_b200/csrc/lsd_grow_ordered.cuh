// LSD region growing (k_lsd_grow_ordered): one warp walks one frame's seeds in order, the 32 lanes cooperate on ONE region.
// Produces the oracle's segment list bit for bit.  Included by line.cu only, after LineParams and the shared helpers
// (kFree / kNotDef, kPI / kDegToRads, fast_atan2_deg, angle_diff_signed, dist_d, dist_sq).
//
// Pixel records {own, angle, cos, sin}, 16 bytes (k_lsd_front): the ownership word says free (kFree) / undefined (kNotDef) /
// used (0), and is written with plain stores by the lane that owns the pixel.
//
// Exactness of the fp64 parts (what round 1 did not have): LineSegmentDetectorImpl::region2rect / get_theta / refine sum over
// the region IN LIST ORDER on the CPU.  The lanes load and form the per-pixel terms in parallel (32 pixels per batch), then
// the three running sums are advanced in list order, one sum per lane, reading the terms from shared memory (ordered_add3) -
// the order of the additions is the oracle's, so the rectangle is bit-identical.  reduce_region_radius() swap-removes; the order of the
// survivors decides the order of the next sums, so it is reproduced exactly: all far flags in parallel (bit mask), then a
// hole / survivor matching (hole r below the final size <- r-th survivor of the tail, counted from the end: what the CPU's
// swap-with-last loop leaves behind), computed with warp prefix sums over the mask words.
#pragma once

namespace pl {
namespace ord {

// recent queue entries in shared memory; older ones are re-read from the region list in global memory (L1 hits).  The L1 share matters
// more than the ring: a small ring leaves more of the SM's shared memory / L1 split to L1
constexpr int kORing = 64;
constexpr int kUsedO = 0;

// Per-frame arrays are addressed as  kernel-parameter base + 32-bit element index (fb = frame * npx + pixel): one IMAD.WIDE per
// access and no 64-bit frame pointers held in registers (the host launches at most 2^31 / npx frames per grid).  The queue
// ring and the term rows of the ordered sums are file-scope __shared__ arrays: addressed directly, not through generic pointers.
struct Ctx {
  int4* REC; const int* SQ; const float2* S2; unsigned* mask;   // global bases (kernel parameters)
  unsigned fb;                                                   // element offset of this frame in the arrays above
  const double* wtab; unsigned* R;
  int sw, sh, fill_off; // fill_off: scratch area inside R (beyond the largest possible region)
};
__shared__ unsigned s_ring[kORing];
__shared__ double s_red[96];          // 3 x 32 doubles: the per-pixel terms of one batch, for the ordered sums
struct RectD { double x1, y1, x2, y2, width; };
#ifdef PL_GROW_STATS
__device__ unsigned long long g_grow_stats[24];
#define GSTAT(i, v) do { if (lane == 0) atomicAdd(&g_grow_stats[i], (unsigned long long)(v)); } while (0)
#define GSTAT_ALL(i, v) atomicAdd(&g_grow_stats[i], (unsigned long long)(v))
#else
#define GSTAT_ALL(i, v) do { } while (0)
#define GSTAT(i, v) do { } while (0)
#endif

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ int& own_of(const Ctx& C, int idx) { return reinterpret_cast<int*>(&C.REC[C.fb + (unsigned)idx])[0]; }
__device__ __forceinline__ int angle_bits(const Ctx& C, int idx) { return reinterpret_cast<const int*>(&C.REC[C.fb + (unsigned)idx])[1]; }
// One 16-byte request per record.  (Written as "int4 v = REC[i]; if (v.x == free) use v.y, v.z, v.w" the compiler splits the load
// into LDG.32 + branch + LDG.32 + LDG.64: two dependent round trips per step for every candidate that is free.)
__device__ __forceinline__ int4 ld_rec(const Ctx& C, int idx) {
  int4 v;
  asm volatile("ld.global.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(&C.REC[C.fb + (unsigned)idx]) : "memory");
  return v;
}
__device__ __forceinline__ unsigned lanemask_lt() { unsigned m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }
__device__ __forceinline__ double shfl_d(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }
// Three running sums advanced in LIST ORDER over one batch of up to 32 pixels.  Every lane has put its three terms into
// shared memory; lane j < 3 then walks row j (one LDS + one DADD per pixel for the whole warp - the three chains run in
// three lanes of the same instruction), so the order of the additions is exactly the CPU's and the cost is 2 instructions
// per pixel.  acc lives in lanes 0..2 (acc of lane j = sum j); ordered_get() hands a finished sum to every lane.
__device__ __forceinline__ void ordered_add3(const Ctx& C, double t0, double t1, double t2, int m, double& acc, int lane) {
  s_red[lane] = t0; s_red[32 + lane] = t1; s_red[64 + lane] = t2;
  __syncwarp();
  const double* row = s_red + 32 * min(lane, 2);
  if (m == 32) {
#pragma unroll
    for (int k = 0; k < 32; k++) acc += row[k];
  } else {
#pragma unroll 1                        // (a partially unrolled remainder loop measured 2.5 % slower: code size)
    for (int k = 0; k < m; k++) acc += row[k];
  }
  __syncwarp();
}
__device__ __forceinline__ double ordered_get(double acc, int j) { return shfl_d(acc, j); }
__device__ __noinline__ double wmax_d(double v) {          // out of line on purpose (4 uses per rectangle; code size, see §6 of DESIGN.md)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __noinline__ double wmin_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __noinline__ float fast_atan2_cold(float y, float x) { return fast_atan2_deg(y, x); }
__device__ __forceinline__ bool is_aligned_generic(double a, double theta, double prec) {
  const double n1 = fabs(theta - a);
  const double n2 = fabs(n1 - 2 * kPI);
  return ((n1 > (3 * kPI) / 2) ? n2 : n1) <= prec;
}

// LineSegmentDetectorImpl::region_grow - exact visiting order; returns the region size, region in C.R[0..n).
// Four queue entries are expanded per step: lanes 8g..8g+7 fetch the 8 neighbours of entry i+g (one 16-byte record each),
// then the candidates are committed in the reference's order (queue order, then row-major inside the 3x3): every
// remaining candidate is tested against the CURRENT region angle at once, the first aligned one is added, which changes
// the angle; a pixel added earlier in the same step invalidates its duplicates in the later neighbourhoods.
// kFast: prec < pi/2, isAligned folded to  n <= prec || n >= prec_hi  (prec_hi = smallest double with 2pi - n <= prec; 2pi - n
// is exact for n in [pi, 4pi], so both forms agree bit for bit).
// Alignment WITHOUT the arctangent for the clear cases (kFast only).  The exact test compares the candidate's angle a with
// reg_angle = fastAtan2(sumdy, sumdx); the candidate's record also carries (cos a, sin a), so the TRUE angle D between the sum
// vector and the candidate is known from one dot product: cos D = (sumdx*c + sumdy*s) / |sum|.  fastAtan2's polynomial is within
// 0.0096 degrees of the true arctangent (measured over 4e7 vectors, tests/test_oracle_line.py pins the bound), float(angle)
// rounding is < 1e-4 degrees, so with a margin M = 0.05 degrees:  D <= prec - M  implies the exact test says aligned, D >= prec + M
// implies it says not aligned.  Only candidates inside the 2M band need the exact arctangent (kSure.ca2 / cn2 = cos^2(prec -/+ M)).
struct Sure { float ca2, cn2; };
// sure: D <= prec - M, the exact test says aligned; !maybe: D >= prec + M (or the candidate faces away), it says not aligned.
// (|sum| >= 1 in region_grow: the seed is a unit vector and every added unit vector is within prec < 90 degrees of the sum)
__device__ __forceinline__ void align_shortcut(float sumdx, float sumdy, float2 cs, Sure sure, bool& sure_al, bool& maybe) {
  const float n2 = __fmaf_rn(sumdx, sumdx, __fmul_rn(sumdy, sumdy));
  const float dot = __fmaf_rn(sumdx, cs.x, __fmul_rn(sumdy, cs.y)), d2 = __fmul_rn(dot, dot);
  sure_al = dot > 0.f && d2 >= __fmul_rn(sure.ca2, n2);
  maybe = dot > 0.f && d2 > __fmul_rn(sure.cn2, n2);
}
// the exact test of the fast path (prec < pi/2): isAligned folded with prec_hi, see region_grow
__device__ __forceinline__ bool aligned_fold(double reg_angle, double a, double prec, double prec_hi) {
  const double n1 = fabs(reg_angle - a);
  return (n1 <= prec) || (n1 >= prec_hi);
}

// need_n: the caller reads reg_angle_out only for regions of at least this many pixels (min_reg_size in the seed loop, 2 in refine)
template <bool kFast>
__device__ __forceinline__ int region_grow(const Ctx& C, unsigned seed, double prec, double prec_hi, Sure sure, double& reg_angle_out, int lane, int need_n) {
  const int sidx = (int)(seed >> 16) * C.sw + (int)(seed & 0xffffu);
  const float2 s0 = __ldg(&C.S2[C.fb + (unsigned)sidx]);
  double reg_angle = (double)__int_as_float(angle_bits(C, sidx)) * kDegToRads;
  float sumdx = s0.x, sumdy = s0.y;
  bool dirty = false;          // reg_angle lags the sums (it is the seed's own angle until the first pixel is added)
  if (lane == 0) { C.R[0] = seed; s_ring[0] = seed; own_of(C, sidx) = kUsedO; }
  int cnt = 1;
  __syncwarp();
  const int grp = lane >> 3, kk8 = lane & 7, kk = kk8 + (kk8 >= 4);
  const int ox = kk % 3 - 1, oy = kk / 3 - 1;
  for (int i = 0; i < cnt;) {
    const int m = min(4, cnt - i);
    GSTAT(kFast ? 1 : 10, 1);
    bool valid = false;
    int idx = -1;
    unsigned pk = 0xffff0000u | (unsigned)lane;      // unique per lane unless it names a real pixel
    int ab = 0;
    float2 csv = make_float2(0.f, 0.f);
    if (grp < m) {
      const int qi = i + grp;
      const unsigned p = (cnt - qi <= kORing) ? s_ring[qi & (kORing - 1)] : C.R[qi];
      const int xx = (int)(p & 0xffffu) + ox, yy = (int)(p >> 16) + oy;
      if (xx >= 0 && yy >= 0 && xx < C.sw && yy < C.sh) {
        idx = yy * C.sw + xx;
        GSTAT_ALL(kFast ? 16 : 17, 1);
        const int4 v = ld_rec(C, idx);
        if (v.x == kFree) {                           // defined and not USED
          valid = true; ab = v.y;
          csv = make_float2(__int_as_float(v.z), __int_as_float(v.w));
          pk = (unsigned)xx | ((unsigned)yy << 16);
        }
      }
    }
    i += m;
    unsigned live = __ballot_sync(0xffffffffu, valid);
    if (live == 0u) continue;
    GSTAT(2, 1);
    // lanes that name the same pixel (a free pixel sits in up to four of the 3x3 windows of one step); invalid lanes are unique
    // (skipping the MATCH when a single entry is expanded - its 8 neighbours are distinct - was measured slower)
    const unsigned dups = __match_any_sync(0xffffffffu, pk);
    unsigned acc = 0u;                                 // lanes accepted in this step, in order
    const int cnt0 = cnt;
    while (live) {
      GSTAT(3, 1);
      unsigned A;
      bool exact = !kFast;
      if (kFast) {
        bool sure_al, maybe;
        align_shortcut(sumdx, sumdy, csv, sure, sure_al, maybe);
        const unsigned MB = __ballot_sync(0xffffffffu, maybe) & live;
        if (MB == 0u) break;
        const unsigned SA = __ballot_sync(0xffffffffu, sure_al);
        if ((MB & (0u - MB)) & SA) A = MB;            // the first candidate that may be aligned surely is: no arctangent
        else exact = true;
      }
      if (exact) {
        GSTAT(5, 1);
        if (dirty) { reg_angle = (double)fast_atan2_deg(sumdy, sumdx) * kDegToRads; dirty = false; }
        const double a = (double)__int_as_float(ab) * kDegToRads;
        bool al;
        if (kFast) al = aligned_fold(reg_angle, a, prec, prec_hi);
        else al = is_aligned_generic(a, reg_angle, prec);
        A = __ballot_sync(0xffffffffu, al) & live;
        if (!A) break;
      }
      const int k = __ffs(A) - 1;
      GSTAT(kFast ? 4 : 11, 1);
      acc |= 1u << k;
      cnt++;
      sumdx = __fadd_rn(sumdx, __shfl_sync(0xffffffffu, csv.x, k));
      sumdy = __fadd_rn(sumdy, __shfl_sync(0xffffffffu, csv.y, k));
      dirty = true;
      // everything up to k has been decided; the same pixel in a later 3x3 is now USED
      live &= ~(((2u << k) - 1u) | __shfl_sync(0xffffffffu, dups, k));
    }
    if ((acc >> lane) & 1u) {      // publish: every accepted lane owns its pixel
      const int mypos = cnt0 + __popc(acc & lanemask_lt());
      own_of(C, idx) = kUsedO;
      C.R[mypos] = pk;
      s_ring[mypos & (kORing - 1)] = pk;
    }
    __syncwarp();
  }
  // most regions end below need_n and their angle is never read
  if (dirty && cnt >= need_n) reg_angle = (double)fast_atan2_deg(sumdy, sumdx) * kDegToRads;
  reg_angle_out = reg_angle;
  return cnt;
}
__device__ __noinline__ int region_grow_cold(const Ctx& C, unsigned seed, double prec, double& reg_angle, int lane) {
  return region_grow<false>(C, seed, prec, 0.0, Sure{0.f, 0.f}, reg_angle, lane, 2);
}

// region2rect + get_theta: sums in list order (see the header), extents by exact max / min
__device__ __forceinline__ double pixel_weight(const Ctx& C, int px, int py) {
  // the gradient magnitude sqrt((gx^2 + gy^2) / 4) of the reference from the integer sum of squares, through the table of
  // exact square roots (cheaper than an in-kernel fp64 sqrt)
  return __ldg(&C.wtab[__ldg(&C.SQ[C.fb + (unsigned)(py * C.sw + px)])]);
}
__device__ __noinline__ void region2rect(const Ctx& C, int n, double reg_angle, double prec, RectD& rec, int lane) {
  double acc = 0;                       // lanes 0, 1, 2: sum x*w, sum y*w, sum w
  GSTAT(9, n); GSTAT(12, 1);
  // the first two batches (64 pixels: most regions) stay in registers for the second and third pass
  unsigned pc0 = 0, pc1 = 0;
  double wc0 = 0, wc1 = 0;
#pragma unroll 1
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    double tx = 0, ty = 0, w = 0;
    if (i < n) {
      const unsigned p = C.R[i];
      const int px = (int)(p & 0xffffu), py = (int)(p >> 16);
      w = pixel_weight(C, px, py);
      tx = (double)px * w; ty = (double)py * w;
      if (i0 == 0) { pc0 = p; wc0 = w; } else if (i0 == 32) { pc1 = p; wc1 = w; }
    }
    ordered_add3(C, tx, ty, w, min(32, n - i0), acc, lane);
  }
  const double sw_ = ordered_get(acc, 2);
  const double x = ordered_get(acc, 0) / sw_, y = ordered_get(acc, 1) / sw_;
  acc = 0;                              // lanes 0, 1, 2: Ixx, Iyy, -Ixy  (Ixy -= t  ==  (-Ixy) += t, negated once at the end: exact)
#pragma unroll 1
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    double t1 = 0, t2 = 0, t3 = 0;
    if (i < n) {
      unsigned p; double w;
      if (i0 == 0) { p = pc0; w = wc0; } else if (i0 == 32) { p = pc1; w = wc1; }
      else { p = C.R[i]; w = pixel_weight(C, (int)(p & 0xffffu), (int)(p >> 16)); }
      const int px = (int)(p & 0xffffu), py = (int)(p >> 16);
      const double dx = (double)px - x, dy = (double)py - y;
      t1 = dy * dy * w; t2 = dx * dx * w; t3 = dx * dy * w;
    }
    ordered_add3(C, t1, t2, t3, min(32, n - i0), acc, lane);
  }
  const double Ixx = ordered_get(acc, 0), Iyy = ordered_get(acc, 1), Ixy = -ordered_get(acc, 2);
  const double lambda = 0.5 * (Ixx + Iyy - sqrt((Ixx - Iyy) * (Ixx - Iyy) + 4.0 * Ixy * Ixy));
  double theta = (fabs(Ixx) > fabs(Iyy)) ? (double)fast_atan2_cold((float)(lambda - Ixx), (float)Ixy)
                                         : (double)fast_atan2_cold((float)Ixy, (float)(lambda - Iyy));
  theta *= kDegToRads;
  if (fabs(angle_diff_signed(theta, reg_angle)) > prec) theta += kPI;
  double dx, dy;
  sincos(theta, &dy, &dx);              // one range reduction; same results as cos() / sin() (CUDA's sincos is the pair of them)
  double l_min = 0, l_max = 0, w_min = 0, w_max = 0;
#pragma unroll 1
  for (int i = lane; i < n; i += 32) {
    const unsigned p = (i < 32) ? pc0 : (i < 64) ? pc1 : C.R[i];
    const double rdx = (double)(int)(p & 0xffffu) - x, rdy = (double)(int)(p >> 16) - y;
    const double l = rdx * dx + rdy * dy, w = -rdx * dy + rdy * dx;
    l_max = fmax(l_max, l); l_min = fmin(l_min, l);
    w_max = fmax(w_max, w); w_min = fmin(w_min, w);
  }
  l_max = wmax_d(l_max); l_min = wmin_d(l_min); w_max = wmax_d(w_max); w_min = wmin_d(w_min);
  rec.x1 = x + l_min * dx; rec.y1 = y + l_min * dy;
  rec.x2 = x + l_max * dx; rec.y2 = y + l_max * dy;
  rec.width = w_max - w_min;
  if (rec.width < 1.0) rec.width = 1.0;
}

// reduce_region_radius(), one round: drop the pixels beyond radSq with the reference's swap-remove order.
// Every pixel is tested exactly once by the CPU loop, so the removed set is "all far pixels" (released in parallel);
// the survivors end up as: kept elements below the final size K stay, each hole below K (in increasing order) receives
// the last kept element of the shrinking tail (in decreasing order); both rankings come from prefix sums over the bit mask.
__device__ __noinline__ int reduce_round(const Ctx& C, int n, double xc, double yc, double radSq, int lane) {
  int kept = 0;
  GSTAT(8, 1); GSTAT(13, n);
#pragma unroll 1
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    bool far = false;
    if (i < n) {
      const unsigned p = C.R[i];
      const double px = (double)(int)(p & 0xffffu), py = (double)(int)(p >> 16);
      far = (px - xc) * (px - xc) + (py - yc) * (py - yc) > radSq;
      if (far) own_of(C, (int)(p >> 16) * C.sw + (int)(p & 0xffffu)) = kFree;
    }
    const unsigned mw = __ballot_sync(0xffffffffu, far);
    if (lane == 0) C.mask[C.fb + (unsigned)(i0 >> 5)] = mw;
    kept += __popc(~mw & (n - i0 >= 32 ? 0xffffffffu : ((1u << (n - i0)) - 1u)));
  }
  __syncwarp();
  if (kept == n) return n;
  // survivors: kept elements below K = kept stay; hole number r below K (increasing position) receives kept element
  // number r of the tail [K, n) counted FROM THE END - exactly what the CPU's swap-with-last loop leaves behind.
  // Both rankings are prefix sums over the mask words: a warp scan per 32 words, no serial walk over the pixels.
  const int K = kept, nw = (n + 31) >> 5, wK = K >> 5;
  unsigned* fill = C.R + C.fill_off;                 // scratch: position of the r-th kept tail element from the end
  int ntail = 0;                                     // kept elements in [K, n)
#pragma unroll 1
  for (int w0 = wK; w0 < nw; w0 += 32) {
    const int w = w0 + lane;
    unsigned km = 0u;
    if (w < nw) {
      km = ~C.mask[C.fb + w];
      if (w == wK) km &= ~((1u << (K & 31)) - 1u);                       // positions >= K only
      if (w == nw - 1 && (n & 31)) km &= (1u << (n & 31)) - 1u;          // positions < n only
    }
    int c = __popc(km), incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    int rank = ntail + incl - c;                     // rank from the START of the tail of this word's first kept element
    while (km) {
      const int bit = __ffs(km) - 1;
      km &= km - 1u;
      fill[rank++] = (unsigned)(w * 32 + bit);
    }
    ntail += __shfl_sync(0xffffffffu, incl, 31);
  }
  __syncwarp();
  int nholes = 0;
#pragma unroll 1
  for (int w0 = 0; w0 * 32 < K; w0 += 32) {
    const int w = w0 + lane;
    unsigned hm = 0u;
    if (w * 32 < K) {
      hm = C.mask[C.fb + w];
      if (w == wK) hm &= (1u << (K & 31)) - 1u;                          // holes below K only
    }
    int c = __popc(hm), incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    int r = nholes + incl - c;
    while (hm) {
      const int bit = __ffs(hm) - 1;
      hm &= hm - 1u;
      C.R[w * 32 + bit] = C.R[fill[ntail - 1 - r]];  // r-th hole <- r-th kept tail element from the end
      r++;
    }
    nholes += __shfl_sync(0xffffffffu, incl, 31);
  }
  __syncwarp();
  return kept;
}

// LineSegmentDetectorImpl::refine + reduce_region_radius; n is updated; returns false if the region is rejected
__device__ __noinline__ bool refine(const Ctx& C, int& n, double reg_angle, double prec, RectD& rec, double density_th, int lane, bool& released) {
  double density = (double)n / (dist_d(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
  if (density >= density_th) return true;
  released = true;              // from here on USED flags are cleared
  GSTAT(7, 1);
  const unsigned p0 = C.R[0];
  const double xc = (double)(int)(p0 & 0xffffu), yc = (double)(int)(p0 >> 16);
  const double ang_c = (double)__int_as_float(angle_bits(C, (int)(p0 >> 16) * C.sw + (int)(p0 & 0xffffu))) * kDegToRads;
  double sum = 0, s_sum = 0, sacc = 0;
  int cnt = 0;
#pragma unroll 1
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    bool in = false;
    double ad = 0, ad2 = 0;
    if (i < n) {
      const unsigned p = C.R[i];
      const int pidx = (int)(p >> 16) * C.sw + (int)(p & 0xffffu);
      own_of(C, pidx) = kFree;
      const double px = (double)(int)(p & 0xffffu), py = (double)(int)(p >> 16);
      if (dist_d(xc, yc, px, py) < rec.width) {
        in = true;
        ad = angle_diff_signed((double)__int_as_float(angle_bits(C, pidx)) * kDegToRads, ang_c);
        ad2 = ad * ad;
      }
    }
    unsigned mi = __ballot_sync(0xffffffffu, in);
    cnt += __popc(mi);
    s_red[lane] = ad; s_red[32 + lane] = ad2;
    __syncwarp();
    const double* row = s_red + 32 * (lane & 1);       // lane 0: sum, lane 1: s_sum (the additions in list order)
    while (mi) {
      const int k = __ffs(mi) - 1;
      mi &= mi - 1u;
      sacc += row[k];
    }
    __syncwarp();
  }
  sum = shfl_d(sacc, 0); s_sum = shfl_d(sacc, 1);
  __syncwarp();
  const double mean_angle = sum / (double)cnt;
  const double tau = 2.0 * sqrt((s_sum - 2.0 * mean_angle * sum) / (double)cnt + mean_angle * mean_angle);
  n = region_grow_cold(C, p0, tau, reg_angle, lane);
  if (n < 2) return false;
  region2rect(C, n, reg_angle, prec, rec, lane);
  density = (double)n / (dist_d(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
  if (density >= density_th) return true;
  const double r1 = dist_sq(xc, yc, rec.x1, rec.y1), r2 = dist_sq(xc, yc, rec.x2, rec.y2);
  double radSq = r1 > r2 ? r1 : r2;
  while (density < density_th) {
    radSq *= 0.75 * 0.75;
    n = reduce_round(C, n, xc, yc, radSq, lane);
    if (n < 2) return false;
    region2rect(C, n, reg_angle, prec, rec, lane);
    density = (double)n / (dist_d(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
  }
  return true;
}

}  // namespace ord

// One warp per frame; grid = frames (32 one-warp CTAs resident per SM: 4224 frames in one wave on the 132 SMs of an H100).
// kPre: examine the neighbourhoods of a whole batch of seeds up front (see below): fewer dependent round trips per frame, but
// more requests - it pays when the GPU is not full of frames (small batches) and costs when it is.
template <bool kPre>
__global__ void __launch_bounds__(32, 32) k_lsd_grow_ordered(LineParams P, int4* __restrict__ REC, const int* __restrict__ SQ, const float2* __restrict__ seedcs,
                                                             const unsigned* __restrict__ order, const int* __restrict__ ndef,
                                                             unsigned* __restrict__ reg, int reg_stride, unsigned* __restrict__ mask, const double* __restrict__ wtab,
                                                             float4* __restrict__ segs, int* __restrict__ nseg, int* __restrict__ overflow, int nframes) {
  using namespace ord;
  const int lane = threadIdx.x & 31;
  for (int f = blockIdx.x; f < nframes; f += gridDim.x) {
    const Ctx C = {REC, SQ, seedcs, mask, (unsigned)f * (unsigned)P.npx, wtab, reg + (long long)f * reg_stride, P.sw, P.sh, P.npx};
    const unsigned* O = order + (long long)f * P.npx;
    float4* S = segs + (long long)f * P.seg_cap;
    const int n = ndef[f];
    int ns = 0;
    for (int i0 = 0; i0 < n; i0 += 32) {
      const int i = i0 + lane;
      const unsigned pix = (i < n) ? O[i] : 0u;
      const int pidx = (int)(pix >> 16) * P.sw + (int)(pix & 0xffffu);
      const int4 me = (i < n) ? ld_rec(C, pidx) : make_int4(0, 0, 0, 0);
      unsigned todo = __ballot_sync(0xffffffffu, i < n && me.x == kFree);
      // Seeds of this batch whose region cannot get past the seed itself: no FREE neighbour is aligned with the seed's own angle
      // (the region angle of the first step).  Between two regions the set of free pixels only shrinks (a region releases only
      // pixels it took itself), so "no free aligned neighbour now" still holds when the seed's turn comes: the region is the
      // seed alone, below min_reg_size, and all that happens is that the seed becomes USED - at ITS turn, not earlier (an
      // earlier seed of the batch may still grow over it).  The 8 records per seed are loaded by 32 lanes at once here instead
      // of one region at a time; they also warm the lines the regions that do grow start from.
      bool single = false;
      if (kPre && ((todo >> lane) & 1u)) {
        const int sx = (int)(pix & 0xffffu), sy = (int)(pix >> 16);
        const double a0 = (double)__int_as_float(me.y) * kDegToRads;
        bool any = false;
#pragma unroll
        for (int q = 0; q < 8; q++) {
          const int kq = q + (q >= 4), xx = sx + kq % 3 - 1, yy = sy + kq / 3 - 1;
          if (xx >= 0 && yy >= 0 && xx < P.sw && yy < P.sh) {
            const int4 v = ld_rec(C, yy * P.sw + xx);
            any |= (v.x == kFree) && aligned_fold(a0, (double)__int_as_float(v.y) * kDegToRads, P.prec, P.prec_hi);
          }
        }
        single = !any;
        prefetch_l2(&C.S2[C.fb + (unsigned)pidx]);
      }
      if (!kPre && ((todo >> lane) & 1u)) {   // this batch's seeds that will grow: their seed record and 3x3 rows into L2
        prefetch_l2(&C.S2[C.fb + (unsigned)pidx]);
        const int up = max(pidx - P.sw, 1), dn = min(pidx + P.sw, P.npx - 2);
        prefetch_l2(&C.REC[C.fb + (unsigned)(up - 1)]); prefetch_l2(&C.REC[C.fb + (unsigned)(up + 1)]); prefetch_l2(&C.REC[C.fb + (unsigned)(dn - 1)]); prefetch_l2(&C.REC[C.fb + (unsigned)(dn + 1)]);
        prefetch_l2(&C.REC[C.fb + (unsigned)(max(pidx, 1) - 1)]); prefetch_l2(&C.REC[C.fb + (unsigned)(min(pidx, P.npx - 2) + 1)]);
      }
      const unsigned singles = __ballot_sync(0xffffffffu, single);
      if (i + 32 < n) { const unsigned pn = O[i + 32]; prefetch_l2(&C.REC[C.fb + (unsigned)((int)(pn >> 16) * P.sw + (int)(pn & 0xffffu))]); }
      while (todo) {
        {   // the lone seeds in front of the next seed that may grow: USED, nothing else
          const unsigned grow = todo & ~singles;
          const unsigned below = grow ? ((grow & (0u - grow)) - 1u) : 0xffffffffu;
          if ((todo & singles & below) >> lane & 1u) own_of(C, pidx) = kUsedO;
          todo &= ~below;
          __syncwarp();
          if (!todo) break;
        }
        const int k = __ffs(todo) - 1;
        const unsigned seed = __shfl_sync(0xffffffffu, pix, k);
        double reg_angle;
        bool released = false;
        GSTAT(0, 1);
        int cnt = region_grow<true>(C, seed, P.prec, P.prec_hi, Sure{P.sure_ca2, P.sure_cn2}, reg_angle, lane, P.min_reg_size);
        if (cnt == 1) GSTAT(14, 1);
        if (cnt <= 4) GSTAT(15, 1);
        if (cnt >= P.min_reg_size) {
          GSTAT(6, 1);
          RectD rec;
          region2rect(C, cnt, reg_angle, P.prec, rec, lane);
          if (refine(C, cnt, reg_angle, P.prec, rec, P.density_th, lane, released)) {
            if (lane == 0 && ns < P.seg_cap)
              S[ns] = make_float4((float)((rec.x1 + 0.5) / 0.8), (float)((rec.y1 + 0.5) / 0.8), (float)((rec.x2 + 0.5) / 0.8),
                                  (float)((rec.y2 + 0.5) / 0.8));
            ns++;
          }
        }
        __syncwarp();
        // seeds later in this batch may have been consumed (or released by refine): re-read their words - unless the region was
        // the seed alone (36 % of the regions), which touched no other pixel
        if (cnt == 1) todo &= ~((2u << k) - 1u);
        else todo = __ballot_sync(0xffffffffu, i < n && lane > k && own_of(C, pidx) == kFree);
      }
    }
    if (lane == 0) { nseg[f] = min(ns, P.seg_cap); if (ns > P.seg_cap) atomicOr(overflow, 1); }
    __syncwarp();
  }
}

}  // namespace pl
