// Float elementary functions as the reference gets them from its C library.
//
// The reference calls  atan2(float, float)  (LSDDetector_custom.cpp:187, KeyLine::angle) and  cos / sin  of a float
// (binary_descriptor_custom.cpp:1130-1131, the LBD line direction; ORBextractor.cc:113, the rBRIEF steering) with <cmath>'s
// overloads, i.e. the FLOAT functions of libm: atan2f and sincosf (nm -u of the reference objects compiled by the test tooling
// shows exactly these).  Their last bit is not what rounding the double function gives (about 16 % of KeyLine angles differ
// by one ulp), so byte parity with the reference needs the same algorithms.  These are restatements of the published algorithms
// glibc 2.39 (the C library of this image and of the GPU box) uses:
//   atan2f / atanf : FreeBSD msun / fdlibm e_atan2f.c, s_atanf.c (Sun Microsystems 1993), all arithmetic in fp32;
//   logf           : Arm Optimized Routines logf.c (16-entry table, degree-3 polynomial, fp64; MapPoint / MapLine::PredictScale call
//                    log() on a float, MapPoint.cc:404, MapLine.cpp:403);
//   sincosf        : Arm Optimized Routines sincosf.c (Szabolcs Nagy, Wilco Dijkstra 2018), argument reduction and the two
//                    minimax polynomials in fp64, one rounding to fp32; the fused multiply-adds are those of the x86-64 FMA build
//                    glibc selects on every CPU with FMA3 (a different contraction can only change the result when the fp64 value
//                    lies within 1e-16 of an fp32 rounding boundary: a 1e-8 event).
// tests/test_libm_glibc.py compiles this header for the host and compares it with the running libm on 2e7 random arguments plus
// the special values: zero mismatches.  Only the argument ranges the path produces are covered (finite, |x| < 120 for sincosf);
// the device build relies on -fmad=false (pl-slam_b200/csrc/Makefile) so that no other product is contracted, and
// tests/test_float_math_gpu.py compares it with the host build and the running libm on the same arguments.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>
#ifdef __CUDACC__
#define PL_LIBM_HD __host__ __device__ __forceinline__
#else
#define PL_LIBM_HD inline
#endif

namespace pl {
namespace glibc {

PL_LIBM_HD uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
PL_LIBM_HD float u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

// s_atanf.c
PL_LIBM_HD float atanf_(float x) {
  const float atanhi[4] = {u2f(0x3eed6338u), u2f(0x3f490fdau), u2f(0x3f7b985eu), u2f(0x3fc90fdau)};
  const float atanlo[4] = {u2f(0x31ac3769u), u2f(0x33222168u), u2f(0x33140fb4u), u2f(0x33a22168u)};
  const float aT[11] = {u2f(0x3eaaaaabu), u2f(0xbe4ccccdu), u2f(0x3e124925u), u2f(0xbde38e38u), u2f(0x3dba2e6eu), u2f(0xbd9d8795u),
                        u2f(0x3d886b35u), u2f(0xbd6ef16bu), u2f(0x3d4bda59u), u2f(0xbd15a221u), u2f(0x3c8569d7u)};
  const float one = 1.0f;
  const int32_t hx = (int32_t)f2u(x), ix = hx & 0x7fffffff;
  int id;
  if (ix >= 0x4c000000) {                     // |x| >= 2^25
    if (ix > 0x7f800000) return x + x;
    return hx > 0 ? atanhi[3] + atanlo[3] : -atanhi[3] - atanlo[3];
  }
  if (ix < 0x3ee00000) {                      // |x| < 0.4375
    if (ix < 0x31000000) return x;            // |x| < 2^-29
    id = -1;
  } else {
    x = fabsf(x);
    if (ix < 0x3f980000) {                    // |x| < 1.1875
      if (ix < 0x3f300000) { id = 0; x = (2.0f * x - one) / (2.0f + x); }
      else { id = 1; x = (x - one) / (x + one); }
    } else {
      if (ix < 0x401c0000) { id = 2; x = (x - 1.5f) / (one + 1.5f * x); }
      else { id = 3; x = -1.0f / x; }
    }
  }
  const float z = x * x, w = z * z;
  const float s1 = z * (aT[0] + w * (aT[2] + w * (aT[4] + w * (aT[6] + w * (aT[8] + w * aT[10])))));
  const float s2 = w * (aT[1] + w * (aT[3] + w * (aT[5] + w * (aT[7] + w * aT[9]))));
  if (id < 0) return x - x * (s1 + s2);
  const float r = atanhi[id] - ((x * (s1 + s2) - atanlo[id]) - x);
  return hx < 0 ? -r : r;
}

// e_atan2f.c (finite arguments; infinities and NaN do not occur on the path and take the generic branch)
PL_LIBM_HD float atan2f_(float y, float x) {
  const float tiny = 1.0e-30f, pi_o_2 = u2f(0x3fc90fdbu), pi = u2f(0x40490fdbu), pi_lo = u2f(0xb3bbbd2eu);
  const int32_t hx = (int32_t)f2u(x), hy = (int32_t)f2u(y), ix = hx & 0x7fffffff, iy = hy & 0x7fffffff;
  if (ix > 0x7f800000 || iy > 0x7f800000) return x + y;
  if (hx == 0x3f800000) return atanf_(y);
  const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);
  if (iy == 0) return m < 2 ? y : (m == 2 ? pi + tiny : -pi - tiny);
  if (ix == 0) return hy < 0 ? -pi_o_2 - tiny : pi_o_2 + tiny;
  const int k = (iy - ix) >> 23;
  float z;
  if (k > 60) z = pi_o_2 + 0.5f * pi_lo;
  else if (hx < 0 && k < -60) z = 0.0f;
  else z = atanf_(fabsf(y / x));
  switch (m) {
    case 0: return z;
    case 1: return u2f(f2u(z) ^ 0x80000000u);
    case 2: return pi - (z - pi_lo);
    default: return (z - pi_lo) - pi;
  }
}

// sincosf.c: |y| < 120 (the path passes angles in [-pi, 2 pi)); larger arguments are outside this restatement
PL_LIBM_HD void sincosf_(float y, float* sinp, float* cosp) {
  const double hpi_inv = 0x1.45f306dc9c883p+23, hpi = 0x1.921fb54442d18p+0;   // 2/pi * 2^24, pi/2
  const double C0 = 1.0, C1 = -0x1.ffffffd0c621cp-2, C2 = 0x1.55553e1068f19p-5, C3 = -0x1.6c087e89a359dp-10, C4 = 0x1.99343027bf8c3p-16;
  const double S1 = -0x1.555545995a603p-3, S2 = 0x1.1107605230bc4p-7, S3 = -0x1.994eb3774cf24p-13;
  const uint32_t top = (f2u(y) >> 20) & 0x7ffu;
  double x = (double)y, x2, cs = 1.0;    // cs: sign of the cosine polynomial (the second table of the original negates c0..c4)
  int n = 0;
  if (top < ((0x3f490fdbu >> 20) & 0x7ffu)) {          // |y| < pi/4
    x2 = x * x;
    if (top < ((0x39800000u >> 20) & 0x7ffu)) { *sinp = y; *cosp = 1.0f; return; }   // |y| < 2^-12
  } else {
    const double r = x * hpi_inv;
    n = ((int32_t)r + 0x800000) >> 24;
    x = fma(-(double)n, hpi, x);
    const double s = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
    if (n & 2) cs = -1.0;
    x2 = x * x;
    x = x * s;
  }
  const double x4 = x2 * x2, x3 = x2 * x;
  const double c2 = fma(x2, cs * C4, cs * C3), s1 = fma(x2, S3, S2), c1 = fma(x2, cs * C1, cs * C0);
  const double x5 = x3 * x2, x6 = x4 * x2;
  const double s = fma(x3, S1, x), c = fma(x4, cs * C2, c1);
  const float sv = (float)fma(x5, s1, s), cv = (float)fma(x6, c2, c);
  if (n & 1) { *sinp = cv; *cosp = sv; } else { *sinp = sv; *cosp = cv; }
}

// logf.c: positive normal arguments (the path passes distance ratios); zero, negatives, subnormals, inf / NaN are outside this restatement
PL_LIBM_HD float logf_(float x) {
  const double invc[16] = {0x1.661ec79f8f3bep+0, 0x1.571ed4aaf883dp+0, 0x1.49539f0f010bp+0, 0x1.3c995b0b80385p+0, 0x1.30d190c8864a5p+0, 0x1.25e227b0b8eap+0,
                           0x1.1bb4a4a1a343fp+0, 0x1.12358f08ae5bap+0, 0x1.0953f419900a7p+0, 0x1p+0, 0x1.e608cfd9a47acp-1, 0x1.ca4b31f026aap-1,
                           0x1.b2036576afce6p-1, 0x1.9c2d163a1aa2dp-1, 0x1.886e6037841edp-1, 0x1.767dcf5534862p-1};
  const double logc[16] = {-0x1.57bf7808caadep-2, -0x1.2bef0a7c06ddbp-2, -0x1.01eae7f513a67p-2, -0x1.b31d8a68224e9p-3, -0x1.6574f0ac07758p-3, -0x1.1aa2bc79c81p-3,
                           -0x1.a4e76ce8c0e5ep-4, -0x1.1973c5a611cccp-4, -0x1.252f438e10c1ep-5, 0x0p+0, 0x1.aa5aa5df25984p-5, 0x1.c5e53aa362eb4p-4,
                           0x1.526e57720db08p-3, 0x1.bc2860d22477p-3, 0x1.1058bc8a07ee1p-2, 0x1.4043057b6ee09p-2};
  const double Ln2 = 0x1.62e42fefa39efp-1, A0 = -0x1.00ea348b88334p-2, A1 = 0x1.5575b0be00b6ap-2, A2 = -0x1.ffffef20a4123p-2;
  const uint32_t ix = f2u(x);
  if (ix == 0x3f800000u) return 0.0f;
  const uint32_t tmp = ix - 0x3f330000u;
  const int i = (int)((tmp >> 19) & 15u), k = (int32_t)tmp >> 23;
  const uint32_t iz = ix - (tmp & 0xff800000u);
  const double z = (double)u2f(iz);
  const double r = fma(z, invc[i], -1.0), y0 = fma((double)k, Ln2, logc[i]);
  const double r2 = r * r;
  double y = fma(A1, r, A2);
  y = fma(A0, r2, y);
  y = fma(y, r2, y0 + r);
  return (float)y;
}

}  // namespace glibc
}  // namespace pl
