// The arguments of the float libm checks and the running C library's answers for them: one fixed sequence, so the host check
// (libm_check.cpp) and the device check (libm_args.cpp, tests/test_float_math_gpu.py) see the same arguments.
// Case i draws an atan2f pair from one of eight families (i & 7), a sincosf angle and a logf ratio; only the domains the
// restatements cover are drawn: sincosf |t| < 120, logf positive normals.
#pragma once
#include <cmath>
#include <cstdint>
#include "../../pl-slam_b200/csrc/libm_glibc.cuh"

struct LibmCase {
  float y, x, atan2;   // atan2f(y, x)
  float t, sin, cos;   // sincosf(t)
  float q, log;        // logf(q)
};

struct LibmArgs {
  uint64_t st = 0x9E3779B97F4A7C15ull;
  uint64_t rnd() { st ^= st << 13; st ^= st >> 7; st ^= st << 17; return st; }
  float urand(float lo, float hi) { return lo + (hi - lo) * (float)((rnd() >> 40) * (1.0 / 16777216.0)); }

  // case i of the sequence (call with i = 0, 1, 2, ... in order); false when the atan2f pair is not finite, and then the
  // case is skipped whole
  bool next(long i, LibmCase& c) {
    float y, x;
    switch (i & 7) {
      case 0: y = urand(-640.f, 640.f); x = urand(-640.f, 640.f); break;                 // end-point differences of a KeyLine
      case 1: y = (float)((int)(rnd() % 1281) - 640); x = (float)((int)(rnd() % 1281) - 640); break;   // integers, zeros, axes
      case 2: y = urand(-1.f, 1.f); x = urand(-1e-3f, 1e-3f); break;
      case 3: y = urand(-1e-3f, 1e-3f); x = urand(-1.f, 1.f); break;
      case 4: y = urand(-2000.f, 2000.f) * 0.25f; x = urand(-2000.f, 2000.f) * 0.25f; break;
      case 5: y = pl::glibc::u2f((uint32_t)rnd() & 0xbfffffffu); x = pl::glibc::u2f((uint32_t)rnd() & 0xbfffffffu); break;   // any finite bit pattern below 2
      default: y = urand(-10.f, 10.f); x = urand(-10.f, 10.f); break;
    }
    if (!std::isfinite(y) || !std::isfinite(x)) return false;
    volatile float vy, vx;   // volatile: the compiler must call libm, not fold
    vy = y; vx = x;
    c.y = y; c.x = x; c.atan2 = atan2f(vy, vx);
    // angles: atan2f results, degrees * pi/180 in [0, 2 pi), and anything below 120
    c.t = (i & 1) ? c.atan2 : ((i & 2) ? urand(0.f, 360.f) * (float)(3.14159265358979323846 / 180.f) : urand(-119.f, 119.f));
    vy = c.t;
    sincosf(vy, &c.sin, &c.cos);
    // logf: distance ratios around 1 (PredictScale), powers of the scale factor, and any positive normal float
    switch (i & 3) {
      case 0: c.q = urand(0.05f, 20.f); break;
      case 1: c.q = powf(1.2f, (float)((int)(rnd() % 17) - 8)) * (1.0f + urand(-2e-6f, 2e-6f)); break;
      case 2: c.q = pl::glibc::u2f(0x00800000u + (uint32_t)(rnd() % (0x7f800000u - 0x00800000u))); break;
      default: c.q = urand(0.5f, 2.f); break;
    }
    vy = c.q;
    c.log = logf(vy);
    return true;
  }
};
