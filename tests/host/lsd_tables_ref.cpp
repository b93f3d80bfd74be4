// Host reference of LSD region growing's gradient table (pl-slam_b200/csrc/line.cu grad_record), as a shared library for
// tests/test_lsd_tables_gpu.py (ctypes).  For the fastAtan2 angle deg of each gradient (computed by the oracle), what the reference
// lsd.cpp computes from it: region_grow adds cos(float(angle)), sin(float(angle)) with <cmath>'s float overloads (the C library's
// cosf / sinf) and starts a region from float(std::cos(angle)), float(std::sin(angle)) of the fp64 angle.
#include <cmath>

extern "C" void lsd_table_ref(const float* deg, long n, float* rec /*[n][4]*/, float* seed /*[n][2]*/) {
  const double deg_to_rads = 3.14159265358979323846 / 180;
  for (long i = 0; i < n; i++) {
    const double angle = deg[i] * deg_to_rads;
    const float af = float(angle);
    rec[4 * i] = deg[i];
    rec[4 * i + 1] = cosf(af);
    rec[4 * i + 2] = sinf(af);
    rec[4 * i + 3] = 0.f;
    seed[2 * i] = float(std::cos(angle));
    seed[2 * i + 1] = float(std::sin(angle));
  }
}
