// The libm argument sequence of libm_args.h and the host build of pl-slam_b200/csrc/libm_glibc.cuh, as a shared library for
// tests/test_float_math_gpu.py (ctypes), which runs the device build on the same arguments.
#include "libm_args.h"

// cases i0 .. i0 + n - 1 of the sequence whose generator state *st holds (0: the start of the sequence, i0 = 0), as up to n
// LibmCase records in out; writes the state back and returns how many records it wrote (cases with a non-finite atan2f pair
// are skipped)
extern "C" long libm_cases(uint64_t* st, long i0, long n, LibmCase* out) {
  LibmArgs args;
  if (*st) args.st = *st;
  long m = 0;
  for (long i = i0; i < i0 + n; i++)
    if (args.next(i, out[m])) m++;
  *st = args.st;
  return m;
}

// the host build of the header on n arguments: fn 0 out0 = atan2f_(a, b), 1 out0, out1 = sincosf_(a), 2 out0 = logf_(a)
extern "C" void libm_header(int fn, const float* a, const float* b, long n, float* out0, float* out1) {
  for (long i = 0; i < n; i++) {
    if (fn == 0) out0[i] = pl::glibc::atan2f_(a[i], b[i]);
    else if (fn == 1) pl::glibc::sincosf_(a[i], out0 + i, out1 + i);
    else out0[i] = pl::glibc::logf_(a[i]);
  }
}
