// Host check of pl-slam_b200/csrc/libm_glibc.cuh against the running C library (tests/test_libm_glibc.py).
// Prints "mismatches <atan2f> <sinf> <cosf> <logf> of <n>"; exit code 0 only when all four are zero.
#include <cstdio>
#include <cstdlib>
#include "libm_args.h"
int main(int argc, char** argv) {
  const long n = argc > 1 ? atol(argv[1]) : 20000000;
  long bad_a = 0, bad_s = 0, bad_c = 0, bad_l = 0;
  LibmArgs args;
  LibmCase c;
  for (long i = 0; i < n; i++) {
    if (!args.next(i, c)) continue;
    const float b = pl::glibc::atan2f_(c.y, c.x);
    if (pl::glibc::f2u(c.atan2) != pl::glibc::f2u(b)) { if (bad_a < 5) fprintf(stderr, "atan2f(%a, %a): libm %a here %a\n", c.y, c.x, c.atan2, b); bad_a++; }
    float s1, c1;
    pl::glibc::sincosf_(c.t, &s1, &c1);
    if (pl::glibc::f2u(c.sin) != pl::glibc::f2u(s1)) { if (bad_s < 5) fprintf(stderr, "sinf(%a): libm %a here %a\n", c.t, c.sin, s1); bad_s++; }
    if (pl::glibc::f2u(c.cos) != pl::glibc::f2u(c1)) { if (bad_c < 5) fprintf(stderr, "cosf(%a): libm %a here %a\n", c.t, c.cos, c1); bad_c++; }
    const float l1 = pl::glibc::logf_(c.q);
    if (pl::glibc::f2u(c.log) != pl::glibc::f2u(l1)) { if (bad_l < 5) fprintf(stderr, "logf(%a): libm %a here %a\n", c.q, c.log, l1); bad_l++; }
  }
  printf("mismatches %ld %ld %ld %ld of %ld\n", bad_a, bad_s, bad_c, bad_l, n);
  return (bad_a || bad_s || bad_c || bad_l) ? 1 : 0;
}
