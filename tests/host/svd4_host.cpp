// pl-slam_b200/csrc/svd4.cuh compiled for the host (tests/test_triangulate_svd.py loads it with ctypes and compares it with cv2).
#include "../../pl-slam_b200/csrc/svd4.cuh"
extern "C" void svd4_batch(const float* A, int n, float* w, float* vt) {
  for (int i = 0; i < n; i++) pl::svd4(A + 16 * i, w + 4 * i, vt + 16 * i);
}
