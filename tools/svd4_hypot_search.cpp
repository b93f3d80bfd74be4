// Search for 4x4 fp32 matrices on which cv::SVD's one-sided Jacobi (pl-slam_b200/csrc/svd4.cuh) gives a different vt when its
// rotation takes gamma from the C library's hypot instead of OpenCV's own hypot template.  Such matrices are rare (about one
// uniform random matrix in 1e7 to 1e8), so the random families of tests/golden/orb_cv2_svd4.npz cannot tell the two hypots apart; the
// ones found here are added to it (tools/gen_svd4_cv2.py), where cv2.SVDecomp decides which hypot is right.
//
//   g++ -O2 -std=c++17 -ffp-contract=off -pthread tools/svd4_hypot_search.cpp -o /tmp/svd4_hypot_search
//   /tmp/svd4_hypot_search [matrices = 2e8] [wanted = 12] [seed = 1]
// Prints one line per matrix found: its 16 fp32 bit patterns, row-major.
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>
#include "../pl-slam_b200/csrc/svd4.cuh"

// The same Jacobi as svd4.cuh with the C library's hypot; returns vt (row-major).
static void svd4_libm_hypot(const float* A, float* vt) {
  float At[4][4], V[4][4];
  double W[4];
  auto dot = [](const float* x, const float* y) { double s = 0; for (int k = 0; k < 4; k++) s += (double)x[k] * (double)y[k]; return s; };
  auto rot = [](float* x, float* y, float c, float s) {
    for (int k = 0; k < 4; k++) { const float t0 = c * x[k] + s * y[k], t1 = -s * x[k] + c * y[k]; x[k] = t0; y[k] = t1; }
  };
  for (int i = 0; i < 4; i++) {
    for (int k = 0; k < 4; k++) { At[i][k] = A[4 * k + i]; V[i][k] = i == k; }
    W[i] = dot(At[i], At[i]);
  }
  const double eps = (double)(2.0f * 1.1920928955078125e-07f);
  for (int iter = 0; iter < 30; iter++) {
    bool changed = false;
    for (int i = 0; i < 3; i++)
      for (int j = i + 1; j < 4; j++) {
        const double a = W[i], b = W[j];
        double p = dot(At[i], At[j]);
        if (std::fabs(p) <= eps * std::sqrt(a * b)) continue;
        p *= 2;
        const double beta = a - b, gamma = ::hypot(p, beta);
        float c, s;
        if (beta < 0) { s = (float)std::sqrt((gamma - beta) * 0.5 / gamma); c = (float)(p / (gamma * s * 2)); }
        else { c = (float)std::sqrt((gamma + beta) / (gamma * 2)); s = (float)(p / (gamma * c * 2)); }
        rot(At[i], At[j], c, s);
        W[i] = dot(At[i], At[i]); W[j] = dot(At[j], At[j]);
        rot(V[i], V[j], c, s);
        changed = true;
      }
    if (!changed) break;
  }
  for (int i = 0; i < 4; i++) W[i] = std::sqrt(dot(At[i], At[i]));
  for (int i = 0; i < 3; i++) {
    int j = i;
    for (int k = i + 1; k < 4; k++) if (W[j] < W[k]) j = k;
    if (j != i) { std::swap(W[i], W[j]); for (int m = 0; m < 4; m++) std::swap(V[i][m], V[j][m]); }
  }
  memcpy(vt, V, sizeof V);
}

int main(int argc, char** argv) {
  const long long n = argc > 1 ? (long long)atof(argv[1]) : 200000000LL;
  const int wanted = argc > 2 ? atoi(argv[2]) : 12;
  const uint64_t seed = argc > 3 ? strtoull(argv[3], nullptr, 10) : 1;
  const int T = std::max(1u, std::thread::hardware_concurrency());
  std::atomic<int> found{0};
  std::mutex mu;
  std::vector<std::thread> pool;
  for (int t = 0; t < T; t++)
    pool.emplace_back([&, t] {
      uint64_t st = 0x9E3779B97F4A7C15ull * (seed * 1000003ull + t + 1);
      auto rnd = [&] { st ^= st << 13; st ^= st >> 7; st ^= st << 17; return st; };
      float A[16], w[4], v1[16], v2[16];
      for (long long i = t; i < n && found.load() < wanted; i += T) {
        for (float& a : A) a = (float)((rnd() >> 40) * (2.0 / 16777216.0) - 1.0);     // uniform in [-1, 1)
        pl::svd4(A, w, v1);
        svd4_libm_hypot(A, v2);
        if (memcmp(v1, v2, sizeof v1) == 0) continue;
        std::lock_guard<std::mutex> lock(mu);
        if (found.fetch_add(1) >= wanted) break;
        for (float a : A) { uint32_t u; memcpy(&u, &a, 4); printf("%u ", u); }
        printf("\n");
        fflush(stdout);
      }
    });
  for (auto& th : pool) th.join();
  return 0;
}
