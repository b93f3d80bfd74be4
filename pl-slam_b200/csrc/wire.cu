// Wire / disk formats around the path (SURVEY.md §8 f.4): the pose record the ranks exchange and the monocular trajectory
// writers of the reference, System::SaveKeyFrameTrajectoryTUM (src/System.cc:396-431) and SaveKeyFrameTrajectoryMonoKitti
// (:433-464), plus the flat binary dump of one front-end step for offline replay (same container as pl-slam_b200/trajectory.py).
//
// A pose record is what both writers print for a keyframe: Rwc = KeyFrame::GetRotation().t(), Ow = GetCameraCenter()
// (= -Rcw^T tcw, fp32 in cv::gemm's accumulation order, KeyFrame.cc:52-66) and Converter::toQuaternion(Rwc) (Converter.cc:
// 141-153: Eigen::Quaterniond from the fp64 copy of the matrix, returned as x y z w).  One thread per pose computes it on the
// device, so the N-rank all-gather can ship 16 floats per frame that every rank writes out without touching the poses again.
#include "common.cuh"
#include <cstdio>
#include <string>
#include <vector>

namespace pl {
__global__ void k_pose_records(const float* __restrict__ Tcw, int n, float* __restrict__ rec) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* T = Tcw + 16 * (long long)i;
  float* o = rec + 16 * (long long)i;
  float R[3][3];
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) R[r][c] = T[4 * c + r];      // Rwc = Rcw^T
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) o[3 * r + c] = R[r][c];
    o[9 + r] = -__fadd_rn(__fadd_rn(__fmul_rn(R[r][0], T[3]), __fmul_rn(R[r][1], T[7])), __fmul_rn(R[r][2], T[11]));
  }
  double m[3][3], q[4] = {0, 0, 0, 0};                                                   // x y z w
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) m[r][c] = (double)R[r][c];
  double t = m[0][0] + m[1][1] + m[2][2];
  if (t > 0) {
    t = sqrt(t + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m[2][1] - m[1][2]) * t; q[1] = (m[0][2] - m[2][0]) * t; q[2] = (m[1][0] - m[0][1]) * t;
  } else {
    int a = 0;
    if (m[1][1] > m[0][0]) a = 1;
    if (m[2][2] > m[a][a]) a = 2;
    const int b = (a + 1) % 3, c = (b + 1) % 3;
    t = sqrt(m[a][a] - m[b][b] - m[c][c] + 1.0);
    q[a] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (m[c][b] - m[b][c]) * t; q[b] = (m[b][a] + m[a][b]) * t; q[c] = (m[c][a] + m[a][c]) * t;
  }
  for (int k = 0; k < 4; k++) o[12 + k] = (float)q[k];
}
}  // namespace pl
using namespace pl;

extern "C" int pl_pose_records_dev(const float* Tcw_dev, int n, float* records_dev, void* stream) {
  PL_ARG(Tcw_dev && records_dev && n >= 0);
  if (n == 0) return PL_OK;
  k_pose_records<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(Tcw_dev, n, records_dev);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

static int pose_records_host(const float* poses, int n, std::vector<float>& rec) {
  int rc = require_device();
  if (rc) return rc;
  rec.assign((size_t)std::max(n, 1) * 16, 0.f);
  if (n == 0) return PL_OK;
  Staging s;
  float* d_T = s.in(poses, (size_t)n * 16); float* d_r = s.out(rec.data(), (size_t)n * 16);
  if ((rc = s.status())) return rc;
  k_pose_records<<<(n + 127) / 128, 128>>>(d_T, n, d_r);
  PL_LAUNCH_CHECK();
  return s.fetch();
}

static long long emit(const std::string& s, char* out, size_t cap) {
  if (out && cap > s.size()) { memcpy(out, s.data(), s.size()); out[s.size()] = 0; }
  return (long long)s.size();
}

// `f << setprecision(6) << pKF->mTimeStamp << setprecision(7) << " " << t0 << " " << t1 << " " << t2 << " " << q0 .. q3 << endl` with
// f << fixed (System.cc:403,425-428).  Returns the number of bytes of the text (written with a terminating NUL if cap is larger), < 0 on error.
extern "C" long long pl_trajectory_format_tum(const double* timestamps, const float* poses_Tcw, const uint8_t* bad, int n, char* out, size_t cap) {
  if (!(timestamps && poses_Tcw && n >= 0)) { set_error("pl_trajectory_format_tum: bad argument"); return PL_ERR_ARG; }
  std::vector<float> rec;
  const int rc = pose_records_host(poses_Tcw, n, rec);
  if (rc) return rc;
  std::string s;
  char buf[64];
  for (int i = 0; i < n; i++) {
    if (bad && bad[i]) continue;                       // if(pKF->isBad()) continue;  (System.cc:418-419)
    const float* r = &rec[(size_t)i * 16];
    snprintf(buf, sizeof buf, "%.6f", timestamps[i]); s += buf;
    for (int k = 9; k < 16; k++) { snprintf(buf, sizeof buf, " %.7f", (double)r[k]); s += buf; }
    s += "\n";
  }
  return emit(s, out, cap);
}
// `f << setprecision(9) << R(0,0) << " " << R(0,1) << " " << R(0,2) << " " << t(0) << " " << R(1,0) ... << t(2) << endl` (System.cc:455-459)
extern "C" long long pl_trajectory_format_mono_kitti(const float* poses_Tcw, const uint8_t* bad, int n, char* out, size_t cap) {
  if (!(poses_Tcw && n >= 0)) { set_error("pl_trajectory_format_mono_kitti: bad argument"); return PL_ERR_ARG; }
  std::vector<float> rec;
  const int rc = pose_records_host(poses_Tcw, n, rec);
  if (rc) return rc;
  std::string s;
  char buf[64];
  for (int i = 0; i < n; i++) {
    if (bad && bad[i]) continue;
    const float* r = &rec[(size_t)i * 16];
    for (int row = 0; row < 3; row++)
      for (int c = 0; c < 4; c++) {
        snprintf(buf, sizeof buf, "%s%.9f", (row || c) ? " " : "", (double)(c < 3 ? r[3 * row + c] : r[9 + row]));
        s += buf;
      }
    s += "\n";
  }
  return emit(s, out, cap);
}
static int write_text(const char* filename, const std::string& s) {
  FILE* f = fopen(filename, "w");
  if (!f) { set_error("cannot open %s", filename); return PL_ERR_ARG; }
  const bool ok = fwrite(s.data(), 1, s.size(), f) == s.size();
  fclose(f);
  if (!ok) { set_error("short write to %s", filename); return PL_ERR_ARG; }
  return PL_OK;
}
extern "C" int pl_save_keyframe_trajectory_tum(const char* filename, const double* timestamps, const float* poses_Tcw, const uint8_t* bad, int n) {
  PL_ARG(filename);
  const long long need = pl_trajectory_format_tum(timestamps, poses_Tcw, bad, n, nullptr, 0);
  if (need < 0) return (int)need;
  std::string s((size_t)need + 1, '\0');
  pl_trajectory_format_tum(timestamps, poses_Tcw, bad, n, &s[0], s.size());
  s.resize((size_t)need);
  return write_text(filename, s);
}
extern "C" int pl_save_keyframe_trajectory_mono_kitti(const char* filename, const float* poses_Tcw, const uint8_t* bad, int n) {
  PL_ARG(filename);
  const long long need = pl_trajectory_format_mono_kitti(poses_Tcw, bad, n, nullptr, 0);
  if (need < 0) return (int)need;
  std::string s((size_t)need + 1, '\0');
  pl_trajectory_format_mono_kitti(poses_Tcw, bad, n, &s[0], s.size());
  s.resize((size_t)need);
  return write_text(filename, s);
}

