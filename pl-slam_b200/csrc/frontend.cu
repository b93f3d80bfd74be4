// Per-frame front-end pipeline for a batch of frames: the sequence of hot-path calls that Tracking makes for one
// frame (SURVEY.md §3.1), chained on one stream with every intermediate resident in HBM:
//   Frame::ExtractORB  -> pl_orb_extract_batch_dev          (Frame.cc:224 -> ORBextractor::operator(), on the RAW image)
//   undistort + remap  -> pl_undistort_remap_batch_dev      (Frame.cc:220-222; only with pl_frontend_set_camera, k1 != 0)
//   Frame::ExtractLSD  -> pl_line_extract_batch_dev         (Frame.cc:225 -> LINEextractor::operator(), on the UNDISTORTED image)
//   UndistortKeyPoints -> pl_undistort_keypoints_dev        (Frame.cc:233, :915-945; mvKeysUn feed the matcher)
//   point matching     -> pl_orb_search_for_initialization_dev  frame k-1 -> frame k (ORBmatcher.cc:455-572 scheme)
//   line matching      -> pl_lsd_search_double_dev               frame k-1 <-> frame k (LSDmatcher.cpp:440-486)
//   2 x Optimizer::PoseOptimization -> pl_pose_optimization_dev  (Tracking.cc:1372 and :1503)
// This is the measured "step" of bench.py and the e2e entry point (host buffers in, host buffers out).

#include "common.cuh"
#include <vector>
#include <string>
#include <cstdio>
#include <string.h>

namespace pl {
__global__ void k_prev_matched_init(const PLKeyPoint* __restrict__ kps_prev, const int* __restrict__ n_prev, int cap, int B,
                                    float* __restrict__ pm) {
  // vbPrevMatched[i] = F1.mvKeysUn[i].pt with F1 = the predecessor of frame b = slot b of the (B+1)-slot arrays
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_prev[b]) { pm[((long long)b * cap + i) * 2] = kps_prev[(long long)b * cap + i].x; pm[((long long)b * cap + i) * 2 + 1] = kps_prev[(long long)b * cap + i].y; }
}

// ---- steady-state tracking stage: the inputs the reference's tracker takes from its map, synthesised from the PREVIOUS frame.
// TrackWithMotionModel projects the map points / lines seen in the last frame (Tracking.cc:1345-1357), SearchLocalPoints /
// SearchLocalLines the local map (:1799, :1855).  The batch step has no map, so frame b's "map" is frame b-1's features: a map
// point per previous keypoint, placed on its viewing ray (depth 1.5 .. 5.25 m) in the world frame of the pose guess Tcw0[b], with
// the keypoint's descriptor, octave and angle; a map line per previous keyline with its end points as the projection.  The matchers
// then do exactly the reference's work: project with the pose guess, search the th * scale window, keep the best Hamming
// distance.  Slot b of the (B+1)-slot arrays is frame b's predecessor.
__global__ void k_track_points(const PLKeyPoint* __restrict__ ku_prev, const PLKeyPoint* __restrict__ kraw_prev, const int* __restrict__ n_prev,
                               int cap, const float* __restrict__ Tcw0, const float* __restrict__ K, uint8_t* __restrict__ valid,
                               float* __restrict__ pos, int* __restrict__ oct, float* __restrict__ ang, float* __restrict__ proj,
                               float* __restrict__ vcos) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap) return;
  const long long o = (long long)b * cap + i;
  const bool v = i < min(n_prev[b], cap);
  valid[o] = v ? 1 : 0;
  if (!v) return;
  const PLKeyPoint k = ku_prev[o];
  const float* T = Tcw0 + 16 * b;
  const float fx = K[4 * b], fy = K[4 * b + 1], cx = K[4 * b + 2], cy = K[4 * b + 3];
  const float z = __fadd_rn(1.5f, __fmul_rn(0.25f, (float)(i & 15)));
  const float xc = __fmul_rn(__fdiv_rn(__fsub_rn(k.x, cx), fx), z), yc = __fmul_rn(__fdiv_rn(__fsub_rn(k.y, cy), fy), z);
  const float dx = __fsub_rn(xc, T[3]), dy = __fsub_rn(yc, T[7]), dz = __fsub_rn(z, T[11]);
  for (int a = 0; a < 3; a++)      // Xw = R^T (Xc - t)
    pos[o * 3 + a] = __fadd_rn(__fadd_rn(__fmul_rn(T[a], dx), __fmul_rn(T[4 + a], dy)), __fmul_rn(T[8 + a], dz));
  oct[o] = kraw_prev[o].octave; ang[o] = k.angle;
  proj[o * 2] = k.x; proj[o * 2 + 1] = k.y; vcos[o] = 1.0f;
}
struct KL68 { float angle; int class_id, octave; float ptx, pty, response, size, sx, sy, ex, ey, sox, soy, eox, eoy, length; int npix; };
static_assert(sizeof(KL68) == 68, "KeyLine layout");
__global__ void k_track_lines(const KL68* __restrict__ kl_prev, const int* __restrict__ nl_prev, int cap, uint8_t* __restrict__ valid,
                              float* __restrict__ proj, float* __restrict__ len, float* __restrict__ vcos) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap) return;
  const long long o = (long long)b * cap + i;
  const bool v = i < min(nl_prev[b], cap);
  valid[o] = v ? 1 : 0;
  if (!v) return;
  const KL68& k = kl_prev[o];
  proj[o * 4] = k.sx; proj[o * 4 + 1] = k.sy; proj[o * 4 + 2] = k.ex; proj[o * 4 + 3] = k.ey;
  len[o] = k.length; vcos[o] = 1.0f;
}
// after the motion-model search: a map element already matched is not searched again in the local-map pass
// (mnLastFrameSeen == mCurrentFrame.mnId, Tracking.cc:1762-1776), a feature that holds a match is skipped (ORBmatcher.cc:100-102)
__global__ void __launch_bounds__(256) k_track_mark(const int* __restrict__ match1, const int* __restrict__ n_cur, const uint8_t* __restrict__ valid,
                                                    int cap, uint8_t* __restrict__ view, uint8_t* __restrict__ pre) {
  const int b = blockIdx.x;
  const long long o = (long long)b * cap;
  for (int i = threadIdx.x; i < cap; i += 256) view[o + i] = valid[o + i];
  __syncthreads();
  const int n = min(n_cur[b], cap);
  for (int j = threadIdx.x; j < cap; j += 256) {
    const int m = j < n ? match1[o + j] : -1;
    pre[o + j] = m >= 0 ? 1 : 0;
    if (m >= 0 && m < cap) view[o + m] = 0;
  }
}
}  // namespace pl
using namespace pl;

struct PLFrontend {
  PLFrontendConfig cfg;
  PLOrb* orb = nullptr;
  PLLine* line = nullptr;
  cudaStream_t stream = nullptr;
  cudaStream_t sLine = nullptr, sLm = nullptr;      // side streams: LSD/LBD chain and the LM run beside the ORB chain
  cudaEvent_t evStart = nullptr, evLine = nullptr, evLm = nullptr;
  int overlap = 0;
  int serial_batch = 0;          // batches of at least this many frames run the three chains on one stream (see pl_frontend_create)
  int B = 0, capK = 0, capL = 0;
  // device-resident per-batch state
  uint8_t* d_img = nullptr;
  PLKeyPoint* d_kps = nullptr; uint8_t* d_desc = nullptr; int* d_n = nullptr;
  void* d_kl = nullptr; uint8_t* d_ldesc = nullptr; double* d_lf = nullptr; int* d_nl = nullptr;
  float* d_bounds = nullptr; float* d_pm = nullptr; int* d_m12 = nullptr; int* d_nm = nullptr; int* d_scr = nullptr;
  int* d_lm = nullptr; int* d_nlm = nullptr;
  // rotated views so that "previous frame" is a plain pointer offset: copies of frame B-1 placed before frame 0
  PLKeyPoint* d_kps_prev = nullptr; uint8_t* d_desc_prev = nullptr; int* d_n_prev = nullptr;
  uint8_t* d_ldesc_prev = nullptr; int* d_nl_prev = nullptr;
  uint8_t* d_kl_prev = nullptr;          // keylines hold B+1 slots like the descriptors (d_kl = slot 1)
  char order[4] = {'L', 'O', 'M', 0};
  // steady-state tracking stage (pl_frontend_set_tracking): the map seen from frame b is frame b-1's features (see k_track_points)
  int tracking = 0;
  float* d_sf = nullptr;
  float *d_tpos = nullptr, *d_tang = nullptr, *d_tproj = nullptr, *d_tvcos = nullptr;
  int *d_toct = nullptr, *d_tm1 = nullptr, *d_tnm1 = nullptr, *d_tm2 = nullptr, *d_tnm2 = nullptr;
  uint8_t *d_tvalid = nullptr, *d_tview = nullptr, *d_tpre = nullptr;
  float *d_lqproj = nullptr, *d_lqlen = nullptr, *d_lqvcos = nullptr;
  int *d_lm1 = nullptr, *d_lnm1 = nullptr, *d_lm2 = nullptr, *d_lnm2 = nullptr;
  uint8_t *d_lqvalid = nullptr, *d_lqview = nullptr, *d_lpre = nullptr, *d_lscratch = nullptr;
  // LM problems
  float *d_T0 = nullptr, *d_K = nullptr, *d_pobs = nullptr, *d_pw = nullptr, *d_pX = nullptr, *d_Tout = nullptr;
  double *d_lfun = nullptr, *d_lX = nullptr, *d_scratch = nullptr;
  int *d_np = nullptr, *d_nl_lm = nullptr, *d_inl = nullptr, *d_its = nullptr;
  uint8_t *d_pout = nullptr, *d_lout = nullptr;
  // camera (pl_frontend_set_camera): undistortion map, undistorted frames, undistorted keypoints (B+1 slots like d_kps)
  PLUndistort* und = nullptr;
  uint8_t* d_und = nullptr;
  PLKeyPoint* d_kpsu_prev = nullptr;
  // streaming (pl_frontend_submit / pl_frontend_wait): two input buffers, one output snapshot, copy streams
  uint8_t* d_in[2] = {nullptr, nullptr};
  uint8_t* d_stage = nullptr;
  cudaStream_t sUp = nullptr, sDown = nullptr;
  cudaEvent_t evUp[2] = {nullptr, nullptr}, evFree[2] = {nullptr, nullptr}, evSnap = nullptr, evOut = nullptr;
  cudaEvent_t evStep[2] = {nullptr, nullptr};   // host outputs of submit #c are complete when evStep[c & 1] fires
  int slot = 0;
  long long submitted = 0, completed = 0;
  int wrap = 0;       // 1: frame 0 is matched against the LAST frame of the same batch (closed loop); 0: against the last frame of the previous step
};

extern "C" void pl_frontend_destroy(PLFrontend* h) {
  if (!h) return;
  pl_orb_destroy(h->orb); pl_line_destroy(h->line); pl_undistort_destroy(h->und);
  cudaFree(h->d_und); cudaFree(h->d_kpsu_prev);
  cudaFree(h->d_in[0]); cudaFree(h->d_in[1]); cudaFree(h->d_stage);
  if (h->sUp) cudaStreamDestroy(h->sUp);
  if (h->sDown) cudaStreamDestroy(h->sDown);
  for (cudaEvent_t e : {h->evUp[0], h->evUp[1], h->evFree[0], h->evFree[1], h->evSnap, h->evOut, h->evStep[0], h->evStep[1]}) if (e) cudaEventDestroy(e);
  void* ptrs[] = {h->d_img, h->d_kl_prev, h->d_sf, h->d_tpos, h->d_tang, h->d_tproj, h->d_tvcos, h->d_toct, h->d_tm1, h->d_tnm1, h->d_tm2, h->d_tnm2,
                  h->d_tvalid, h->d_tview, h->d_tpre, h->d_lqproj, h->d_lqlen, h->d_lqvcos, h->d_lm1, h->d_lnm1, h->d_lm2, h->d_lnm2,
                  h->d_lqvalid, h->d_lqview, h->d_lpre, h->d_lscratch, h->d_lf, h->d_bounds, h->d_pm, h->d_m12,
                  h->d_nm, h->d_scr, h->d_lm, h->d_nlm, h->d_kps_prev, h->d_desc_prev, h->d_n_prev, h->d_ldesc_prev, h->d_nl_prev,
                  h->d_T0, h->d_K, h->d_pobs, h->d_pw, h->d_pX, h->d_Tout, h->d_lfun, h->d_lX, h->d_scratch, h->d_np, h->d_nl_lm,
                  h->d_inl, h->d_its, h->d_pout, h->d_lout};
  for (void* p : ptrs) cudaFree(p);
  if (h->stream) cudaStreamDestroy(h->stream);
  if (h->sLine) cudaStreamDestroy(h->sLine);
  if (h->sLm) cudaStreamDestroy(h->sLm);
  if (h->evStart) cudaEventDestroy(h->evStart);
  if (h->evLine) cudaEventDestroy(h->evLine);
  if (h->evLm) cudaEventDestroy(h->evLm);
  delete h;
}

extern "C" int pl_frontend_create(const PLFrontendConfig* cfg, PLFrontend** out) {
  PL_ARG(cfg && out && cfg->max_batch >= 1 && cfg->lm_cap_points >= 1 && cfg->lm_cap_lines >= 1);
  int rc = require_device();
  if (rc) return rc;
  PLFrontend* h = new PLFrontend;
  h->cfg = *cfg;
  h->B = cfg->max_batch;
#define FE_TRY(e) do { int _r = (e); if (_r) { pl_frontend_destroy(h); return _r; } } while (0)
#define FE_CUDA(e) do { cudaError_t _e = (e); if (_e != cudaSuccess) { set_error("%s -> %s", #e, cudaGetErrorString(_e)); pl_frontend_destroy(h); return PL_ERR_CUDA; } } while (0)
  PLOrbConfig oc = {cfg->width, cfg->height, cfg->orb_nfeatures, cfg->orb_scale_factor, cfg->orb_nlevels, cfg->orb_ini_th, cfg->orb_min_th, cfg->max_batch, 0};
  FE_TRY(pl_orb_create(&oc, &h->orb));
  PLLineConfig lc = {cfg->width, cfg->height, cfg->line_nfeatures, cfg->line_min_length, cfg->max_batch, 0, 0};
  FE_TRY(pl_line_create(&lc, &h->line));
  h->capK = pl_orb_capacity(h->orb); h->capL = pl_line_capacity(h->line);
  FE_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  FE_CUDA(cudaStreamCreateWithFlags(&h->sLine, cudaStreamNonBlocking));
  FE_CUDA(cudaStreamCreateWithFlags(&h->sLm, cudaStreamNonBlocking));
  FE_CUDA(cudaEventCreateWithFlags(&h->evStart, cudaEventDisableTiming));
  FE_CUDA(cudaEventCreateWithFlags(&h->evLine, cudaEventDisableTiming));
  FE_CUDA(cudaEventCreateWithFlags(&h->evLm, cudaEventDisableTiming));
  // The three chains run on separate streams (PLSLAM_FRONTEND_OVERLAP=0: one stream): the low-occupancy kernels (matchers,
  // quadtree, pose optimisation) fill the tails of the others.  Not from 32 frames per SM on: there k_lsd_grow_ordered is one
  // wave of one-warp CTAs that holds all 32 block slots and the whole register file of every SM, so the other chains are only
  // placed in its tail, where they slow the grow's last frames by more than they gain (DESIGN.md §7: 402 ms with three streams,
  // 392 ms with one, at 4224 frames on an H100).
  { const char* e = getenv("PLSLAM_FRONTEND_OVERLAP"); h->overlap = !(e && e[0] == '0'); }
  {
    int dev = 0, sms = 132;
    FE_CUDA(cudaGetDevice(&dev));
    FE_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    h->serial_batch = 32 * sms;
  }
  if (const char* e = getenv("PLSLAM_FRONTEND_ORDER")) {
    const std::string o(e);
    if (o.size() == 3 && o.find('L') != std::string::npos && o.find('O') != std::string::npos && o.find('M') != std::string::npos) memcpy(h->order, o.data(), 3);
  }
  const size_t B = h->B, cK = h->capK, cL = h->capL, cp = cfg->lm_cap_points, cl = cfg->lm_cap_lines;
  FE_TRY(dev_alloc(&h->d_img, (size_t)cfg->width * cfg->height * B));
  // feature arrays hold B+1 frames: slot 0 = copy of the batch's last frame ("previous" of frame 0), slots 1..B = frames
  FE_TRY(dev_alloc(&h->d_kps_prev, cK * (B + 1))); h->d_kps = h->d_kps_prev + cK;
  FE_TRY(dev_alloc(&h->d_desc_prev, cK * 32 * (B + 1))); h->d_desc = h->d_desc_prev + cK * 32;
  FE_TRY(dev_alloc(&h->d_n_prev, B + 1)); h->d_n = h->d_n_prev + 1;
  FE_CUDA(cudaMemset(h->d_n_prev, 0, sizeof(int) * (B + 1)));      // before the first step frame 0 has no predecessor
  FE_TRY(dev_alloc(&h->d_ldesc_prev, cL * 32 * (B + 1))); h->d_ldesc = h->d_ldesc_prev + cL * 32;
  FE_TRY(dev_alloc(&h->d_nl_prev, B + 1)); h->d_nl = h->d_nl_prev + 1;
  FE_CUDA(cudaMemset(h->d_nl_prev, 0, sizeof(int) * (B + 1)));
  FE_TRY(dev_alloc(&h->d_kl_prev, cL * 68 * (B + 1))); h->d_kl = h->d_kl_prev + cL * 68;
  FE_TRY(dev_alloc(&h->d_lf, cL * 3 * B));
  FE_TRY(dev_alloc(&h->d_bounds, 4)); FE_TRY(dev_alloc(&h->d_pm, cK * 2 * B)); FE_TRY(dev_alloc(&h->d_m12, cK * B));
  FE_TRY(dev_alloc(&h->d_nm, B)); FE_TRY(dev_alloc(&h->d_scr, cK * 2 * B)); FE_TRY(dev_alloc(&h->d_lm, cL * B)); FE_TRY(dev_alloc(&h->d_nlm, B));
  float bounds[4] = {0.f, 0.f, (float)cfg->width, (float)cfg->height};   // Frame::ComputeImageBounds without distortion
  FE_CUDA(cudaMemcpy(h->d_bounds, bounds, sizeof(bounds), cudaMemcpyHostToDevice));
  FE_TRY(dev_alloc(&h->d_T0, 16 * B)); FE_TRY(dev_alloc(&h->d_K, 4 * B)); FE_TRY(dev_alloc(&h->d_pobs, cp * 2 * B));
  FE_TRY(dev_alloc(&h->d_pw, cp * B)); FE_TRY(dev_alloc(&h->d_pX, cp * 3 * B)); FE_TRY(dev_alloc(&h->d_Tout, 16 * B * 2));
  FE_TRY(dev_alloc(&h->d_lfun, cl * 3 * B)); FE_TRY(dev_alloc(&h->d_lX, cl * 6 * B));
  FE_TRY(dev_alloc(&h->d_scratch, pl_pose_optimization_scratch_doubles((int)B, (int)cp, (int)cl)));
  FE_TRY(dev_alloc(&h->d_np, B)); FE_TRY(dev_alloc(&h->d_nl_lm, B)); FE_TRY(dev_alloc(&h->d_inl, B * 2)); FE_TRY(dev_alloc(&h->d_its, B * 2));
  FE_TRY(dev_alloc(&h->d_pout, cp * B * 2)); FE_TRY(dev_alloc(&h->d_lout, cl * B * 2));
  *out = h;
  return PL_OK;
}

extern "C" int pl_frontend_capacities(const PLFrontend* h, int* cap_keypoints, int* cap_lines) {
  PL_ARG(h);
  if (cap_keypoints) *cap_keypoints = h->capK;
  if (cap_lines) *cap_lines = h->capL;
  return PL_OK;
}

// A problem over the configured capacities would lose its surplus correspondences without a word (the kernel clamps): refused.
static int check_pose_problem_sizes(const PLFrontend* h, int B, const int* n_points, const int* n_lines) {
  for (int b = 0; b < B; b++)
    if (n_points[b] < 0 || n_points[b] > h->cfg.lm_cap_points || n_lines[b] < 0 || n_lines[b] > h->cfg.lm_cap_lines) {
      set_error("pose problem %d has %d points and %d lines; the capacities are %d and %d", b, n_points[b], n_lines[b],
                h->cfg.lm_cap_points, h->cfg.lm_cap_lines);
      return PL_ERR_ARG;
    }
  return PL_OK;
}

// LM problems of the batch (device-resident until replaced).  Host pointers; [B][cap] layouts.
extern "C" int pl_frontend_set_pose_problems(PLFrontend* h, int B, const float* Tcw0, const float* K, const int* n_points,
                                             const float* pt_obs, const float* pt_inv_sigma2, const float* pt_Xw,
                                             const int* n_lines, const double* line_func, const double* line_Xw) {
  PL_ARG(h && B >= 1 && B <= h->B && Tcw0 && K && n_points && pt_obs && pt_inv_sigma2 && pt_Xw && n_lines && line_func && line_Xw);
  if (int rc = check_pose_problem_sizes(h, B, n_points, n_lines)) return rc;
  const size_t cp = h->cfg.lm_cap_points, cl = h->cfg.lm_cap_lines, b = B;
  cudaStream_t st = h->stream;
  PL_CUDA(cudaMemcpyAsync(h->d_T0, Tcw0, 64 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_K, K, 16 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_np, n_points, 4 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_nl_lm, n_lines, 4 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_pobs, pt_obs, cp * 8 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_pw, pt_inv_sigma2, cp * 4 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_pX, pt_Xw, cp * 12 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_lfun, line_func, cl * 24 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_lX, line_Xw, cl * 48 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaStreamSynchronize(st));
  return PL_OK;
}
extern "C" long long pl_frontend_set_pose_problems_async(PLFrontend* h, int B, const float* Tcw0, const float* K, const int* n_points,
                                                         const float* pt_obs, const float* pt_inv_sigma2, const float* pt_Xw,
                                                         const int* n_lines, const double* line_func, const double* line_Xw, void* stream_) {
  PL_ARG(h && B >= 1 && B <= h->B && Tcw0 && K && n_points && pt_obs && pt_inv_sigma2 && pt_Xw && n_lines && line_func && line_Xw);
  if (int rc = check_pose_problem_sizes(h, B, n_points, n_lines)) return rc;
  const size_t cp = h->cfg.lm_cap_points, cl = h->cfg.lm_cap_lines, b = B;
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : h->stream;
  PL_CUDA(cudaMemcpyAsync(h->d_T0, Tcw0, 64 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_K, K, 16 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_np, n_points, 4 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_nl_lm, n_lines, 4 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_pobs, pt_obs, cp * 8 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_pw, pt_inv_sigma2, cp * 4 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_pX, pt_Xw, cp * 12 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_lfun, line_func, cl * 24 * b, cudaMemcpyHostToDevice, st));
  PL_CUDA(cudaMemcpyAsync(h->d_lX, line_Xw, cl * 48 * b, cudaMemcpyHostToDevice, st));
  return (long long)((64 + 16 + 4 + 4 + cp * (8 + 4 + 12) + cl * (24 + 48)) * b);
}
// Steady-state tracking stage on / off (default off).  Allocates its arrays on first use.
extern "C" int pl_frontend_set_tracking(PLFrontend* h, int on) {
  PL_ARG(h);
  if (on && !h->d_sf) {
    const size_t B = h->B, cK = h->capK, cL = h->capL;
    std::vector<float> sf(std::max(h->cfg.orb_nlevels, 1), 1.0f);
    for (size_t i = 1; i < sf.size(); i++) sf[i] = sf[i - 1] * h->cfg.orb_scale_factor;     // ORBextractor.cc:419-426
    int rc;
#define TR_TRY(e) do { if ((rc = (e))) return rc; } while (0)
    TR_TRY(dev_alloc(&h->d_sf, sf.size()));
    PL_CUDA(cudaMemcpy(h->d_sf, sf.data(), sf.size() * sizeof(float), cudaMemcpyHostToDevice));
    TR_TRY(dev_alloc(&h->d_tpos, cK * 3 * B)); TR_TRY(dev_alloc(&h->d_tang, cK * B)); TR_TRY(dev_alloc(&h->d_tproj, cK * 2 * B));
    TR_TRY(dev_alloc(&h->d_tvcos, cK * B)); TR_TRY(dev_alloc(&h->d_toct, cK * B)); TR_TRY(dev_alloc(&h->d_tm1, cK * B)); TR_TRY(dev_alloc(&h->d_tnm1, B));
    TR_TRY(dev_alloc(&h->d_tm2, cK * B)); TR_TRY(dev_alloc(&h->d_tnm2, B)); TR_TRY(dev_alloc(&h->d_tvalid, cK * B)); TR_TRY(dev_alloc(&h->d_tview, cK * B));
    TR_TRY(dev_alloc(&h->d_tpre, cK * B));
    TR_TRY(dev_alloc(&h->d_lqproj, cL * 4 * B)); TR_TRY(dev_alloc(&h->d_lqlen, cL * B)); TR_TRY(dev_alloc(&h->d_lqvcos, cL * B));
    TR_TRY(dev_alloc(&h->d_lm1, cL * B)); TR_TRY(dev_alloc(&h->d_lnm1, B)); TR_TRY(dev_alloc(&h->d_lm2, cL * B)); TR_TRY(dev_alloc(&h->d_lnm2, B));
    TR_TRY(dev_alloc(&h->d_lqvalid, cL * B)); TR_TRY(dev_alloc(&h->d_lqview, cL * B)); TR_TRY(dev_alloc(&h->d_lpre, cL * B));
    TR_TRY(dev_alloc(&h->d_lscratch, pl_lsd_search_scratch_bytes((int)cL, (int)B)));
#undef TR_TRY
  }
  h->tracking = on ? 1 : 0;
  return PL_OK;
}
// Results and inputs of the tracking stage of the last step (host arrays, NULL = skip): matches [B][capK] / [B][capL] hold the index
// of the previous frame's feature (-1 none); which: 0 = motion-model search, 1 = local-map search.
extern "C" int pl_frontend_fetch_tracking(PLFrontend* h, int B, int which, int* point_match, int* n_point_matches, int* line_match,
                                          int* n_line_matches, float* map_pos, uint8_t* point_in_view, uint8_t* line_in_view) {
  PL_ARG(h && h->tracking && h->d_sf && B >= 1 && B <= h->B && (which == 0 || which == 1));
  const size_t cK = h->capK, cL = h->capL;
  PL_CUDA(cudaStreamSynchronize(h->stream));
  if (point_match) PL_CUDA(cudaMemcpy(point_match, which ? h->d_tm2 : h->d_tm1, cK * B * sizeof(int), cudaMemcpyDeviceToHost));
  if (n_point_matches) PL_CUDA(cudaMemcpy(n_point_matches, which ? h->d_tnm2 : h->d_tnm1, B * sizeof(int), cudaMemcpyDeviceToHost));
  if (line_match) PL_CUDA(cudaMemcpy(line_match, which ? h->d_lm2 : h->d_lm1, cL * B * sizeof(int), cudaMemcpyDeviceToHost));
  if (n_line_matches) PL_CUDA(cudaMemcpy(n_line_matches, which ? h->d_lnm2 : h->d_lnm1, B * sizeof(int), cudaMemcpyDeviceToHost));
  if (map_pos) PL_CUDA(cudaMemcpy(map_pos, h->d_tpos, cK * 3 * B * sizeof(float), cudaMemcpyDeviceToHost));
  if (point_in_view) PL_CUDA(cudaMemcpy(point_in_view, which ? h->d_tview : h->d_tvalid, cK * B, cudaMemcpyDeviceToHost));
  if (line_in_view) PL_CUDA(cudaMemcpy(line_in_view, which ? h->d_lqview : h->d_lqvalid, cL * B, cudaMemcpyDeviceToHost));
  return PL_OK;
}
extern "C" int pl_frontend_set_wrap(PLFrontend* h, int on) { PL_ARG(h); h->wrap = on ? 1 : 0; return PL_OK; }
extern "C" int pl_frontend_check_overflow(PLFrontend* h) {
  PL_ARG(h);
  int rc = pl_orb_check_overflow(h->orb);
  const int rc2 = pl_line_check_overflow(h->line);
  return rc ? rc : rc2;
}

// The timed device-resident step: frames already in HBM (imgs = device pointer, or NULL = the frames uploaded by the
// last pl_frontend_run()).  Everything asynchronous on `stream` (NULL = the handle's own stream).
extern "C" int pl_frontend_run_dev(PLFrontend* h, const uint8_t* imgs, int stride, size_t frame_stride, int B, void* stream_) {
  PL_ARG(h && B >= 1 && B <= h->B);
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : h->stream;
  if (!imgs) { imgs = h->d_img; stride = h->cfg.width; frame_stride = (size_t)h->cfg.width * h->cfg.height; }
  const size_t cK = h->capK, cL = h->capL;
  int rc;
  const size_t cp = h->cfg.lm_cap_points, cl = h->cfg.lm_cap_lines;
  // Three independent chains, like the reference's per-frame std::threads (Frame.cc:224-227): the line chain (LSD grow is
  // latency bound and leaves issue slots free), the ORB + point-matching chain, and the two pose optimisations.
  const bool overlap = h->overlap && B < h->serial_batch;
  cudaStream_t sL = overlap ? h->sLine : st, sM = overlap ? h->sLm : st;
  if (overlap) {
    PL_CUDA(cudaEventRecord(h->evStart, st));
    PL_CUDA(cudaStreamWaitEvent(sL, h->evStart, 0));
    PL_CUDA(cudaStreamWaitEvent(sM, h->evStart, 0));
  }
  auto line_chain = [&]() -> int {
  // --- line chain (on the undistorted frames when the camera has distortion, Frame.cc:220-225)
  const uint8_t* limgs = imgs; int lstride = stride; size_t lframe = frame_stride;
  if (h->und) {
    const size_t fb = (size_t)h->cfg.width * h->cfg.height;
    if ((rc = pl_undistort_remap_batch_dev(h->und, imgs, stride, frame_stride, B, h->d_und, h->cfg.width, fb, sL))) return rc;
    limgs = h->d_und; lstride = h->cfg.width; lframe = fb;
  }
  if ((rc = pl_line_extract_batch_dev(h->line, limgs, lstride, lframe, B, nullptr, h->d_kl, h->d_ldesc, h->d_lf, h->d_nl, sL))) return rc;
  // slot 0 of every feature array is "the frame before frame 0": the last frame of the PREVIOUS step (sequence replay: the
  // copy follows the matching), or, in wrap mode, the last frame of this batch (the copy precedes the matching)
  auto carry_lines = [&]() -> int {
    PL_CUDA(cudaMemcpyAsync(h->d_ldesc_prev, h->d_ldesc + cL * 32 * (B - 1), cL * 32, cudaMemcpyDeviceToDevice, sL));
    PL_CUDA(cudaMemcpyAsync(h->d_nl_prev, h->d_nl + (B - 1), sizeof(int), cudaMemcpyDeviceToDevice, sL));
    PL_CUDA(cudaMemcpyAsync(h->d_kl_prev, (const uint8_t*)h->d_kl + cL * 68 * (B - 1), cL * 68, cudaMemcpyDeviceToDevice, sL));
    return PL_OK;
  };
  if (h->wrap && (rc = carry_lines())) return rc;
  if ((rc = pl_lsd_search_double_dev(h->d_ldesc_prev, h->d_nl_prev, h->d_ldesc, h->d_nl, (int)cL, (int)cL, B, 50.f, 0.7f, 1, h->d_lm,
                                     h->d_nlm, sL))) return rc;
  if (h->tracking) {   // lines: TrackWithMotionModel (Tracking.cc:1347, th = 15) then SearchLocalLines (:1855, th = 1), LSDmatcher(0.7)
    const dim3 g((unsigned)((cL + 127) / 128), B);
    k_track_lines<<<g, 128, 0, sL>>>((const KL68*)h->d_kl_prev, h->d_nl_prev, (int)cL, h->d_lqvalid, h->d_lqproj, h->d_lqlen, h->d_lqvcos);
    PL_LAUNCH_CHECK();
    if ((rc = pl_lsd_search_by_projection_dev(0, h->d_kl, h->d_lf, h->d_ldesc, h->d_nl, (int)cL, B, h->d_bounds, h->d_nl_prev, (int)cL, h->d_lqvalid,
                                              h->d_lqproj, h->d_ldesc_prev, h->d_lqlen, 15.f, 0.7f, nullptr, h->d_lm1, h->d_lnm1, h->d_lscratch, sL))) return rc;
    k_track_mark<<<B, 256, 0, sL>>>(h->d_lm1, h->d_nl, h->d_lqvalid, (int)cL, h->d_lqview, h->d_lpre);
    PL_LAUNCH_CHECK();
    if ((rc = pl_lsd_search_by_projection_dev(1, h->d_kl, h->d_lf, h->d_ldesc, h->d_nl, (int)cL, B, h->d_bounds, h->d_nl_prev, (int)cL, h->d_lqview,
                                              h->d_lqproj, h->d_ldesc_prev, h->d_lqvcos, 1.f, 0.7f, h->d_lpre, h->d_lm2, h->d_lnm2, h->d_lscratch, sL))) return rc;
  }
  if (!h->wrap && (rc = carry_lines())) return rc;
  return PL_OK;
  };
  auto orb_chain = [&]() -> int {
  // --- ORB chain (slot 0 <- frame B-1 so that frame b's predecessor is slot b, a plain offset)
  if ((rc = pl_orb_extract_batch_dev(h->orb, imgs, stride, frame_stride, B, h->d_kps, h->d_desc, h->d_n, st))) return rc;
  // mvKeysUn: the matcher works on undistorted keypoints (aliases of the raw ones without a distorting camera)
  const PLKeyPoint *ku_prev = h->d_kps_prev, *ku = h->d_kps;
  PLKeyPoint* kudst = nullptr;
  if (h->und) {
    kudst = h->d_kpsu_prev + cK;
    if ((rc = pl_undistort_keypoints_dev(h->und, h->d_kps, h->d_n, (int)cK, B, kudst, st))) return rc;
    ku_prev = h->d_kpsu_prev; ku = kudst;
  }
  auto carry_points = [&]() -> int {
    PL_CUDA(cudaMemcpyAsync(h->d_kps_prev, h->d_kps + cK * (B - 1), cK * sizeof(PLKeyPoint), cudaMemcpyDeviceToDevice, st));
    PL_CUDA(cudaMemcpyAsync(h->d_desc_prev, h->d_desc + cK * 32 * (B - 1), cK * 32, cudaMemcpyDeviceToDevice, st));
    PL_CUDA(cudaMemcpyAsync(h->d_n_prev, h->d_n + (B - 1), sizeof(int), cudaMemcpyDeviceToDevice, st));
    if (kudst) PL_CUDA(cudaMemcpyAsync(h->d_kpsu_prev, kudst + cK * (B - 1), cK * sizeof(PLKeyPoint), cudaMemcpyDeviceToDevice, st));
    return PL_OK;
  };
  if (h->wrap && (rc = carry_points())) return rc;
  k_prev_matched_init<<<dim3((unsigned)((cK + 127) / 128), B), 128, 0, st>>>(ku_prev, h->d_n_prev, (int)cK, B, h->d_pm);
  PL_LAUNCH_CHECK();
  if ((rc = pl_orb_search_for_initialization_dev(ku_prev, h->d_desc_prev, h->d_n_prev, ku, h->d_desc, h->d_n, (int)cK, B,
                                                 h->d_bounds, h->d_pm, h->d_m12, h->d_nm, 100, 0.9f, 1, h->d_scr, st))) return rc;
  if (h->tracking) {   // points: TrackWithMotionModel (Tracking.cc:1345-1357: th = 15, again with 2 th if < 20 matches), SearchLocalPoints (:1799)
    const PLKeyPoint* kraw_prev = h->d_kps_prev;
    const dim3 g((unsigned)((cK + 127) / 128), B);
    k_track_points<<<g, 128, 0, st>>>(ku_prev, kraw_prev, h->d_n_prev, (int)cK, h->d_T0, h->d_K, h->d_tvalid, h->d_tpos, h->d_toct, h->d_tang,
                                      h->d_tproj, h->d_tvcos);
    PL_LAUNCH_CHECK();
    for (int pass = 0; pass < 2; pass++)
      if ((rc = pl_orb_search_by_projection_last_dev(ku, h->d_desc, h->d_n, (int)cK, B, h->d_bounds, h->d_T0, h->d_K, h->d_sf, h->cfg.orb_nlevels,
                                                     h->d_n_prev, (int)cK, h->d_tvalid, h->d_tpos, h->d_desc_prev, h->d_toct, h->d_tang,
                                                     pass ? 30.f : 15.f, 1, nullptr, pass ? h->d_tnm1 : nullptr, 20, h->d_tm1, h->d_tnm1, st))) return rc;
    k_track_mark<<<B, 256, 0, st>>>(h->d_tm1, h->d_n, h->d_tvalid, (int)cK, h->d_tview, h->d_tpre);
    PL_LAUNCH_CHECK();
    if ((rc = pl_orb_search_by_projection_points_dev(ku, h->d_desc, h->d_n, (int)cK, B, h->d_bounds, h->d_sf, h->d_n_prev, (int)cK, h->d_tview,
                                                     h->d_tproj, h->d_toct, h->d_tvcos, h->d_desc_prev, 1.f, 0.8f, h->d_tpre, h->d_tm2, h->d_tnm2, st))) return rc;
  }
  if (!h->wrap && (rc = carry_points())) return rc;
  return PL_OK;
  };
  auto lm_chain = [&]() -> int {
  // --- pose optimisations: TrackWithMotionModel (Tracking.cc:1372) and TrackLocalMapWithLines (:1503)
  for (int call = 0; call < 2; call++)
    if ((rc = pl_pose_optimization_dev(0, B, h->d_T0, h->d_K, h->d_np, (int)cp, h->d_pobs, h->d_pw, h->d_pX, h->d_nl_lm, (int)cl,
                                       h->d_lfun, h->d_lX, h->d_Tout + 16 * (size_t)B * call, h->d_pout + cp * B * call,
                                       h->d_lout + cl * B * call, h->d_inl + (size_t)B * call, h->d_its + (size_t)B * call,
                                       h->d_scratch, sM))) return rc;
  return PL_OK;
  };
  // enqueue order of the chains (it only matters with overlap on: the block scheduler serves the streams in launch order)
  for (const char* o = h->order; *o; o++) {
    rc = *o == 'L' ? line_chain() : *o == 'O' ? orb_chain() : lm_chain();
    if (rc) return rc;
  }
  if (overlap) {
    PL_CUDA(cudaEventRecord(h->evLine, sL));
    PL_CUDA(cudaEventRecord(h->evLm, sM));
    PL_CUDA(cudaStreamWaitEvent(st, h->evLine, 0));
    PL_CUDA(cudaStreamWaitEvent(st, h->evLm, 0));
  }
  return PL_OK;
}

// Camera of the sequence (Tracking.cc:53-120: mK, mDistCoef).  With k1 != 0 the step undistorts every frame for the line
// extractor and the keypoints for the matcher, and the grid bounds become Frame::ComputeImageBounds'; with k1 == 0 (or never
// called) the step is the undistorted-camera path (KITTI-style configs).
extern "C" int pl_frontend_set_camera(PLFrontend* h, const float* K, const float* dist5) {
  PL_ARG(h && K && dist5);
  PL_CUDA(cudaDeviceSynchronize());
  pl_undistort_destroy(h->und); h->und = nullptr;
  float bounds[4];
  int rc = pl_frame_image_bounds(K, dist5, h->cfg.width, h->cfg.height, bounds);
  if (rc) return rc;
  if (dist5[0] != 0.0f) {
    if ((rc = pl_undistort_create(K, dist5, h->cfg.width, h->cfg.height, &h->und))) return rc;
    if (!h->d_und && (rc = dev_alloc(&h->d_und, (size_t)h->cfg.width * h->cfg.height * h->B))) return rc;
    if (!h->d_kpsu_prev && (rc = dev_alloc(&h->d_kpsu_prev, (size_t)h->capK * (h->B + 1)))) return rc;
  }
  PL_CUDA(cudaMemcpy(h->d_bounds, bounds, sizeof(bounds), cudaMemcpyHostToDevice));
  return PL_OK;
}
// mvKeysUn of the last step (equal to the raw keypoints without a distorting camera)
extern "C" int pl_frontend_fetch_keys_un(PLFrontend* h, int B, PLKeyPoint* out) {
  PL_ARG(h && out && B >= 1 && B <= h->B);
  PL_CUDA(cudaDeviceSynchronize());
  const PLKeyPoint* src = h->und ? h->d_kpsu_prev + h->capK : h->d_kps;
  PL_CUDA(cudaMemcpy(out, src, (size_t)h->capK * B * sizeof(PLKeyPoint), cudaMemcpyDeviceToHost));
  return PL_OK;
}

// End-to-end step on HOST buffers: H2D of the frames, the device step, D2H of every per-frame result.
extern "C" int pl_frontend_run(PLFrontend* h, const uint8_t* imgs, int stride, size_t frame_stride, int B, PLKeyPoint* kps,
                               uint8_t* desc, int* n, void* keylines, uint8_t* ldesc, double* linefunc, int* nl,
                               int* pt_matches, int* n_pt_matches, int* line_matches, int* n_line_matches, float* poses,
                               int* inliers) {
  PL_ARG(h && imgs && B >= 1 && B <= h->B && kps && desc && n && keylines && ldesc && linefunc && nl && pt_matches &&
         n_pt_matches && line_matches && n_line_matches && poses && inliers);
  const int W = h->cfg.width, H = h->cfg.height;
  cudaStream_t st = h->stream;
  if (stride == W && frame_stride == (size_t)W * H)
    PL_CUDA(cudaMemcpyAsync(h->d_img, imgs, (size_t)W * H * B, cudaMemcpyHostToDevice, st));
  else
    for (int b = 0; b < B; b++)
      PL_CUDA(cudaMemcpy2DAsync(h->d_img + (size_t)b * W * H, W, imgs + (size_t)b * frame_stride, stride, W, H, cudaMemcpyHostToDevice, st));
  int rc = pl_frontend_run_dev(h, nullptr, 0, 0, B, st);
  if (rc) return rc;
  const size_t cK = h->capK, cL = h->capL, b = B;
  PL_CUDA(cudaMemcpyAsync(kps, h->d_kps, cK * b * sizeof(PLKeyPoint), cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaMemcpyAsync(desc, h->d_desc, cK * b * 32, cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaMemcpyAsync(n, h->d_n, b * 4, cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaMemcpyAsync(keylines, h->d_kl, cL * b * 68, cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaMemcpyAsync(ldesc, h->d_ldesc, cL * b * 32, cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaMemcpyAsync(linefunc, h->d_lf, cL * b * 24, cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaMemcpyAsync(nl, h->d_nl, b * 4, cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaMemcpyAsync(pt_matches, h->d_m12, cK * b * 4, cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaMemcpyAsync(n_pt_matches, h->d_nm, b * 4, cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaMemcpyAsync(line_matches, h->d_lm, cL * b * 4, cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaMemcpyAsync(n_line_matches, h->d_nlm, b * 4, cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaMemcpyAsync(poses, h->d_Tout, 64 * b * 2, cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaMemcpyAsync(inliers, h->d_inl, 4 * b * 2, cudaMemcpyDeviceToHost, st));
  PL_CUDA(cudaStreamSynchronize(st));
  return pl_frontend_check_overflow(h);    // a truncated frame is an error here, not a sticky flag for a later call
}


// ---- streaming form of pl_frontend_run: the H2D copy of step i+1 and the D2H copy of step i-1 run beside the kernels of
// step i.  submit() returns as soon as the work is enqueued; the host output buffers of a step are valid after the wait()
// that follows the NEXT submit (or any wait() with nothing in flight after it).  At most two steps are in flight; the
// caller alternates two sets of (pinned) output buffers.
static size_t fe_out_bytes(const PLFrontend* h, int B, size_t off[14]) {
  const size_t cK = h->capK, cL = h->capL, b = B;
  const size_t sz[13] = {cK * b * sizeof(PLKeyPoint), cK * b * 32, b * 4, cL * b * 68, cL * b * 32, cL * b * 24, b * 4, cK * b * 4, b * 4,
                         cL * b * 4, b * 4, 64 * b * 2, 4 * b * 2};
  size_t o = 0;
  for (int i = 0; i < 13; i++) { off[i] = o; o += (sz[i] + 255) / 256 * 256; }
  off[13] = o;
  return o;
}
extern "C" int pl_frontend_wait(PLFrontend* h, int keep_in_flight) {
  PL_ARG(h && keep_in_flight >= 0 && keep_in_flight <= 1);
  bool finished = false;
  while (h->submitted - h->completed > keep_in_flight) {      // steps complete in submission order
    PL_CUDA(cudaEventSynchronize(h->evStep[h->completed & 1]));
    h->completed++;
    finished = true;
  }
  return finished ? pl_frontend_check_overflow(h) : PL_OK;
}
extern "C" int pl_frontend_submit(PLFrontend* h, const uint8_t* imgs, int stride, size_t frame_stride, int B, PLKeyPoint* kps,
                                  uint8_t* desc, int* n, void* keylines, uint8_t* ldesc, double* linefunc, int* nl,
                                  int* pt_matches, int* n_pt_matches, int* line_matches, int* n_line_matches, float* poses,
                                  int* inliers) {
  PL_ARG(h && imgs && B >= 1 && B <= h->B && kps && desc && n && keylines && ldesc && linefunc && nl && pt_matches &&
         n_pt_matches && line_matches && n_line_matches && poses && inliers);
  const int W = h->cfg.width, H = h->cfg.height;
  size_t off[14];
  if (!h->sUp) {   // first use: allocate the streaming state
    const size_t fb = (size_t)W * H * h->B;
    int rc;
    if ((rc = dev_alloc(&h->d_in[0], fb)) || (rc = dev_alloc(&h->d_in[1], fb)) || (rc = dev_alloc(&h->d_stage, fe_out_bytes(h, h->B, off)))) return rc;
    PL_CUDA(cudaStreamCreateWithFlags(&h->sUp, cudaStreamNonBlocking));
    PL_CUDA(cudaStreamCreateWithFlags(&h->sDown, cudaStreamNonBlocking));
    for (cudaEvent_t* e : {&h->evUp[0], &h->evUp[1], &h->evFree[0], &h->evFree[1], &h->evSnap, &h->evOut, &h->evStep[0], &h->evStep[1]})
      PL_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    for (int k = 0; k < 2; k++) PL_CUDA(cudaEventRecord(h->evFree[k], h->stream));
    PL_CUDA(cudaEventRecord(h->evOut, h->sDown));
  }
  if (h->submitted - h->completed >= 2) { int rc = pl_frontend_wait(h, 1); if (rc) return rc; }   // at most two steps in flight
  fe_out_bytes(h, B, off);
  const int k = h->slot;
  cudaStream_t st = h->stream;
  // upload into buffer k once the step that last read it has finished
  PL_CUDA(cudaStreamWaitEvent(h->sUp, h->evFree[k], 0));
  if (stride == W && frame_stride == (size_t)W * H)
    PL_CUDA(cudaMemcpyAsync(h->d_in[k], imgs, (size_t)W * H * B, cudaMemcpyHostToDevice, h->sUp));
  else
    for (int b = 0; b < B; b++)
      PL_CUDA(cudaMemcpy2DAsync(h->d_in[k] + (size_t)b * W * H, W, imgs + (size_t)b * frame_stride, stride, W, H, cudaMemcpyHostToDevice, h->sUp));
  PL_CUDA(cudaEventRecord(h->evUp[k], h->sUp));
  // compute
  PL_CUDA(cudaStreamWaitEvent(st, h->evUp[k], 0));
  int rc = pl_frontend_run_dev(h, h->d_in[k], W, (size_t)W * H, B, st);
  if (rc) return rc;
  PL_CUDA(cudaEventRecord(h->evFree[k], st));
  // snapshot of the step's outputs (device to device), once the previous snapshot has left for the host
  PL_CUDA(cudaStreamWaitEvent(st, h->evOut, 0));
  const size_t cK = h->capK, cL = h->capL, b = B;
  const void* src[13] = {h->d_kps, h->d_desc, h->d_n, h->d_kl, h->d_ldesc, h->d_lf, h->d_nl, h->d_m12, h->d_nm, h->d_lm, h->d_nlm, h->d_Tout, h->d_inl};
  void* dst[13] = {kps, desc, n, keylines, ldesc, linefunc, nl, pt_matches, n_pt_matches, line_matches, n_line_matches, poses, inliers};
  const size_t sz[13] = {cK * b * sizeof(PLKeyPoint), cK * b * 32, b * 4, cL * b * 68, cL * b * 32, cL * b * 24, b * 4, cK * b * 4, b * 4,
                         cL * b * 4, b * 4, 64 * b * 2, 4 * b * 2};
  for (int i = 0; i < 13; i++) PL_CUDA(cudaMemcpyAsync(h->d_stage + off[i], src[i], sz[i], cudaMemcpyDeviceToDevice, st));
  PL_CUDA(cudaEventRecord(h->evSnap, st));
  // download
  PL_CUDA(cudaStreamWaitEvent(h->sDown, h->evSnap, 0));
  for (int i = 0; i < 13; i++) PL_CUDA(cudaMemcpyAsync(dst[i], h->d_stage + off[i], sz[i], cudaMemcpyDeviceToHost, h->sDown));
  PL_CUDA(cudaEventRecord(h->evOut, h->sDown));
  PL_CUDA(cudaEventRecord(h->evStep[h->submitted & 1], h->sDown));
  h->slot ^= 1;
  h->submitted++;
  return PL_OK;
}

// bytes moved per frame by pl_frontend_run (for bench.py's e2e accounting)
extern "C" int pl_frontend_io_bytes(const PLFrontend* h, long long* h2d_per_frame, long long* d2h_per_frame) {
  PL_ARG(h && h2d_per_frame && d2h_per_frame);
  const long long cK = h->capK, cL = h->capL;
  *h2d_per_frame = (long long)h->cfg.width * h->cfg.height;
  *d2h_per_frame = cK * (28 + 32 + 4) + 4 + cL * (68 + 32 + 24 + 4) + 4 + 8 + 128 + 8;
  return PL_OK;
}

// copy device-resident results of the last run to host (used by tests to check the device path)
extern "C" int pl_frontend_fetch(PLFrontend* h, int B, PLKeyPoint* kps, uint8_t* desc, int* n, void* keylines, uint8_t* ldesc,
                                 int* nl, int* pt_matches, int* n_pt_matches, int* line_matches, int* n_line_matches,
                                 float* poses, int* inliers) {
  PL_ARG(h && B >= 1 && B <= h->B);
  const size_t cK = h->capK, cL = h->capL, b = B;
  PL_CUDA(cudaStreamSynchronize(h->stream));
  PL_CUDA(cudaDeviceSynchronize());
  if (kps) PL_CUDA(cudaMemcpy(kps, h->d_kps, cK * b * sizeof(PLKeyPoint), cudaMemcpyDeviceToHost));
  if (desc) PL_CUDA(cudaMemcpy(desc, h->d_desc, cK * b * 32, cudaMemcpyDeviceToHost));
  if (n) PL_CUDA(cudaMemcpy(n, h->d_n, b * 4, cudaMemcpyDeviceToHost));
  if (keylines) PL_CUDA(cudaMemcpy(keylines, h->d_kl, cL * b * 68, cudaMemcpyDeviceToHost));
  if (ldesc) PL_CUDA(cudaMemcpy(ldesc, h->d_ldesc, cL * b * 32, cudaMemcpyDeviceToHost));
  if (nl) PL_CUDA(cudaMemcpy(nl, h->d_nl, b * 4, cudaMemcpyDeviceToHost));
  if (pt_matches) PL_CUDA(cudaMemcpy(pt_matches, h->d_m12, cK * b * 4, cudaMemcpyDeviceToHost));
  if (n_pt_matches) PL_CUDA(cudaMemcpy(n_pt_matches, h->d_nm, b * 4, cudaMemcpyDeviceToHost));
  if (line_matches) PL_CUDA(cudaMemcpy(line_matches, h->d_lm, cL * b * 4, cudaMemcpyDeviceToHost));
  if (n_line_matches) PL_CUDA(cudaMemcpy(n_line_matches, h->d_nlm, b * 4, cudaMemcpyDeviceToHost));
  if (poses) PL_CUDA(cudaMemcpy(poses, h->d_Tout, 64 * b * 2, cudaMemcpyDeviceToHost));
  if (inliers) PL_CUDA(cudaMemcpy(inliers, h->d_inl, 4 * b * 2, cudaMemcpyDeviceToHost));
  return pl_frontend_check_overflow(h);
}

// hooks used by bench.py: timing of the dominant kernel and a device-to-device copy of the pose records that the
// multi-GPU run all-gathers (SURVEY.md §8e)
extern "C" int pl_frontend_set_timing(PLFrontend* h, int on) { PL_ARG(h); return pl_line_set_timing(h->line, on); }
extern "C" int pl_frontend_grow_ms(PLFrontend* h, float* ms) { PL_ARG(h); return pl_line_grow_ms(h->line, ms); }
extern "C" long long pl_frontend_grow_bytes_per_frame(const PLFrontend* h) { return h ? pl_line_grow_bytes_per_frame(h->line) : 0; }
extern "C" int pl_frontend_copy_poses_dev(PLFrontend* h, int B, float* dst, void* stream) {
  PL_ARG(h && dst && B >= 1 && B <= h->B);
  PL_CUDA(cudaMemcpyAsync(dst, h->d_Tout + 16 * (size_t)B, 64 * (size_t)B, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return PL_OK;
}

// ---- flat binary dump of one front-end step (the arrays pl_frontend_fetch returns), the container trajectory.load_frontend reads:
// magic "PLSB200\x01", int32 B, then per field: int32 name length, name, int32 dtype length, dtype text (numpy descr), int32 ndim,
// int64 shape[ndim], raw little-endian bytes.
extern "C" int pl_frontend_dump(PLFrontend* h, int B, const char* path) {
  PL_ARG(h && path && B >= 1);
  int cK = 0, cL = 0;
  int rc = pl_frontend_capacities(h, &cK, &cL);
  if (rc) return rc;
  std::vector<PLKeyPoint> kps((size_t)B * cK); std::vector<uint8_t> desc((size_t)B * cK * 32), kl((size_t)B * cL * 68), ldesc((size_t)B * cL * 32);
  std::vector<int> n(B), nl(B), m12((size_t)B * cK), nm(B), lm((size_t)B * cL), nlm(B), inl((size_t)2 * B);
  std::vector<double> lf((size_t)B * cL * 3); std::vector<float> poses((size_t)2 * B * 16);
  rc = pl_frontend_fetch(h, B, kps.data(), desc.data(), n.data(), kl.data(), ldesc.data(), nl.data(), m12.data(), nm.data(), lm.data(),
                         nlm.data(), poses.data(), inl.data());
  if (rc) return rc;
  PL_CUDA(cudaMemcpy(lf.data(), h->d_lf, lf.size() * sizeof(double), cudaMemcpyDeviceToHost));
  FILE* f = fopen(path, "wb");
  if (!f) { set_error("cannot open %s", path); return PL_ERR_ARG; }
  bool ok = fwrite("PLSB200\x01", 1, 8, f) == 8;
  const int32_t b32 = B;
  ok = ok && fwrite(&b32, 4, 1, f) == 1;
  auto field = [&](const char* name, const char* dtype, std::vector<long long> shape, const void* data, size_t bytes) {
    const int32_t ln = (int32_t)strlen(name), ld = (int32_t)strlen(dtype), nd = (int32_t)shape.size();
    ok = ok && fwrite(&ln, 4, 1, f) == 1 && fwrite(name, 1, ln, f) == (size_t)ln && fwrite(&ld, 4, 1, f) == 1 && fwrite(dtype, 1, ld, f) == (size_t)ld;
    ok = ok && fwrite(&nd, 4, 1, f) == 1 && fwrite(shape.data(), 8, nd, f) == (size_t)nd && (bytes == 0 || fwrite(data, 1, bytes, f) == bytes);
  };
  const char* kp_dt = "[('x', '<f4'), ('y', '<f4'), ('size', '<f4'), ('angle', '<f4'), ('response', '<f4'), ('octave', '<i4'), ('class_id', '<i4')]";
  const char* kl_dt = "[('angle', '<f4'), ('class_id', '<i4'), ('octave', '<i4'), ('ptx', '<f4'), ('pty', '<f4'), ('response', '<f4'), ('size', '<f4'), "
                      "('startPointX', '<f4'), ('startPointY', '<f4'), ('endPointX', '<f4'), ('endPointY', '<f4'), ('sPointInOctaveX', '<f4'), "
                      "('sPointInOctaveY', '<f4'), ('ePointInOctaveX', '<f4'), ('ePointInOctaveY', '<f4'), ('lineLength', '<f4'), ('numOfPixels', '<i4')]";
  field("kps", kp_dt, {B, cK}, kps.data(), kps.size() * sizeof(PLKeyPoint));
  field("desc", "'|u1'", {B, cK, 32}, desc.data(), desc.size());
  field("n", "'<i4'", {B}, n.data(), n.size() * 4);
  field("keylines", kl_dt, {B, cL}, kl.data(), kl.size());
  field("ldesc", "'|u1'", {B, cL, 32}, ldesc.data(), ldesc.size());
  field("linefunc", "'<f8'", {B, cL, 3}, lf.data(), lf.size() * 8);
  field("nl", "'<i4'", {B}, nl.data(), nl.size() * 4);
  field("pt_matches", "'<i4'", {B, cK}, m12.data(), m12.size() * 4);
  field("n_pt_matches", "'<i4'", {B}, nm.data(), nm.size() * 4);
  field("line_matches", "'<i4'", {B, cL}, lm.data(), lm.size() * 4);
  field("n_line_matches", "'<i4'", {B}, nlm.data(), nlm.size() * 4);
  field("poses", "'<f4'", {2, B, 16}, poses.data(), poses.size() * 4);
  field("inliers", "'<i4'", {2, B}, inl.data(), inl.size() * 4);
  fclose(f);
  if (!ok) { set_error("short write to %s", path); return PL_ERR_ARG; }
  return PL_OK;
}
