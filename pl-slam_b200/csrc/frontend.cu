// Per-frame front-end pipeline for a batch of frames: the sequence of hot-path calls that Tracking makes for one
// frame (SURVEY.md §3.1), chained on one stream with every intermediate resident in HBM:
//   Frame::ExtractORB  -> pl_orb_extract_batch_dev          (Frame.cc:224 -> ORBextractor::operator(), on the RAW image)
//   undistort + remap  -> the line handle (pl_line_set_undistort) (Frame.cc:220-222; only with pl_frontend_set_camera, k1 != 0)
//   Frame::ExtractLSD  -> pl_line_extract_batch_dev         (Frame.cc:225 -> LINEextractor::operator(), on the UNDISTORTED image)
//   UndistortKeyPoints -> pl_undistort_keypoints_dev        (Frame.cc:233, :915-945; mvKeysUn feed the matcher)
//   point matching     -> pl_orb_search_for_initialization_dev  frame k-1 -> frame k (ORBmatcher.cc:455-572 scheme)
//   line matching      -> pl_lsd_search_double_dev               frame k-1 <-> frame k (LSDmatcher.cpp:440-486)
//   2 x Optimizer::PoseOptimization -> pl_pose_optimization_dev  (Tracking.cc:1372 and :1503)
// This is the measured "step" of bench.py and the e2e entry point (host buffers in, host buffers out).

#include "common.cuh"
#include "search.cuh"
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
  Owned<PLOrb, pl_orb_destroy> orb;
  Owned<PLLine, pl_line_destroy> line;
  Stream stream;
  Stream sLine, sLm;      // side streams: LSD/LBD chain and the LM run beside the ORB chain
  Event evStart, evLine, evLm;
  int overlap = 0;
  int serial_batch = 0;          // batches of at least this many frames run the three chains on one stream (see pl_frontend_create)
  int B = 0, capK = 0, capL = 0;
  // device-resident per-batch state
  DevBuf<uint8_t> d_img;
  PLKeyPoint* d_kps = nullptr; uint8_t* d_desc = nullptr; int* d_n = nullptr;
  void* d_kl = nullptr; uint8_t* d_ldesc = nullptr; DevBuf<double> d_lf; int* d_nl = nullptr;
  DevBuf<float> d_bounds, d_pm; DevBuf<int> d_m12, d_nm, d_scr;
  DevBuf<int> d_lm, d_nlm;
  // rotated views so that "previous frame" is a plain pointer offset: copies of frame B-1 placed before frame 0
  DevBuf<PLKeyPoint> d_kps_prev; DevBuf<uint8_t> d_desc_prev; DevBuf<int> d_n_prev;
  DevBuf<uint8_t> d_ldesc_prev; DevBuf<int> d_nl_prev;
  DevBuf<uint8_t> d_kl_prev;             // keylines hold B+1 slots like the descriptors (d_kl = slot 1)
  char order[4] = {'L', 'O', 'M', 0};
  // steady-state tracking stage (pl_frontend_set_tracking): the map seen from frame b is frame b-1's features (see k_track_points)
  int tracking = 0;
  struct Tracking {
    DevBuf<float> d_sf, d_tpos, d_tang, d_tproj, d_tvcos;
    DevBuf<int> d_toct, d_tm1, d_tnm1, d_tm2, d_tnm2;
    DevBuf<uint8_t> d_tvalid, d_tview, d_tpre;
    DevBuf<float> d_lqproj, d_lqlen, d_lqvcos;
    DevBuf<int> d_lm1, d_lnm1, d_lm2, d_lnm2;
    DevBuf<uint8_t> d_lqvalid, d_lqview, d_lpre, d_lscratch;
  };
  std::unique_ptr<Tracking> tr;          // made on the first pl_frontend_set_tracking(h, 1)
  // LM problems
  DevBuf<float> d_T0, d_K, d_pobs, d_pw, d_pX, d_Tout;
  DevBuf<double> d_lfun, d_lX, d_scratch;
  DevBuf<int> d_np, d_nl_lm, d_inl, d_its;
  DevBuf<uint8_t> d_pout, d_lout;
  // camera (pl_frontend_set_camera): undistortion map (bound to the line handle), undistorted keypoints (B+1 slots like d_kps)
  Owned<PLUndistort, pl_undistort_destroy> und;
  DevBuf<PLKeyPoint> d_kpsu_prev;
  // streaming (pl_frontend_submit / pl_frontend_wait): two input buffers, one output snapshot, copy streams; made on first use
  struct Streaming {
    DevBuf<uint8_t> d_in[2], d_stage;
    Stream sUp, sDown;
    Event evUp[2], evFree[2], evSnap, evOut;
    Event evStep[2];   // host outputs of submit #c are complete when evStep[c & 1] fires
  };
  std::unique_ptr<Streaming> io;
  int slot = 0;
  long long submitted = 0, completed = 0;
  int wrap = 0;       // 1: frame 0 is matched against the LAST frame of the same batch (closed loop); 0: against the last frame of the previous step
  DevBuf<float> d_orb_tab;
  int last_B = 0;                       // frames of the last step (0: none yet) and where its mvKeysUn are
  const PLKeyPoint* last_ku = nullptr;   // mvScaleFactors, mvInvLevelSigma2 for pl_frontend_track_local_map_dev (made on first use)
};

extern "C" void pl_frontend_destroy(PLFrontend* h) {
  if (!h) return;
  delete h;
}

extern "C" int pl_frontend_create(const PLFrontendConfig* cfg, PLFrontend** out) {
  PL_ARG(cfg && out && cfg->max_batch >= 1 && cfg->lm_cap_points >= 1 && cfg->lm_cap_lines >= 1);
  int rc = require_device();
  if (rc) return rc;
  std::unique_ptr<PLFrontend> h(new PLFrontend);
  h->cfg = *cfg;
  h->B = cfg->max_batch;
  PLOrbConfig oc = {cfg->width, cfg->height, cfg->orb_nfeatures, cfg->orb_scale_factor, cfg->orb_nlevels, cfg->orb_ini_th, cfg->orb_min_th, cfg->max_batch, 0};
  PLOrb* orb = nullptr;
  PL_TRY(pl_orb_create(&oc, &orb));
  h->orb.reset(orb);
  PLLineConfig lc = {cfg->width, cfg->height, cfg->line_nfeatures, cfg->line_min_length, cfg->max_batch, 0, 0};
  PLLine* line = nullptr;
  PL_TRY(pl_line_create(&lc, &line));
  h->line.reset(line);
  h->capK = pl_orb_capacity(orb); h->capL = pl_line_capacity(line);
  // every step matches consecutive frames at these capacities: refuse the ones the matchers cannot take here, not in each run
  if (h->capK > kMatchMaxKeys) {
    set_error("orb_nfeatures %d at %d levels gives a keypoint capacity of %d, over the matchers' %d; at most %d features fit at "
              "%d levels", cfg->orb_nfeatures, cfg->orb_nlevels, h->capK, kMatchMaxKeys, kMatchMaxKeys - (h->capK - cfg->orb_nfeatures),
              cfg->orb_nlevels);
    return PL_ERR_ARG;
  }
  PL_TRY(search_double_fits(h->capL, h->capL));
  for (Stream* s : {&h->stream, &h->sLine, &h->sLm}) PL_TRY(s->create(cudaStreamNonBlocking));
  for (Event* e : {&h->evStart, &h->evLine, &h->evLm}) PL_TRY(e->create(cudaEventDisableTiming));
  // The three chains run on separate streams (PLSLAM_FRONTEND_OVERLAP=0: one stream): the low-occupancy kernels (matchers,
  // quadtree, pose optimisation) fill the tails of the others.  Not from 32 frames per SM on: there k_lsd_grow_ordered is one
  // wave of one-warp CTAs that holds all 32 block slots and the whole register file of every SM, so the other chains are only
  // placed in its tail, where they slow the grow's last frames by more than they gain (DESIGN.md §7: 402 ms with three streams,
  // 392 ms with one, at 4224 frames on an H100).
  { const char* e = getenv("PLSLAM_FRONTEND_OVERLAP"); h->overlap = !(e && e[0] == '0'); }
  {
    int dev = 0, sms = 132;
    PL_CUDA(cudaGetDevice(&dev));
    PL_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    h->serial_batch = pl::kSerialFramesPerSM * sms;
  }
  if (const char* e = getenv("PLSLAM_FRONTEND_ORDER")) {
    const std::string o(e);
    if (o.size() == 3 && o.find('L') != std::string::npos && o.find('O') != std::string::npos && o.find('M') != std::string::npos) memcpy(h->order, o.data(), 3);
  }
  const size_t B = h->B, cK = h->capK, cL = h->capL, cp = cfg->lm_cap_points, cl = cfg->lm_cap_lines;
  PL_TRY(h->d_img.alloc((size_t)cfg->width * cfg->height * B));
  // feature arrays hold B+1 frames: slot 0 = copy of the batch's last frame ("previous" of frame 0), slots 1..B = frames
  PL_TRY(h->d_kps_prev.alloc(cK * (B + 1))); h->d_kps = h->d_kps_prev + cK;
  PL_TRY(h->d_desc_prev.alloc(cK * 32 * (B + 1))); h->d_desc = h->d_desc_prev + cK * 32;
  PL_TRY(h->d_n_prev.alloc(B + 1)); h->d_n = h->d_n_prev + 1;
  PL_CUDA(cudaMemset(h->d_n_prev, 0, sizeof(int) * (B + 1)));      // before the first step frame 0 has no predecessor
  PL_TRY(h->d_ldesc_prev.alloc(cL * 32 * (B + 1))); h->d_ldesc = h->d_ldesc_prev + cL * 32;
  PL_TRY(h->d_nl_prev.alloc(B + 1)); h->d_nl = h->d_nl_prev + 1;
  PL_CUDA(cudaMemset(h->d_nl_prev, 0, sizeof(int) * (B + 1)));
  PL_TRY(h->d_kl_prev.alloc(cL * 68 * (B + 1))); h->d_kl = h->d_kl_prev + cL * 68;
  PL_TRY(h->d_lf.alloc(cL * 3 * B));
  PL_TRY(h->d_bounds.alloc(4)); PL_TRY(h->d_pm.alloc(cK * 2 * B)); PL_TRY(h->d_m12.alloc(cK * B));
  PL_TRY(h->d_nm.alloc(B)); PL_TRY(h->d_scr.alloc(cK * 2 * B)); PL_TRY(h->d_lm.alloc(cL * B)); PL_TRY(h->d_nlm.alloc(B));
  float bounds[4] = {0.f, 0.f, (float)cfg->width, (float)cfg->height};   // Frame::ComputeImageBounds without distortion
  PL_CUDA(cudaMemcpy(h->d_bounds, bounds, sizeof(bounds), cudaMemcpyHostToDevice));
  PL_TRY(h->d_T0.alloc(16 * B)); PL_TRY(h->d_K.alloc(4 * B)); PL_TRY(h->d_pobs.alloc(cp * 2 * B));
  PL_TRY(h->d_pw.alloc(cp * B)); PL_TRY(h->d_pX.alloc(cp * 3 * B)); PL_TRY(h->d_Tout.alloc(16 * B * 2));
  PL_TRY(h->d_lfun.alloc(cl * 3 * B)); PL_TRY(h->d_lX.alloc(cl * 6 * B));
  PL_TRY(h->d_scratch.alloc(pl_pose_optimization_scratch_doubles((int)B, (int)cp, (int)cl)));
  PL_TRY(h->d_np.alloc(B)); PL_TRY(h->d_nl_lm.alloc(B)); PL_TRY(h->d_inl.alloc(B * 2)); PL_TRY(h->d_its.alloc(B * 2));
  PL_TRY(h->d_pout.alloc(cp * B * 2)); PL_TRY(h->d_lout.alloc(cl * B * 2));
  *out = h.release();
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
  if (on && !h->tr) {
    const size_t B = h->B, cK = h->capK, cL = h->capL;
    std::vector<float> sf(std::max(h->cfg.orb_nlevels, 1), 1.0f);
    for (size_t i = 1; i < sf.size(); i++) sf[i] = sf[i - 1] * h->cfg.orb_scale_factor;     // ORBextractor.cc:419-426
    auto t = std::make_unique<PLFrontend::Tracking>();
    PL_TRY(t->d_sf.alloc(sf.size()));
    PL_CUDA(cudaMemcpy(t->d_sf, sf.data(), sf.size() * sizeof(float), cudaMemcpyHostToDevice));
    PL_TRY(t->d_tpos.alloc(cK * 3 * B)); PL_TRY(t->d_tang.alloc(cK * B)); PL_TRY(t->d_tproj.alloc(cK * 2 * B));
    PL_TRY(t->d_tvcos.alloc(cK * B)); PL_TRY(t->d_toct.alloc(cK * B)); PL_TRY(t->d_tm1.alloc(cK * B)); PL_TRY(t->d_tnm1.alloc(B));
    PL_TRY(t->d_tm2.alloc(cK * B)); PL_TRY(t->d_tnm2.alloc(B)); PL_TRY(t->d_tvalid.alloc(cK * B)); PL_TRY(t->d_tview.alloc(cK * B));
    PL_TRY(t->d_tpre.alloc(cK * B));
    PL_TRY(t->d_lqproj.alloc(cL * 4 * B)); PL_TRY(t->d_lqlen.alloc(cL * B)); PL_TRY(t->d_lqvcos.alloc(cL * B));
    PL_TRY(t->d_lm1.alloc(cL * B)); PL_TRY(t->d_lnm1.alloc(B)); PL_TRY(t->d_lm2.alloc(cL * B)); PL_TRY(t->d_lnm2.alloc(B));
    PL_TRY(t->d_lqvalid.alloc(cL * B)); PL_TRY(t->d_lqview.alloc(cL * B)); PL_TRY(t->d_lpre.alloc(cL * B));
    PL_TRY(t->d_lscratch.alloc(pl_lsd_search_scratch_bytes((int)cL, (int)B)));
    h->tr = std::move(t);
  }
  h->tracking = on ? 1 : 0;
  return PL_OK;
}
// Results and inputs of the tracking stage of the last step (host arrays, NULL = skip): matches [B][capK] / [B][capL] hold the index
// of the previous frame's feature (-1 none); which: 0 = motion-model search, 1 = local-map search.
extern "C" int pl_frontend_fetch_tracking(PLFrontend* h, int B, int which, int* point_match, int* n_point_matches, int* line_match,
                                          int* n_line_matches, float* map_pos, uint8_t* point_in_view, uint8_t* line_in_view) {
  PL_ARG(h && h->tracking && B >= 1 && B <= h->B && (which == 0 || which == 1));
  const PLFrontend::Tracking& t = *h->tr;
  const size_t cK = h->capK, cL = h->capL;
  PL_CUDA(cudaStreamSynchronize(h->stream));
  if (point_match) PL_CUDA(cudaMemcpy(point_match, which ? t.d_tm2 : t.d_tm1, cK * B * sizeof(int), cudaMemcpyDeviceToHost));
  if (n_point_matches) PL_CUDA(cudaMemcpy(n_point_matches, which ? t.d_tnm2 : t.d_tnm1, B * sizeof(int), cudaMemcpyDeviceToHost));
  if (line_match) PL_CUDA(cudaMemcpy(line_match, which ? t.d_lm2 : t.d_lm1, cL * B * sizeof(int), cudaMemcpyDeviceToHost));
  if (n_line_matches) PL_CUDA(cudaMemcpy(n_line_matches, which ? t.d_lnm2 : t.d_lnm1, B * sizeof(int), cudaMemcpyDeviceToHost));
  if (map_pos) PL_CUDA(cudaMemcpy(map_pos, t.d_tpos, cK * 3 * B * sizeof(float), cudaMemcpyDeviceToHost));
  if (point_in_view) PL_CUDA(cudaMemcpy(point_in_view, which ? t.d_tview : t.d_tvalid, cK * B, cudaMemcpyDeviceToHost));
  if (line_in_view) PL_CUDA(cudaMemcpy(line_in_view, which ? t.d_lqview : t.d_lqvalid, cL * B, cudaMemcpyDeviceToHost));
  return PL_OK;
}
extern "C" int pl_frontend_set_wrap(PLFrontend* h, int on) { PL_ARG(h); h->wrap = on ? 1 : 0; return PL_OK; }
extern "C" int pl_frontend_check_overflow(PLFrontend* h) {
  PL_ARG(h);
  int rc = pl_orb_check_overflow(h->orb.get());
  const int rc2 = pl_line_check_overflow(h->line.get());
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
  // --- line chain (on the undistorted frames when the camera has distortion, Frame.cc:220-225: the line handle undistorts the
  // raw frames with the camera's map, pl_frontend_set_camera)
  if ((rc = pl_line_extract_batch_dev(h->line.get(), imgs, stride, frame_stride, B, nullptr, h->d_kl, h->d_ldesc, h->d_lf, h->d_nl, sL))) return rc;
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
    const PLFrontend::Tracking& t = *h->tr;
    const dim3 g((unsigned)((cL + 127) / 128), B);
    k_track_lines<<<g, 128, 0, sL>>>((const KL68*)h->d_kl_prev.get(), h->d_nl_prev, (int)cL, t.d_lqvalid, t.d_lqproj, t.d_lqlen, t.d_lqvcos);
    PL_LAUNCH_CHECK();
    if ((rc = pl_lsd_search_by_projection_dev(0, h->d_kl, h->d_lf, h->d_ldesc, h->d_nl, (int)cL, B, h->d_bounds, h->d_nl_prev, (int)cL, t.d_lqvalid,
                                              t.d_lqproj, h->d_ldesc_prev, t.d_lqlen, 15.f, 0.7f, nullptr, t.d_lm1, t.d_lnm1, t.d_lscratch, sL))) return rc;
    k_track_mark<<<B, 256, 0, sL>>>(t.d_lm1, h->d_nl, t.d_lqvalid, (int)cL, t.d_lqview, t.d_lpre);
    PL_LAUNCH_CHECK();
    if ((rc = pl_lsd_search_by_projection_dev(1, h->d_kl, h->d_lf, h->d_ldesc, h->d_nl, (int)cL, B, h->d_bounds, h->d_nl_prev, (int)cL, t.d_lqview,
                                              t.d_lqproj, h->d_ldesc_prev, t.d_lqvcos, 1.f, 0.7f, t.d_lpre, t.d_lm2, t.d_lnm2, t.d_lscratch, sL))) return rc;
  }
  if (!h->wrap && (rc = carry_lines())) return rc;
  return PL_OK;
  };
  auto orb_chain = [&]() -> int {
  // --- ORB chain (slot 0 <- frame B-1 so that frame b's predecessor is slot b, a plain offset)
  if ((rc = pl_orb_extract_batch_dev(h->orb.get(), imgs, stride, frame_stride, B, h->d_kps, h->d_desc, h->d_n, st))) return rc;
  // mvKeysUn: the matcher works on undistorted keypoints (aliases of the raw ones without a distorting camera)
  const PLKeyPoint *ku_prev = h->d_kps_prev, *ku = h->d_kps;
  PLKeyPoint* kudst = nullptr;
  if (h->und) {
    kudst = h->d_kpsu_prev + cK;
    if ((rc = pl_undistort_keypoints_dev(h->und.get(), h->d_kps, h->d_n, (int)cK, B, kudst, st))) return rc;
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
    const PLFrontend::Tracking& t = *h->tr;
    const PLKeyPoint* kraw_prev = h->d_kps_prev;
    const dim3 g((unsigned)((cK + 127) / 128), B);
    k_track_points<<<g, 128, 0, st>>>(ku_prev, kraw_prev, h->d_n_prev, (int)cK, h->d_T0, h->d_K, t.d_tvalid, t.d_tpos, t.d_toct, t.d_tang,
                                      t.d_tproj, t.d_tvcos);
    PL_LAUNCH_CHECK();
    for (int pass = 0; pass < 2; pass++)
      if ((rc = pl_orb_search_by_projection_last_dev(ku, h->d_desc, h->d_n, (int)cK, B, h->d_bounds, h->d_T0, h->d_K, t.d_sf, h->cfg.orb_nlevels,
                                                     h->d_n_prev, (int)cK, t.d_tvalid, t.d_tpos, h->d_desc_prev, t.d_toct, t.d_tang,
                                                     pass ? 30.f : 15.f, 1, nullptr, pass ? t.d_tnm1.get() : nullptr, 20, t.d_tm1, t.d_tnm1, st))) return rc;
    k_track_mark<<<B, 256, 0, st>>>(t.d_tm1, h->d_n, t.d_tvalid, (int)cK, t.d_tview, t.d_tpre);
    PL_LAUNCH_CHECK();
    if ((rc = pl_orb_search_by_projection_points_dev(ku, h->d_desc, h->d_n, (int)cK, B, h->d_bounds, t.d_sf, h->d_n_prev, (int)cK, t.d_tview,
                                                     t.d_tproj, t.d_toct, t.d_tvcos, h->d_desc_prev, 1.f, 0.8f, t.d_tpre, t.d_tm2, t.d_tnm2, st))) return rc;
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
  h->last_B = B; h->last_ku = h->und ? h->d_kpsu_prev + cK : h->d_kps;
  return PL_OK;
}

// Camera of the sequence (Tracking.cc:53-120: mK, mDistCoef).  With k1 != 0 the step undistorts every frame for the line
// extractor and the keypoints for the matcher, and the grid bounds become Frame::ComputeImageBounds'; with k1 == 0 (or never
// called) the step is the undistorted-camera path (KITTI-style configs).
extern "C" int pl_frontend_set_camera(PLFrontend* h, const float* K, const float* dist5) {
  PL_ARG(h && K && dist5);
  PL_CUDA(cudaDeviceSynchronize());
  pl_line_set_undistort(h->line.get(), nullptr);
  h->und.reset();
  float bounds[4];
  int rc = pl_frame_image_bounds(K, dist5, h->cfg.width, h->cfg.height, bounds);
  if (rc) return rc;
  if (dist5[0] != 0.0f) {
    if (!h->d_kpsu_prev && (rc = h->d_kpsu_prev.alloc((size_t)h->capK * (h->B + 1)))) return rc;
    PLUndistort* und = nullptr;
    if ((rc = pl_undistort_create(K, dist5, h->cfg.width, h->cfg.height, &und))) return rc;
    h->und.reset(und);
    if ((rc = pl_line_set_undistort(h->line.get(), und))) return rc;
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
    PL_CUDA(cudaEventSynchronize(h->io->evStep[h->completed & 1]));
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
  if (!h->io) {   // first use: allocate the streaming state
    const size_t fb = (size_t)W * H * h->B;
    auto io = std::make_unique<PLFrontend::Streaming>();
    PL_TRY(io->d_in[0].alloc(fb)); PL_TRY(io->d_in[1].alloc(fb)); PL_TRY(io->d_stage.alloc(fe_out_bytes(h, h->B, off)));
    PL_TRY(io->sUp.create(cudaStreamNonBlocking)); PL_TRY(io->sDown.create(cudaStreamNonBlocking));
    for (Event* e : {&io->evUp[0], &io->evUp[1], &io->evFree[0], &io->evFree[1], &io->evSnap, &io->evOut, &io->evStep[0], &io->evStep[1]})
      PL_TRY(e->create(cudaEventDisableTiming));
    for (int k = 0; k < 2; k++) PL_CUDA(cudaEventRecord(io->evFree[k], h->stream));
    PL_CUDA(cudaEventRecord(io->evOut, io->sDown));
    h->io = std::move(io);
  }
  PLFrontend::Streaming& io = *h->io;
  if (h->submitted - h->completed >= 2) { int rc = pl_frontend_wait(h, 1); if (rc) return rc; }   // at most two steps in flight
  fe_out_bytes(h, B, off);
  const int k = h->slot;
  cudaStream_t st = h->stream;
  // upload into buffer k once the step that last read it has finished
  PL_CUDA(cudaStreamWaitEvent(io.sUp, io.evFree[k], 0));
  if (stride == W && frame_stride == (size_t)W * H)
    PL_CUDA(cudaMemcpyAsync(io.d_in[k], imgs, (size_t)W * H * B, cudaMemcpyHostToDevice, io.sUp));
  else
    for (int b = 0; b < B; b++)
      PL_CUDA(cudaMemcpy2DAsync(io.d_in[k] + (size_t)b * W * H, W, imgs + (size_t)b * frame_stride, stride, W, H, cudaMemcpyHostToDevice, io.sUp));
  PL_CUDA(cudaEventRecord(io.evUp[k], io.sUp));
  // compute
  PL_CUDA(cudaStreamWaitEvent(st, io.evUp[k], 0));
  int rc = pl_frontend_run_dev(h, io.d_in[k], W, (size_t)W * H, B, st);
  if (rc) return rc;
  PL_CUDA(cudaEventRecord(io.evFree[k], st));
  // snapshot of the step's outputs (device to device), once the previous snapshot has left for the host
  PL_CUDA(cudaStreamWaitEvent(st, io.evOut, 0));
  const size_t cK = h->capK, cL = h->capL, b = B;
  const void* src[13] = {h->d_kps, h->d_desc, h->d_n, h->d_kl, h->d_ldesc, h->d_lf, h->d_nl, h->d_m12, h->d_nm, h->d_lm, h->d_nlm, h->d_Tout, h->d_inl};
  void* dst[13] = {kps, desc, n, keylines, ldesc, linefunc, nl, pt_matches, n_pt_matches, line_matches, n_line_matches, poses, inliers};
  const size_t sz[13] = {cK * b * sizeof(PLKeyPoint), cK * b * 32, b * 4, cL * b * 68, cL * b * 32, cL * b * 24, b * 4, cK * b * 4, b * 4,
                         cL * b * 4, b * 4, 64 * b * 2, 4 * b * 2};
  for (int i = 0; i < 13; i++) PL_CUDA(cudaMemcpyAsync(io.d_stage + off[i], src[i], sz[i], cudaMemcpyDeviceToDevice, st));
  PL_CUDA(cudaEventRecord(io.evSnap, st));
  // download
  PL_CUDA(cudaStreamWaitEvent(io.sDown, io.evSnap, 0));
  for (int i = 0; i < 13; i++) PL_CUDA(cudaMemcpyAsync(dst[i], io.d_stage + off[i], sz[i], cudaMemcpyDeviceToHost, io.sDown));
  PL_CUDA(cudaEventRecord(io.evOut, io.sDown));
  PL_CUDA(cudaEventRecord(io.evStep[h->submitted & 1], io.sDown));
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
extern "C" int pl_frontend_set_timing(PLFrontend* h, int on) { PL_ARG(h); return pl_line_set_timing(h->line.get(), on); }
extern "C" int pl_frontend_grow_ms(PLFrontend* h, float* ms) { PL_ARG(h); return pl_line_grow_ms(h->line.get(), ms); }
extern "C" long long pl_frontend_grow_bytes_per_frame(const PLFrontend* h) { return h ? pl_line_grow_bytes_per_frame(h->line.get()) : 0; }
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

// Tracking::TrackLocalMapWithLines on the frames of the last step (track.cu): mvKeysUn, descriptors, keylines, line functions and line
// descriptors stay where the step left them; mvScaleFactors / mvInvLevelSigma2 / mfLogScaleFactor are the handle's ORB tables.
extern "C" int pl_frontend_track_local_map_dev(PLFrontend* h, PLMap* map, int B, const float* Tcw0, const float* K, const int* point_map_in,
                                               const int* line_map_in, const PLTrackLocal* local, const PLTrackOut* out, void* scratch,
                                               void* stream) {
  // only the frames the last step produced: later slots hold an older step's features, or none
  PL_ARG(h && B >= 1 && B <= h->last_B);
  const int nlev = h->cfg.orb_nlevels;
  if (!h->d_orb_tab) {
    std::vector<float> tab(2 * (size_t)nlev);
    int rc = pl_orb_tables(h->orb.get(), tab.data(), nullptr, nullptr, tab.data() + nlev, nullptr, nullptr, nullptr);
    if (rc) return rc;
    if ((rc = h->d_orb_tab.alloc(tab.size()))) return rc;
    PL_CUDA(cudaMemcpy(h->d_orb_tab, tab.data(), tab.size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  PLTrackFrames F;
  F.B = B;
  F.keys_un = h->last_ku; F.desc = h->d_desc; F.n = h->d_n; F.cap_points = h->capK;
  F.keylines = h->d_kl; F.line_func = h->d_lf; F.line_desc = h->d_ldesc; F.nl = h->d_nl; F.cap_lines = h->capL;
  F.bounds = h->d_bounds; F.scale_factors = h->d_orb_tab; F.inv_level_sigma2 = h->d_orb_tab + nlev; F.nlevels = nlev;
  F.log_scale_factor = logf(h->cfg.orb_scale_factor);   // Frame: mfLogScaleFactor = log(mfScaleFactor) on a float
  F.Tcw0 = Tcw0; F.K = K; F.point_map_in = point_map_in; F.line_map_in = line_map_in;
  return pl_track_local_map_dev(map, &F, local, out, scratch, stream ? stream : (void*)h->stream);
}
