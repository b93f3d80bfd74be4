/* plslam_b200 — C ABI of the H100-native PL-SLAM front-end / LM hot path.
 *
 * Every entry point replaces one C++ interface of the reference (HarborC/PL-SLAM); the
 * reference has no FFI of its own (SURVEY.md §8b), so these are what a thin C++ class with the
 * reference's signature binds (see pl-slam_b200/host/ and INTEGRATION.md).
 *
 * Conventions: plain pointers and sizes; `_dev` variants take DEVICE pointers (inputs resident
 * in HBM) plus a cudaStream_t passed as void* (NULL = the handle's own stream) and are
 * asynchronous; the plain variants take HOST pointers, copy in/out and synchronise.
 * Return value: 0 = ok, <0 = error (pl_last_error() gives the text).  There is NO CPU fallback:
 * without a usable sm_90 (H100) device every compute entry point fails with PL_ERR_CUDA.
 */
#ifndef PLSLAM_B200_H
#define PLSLAM_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define PL_OK 0
#define PL_ERR_ARG (-1)
#define PL_ERR_CUDA (-2)
#define PL_ERR_CAPACITY (-3)

const char* pl_last_error(void);
int pl_version(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches claim) */
unsigned long long pl_launch_count(void);

/* ------------------------------------------------------------------ ORB extraction
 * replaces ORB_SLAM2::ORBextractor (reference include/ORBextractor.h:45-111,
 * src/ORBextractor.cc:410-470 ctor, :1043-1105 operator()).                         */
typedef struct PLKeyPoint { /* byte-compatible with cv::KeyPoint (28 B) */
  float x, y, size, angle, response;
  int32_t octave, class_id;
} PLKeyPoint;

typedef struct PLOrbConfig {
  int width, height;   /* frame size (fixed per handle)                               */
  int nfeatures;       /* ORBextractor.nFeatures                                      */
  float scale_factor;  /* ORBextractor.scaleFactor                                    */
  int nlevels;         /* ORBextractor.nLevels (<= 12)                                */
  int ini_th_fast;     /* ORBextractor.iniThFAST                                      */
  int min_th_fast;     /* ORBextractor.minThFAST                                      */
  int max_batch;       /* frames per call upper bound (device buffers are sized once) */
  int cell_slot_cap;   /* max NMS maxima kept per FAST cell; 0 = default 128          */
} PLOrbConfig;

typedef struct PLOrb PLOrb;

int pl_orb_create(const PLOrbConfig* cfg, PLOrb** out);
void pl_orb_destroy(PLOrb* h);
/* max keypoints one frame can return (nfeatures + 3 per level overshoot, see DESIGN.md) */
int pl_orb_capacity(const PLOrb* h);
/* ORBextractor::Get{ScaleFactors,InverseScaleFactors,ScaleSigmaSquares,InverseScaleSigmaSquares},
 * mnFeaturesPerLevel and the level sizes; each array has nlevels entries (NULL = skip). */
int pl_orb_tables(const PLOrb* h, float* scale, float* inv_scale, float* sigma2, float* inv_sigma2,
                  int* features_per_level, int* level_w, int* level_h);
/* ORBextractor::operator()(image, mask, keypoints, descriptors) for ONE host frame.
 * kps: capacity pl_orb_capacity(); desc: capacity*32 bytes; *n receives the count.       */
int pl_orb_extract(PLOrb* h, const uint8_t* img, int stride, PLKeyPoint* kps, uint8_t* desc, int* n);
/* B host frames (frame b at imgs + b*frame_stride); outputs are [B][capacity] arrays. */
int pl_orb_extract_batch(PLOrb* h, const uint8_t* imgs, int stride, size_t frame_stride, int B,
                         PLKeyPoint* kps, uint8_t* desc, int* n);
/* Same with every pointer a device pointer; asynchronous on `stream`. */
int pl_orb_extract_batch_dev(PLOrb* h, const uint8_t* imgs, int stride, size_t frame_stride, int B,
                             PLKeyPoint* kps, uint8_t* desc, int* n, void* stream);
/* ORBextractor::mvImagePyramid[level] of frame `frame` of the LAST call, copied to host;
 * with_border != 0 adds the 19-px BORDER_REFLECT_101 frame (reference ORBextractor.cc:1107-1132). */
int pl_orb_get_level(PLOrb* h, int frame, int level, uint8_t* out, int with_border);
/* Capacity flag of the calls since the last check: PL_ERR_CAPACITY if a FAST cell overflowed cell_slot_cap (keypoints were
 * dropped), else PL_OK; clears the flag.  The host-buffer entry points call it themselves; callers of *_dev call it after
 * synchronising their stream. */
int pl_orb_check_overflow(PLOrb* h);
/* Debug / parity taps of the LAST call: pre-quadtree FAST candidates of (frame, level) in the
 * reference's order, coordinates relative to the level's (16,16) detection origin.  Returns count. */
int pl_orb_debug_candidates(PLOrb* h, int frame, int level, PLKeyPoint* out, int cap);

/* ------------------------------------------------------------------ descriptor matching
 * Flat-array forms of the reference's matcher methods.  A "frame" is the triple the matchers read from
 * ORB_SLAM2::Frame: mvKeysUn (PLKeyPoint[]), mDescriptors (n x 32 bytes), and the image bounds
 * bounds[4] = {mnMinX, mnMinY, mnMaxX, mnMaxY} that define the 64x48 bucket grid (Frame.cc:36,116-117,278-294).
 * Host-pointer forms synchronise and return the match count (>= 0) or an error (< 0); `_dev` forms are batched
 * over B frames ([B][cap] arrays, counts n[B]) and asynchronous.                                              */

/* ORBmatcher::DescriptorDistance (ORBmatcher.cc:1764-1780) == LSDmatcher::DescriptorDistance (LSDmatcher.cpp:654-670)
 * for n independent 32-byte pairs. */
int pl_descriptor_distance_batch(const uint8_t* a, const uint8_t* b, int n, int* out);

/* Frame::AssignFeaturesToGrid (Frame.cc:278-294): CSR of mGrid, cell = ix*48+iy; cell_start[3073], cell_items[n]. */
int pl_frame_assign_grid(const PLKeyPoint* keys_un, int n, const float* bounds, int* cell_start, int* cell_items);
int pl_frame_assign_grid_dev(const PLKeyPoint* keys_un, const int* n, int cap, int B, const float* bounds,
                             int* cell_start /*[B][3073]*/, int* cell_items /*[B][cap]*/, void* stream);

/* ORBmatcher::SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize) (ORBmatcher.cc:455-572).
 * prev_matched [n1][2] in/out, matches12 [n1] out. */
int pl_orb_search_for_initialization(const PLKeyPoint* keys1, const uint8_t* desc1, int n1, const PLKeyPoint* keys2,
                                     const uint8_t* desc2, int n2, const float* bounds, float* prev_matched,
                                     int* matches12, int window_size, float nnratio, int check_orientation);
/* batched: scratch = int[B][2*cap] */
int pl_orb_search_for_initialization_dev(const PLKeyPoint* keys1, const uint8_t* desc1, const int* n1,
                                         const PLKeyPoint* keys2, const uint8_t* desc2, const int* n2, int cap, int B,
                                         const float* bounds, float* prev_matched, int* matches12, int* nmatches,
                                         int window_size, float nnratio, int check_orientation, int* scratch,
                                         void* stream);

/* ORBmatcher::SearchByProjection(CurrentFrame, LastFrame, th, bMono=true) (ORBmatcher.cc:1441-1585).
 * Last frame side, per keypoint i: last_valid = (mvpMapPoints[i] && !mvbOutlier[i]), last_pos = GetWorldPos()
 * (3 floats), last_desc = GetDescriptor(), last_octave = mvKeys[i].octave, last_angle = mvKeysUn[i].angle.
 * Tcw: current pose (row-major 4x4 float), K = {fx,fy,cx,cy}.  cur_preassigned (may be NULL): keypoints that
 * already hold an observed map point.  cur_match[n_cur] out: last-frame index, -1 none, -2 pre-assigned. */
int pl_orb_search_by_projection_last(const PLKeyPoint* keys_cur, const uint8_t* desc_cur, int n_cur,
                                     const float* bounds, const float* Tcw, const float* K,
                                     const float* scale_factors, int nlevels, int n_last, const uint8_t* last_valid,
                                     const float* last_pos, const uint8_t* last_desc, const int* last_octave,
                                     const float* last_angle, float th, int check_orientation,
                                     const uint8_t* cur_preassigned, int* cur_match);

/* ORBmatcher::SearchByProjection(F, vpMapPoints, th) (ORBmatcher.cc:56-152).  Per map point: in_view =
 * (mbTrackInView && !isBad()), proj = {mTrackProjX, mTrackProjY}, level = mnTrackScaleLevel, view_cos =
 * mTrackViewCos, mp_desc = GetDescriptor().  match[n] out: map point index, -1, or -2 (pre-assigned). */
int pl_orb_search_by_projection_points(const PLKeyPoint* keys, const uint8_t* desc, int n, const float* bounds,
                                       const float* scale_factors, int nlevels, int n_mp, const uint8_t* in_view,
                                       const float* proj, const int* level, const float* view_cos,
                                       const uint8_t* mp_desc, float th, float nnratio, const uint8_t* preassigned,
                                       int* match);

/* cv::BFMatcher(NORM_HAMMING).knnMatch(d1, d2, k=2) as called at LSDmatcher.cpp:469: idx/dist are [n1][2]. */
int pl_match_bf_knn2(const uint8_t* d1, int n1, const uint8_t* d2, int n2, int* idx, int* dist);
/* LSDmatcher::FrameBFMatch(ldesc1, ldesc2, LineMatches, TH) incl. lineDescriptorMAD (LSDmatcher.cpp:462-486,627-652) */
int pl_lsd_frame_bf_match(const uint8_t* d1, int n1, const uint8_t* d2, int n2, float th, float nnratio, int* matches);
/* LSDmatcher::SearchDouble(InitialFrame, CurrentFrame, LineMatches) (LSDmatcher.cpp:440-460): both directions + mutual */
int pl_lsd_search_double(const uint8_t* d1, int n1, const uint8_t* d2, int n2, float nnratio, int* matches);
int pl_lsd_search_double_dev(const uint8_t* d1, const int* n1, const uint8_t* d2, const int* n2, int cap1, int cap2,
                             int B, float th, float nnratio, int mutual, int* matches /*[B][cap1]*/, int* nmatches,
                             void* stream);

/* ------------------------------------------------------------------ pose-only Levenberg-Marquardt
 * Optimizer::PoseOptimization (mode 0, src/Optimizer.cc:640-975), PoseOptimizationWithPoints (mode 1, :977-1115),
 * PoseOptimizationWithLines (mode 2, :1117-1284) with g2o's LM semantics restated (DESIGN.md §5).
 * One problem = one Frame: Tcw (row-major 4x4 float, pFrame->mTcw), K = {fx,fy,cx,cy};
 * per matched point i: pt_obs = mvKeysUn[i].pt, pt_inv_sigma2 = mvInvLevelSigma2[octave], pt_Xw = GetWorldPos();
 * per matched line i: line_func = mvKeyLineFunctions[i] (3 doubles), line_Xw = MapLine::mWorldPos (6 doubles).
 * Outputs: optimised Tcw, mvbOutlier / mvbLineOutlier flags.  Returns the reference's return value
 * (inlier count; 0 and an untouched pose when fewer than 3 correspondences) or an error < 0.
 * Mode 1 writes only pt_outlier and mode 2 only line_outlier (the other mask is left as the caller passed it, like the
 * reference's WithPoints / WithLines); the same holds per problem for the [B][cap] masks of pl_pose_optimization_dev. */
int pl_pose_optimization(int mode, const float* Tcw_in, const float* K, int n_points, const float* pt_obs,
                         const float* pt_inv_sigma2, const float* pt_Xw, int n_lines, const double* line_func,
                         const double* line_Xw, float* Tcw_out, uint8_t* pt_outlier, uint8_t* line_outlier,
                         int* iterations /* may be NULL: LM iterations executed */);
/* Batched, device pointers: arrays are [B][cap_*]...; scratch holds pl_pose_optimization_scratch_doubles() doubles. */
size_t pl_pose_optimization_scratch_doubles(int B, int cap_points, int cap_lines);
int pl_pose_optimization_dev(int mode, int B, const float* Tcw_in, const float* K, const int* n_points,
                             int cap_points, const float* pt_obs, const float* pt_inv_sigma2, const float* pt_Xw,
                             const int* n_lines, int cap_lines, const double* line_func, const double* line_Xw,
                             float* Tcw_out, uint8_t* pt_outlier, uint8_t* line_outlier, int* inliers,
                             int* iterations, double* scratch, void* stream);

/* ------------------------------------------------------------------ line features (LSD + LBD)
 * replaces ORB_SLAM2::LINEextractor (reference include/LineExtractor.h:20-62, src/LineExtractor.cpp:26-93).
 * KeyLine records are byte-compatible with cv::line_descriptor::KeyLine (68 B: angle, class_id, octave, pt.x, pt.y,
 * response, size, startPointX/Y, endPointX/Y, sPointInOctaveX/Y, ePointInOctaveX/Y, lineLength, numOfPixels).   */
typedef struct PLLineConfig {
  int width, height;
  int nfeatures;            /* LINEextractor.nFeatures (nLSDFeature); the reference keeps up to nfeatures+1 lines */
  double min_line_length;   /* LINEextractor.min_line_length                                                    */
  int max_batch;
  int segment_cap;          /* max LSD segments per frame before truncation; 0 = default 8192                     */
  int lsd_used_in_global;   /* region-growing USED map: <0 shared memory, >0 global memory, 0 = global unless env PLSLAM_LSD_USED_GLOBAL=0 */
} PLLineConfig;
typedef struct PLLine PLLine;
int pl_line_create(const PLLineConfig* cfg, PLLine** out);
void pl_line_destroy(PLLine* h);
int pl_line_capacity(const PLLine* h);   /* nfeatures + 1 */
/* LINEextractor::operator()(image, mask, keylines, descriptors, lineVec2d) for ONE host frame; mask may be NULL
 * (8UC1, same size; a line is dropped when both end points lie on mask==0).  keylines: capacity x 68 B,
 * desc: capacity x 32, linefunc: capacity x 3 doubles (normalised sp x ep), *n: number of KeyLines. */
int pl_line_extract(PLLine* h, const uint8_t* img, int stride, const uint8_t* mask, void* keylines, uint8_t* desc,
                    double* linefunc, int* n);
int pl_line_extract_batch(PLLine* h, const uint8_t* imgs, int stride, size_t frame_stride, int B, const uint8_t* mask,
                          void* keylines, uint8_t* desc, double* linefunc, int* n);
int pl_line_extract_batch_dev(PLLine* h, const uint8_t* imgs, int stride, size_t frame_stride, int B,
                              const uint8_t* mask, void* keylines, uint8_t* desc, double* linefunc, int* n, void* stream);
/* parity taps of the LAST call: raw LSD segments (x1,y1,x2,y2 floats, detection order), the 0.8x scaled image,
 * the LBD Sobel pair, and the seed order (pixel indices y*sw+x of the scaled image). */
/* Capacity flags since the last check (segment_cap exceeded / region growing gave a frame up): PL_ERR_CAPACITY or PL_OK;
 * clears them.  For callers of pl_line_extract_batch_dev, after synchronising their stream. */
int pl_line_check_overflow(PLLine* h);
int pl_line_debug_segments(PLLine* h, int frame, float* out, int cap);
int pl_line_debug_scaled(PLLine* h, int frame, uint8_t* out, int* sw, int* sh);
int pl_line_debug_sobel(PLLine* h, int frame, short* dx, short* dy);
int pl_line_debug_order(PLLine* h, int frame, unsigned* out, int cap);
/* control words of the speculative region growing for one frame of the LAST call (counters; post-mortem of the watchdog) */
int pl_line_debug_ctl(PLLine* h, int frame, int* out, int nwords);

/* ------------------------------------------------------------------ per-frame front-end pipeline (batch of frames)
 * The hot-path calls Tracking makes for one frame (SURVEY.md §3.1), chained on one stream with all intermediates in
 * HBM: ORB extract, LSD+LBD extract, point matching frame k-1 -> k (SearchForInitialization scheme, window 100,
 * ratio 0.9), line matching (SearchDouble), and two Optimizer::PoseOptimization calls on the frame's pose problem.
 * Frame 0's predecessor is the LAST frame of the PREVIOUS step (consecutive batches of one sequence; none before the first
 * step), or, after pl_frontend_set_wrap(h, 1), the last frame of the same batch (closed loop).  bench.py's "step".    */
typedef struct PLFrontendConfig {
  int width, height, max_batch;
  int orb_nfeatures; float orb_scale_factor; int orb_nlevels, orb_ini_th, orb_min_th;
  int line_nfeatures; double line_min_length;
  int lm_cap_points, lm_cap_lines;     /* capacity of the per-frame pose problems */
} PLFrontendConfig;
typedef struct PLFrontend PLFrontend;
int pl_frontend_create(const PLFrontendConfig* cfg, PLFrontend** out);
void pl_frontend_destroy(PLFrontend* h);
int pl_frontend_capacities(const PLFrontend* h, int* cap_keypoints, int* cap_lines);
/* upload the batch's pose problems (host pointers, [B][cap] layouts as in pl_pose_optimization_dev); PL_ERR_ARG if a count is
 * negative or any n_points[b] > lm_cap_points or n_lines[b] > lm_cap_lines (nothing is uploaded then; the same holds for the
 * _async form) */
int pl_frontend_set_pose_problems(PLFrontend* h, int B, const float* Tcw0, const float* K, const int* n_points,
                                  const float* pt_obs, const float* pt_inv_sigma2, const float* pt_Xw, const int* n_lines,
                                  const double* line_func, const double* line_Xw);
/* camera of the sequence: K = {fx,fy,cx,cy}, dist5 = {k1,k2,p1,p2,k3} (Tracking.cc:53-120).  k1 != 0: every frame is
 * undistorted for the line extractor (Frame.cc:220-225), keypoints are undistorted for the matcher (Frame.cc:233) and the
 * grid bounds come from ComputeImageBounds; k1 == 0 or never called: no undistortion (the default). */
int pl_frontend_set_camera(PLFrontend* h, const float* K, const float* dist5);
/* the same upload enqueued on `stream` (NULL = the handle's stream) without synchronising: PINNED host arrays that stay
 * valid until the stream has passed; a following pl_frontend_run_dev / submit on the same stream sees the new problems.
 * Returns the bytes enqueued (>= 0) or an error. */
long long pl_frontend_set_pose_problems_async(PLFrontend* h, int B, const float* Tcw0, const float* K, const int* n_points,
                                              const float* pt_obs, const float* pt_inv_sigma2, const float* pt_Xw,
                                              const int* n_lines, const double* line_func, const double* line_Xw, void* stream);
/* PL_ERR_CAPACITY if any step since the last check overflowed an extractor capacity (callers of pl_frontend_run_dev) */
int pl_frontend_check_overflow(PLFrontend* h);
int pl_frontend_set_wrap(PLFrontend* h, int on);
/* Steady-state tracking stage of the step (default off): the four projection searches the reference's tracker runs per frame -
 * ORBmatcher::SearchByProjection(Current, Last, 15, mono) and again with 30 for frames under 20 matches (Tracking.cc:1345-1357),
 * LSDmatcher::SearchByProjection(Current, Last, 15) (:1347), ORBmatcher(0.8)::SearchByProjection(F, local points, 1) (:1799),
 * LSDmatcher::SearchByProjection(F, local lines, 1) (:1855) - on the pose guess Tcw0 / K of pl_frontend_set_pose_problems.
 * The batch step has no map: frame b's map is frame b-1's features (a point on each keypoint's ray, a line per keyline). */
int pl_frontend_set_tracking(PLFrontend* h, int on);
/* which: 0 = motion-model searches, 1 = local-map searches.  Matches index the previous frame's features (-1 none, -2 feature
 * held a match already); map_pos = the synthetic map points [B][capK][3]; *_in_view = the elements each search projected. */
int pl_frontend_fetch_tracking(PLFrontend* h, int B, int which, int* point_match, int* n_point_matches, int* line_match,
                               int* n_line_matches, float* map_pos, uint8_t* point_in_view, uint8_t* line_in_view);
/* mvKeysUn of the last step, [B][cap_keypoints] */
int pl_frontend_fetch_keys_un(PLFrontend* h, int B, PLKeyPoint* out);
/* device-resident step (imgs = device pointer; NULL = frames uploaded by the last pl_frontend_run); asynchronous */
int pl_frontend_run_dev(PLFrontend* h, const uint8_t* imgs, int stride, size_t frame_stride, int B, void* stream);
/* end-to-end step on HOST buffers: H2D frames, device step, D2H of every per-frame result; synchronous.
 * outputs: kps/desc/n [B][capK], keylines/ldesc/linefunc/nl [B][capL], pt_matches [B][capK] (index into frame k of
 * the match of keypoint i of frame k-1, or -1), line_matches [B][capL], poses [2][B][16], inliers [2][B]. */
int pl_frontend_run(PLFrontend* h, const uint8_t* imgs, int stride, size_t frame_stride, int B, PLKeyPoint* kps,
                    uint8_t* desc, int* n, void* keylines, uint8_t* ldesc, double* linefunc, int* nl, int* pt_matches,
                    int* n_pt_matches, int* line_matches, int* n_line_matches, float* poses, int* inliers);
/* Streaming form of pl_frontend_run: returns once the step is enqueued; the H2D copy of the next step and the D2H copy of
 * the previous one overlap the kernels.  Host buffers should be pinned; outputs of submit #i are valid once
 * pl_frontend_wait has let it complete.  At most two steps are in flight (submit blocks otherwise); with two alternating
 * output sets the loop is: submit(i+1); wait(keep_in_flight = 1); consume outputs of step i. */
int pl_frontend_submit(PLFrontend* h, const uint8_t* imgs, int stride, size_t frame_stride, int B, PLKeyPoint* kps,
                       uint8_t* desc, int* n, void* keylines, uint8_t* ldesc, double* linefunc, int* nl, int* pt_matches,
                       int* n_pt_matches, int* line_matches, int* n_line_matches, float* poses, int* inliers);
/* wait until at most keep_in_flight (0 or 1) submitted steps are unfinished; PL_ERR_CAPACITY if a finished step overflowed
 * a capacity (the same check pl_frontend_run and pl_frontend_fetch make) */
int pl_frontend_wait(PLFrontend* h, int keep_in_flight);
int pl_frontend_io_bytes(const PLFrontend* h, long long* h2d_per_frame, long long* d2h_per_frame);
int pl_frontend_fetch(PLFrontend* h, int B, PLKeyPoint* kps, uint8_t* desc, int* n, void* keylines, uint8_t* ldesc, int* nl,
                      int* pt_matches, int* n_pt_matches, int* line_matches, int* n_line_matches, float* poses, int* inliers);

/* ------------------------------------------------------------------ wire / disk formats (SURVEY.md §8 f.4)
 * Pose record of a frame, 16 floats: Rwc (row-major 3x3) = KeyFrame::GetRotation().t(), Ow = GetCameraCenter() (KeyFrame.cc:52-66),
 * Converter::toQuaternion(Rwc) as x y z w (Converter.cc:141-153) - what both trajectory writers print, computed on the device so
 * that the multi-GPU all-gather can ship it as is. */
int pl_pose_records_dev(const float* Tcw_dev /*[n][16]*/, int n, float* records_dev /*[n][16]*/, void* stream);
/* System::SaveKeyFrameTrajectoryTUM (System.cc:396-431): "stamp tx ty tz qx qy qz qw\n", fixed, precision 6 / 7; bad[i] = pKF->isBad().
 * Return: length of the text (>= 0; written NUL-terminated into out if cap is larger - call with out = NULL to size), < 0 = PL_ERR_*. */
long long pl_trajectory_format_tum(const double* timestamps, const float* poses_Tcw, const uint8_t* bad, int n, char* out, size_t cap);
/* System::SaveKeyFrameTrajectoryMonoKitti (System.cc:433-464): the 3x4 [Rwc | Ow] row-major, precision 9. */
long long pl_trajectory_format_mono_kitti(const float* poses_Tcw, const uint8_t* bad, int n, char* out, size_t cap);
int pl_save_keyframe_trajectory_tum(const char* filename, const double* timestamps, const float* poses_Tcw, const uint8_t* bad, int n);
int pl_save_keyframe_trajectory_mono_kitti(const char* filename, const float* poses_Tcw, const uint8_t* bad, int n);
/* Flat little-endian dump of the last step's results (the arrays of pl_frontend_fetch + the line functions) for offline replay:
 * "PLSB200\x01", int32 B, then per field {int32 len, name, int32 len, numpy dtype text, int32 ndim, int64 shape[], bytes}. */
int pl_frontend_dump(PLFrontend* h, int B, const char* path);

/* measurement hooks (bench.py): CUDA-event timing of k_lsd_grow on its launching stream, its algorithmic bytes, and
 * a device copy of the second-call poses [B][16] for the multi-GPU all-gather */
int pl_line_set_timing(PLLine* h, int on);
int pl_line_grow_ms(PLLine* h, float* ms);
long long pl_line_grow_bytes_per_frame(const PLLine* h);
int pl_frontend_set_timing(PLFrontend* h, int on);
int pl_frontend_grow_ms(PLFrontend* h, float* ms);
long long pl_frontend_grow_bytes_per_frame(const PLFrontend* h);
int pl_frontend_copy_poses_dev(PLFrontend* h, int B, float* dst, void* stream);

/* ------------------------------------------------------------------ local bundle adjustment (points + lines)
 * Optimizer::LocalBundleAdjustmentWithLine(pKF, pbStopFlag, pMap) (src/Optimizer.cc:1645-2100; with n_le == 0 it is
 * Optimizer::LocalBundleAdjustment, :1308-1642) on the flattened local window that the reference gathers at
 * :1649-1742.  Keyframes: local (free) and fixed ones (kf_fixed: lFixedCameras and mnId == 0); landmarks: map points
 * and the two end points of every map line; edges in the reference's insertion order.  Host pointers; synchronous. */
typedef struct PLBAProblem {
  int n_kf;  const float* kf_Tcw /*[n_kf][16]*/; const uint8_t* kf_fixed; const float* kf_K /*[n_kf][4] fx fy cx cy*/;
  float K_end[4];                 /* intrinsics the END-point line edges use: the current keyframe's (Optimizer.cc:1939-1942) */
  int n_pt;  const float* pt_Xw /*[n_pt][3] MapPoint::GetWorldPos*/;
  int n_ln;  const double* ln_Xw /*[n_ln][6] MapLine::mWorldPos*/;
  int n_pe;  const int* pe_kf; const int* pe_pt; const float* pe_obs /*[n_pe][2] mvKeysUn.pt*/; const float* pe_inv_sigma2;
  int n_le;  const int* le_kf; const int* le_ln; const double* le_func /*[n_le][3] mvKeyLineFunctions*/;
} PLBAProblem;
/* stop_flag_dev: device-visible int (e.g. mapped pinned memory) polled like g2o's forceStopFlag; NULL = never stop.
 * Outputs: optimised keyframe poses, points, line end points; pe_erase / le_erase = observations the reference would
 * erase (:2005-2043), le_erase_kf = the keyframe index the reference pairs with line observation i (its i/2 quirk). */
int pl_local_ba(const PLBAProblem* p, const int* stop_flag_dev, float* kf_Tcw_out, float* pt_Xw_out, double* ln_Xw_out,
                uint8_t* pe_erase, uint8_t* le_erase, int* le_erase_kf, int* iterations);

/* Optimizer::BundleAdjustment with lines (src/Optimizer.cc:275-638; GlobalBundleAdjustemnt :41-58 passes the whole map):
 * ONE Levenberg-Marquardt optimize(n_iterations) over all keyframes (kf_fixed = mnId == 0), map points and map-line end points,
 * Huber kernels (sqrt(5.99) points, sqrt(3.84) line end points) iff robust, line information = identity, every line edge on
 * the observing keyframe's own intrinsics (K_end of PLBAProblem is not read); no outlier rounds, nothing is erased.
 * stop_flag_host: the reference's pbStopFlag (HOST int, polled between iterations and trials; NULL = never).
 * Outputs: every keyframe's pose (the reference calls SetPose(toCvMat(estimate)) on all of them, :549-556), points (a point
 * without observations keeps its input, :411-416), line end points (through float like Converter::toCvMat, :621-625).
 * The nLoopKF != 0 variant only changes WHERE the caller stores these (mTcwGBA / mPosGBA, :557-562): caller's business.
 * Multi-CTA: reduced pose system built per non-zero 6x6 block in landmark order (no atomics: bit-reproducible), dense
 * blocked Cholesky; solve_ms (may be NULL) = device time of the whole optimisation (CUDA events). */
int pl_global_ba(const PLBAProblem* p, int n_iterations, int robust, const int* stop_flag_host, float* kf_Tcw_out,
                 float* pt_Xw_out, double* ln_Xw_out, int* iterations, float* solve_ms);

/* ------------------------------------------------------------------ line matching by projection
 * Frame::AssignFeaturesToGridForLine (Frame.cc:296-320): CSR of mGridForLine (cell = ix*48+iy); returns #items. */
int pl_frame_assign_grid_lines(const void* keylines_un /*68 B records*/, int n, const float* bounds, int* cell_start /*[3073]*/,
                               int* cell_items, int cap_items);
/* LSDmatcher::SearchByProjection(CurrentFrame, LastFrame, th) (LSDmatcher.cpp:72-176).  Per last-frame line i:
 * last_valid = (mvpMapLines[i] && !mvbLineOutlier[i] && CurrentFrame.isInFrustum(pML, 0.5)), last_proj =
 * {mTrackProjX1, Y1, X2, Y2}, last_desc = GetDescriptor(), last_length = LastFrame.mvKeylinesUn[i].lineLength.
 * (The frustum test itself is Frame glue, SURVEY.md §8f.1.)  cur_match[n_cur]: last index, -1, or -2 pre-assigned. */
int pl_lsd_search_by_projection_last(const void* keylines_cur, const double* linefunc_cur, const uint8_t* desc_cur, int n_cur,
                                     const float* bounds, int n_last, const uint8_t* last_valid, const float* last_proj,
                                     const uint8_t* last_desc, const float* last_length, float th,
                                     const uint8_t* cur_preassigned, int* cur_match);
/* LSDmatcher::SearchByProjection(F, vpMapLines, th) (LSDmatcher.cpp:221-338): in_view = (mbTrackInView && !isBad()),
 * proj = {mTrackProjX1,Y1,X2,Y2}, view_cos = mTrackViewCos, ml_desc = GetDescriptor(). */
int pl_lsd_search_by_projection_lines(const void* keylines, const double* linefunc, const uint8_t* desc, int n,
                                      const float* bounds, int n_ml, const uint8_t* in_view, const float* proj,
                                      const float* view_cos, const uint8_t* ml_desc, float th, float nnratio,
                                      const uint8_t* preassigned, int* match);

/* Batched, device-resident forms of the projection searches ([B][cap] arrays, one launch, asynchronous on `stream`); the
 * host-pointer functions above are their B = 1 case.  gate_nmatches / gate_min: frame b runs only if gate_nmatches[b] < gate_min
 * (the "fill(mvpMapPoints, NULL); search again with 2 * th" retry of Tracking.cc:1352-1357); NULL = every frame runs. */
int pl_orb_search_by_projection_last_dev(const PLKeyPoint* keys_cur, const uint8_t* desc_cur, const int* n_cur, int cap, int B,
                                         const float* bounds, const float* Tcw /*[B][16]*/, const float* K /*[B][4]*/,
                                         const float* scale_factors, int nlevels, const int* n_last, int cap_last,
                                         const uint8_t* last_valid, const float* last_pos, const uint8_t* last_desc,
                                         const int* last_octave, const float* last_angle, float th, int check_orientation,
                                         const uint8_t* cur_preassigned, const int* gate_nmatches, int gate_min, int* cur_match,
                                         int* nmatches, void* stream);
int pl_orb_search_by_projection_points_dev(const PLKeyPoint* keys, const uint8_t* desc, const int* n, int cap, int B,
                                           const float* bounds, const float* scale_factors, const int* n_mp, int cap_mp,
                                           const uint8_t* in_view, const float* proj, const int* level, const float* view_cos,
                                           const uint8_t* mp_desc, float th, float nnratio, const uint8_t* preassigned, int* match,
                                           int* nmatches, void* stream);
size_t pl_lsd_search_scratch_bytes(int cap, int B);
/* variant 0: LSDmatcher::SearchByProjection(CurrentFrame, LastFrame, th), q_length_or_view_cos = last lineLength;
 * variant 1: SearchByProjection(F, vpMapLines, th), q_length_or_view_cos = mTrackViewCos.  scratch: pl_lsd_search_scratch_bytes. */
int pl_lsd_search_by_projection_dev(int variant, const void* keylines, const double* linefunc, const uint8_t* desc, const int* n,
                                    int cap, int B, const float* bounds, const int* n_q, int cap_q, const uint8_t* q_valid,
                                    const float* q_proj, const uint8_t* q_desc, const float* q_length_or_view_cos, float th,
                                    float nnratio, const uint8_t* preassigned, int* match, int* nmatches, void* scratch, void* stream);

/* ------------------------------------------------------------------ Frame glue (SURVEY.md §8f.1)
 * The mono Frame constructor undistorts every frame for the line extractor (initUndistortRectifyMap + remap,
 * src/Frame.cc:220-222), undistorts the keypoints (UndistortKeyPoints, :915-945) and computes the image bounds
 * (:947-985); Tracking then projects local map points / lines with Frame::isInFrustum (:560-702).  K = {fx,fy,cx,cy},
 * dist5 = {k1,k2,p1,p2,k3} exactly as Tracking.cc:53-120 fills mK / mDistCoef (float).                         */
typedef struct PLUndistort PLUndistort;
int pl_undistort_create(const float* K, const float* dist5, int width, int height, PLUndistort** out);   /* builds the map once */
void pl_undistort_destroy(PLUndistort* h);
/* cv::remap(src, dst, mUndistX, mUndistY, INTER_LINEAR) */
int pl_undistort_remap(PLUndistort* h, const uint8_t* src, int sstride, uint8_t* dst, int dstride);
int pl_undistort_remap_batch_dev(PLUndistort* h, const uint8_t* src, int sstride, size_t sframe, int B, uint8_t* dst,
                                 int dstride, size_t dframe, void* stream);
/* Frame::UndistortKeyPoints: only pt.x / pt.y change; k1 == 0 copies */
int pl_undistort_keypoints(PLUndistort* h, const PLKeyPoint* kps, int n, PLKeyPoint* out);
int pl_undistort_keypoints_dev(PLUndistort* h, const PLKeyPoint* kps, const int* n, int cap, int B, PLKeyPoint* out, void* stream);
/* Frame::ComputeImageBounds -> {mnMinX, mnMinY, mnMaxX, mnMaxY} */
int pl_frame_image_bounds(const float* K, const float* dist5, int width, int height, float* bounds);
/* Frame::isInFrustum(MapPoint*, viewingCosLimit) for n map points: pos = GetWorldPos, normal = GetNormal,
 * min/max_dist = the RAW MapPoint::mfMinDistance / mfMaxDistance (the 0.8f / 1.2f factors of Get{Min,Max}DistanceInvariance are
 * applied inside for the range test; PredictScale uses the raw mfMaxDistance, MapPoint.cc:396-428, MapLine.cpp:395-404); Tcw row-major 4x4, Ow = mOw.  Outputs mbTrackInView, {mTrackProjX,Y},
 * mnTrackScaleLevel, mTrackViewCos. */
int pl_frame_is_in_frustum_points(const float* Tcw, const float* Ow, const float* K, const float* bounds, float log_scale_factor,
                                  int n_scale_levels, float viewing_cos_limit, int n, const float* pos, const float* normal,
                                  const float* min_dist, const float* max_dist, uint8_t* inview, float* proj, int* level,
                                  float* viewcos);
/* Frame::isInFrustum(MapLine*, viewingCosLimit): pos = mWorldPos (6 doubles), normal = GetNormal (3 doubles); proj = {X1,Y1,X2,Y2} */
int pl_frame_is_in_frustum_lines(const float* Tcw, const float* Ow, const float* K, const float* bounds, float log_scale_factor,
                                 float viewing_cos_limit, int n, const double* pos, const double* normal, const float* min_dist,
                                 const float* max_dist, uint8_t* inview, float* proj, int* level, float* viewcos);

/* ------------------------------------------------------------------ LocalMapping matchers (SURVEY.md §8f.2)
 * ORBmatcher::SearchForTriangulation(pKF1, pKF2, F12, vMatchedPairs, bOnlyStereo=false) (src/ORBmatcher.cc:720-911), monocular.
 * keys*_un = mvKeysUn, has_mp* = GetMapPoint(i) != NULL, fv* = DBoW2 FeatureVector as CSR (node ids ascending as in std::map,
 * fv_start[nn+1], fv_items = feature indices in insertion order), F12 row-major 3x3, Cw1 = pKF1->GetCameraCenter(),
 * R2w/t2w = pKF2 rotation (row-major 3x3) / translation, K2 = {fx,fy,cx,cy}, scale_factors2 = mvScaleFactors,
 * level_sigma2_2 = mvLevelSigma2.  matches12[i] = idx2 or -1 (vMatchedPairs = the pairs with idx2 >= 0); returns nmatches. */
int pl_orb_search_for_triangulation(const PLKeyPoint* keys1_un, const uint8_t* desc1, const uint8_t* has_mp1, int n1,
                                    const PLKeyPoint* keys2_un, const uint8_t* desc2, const uint8_t* has_mp2, int n2,
                                    const unsigned* fv1_nodes, const int* fv1_start, const int* fv1_items, int nn1,
                                    const unsigned* fv2_nodes, const int* fv2_start, const int* fv2_items, int nn2,
                                    const float* F12, const float* Cw1, const float* R2w, const float* t2w, const float* K2,
                                    const float* scale_factors2, const float* level_sigma2_2, int nlevels,
                                    int check_orientation, int* matches12);
/* ORBmatcher::SearchByProjection(CurrentFrame, pKF, sAlreadyFound, th, ORBdist) (src/ORBmatcher.cc:1587-1716;
 * Tracking::Relocalization Tracking.cc:2194,2208).  kf_valid[i] = pMP && !isBad() && !sAlreadyFound.count(pMP) for the keyframe's
 * map-point matches; pos / mp_desc / min,max_dist = GetWorldPos, GetDescriptor, raw mfMinDistance / mfMaxDistance (see pl_frame_is_in_frustum); kf_angle =
 * pKF->mvKeysUn[i].angle; Ow = camera centre of the current pose; cur_preassigned[i2] = mvpMapPoints[i2] != NULL.
 * cur_match[i2] = keyframe index i, -1, or -2 (was preassigned); returns nmatches. */
int pl_orb_search_by_projection_keyframe(const PLKeyPoint* keys_cur, const uint8_t* desc_cur, int n_cur, const float* bounds,
                                         const float* Tcw, const float* Ow, const float* K, const float* scale_factors, int nlevels,
                                         float log_scale_factor, int n_kf, const uint8_t* kf_valid, const float* pos,
                                         const uint8_t* mp_desc, const float* min_dist, const float* max_dist,
                                         const float* kf_angle, float th, int orb_dist, int check_orientation,
                                         const uint8_t* cur_preassigned, int* cur_match);
/* ORBmatcher::SearchByBoW(pKF, F, vpMapPointMatches) (src/ORBmatcher.cc:187-327; TrackReferenceKeyFrame Tracking.cc:1157,
 * Relocalization :2119): has_mp_kf[i] = vpMapPointsKF[i] && !isBad(); fv* as in pl_orb_search_for_triangulation; keysF = F.mvKeys.
 * matchesF[j] = keyframe feature whose MapPoint frame feature j receives, or -1; returns nmatches. */
int pl_orb_search_by_bow(const PLKeyPoint* keysKF_un, const uint8_t* descKF, const uint8_t* has_mp_kf, int nKF,
                         const PLKeyPoint* keysF, const uint8_t* descF, int nF, const unsigned* fvK_nodes, const int* fvK_start,
                         const int* fvK_items, int nnK, const unsigned* fvF_nodes, const int* fvF_start, const int* fvF_items,
                         int nnF, float nnratio, int check_orientation, int* matchesF);
/* ORBmatcher::SearchByBoW(pKF1, pKF2, vpMatches12) (src/ORBmatcher.cc:574-709; LoopClosing::ComputeSim3): MapPoints required on
 * both sides (has_mp*), vbMatched2 state, gate bestDist1 < TH_LOW.  matches12[i] = idx2 (vpMatches12[i] = vpMapPoints2[idx2]) or -1. */
int pl_orb_search_by_bow_keyframes(const PLKeyPoint* keys1_un, const uint8_t* desc1, const uint8_t* has_mp1, int n1,
                                   const PLKeyPoint* keys2_un, const uint8_t* desc2, const uint8_t* has_mp2, int n2,
                                   const unsigned* fv1_nodes, const int* fv1_start, const int* fv1_items, int nn1,
                                   const unsigned* fv2_nodes, const int* fv2_start, const int* fv2_items, int nn2, float nnratio,
                                   int check_orientation, int* matches12);
/* LSDmatcher::SearchForTriangulation(pKF1, pKF2, vMatchedPairs, isDouble) (src/LSDmatcher.cpp:727-776; LocalMapping.cc:961):
 * FrameBFMatch both ways at th (TH_HIGH = 80 there) with the matcher's nnratio, mutual check when is_double, pairs touching a
 * line that already has a MapLine (has_ml*) removed.  The pair<> overload (:672-725; LocalMapping.cc:679) is th = TH_LOW = 50,
 * is_double = 1.  matched_pairs[i] = j or -1; returns nmatches.
 * LSDmatcher::SearchDouble(KeyFrame*, Frame&) (:375-430; Tracking.cc:1159) is pl_lsd_search_double(F.mLdesc, KF.mLineDescriptors)
 * followed by keeping the pairs whose keyframe line has a MapLine. */
int pl_lsd_search_for_triangulation(const uint8_t* ldesc1, const uint8_t* has_ml1, int n1, const uint8_t* ldesc2,
                                    const uint8_t* has_ml2, int n2, float th, float nnratio, int is_double, int* matched_pairs);
/* The search half of ORBmatcher::Fuse(pKF, vpMapPoints, th) (src/ORBmatcher.cc:914-1034): best keypoint of the keyframe for
 * every map point (best_idx = -1 / best_dist = 256 when skipped or nothing qualifies).  skip[i] = !pMP || isBad || IsInKeyFrame;
 * the caller applies :1036-1061 (Replace / AddObservation) to the points with best_dist <= TH_LOW (50) in order. */
int pl_orb_fuse_search(const PLKeyPoint* keys_un, const uint8_t* desc, int n, const float* bounds, const float* Tcw,
                       const float* Ow, const float* K, const float* scale_factors, const float* inv_level_sigma2, int nlevels,
                       float log_scale_factor, int n_mp, const uint8_t* skip, const float* pos, const float* normal,
                       const float* min_dist, const float* max_dist, const uint8_t* mp_desc, float th, int* best_idx,
                       int* best_dist);

/* MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:249-314) for n_mp map points: the descriptors of point m are rows
 * offsets[m] .. offsets[m+1] of desc (its observations in std::map order, bad keyframes dropped by the caller).  best_idx[m] =
 * index INSIDE the point's list of the descriptor with the least median distance to the others (first wins; -1 for an empty
 * list: the reference keeps mDescriptor); out_desc (may be NULL) receives the chosen 32 bytes per point. */
int pl_mappoint_distinctive_descriptors(const uint8_t* desc, const int* offsets, int n_mp, int* best_idx, uint8_t* out_desc);
/* The search half of LSDmatcher::Fuse(pKF, vpMapLines, th) (src/LSDmatcher.cpp:860-1011; LocalMapping.cc:1600,1627), with the
 * reference's quirks: the first map line with an end point behind the camera ends the call with `return false` (*stop_at = its
 * index, n_ml if none: the caller returns 0 and has applied the surgery of the lines before it); candidates are
 * KeyFrame::GetLinesInArea (KeyFrame.cc:647-682) with kl.octave in [level-1, level], level = unclamped MapLine::PredictScale;
 * the map line's descriptor is compared with row idx of the keyframe's POINT descriptors (:966; rows beyond n_pdesc skipped);
 * mvScaleFactorsLine[level] out of range is restated as scale_line^level.  skip[i] = !pML || isBad() || IsInKeyFrame(pKF);
 * bounds = {mnMinX, mnMinY, mnMaxX, mnMaxY} (IsInImage: min <= x < max); min/max_dist raw.  best_idx = -1 / best_dist = 256 when
 * skipped or nothing qualifies; the caller applies :986-1006 (Replace / AddObservation) to lines with best_dist <= 50 in order. */
int pl_lsd_fuse_search(const void* keylines, int nl, const uint8_t* kf_point_desc, int n_pdesc, const float* bounds, const float* Tcw,
                       const float* Ow, const float* K, float scale_line, float log_scale_factor_line, int n_ml, const uint8_t* skip,
                       const double* pos, const double* normal, const float* min_dist, const float* max_dist, const uint8_t* ml_desc,
                       float th, int* best_idx, int* best_dist, int* stop_at);

/* ------------------------------------------------------------------ multi-GPU exchange (SURVEY.md §8e)
 * Frames shard across the GPUs of one box with no data-path collective; the ONE exchange is an all-gather of the per-frame
 * pose records (64 B per frame) over NCCL / NVLink so that the rank running the sequential Tracking logic (Tracking.cc:329)
 * sees them in frame order.  NCCL is taken from the libnccl.so.2 already in the process (no link-time dependency).
 * pl_comm_unique_id on rank 0 -> ship the 128 bytes to every rank (MPI / torch.distributed / a file) -> pl_comm_create on all. */
typedef struct PLComm PLComm;
int pl_comm_unique_id(void* id128);
int pl_comm_create(const void* id128, int nranks, int rank, PLComm** out);
void pl_comm_destroy(PLComm* c);
int pl_nccl_version(void);
/* every rank contributes floats_per_rank floats (its block of [frames][16] poses, padded to the common block size);
 * recv_dev = [nranks][floats_per_rank] on every rank; asynchronous on `stream`. */
int pl_allgather_poses(PLComm* c, const float* send_dev, float* recv_dev, size_t floats_per_rank, void* stream);
/* the same on a communicator the host already owns (ncclComm_t passed as void*) */
int pl_allgather_poses_nccl(void* nccl_comm, const float* send_dev, float* recv_dev, size_t floats_per_rank, void* stream);

#ifdef __cplusplus
}
#endif
#endif
