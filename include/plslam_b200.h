/* plslam_b200 — C ABI of the H100-native PL-SLAM front-end / LM hot path.
 *
 * Every entry point replaces one C++ interface of the reference (HarborC/PL-SLAM); the
 * reference has no FFI of its own (SURVEY.md §8b), so these are what a thin C++ class with the
 * reference's signature binds (see pl-slam_b200/host/ and INTEGRATION.md).
 *
 * Conventions: plain pointers and sizes; `_dev` variants take DEVICE pointers (inputs resident
 * in HBM) plus a cudaStream_t passed as void* (NULL = the handle's own stream) and are
 * asynchronous; the plain variants take HOST pointers, copy in/out and synchronise.  A plain variant
 * refuses a NULL array whose count is > 0 with PL_ERR_ARG, and reports a failed device allocation
 * or copy while staging its arrays as PL_ERR_CUDA.
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
/* device bytes currently held through the library's owner type: every handle's buffers, not per-call staging */
unsigned long long pl_device_bytes(void);

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
                       /* each level's quota (mnFeaturesPerLevel) must fit one quadtree in shared memory: at most 4878
                        * on a 4:3 frame with the H100's 232448 B per block; pl_orb_create refuses a larger quota with
                        * PL_ERR_ARG and names the largest that fits */
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
 * over B frames ([B][cap] arrays, counts n[B]) and asynchronous.  In a `_dev` form frame b's row of an array with capacity
 * cap starts at b * cap, each side with its own capacity (cap_last, cap_mp, cap_q, cap1, cap2); a count above its capacity
 * is clamped to it.  Rows of an input past its count are never read, and entries of an output row past its count
 * (matches, prev_matched, cell_items past cell_start[3072]) are never written.                                   */

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
/* batched: scratch = int[B][2*cap]; cap at most 6144 (PL_ERR_ARG before any launch above it) */
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
/* batched: mutual = 1 is SearchDouble at threshold th, mutual = 0 FrameBFMatch(d1, d2, th).  One CTA per frame keeps
 * 2 * (cap1 + cap2 + 2 * max(cap1, cap2)) bytes of shared memory; capacities for which that and the kernel's static shared
 * memory exceed the device's opt-in limit per block (about 28,900 lines per side on an H100) return PL_ERR_ARG before any
 * launch, in this form and in the host forms above (whose capacities are n1 and n2). */
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
  int segment_cap;          /* max LSD segments per frame before truncation; 0 = default 8192.  k_keylines sorts
                               pow2(segment_cap) 8-byte keys in one block's shared memory, so the largest cap is the
                               device's opt-in shared memory per block over 8, rounded down to a power of two (16384
                               on H100); a larger or a negative cap is refused with PL_ERR_ARG.  A textured 1920x1080
                               frame can exceed the default 8192 and then needs an explicit cap up to 16384.       */
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
/* Capacity flag since the last check (segment_cap exceeded): PL_ERR_CAPACITY or PL_OK;
 * clears them.  For callers of pl_line_extract_batch_dev, after synchronising their stream. */
int pl_line_check_overflow(PLLine* h);
int pl_line_debug_segments(PLLine* h, int frame, float* out, int cap);
int pl_line_debug_scaled(PLLine* h, int frame, uint8_t* out, int* sw, int* sh);
int pl_line_debug_sobel(PLLine* h, int frame, short* dx, short* dy);
int pl_line_debug_order(PLLine* h, int frame, unsigned* out, int cap);
/* which sort built the seed order of the LAST call: 1 the cluster kernel k_lsd_seed_order, 0 k_lsd_hist/scan/scatter */
int pl_line_debug_seed_path(PLLine* h);
/* fill every byte of the seed order and of its lengths with `byte` (tests: a later call must rewrite all it reports) */
int pl_line_debug_fill_order(PLLine* h, int byte);
/* Test-only: the library's own device build of the float libm restatements and of the 4x4 SVD, one thread per argument on
 * `stream`, all arrays DEVICE pointers of n entries.  fn 0: out0 = atan2f(a, b); fn 1: out0, out1 = sinf(a), cosf(a) (|a| < 120);
 * fn 2: out0 = logf(a) (positive normal a); b and out1 are read / written only where fn uses them.  pl_debug_svd4_dev: w [n][4]
 * and vt [n][4][4] of cv::SVD::compute(A [n][4][4] row-major CV_32F, MODIFY_A | FULL_UV). */
int pl_debug_float_math_dev(int fn, const float* a, const float* b, int n, float* out0, float* out1, void* stream);
int pl_debug_svd4_dev(const float* A, int n, float* w, float* vt, void* stream);
/* Test-only: LSD region growing's tables and alignment decisions, as a line handle's frames use them.
 * pl_line_debug_tables copies the handle's tables to host arrays (NULL = skip): gtab [1021 * 1021][4] floats {deg, cos, sin, 0}
 * and gtab_seed [1021 * 1021][2] {cos, sin} for the gradient (gx, gy) at (gx + 510) * 1021 + gy + 510, wtab [2 * 510^2 + 1]
 * doubles sqrt(i / 4).  pl_debug_lsd_align_dev (DEVICE arrays of n): out[i] bit 0 = the shortcut's "surely aligned", bit 1 its
 * "maybe aligned", bit 2 the exact test, bit 3 the generic isAligned, for the region sum (sumdx, sumdy) and the candidate of
 * gradient (gx, gy); bit 4 flags |gx| or |gy| > 510 (the decisions then use the clamped gradient).  pl_debug_lsd_fold_dev:
 * bit 0 the exact test, bit 1 the generic isAligned, for the region angle reg_deg and the candidate angle deg in degrees.
 * NULL stream = the handle's stream. */
int pl_line_debug_tables(PLLine* h, float* gtab, float* gtab_seed, double* wtab);
int pl_debug_lsd_align_dev(PLLine* h, int n, const float* sumdx, const float* sumdy, const int* gx, const int* gy, uint8_t* out,
                           void* stream);
int pl_debug_lsd_fold_dev(PLLine* h, int n, const float* reg_deg, const float* deg, uint8_t* out, void* stream);

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
/* PL_ERR_ARG when the matchers cannot take the extractors' capacities: a keypoint capacity over 6144 (at most
 * 6144 - 4 * orb_nlevels features), or a line capacity over pl_lsd_search_double_dev's shared-memory limit. */
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

/* measurement hooks (bench.py): CUDA-event timing of k_lsd_grow_ordered on its launching stream, its algorithmic bytes, and
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
 * erase (:2005-2043), le_erase_kf = the keyframe index the reference pairs with line observation i (its i/2 quirk).
 * PL_ERR_ARG for more than 7723 free keyframes (the dense reduced system, (6 n_free)^2 doubles, is indexed with an int). */
int pl_local_ba(const PLBAProblem* p, const int* stop_flag_dev, float* kf_Tcw_out, float* pt_Xw_out, double* ln_Xw_out,
                uint8_t* pe_erase, uint8_t* le_erase, int* le_erase_kf, int* iterations);

/* W local windows in one launch, on device pointers, asynchronous.  Window w is the PLBAProblem made of row w: counts
 * n_*[w] (device arrays [W]) and rows of capacity cap_* in [W][cap] layouts (kf_Tcw [W][cap_kf][16], kf_fixed [W][cap_kf],
 * kf_K [W][cap_kf][4], K_end [W][4], pt_Xw [W][cap_pt][3], ln_Xw [W][cap_ln][6], pe_kf / pe_pt / pe_inv_sigma2 [W][cap_pe],
 * pe_obs [W][cap_pe][2], le_kf / le_ln [W][cap_le], le_func [W][cap_le][3]); edge indices are relative to the window's own
 * rows.  Same meaning and units as PLBAProblem. */
typedef struct PLBAWindows {
  int W;
  int cap_kf, cap_pt, cap_ln, cap_pe, cap_le;
  const int* n_kf; const int* n_pt; const int* n_ln; const int* n_pe; const int* n_le;
  const float* kf_Tcw; const uint8_t* kf_fixed; const float* kf_K; const float* K_end;
  const float* pt_Xw; const double* ln_Xw;
  const int* pe_kf; const int* pe_pt; const float* pe_obs; const float* pe_inv_sigma2;
  const int* le_kf; const int* le_ln; const double* le_func;
} PLBAWindows;
/* Outputs of pl_local_ba_dev (device arrays, all required), in the layouts of the inputs: kf_Tcw [W][cap_kf][16],
 * pt_Xw [W][cap_pt][3], ln_Xw [W][cap_ln][6], pe_erase [W][cap_pe], le_erase / le_erase_kf [W][cap_le], iterations [W],
 * status [W].  Entries past a window's counts are never written.  status[w] = 0: window w ran; 1: one of its counts is
 * negative or over its capacity; 2: one of its edges names a keyframe or landmark outside its counts.  A window with a
 * nonzero status writes only status[w] and iterations[w] = 0; its other outputs keep what they held. */
typedef struct PLBAOut {
  float* kf_Tcw; float* pt_Xw; double* ln_Xw; uint8_t* pe_erase; uint8_t* le_erase; int* le_erase_kf;
  int* iterations; int* status;
} PLBAOut;
/* Device scratch of pl_local_ba_dev: per window, the dense reduced pose system of (6 cap_kf)^2 doubles, the edge Jacobians and
 * the two CSR indices.  0 for arguments pl_local_ba_dev refuses. */
size_t pl_local_ba_scratch_bytes(int W, int cap_kf, int cap_pt, int cap_ln, int cap_pe, int cap_le);
/* pl_local_ba on W windows, one CTA per window, enqueued on `stream` (NULL = the legacy default stream): kernels only, no
 * allocation, copy or synchronisation, so the call can be captured into a CUDA graph.  stop_flag_dev as in pl_local_ba, for
 * every window.  scratch: pl_local_ba_scratch_bytes(W, caps) bytes of device memory, 16-byte aligned; nothing past them is
 * written.  PL_ERR_ARG before anything is enqueued for a NULL windows / out / array / scratch (W > 0), W < 0, or a capacity
 * outside its limits: 1 <= cap_kf <= 7723 (the kernel indexes the (6 cap_kf)^2 reduced system with an int), cap_pt, cap_ln,
 * cap_pe, cap_le in 1 .. 2^24, and W * cap of every capacity within an int.  W = 0 enqueues nothing.  Counts and edge indices
 * are checked on the device (status).  Windows are independent: each one's results equal pl_local_ba's on its problem, up to
 * the last bits the fp64-atomic Schur sum leaves to chance. */
int pl_local_ba_dev(const PLBAWindows* windows, const int* stop_flag_dev, const PLBAOut* out, void* scratch, void* stream);

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
 * (the "fill(mvpMapPoints, NULL); search again with 2 * th" retry of Tracking.cc:1352-1357); NULL = every frame runs.  A frame
 * that does not run writes nothing: its cur_match row and nmatches[b] keep what they held, so the first pass's outputs can be
 * passed as both the gate and the outputs of the retry.  The point searches take cap at most 6144.  The line search's scratch
 * is pl_lsd_search_scratch_bytes(cap, B) bytes of device memory, and nothing past them is touched. */
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
/* Line extraction on raw frames: every later pl_line_extract* call reads each frame through this map (what
 * pl_undistort_remap would have stored) instead of taking the frames as already undistorted.  NULL unbinds it.  The map
 * must have the line handle's size (else PL_ERR_ARG) and the caller keeps it alive while it is bound.  Batches below 32
 * frames per SM are undistorted into a buffer of the handle first (W x H x max_batch bytes, made on first use). */
int pl_line_set_undistort(PLLine* h, const PLUndistort* und);
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
 * level_sigma2_2 = mvLevelSigma2.  matches12[i] = idx2 or -1 (vMatchedPairs = the pairs with idx2 >= 0); returns nmatches.
 * PL_ERR_ARG for a feature vector whose fv_start is not monotone or runs past n, or with an item outside 0 .. n - 1. */
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

/* ------------------------------------------------------------------ many Fuse searches in one launch (LocalMapping::SearchInNeighbors)
 * The search halves of pl_orb_fuse_search / pl_lsd_fuse_search for P problems at once, on device pointers, enqueued on `stream`
 * (NULL = the legacy default stream): kernels only, no allocation, copy or synchronisation, so the calls can be captured into a
 * CUDA graph.  The host-pointer functions above are their P = 1 case.
 *
 * Problem p searches the landmarks of entries offset[p] .. offset[p] + count[p] - 1 against keyframe kf[p] with radius factor
 * th[p], and writes the result of its j-th entry to best_idx / best_dist [out_offset[p] + j].  Entry e names landmark entry_lm[e]
 * and carries its own skip byte entry_skip[e] (skip = !pMP || isBad() || IsInKeyFrame(target): it depends on the target).
 * Problems may share a keyframe and an entry range; their output ranges must not overlap. */
typedef struct PLFuseProblems {
  int P;
  const int* kf; const float* th; const int* offset; const int* count; const int* out_offset;   /* [P] */
  int n_entries; const int* entry_lm; const uint8_t* entry_skip;                                /* [n_entries] */
  int n_out;                                                                                    /* length of the outputs */
} PLFuseProblems;
/* Point keyframes: rows of capacity cap, keys_un [n_kf][cap] (mvKeysUn), desc [n_kf][cap][32], n [n_kf]; per keyframe Tcw
 * [n_kf][16], Ow [n_kf][3], K [n_kf][4] (fx fy cx cy), bounds [n_kf][4]; the scale tables are shared by every keyframe. */
typedef struct PLFuseKeyframes {
  int n_kf, cap;
  const PLKeyPoint* keys_un; const uint8_t* desc; const int* n;
  const float* Tcw; const float* Ow; const float* K; const float* bounds;
  const float* scale_factors; const float* inv_level_sigma2; int nlevels; float log_scale_factor;
} PLFuseKeyframes;
/* Map points, as pl_orb_fuse_search takes them: pos / normal [n][3], raw min / max distance [n], desc [n][32]. */
typedef struct PLFusePoints {
  int n; const float* pos; const float* normal; const float* min_dist; const float* max_dist; const uint8_t* desc;
} PLFusePoints;
/* Line keyframes: keylines [n_kf][cap] (68-byte records), n [n_kf]; the keyframe's POINT descriptors pdesc [n_kf][cap_pdesc][32]
 * with n_pdesc [n_kf] rows (see pl_lsd_fuse_search); Tcw, Ow, K, bounds as PLFuseKeyframes; scale_line / log_scale_factor_line
 * shared. */
typedef struct PLFuseLineKeyframes {
  int n_kf, cap, cap_pdesc;
  const void* keylines; const int* n; const uint8_t* pdesc; const int* n_pdesc;
  const float* Tcw; const float* Ow; const float* K; const float* bounds;
  float scale_line, log_scale_factor_line;
} PLFuseLineKeyframes;
/* Map lines, as pl_lsd_fuse_search takes them: pos [n][6] (start, end), normal [n][3], raw min / max distance [n], desc [n][32]. */
typedef struct PLFuseLines {
  int n; const double* pos; const double* normal; const float* min_dist; const float* max_dist; const uint8_t* desc;
} PLFuseLines;
/* status[p] = 0: problem p ran; 1: kf[p], its entry range or its output range lies outside its table; 2: its keyframe's count
 * (n, or n_pdesc for lines) is negative or over the capacity; 3: one of its entries names a landmark outside the table.  A
 * problem with a nonzero status writes nothing but status[p].  Lines: stop_at[p] = the position j inside the problem of the first
 * entry that is not skipped and has an end point behind the camera (count[p] if none); entries from there on get -1 / 256.
 * stop_at is decided on the skip bytes given: if the caller's surgery at an earlier target has since made that entry skipped,
 * the reference steps over it, so the entries after it must be searched again (INTEGRATION.md, SearchInNeighbors).
 * PL_ERR_ARG before anything is enqueued for P < 0 or n_entries, n_out, landmark count < 0; and, when P > 0, for a NULL table,
 * array or output, n_kf < 1, nlevels < 1, cap outside 1 .. 6144 (points) or 1 .. 32768 (lines), cap_pdesc outside 1 .. 32768,
 * or n_kf * cap beyond an int.  P = 0 enqueues nothing.  Each problem equals pl_orb_fuse_search / pl_lsd_fuse_search on its
 * keyframe and the landmarks of its entries, bit for bit. */
int pl_orb_fuse_search_dev(const PLFuseKeyframes* kfs, const PLFusePoints* points, const PLFuseProblems* problems, int* best_idx,
                           int* best_dist, int* status, void* stream);
int pl_lsd_fuse_search_dev(const PLFuseLineKeyframes* kfs, const PLFuseLines* lines, const PLFuseProblems* problems, int* best_idx,
                           int* best_dist, int* stop_at, int* status, void* stream);

/* ------------------------------------------------------------------ many triangulation searches in one launch
 * (LocalMapping::CreateNewMapPoints and CreateNewMapLinesConstraint)
 * pl_orb_search_for_triangulation / pl_lsd_search_for_triangulation for P (KF1, KF2) problems at once, on device pointers, enqueued
 * on `stream` (NULL = the legacy default stream): kernels only, no allocation, copy or synchronisation, so the calls can be
 * captured into a CUDA graph.  The host-pointer functions above are their P = 1 case.
 *
 * Problem p searches keyframe kf1[p] against keyframe kf2[p] and writes match [out_offset[p] + i] for i < n[kf1[p]] (idx2 or -1),
 * nmatches[p] and status[p].  F12 [P][9] is row-major (LocalMapping::ComputeF12(KF1, KF2)); the line call ignores it (it may be
 * NULL).  Problems may share keyframes; their output ranges must not overlap. */
typedef struct PLTriProblems {
  int P;
  const int* kf1; const int* kf2; const float* F12; const int* out_offset;   /* [P], F12 [P][9] */
  int n_out;                                                                 /* length of the match output */
} PLTriProblems;
/* Point keyframes: rows of capacity cap, keys_un [n_kf][cap] (mvKeysUn), desc [n_kf][cap][32], has_mp [n_kf][cap]
 * (GetMapPoint(i) != NULL at the snapshot), n [n_kf]; mFeatVec as CSR per keyframe: fv_nodes [n_kf][cap_nodes] (ascending and
 * unique, as std::map keeps them), fv_start [n_kf][cap_nodes + 1], fv_items [n_kf][cap], nn [n_kf] nodes; the camera Tcw [n_kf][16]
 * (row-major; R2w and t2w of a KF2), Ow [n_kf][3] (GetCameraCenter() as stored; Cw of a KF1), K [n_kf][4] (fx fy cx cy of a KF2);
 * pl_orb_triangulate_dev reads Tcw, Ow and K of KF1 and of KF2;
 * scale_factors / level_sigma2 [nlevels] (mvScaleFactors, mvLevelSigma2) shared by every keyframe. */
typedef struct PLTriKeyframes {
  int n_kf, cap, cap_nodes;
  const PLKeyPoint* keys_un; const uint8_t* desc; const uint8_t* has_mp; const int* n;
  const unsigned* fv_nodes; const int* fv_start; const int* fv_items; const int* nn;
  const float* Tcw; const float* Ow; const float* K;
  const float* scale_factors; const float* level_sigma2; int nlevels;
} PLTriKeyframes;
/* Line keyframes: ldesc [n_kf][cap][32] (mLineDescriptors), has_ml [n_kf][cap] (GetMapLine(i) != NULL), n [n_kf]. */
typedef struct PLTriLineKeyframes {
  int n_kf, cap;
  const uint8_t* ldesc; const uint8_t* has_ml; const int* n;
} PLTriLineKeyframes;
/* status[p] = 0: problem p ran; 1: kf1[p] or kf2[p] lies outside the table, or its output range [out_offset[p], out_offset[p] +
 * n[kf1[p]]) lies outside n_out; 2: a keyframe's n or nn is negative or over its capacity, or its fv_start is not monotone, starts
 * below 0 or runs past n; 3: an fv_items entry of a keyframe lies outside 0 .. n - 1.  A problem with a nonzero status writes
 * nothing but status[p].
 * check_orientation = 1 keeps the rotation histogram per problem.  LocalMapping::CreateNewMapPoints uses 0, and only then are the
 * keypoints of KF1 independent of each other, so that a caller may search every neighbour against one snapshot of has_mp and
 * drop, at application, the pairs whose idx1 received a map point at an earlier neighbour (INTEGRATION.md, CreateNewMapPoints).
 * PL_ERR_ARG before anything is enqueued for a NULL problem list, P < 0 or n_out < 0; and, when P > 0, for a NULL table, array
 * or output (F12 may be NULL for lines), n_kf < 1, nlevels < 1, cap outside 1 .. 6144 (points) or beyond what pl_lsd_search_double_dev takes (lines: below
 * 32000 and inside the device's shared memory), cap_nodes < 1, or n_kf * cap (n_kf * (cap_nodes + 1)) beyond an int.  P = 0
 * enqueues nothing.  Each problem equals pl_orb_search_for_triangulation / pl_lsd_search_for_triangulation on its two keyframes,
 * bit for bit. */
int pl_orb_search_for_triangulation_dev(const PLTriKeyframes* kfs, const PLTriProblems* problems, int check_orientation,
                                        int* matches12, int* nmatches, int* status, void* stream);
int pl_lsd_search_for_triangulation_dev(const PLTriLineKeyframes* kfs, const PLTriProblems* problems, float th, float nnratio,
                                        int is_double, int* matched_pairs, int* nmatches, int* status, void* stream);

/* The triangulation of LocalMapping::CreateNewMapPoints (src/LocalMapping.cc:417-574, monocular) for the pairs that
 * pl_orb_search_for_triangulation_dev found, with the neighbour-order commit, on the same keyframe table and problem list, enqueued
 * on `stream`: kernels only, no allocation, copy or synchronisation, so the call can be captured into a CUDA graph together with
 * the search.  matches12 and search_status are the search's outputs, read on the device.  It reads keys_un, n, Tcw, Ow, K (of KF1
 * and KF2), scale_factors, level_sigma2 and nlevels of the table, never the descriptors, has_mp or the feature vector.
 * scale_factor is KF1's mfScaleFactor (ratioFactor = 1.5f * scale_factor); scale_factors[1] does not exist when nlevels == 1.
 * The caller guarantees 0 <= octave < nlevels for every keypoint of KF1 and KF2 in a pair (ORBextractor's keypoints satisfy it):
 * scale_factors and level_sigma2 are read at both keypoints' octaves unchecked, as the search reads them at KF2's.
 *
 * Per slot out_offset[p] + idx1, idx1 < n[kf1[p]]: code -1 no pair (matches12 = -1); 0 committed; 1 dropped at commit (the pair
 * passed the gates, but an earlier problem with the same kf1 committed or dropped a pair at the same idx1: the reference searched
 * that neighbour later, when idx1 already held a map point); 2 .. 8 the first gate that rejected it: 2 parallax (cosParallaxRays
 * not in (0, 0.9998)), 3 vt.row(3)[3] == 0, 4 behind camera 1, 5 behind camera 2, 6 reprojection in KF1, 7 reprojection in KF2
 * (5.991 sigma^2 at the keypoint's octave), 8 scale consistency (a zero distance, or the distance ratio off the octave ratio by
 * more than ratioFactor).  x3D [n_out][3] is the triangulated point (world) for codes 0 and 1, bit for bit the reference's.
 * Per problem: nnew[p] = the number of committed slots; status[p] = search_status[p] when that is nonzero, else 1: kf1[p] or
 * kf2[p] outside the table or the output range outside n_out, 2: n[kf1] or n[kf2] negative or over cap, 4: a matches12 entry of
 * the problem outside -1 .. n[kf2] - 1, or 0.  A problem with a nonzero status writes nothing but status[p].
 *
 * A caller applies the committed slots in problem order, then in ascending idx1: that is the reference's creation order when the
 * problems of a kf1 are its neighbours in the reference's order.  Two committed slots of one problem may share an idx2 (the search
 * never marks KF2's keypoints as taken); the reference creates both points, and KF2's slot ends up with the later one
 * (AddMapPoint overwrites it).  Problems with different kf1 are independent.
 * PL_ERR_ARG before anything is enqueued: the argument and capacity rules of pl_orb_search_for_triangulation_dev on kfs, problems
 * and (matches12, nnew, status) in the places of (matches12, nmatches, status), and a NULL search_status, or a NULL x3D or code
 * when n_out > 0.  P = 0 enqueues nothing. */
int pl_orb_triangulate_dev(const PLTriKeyframes* kfs, const PLTriProblems* problems, const int* matches12, const int* search_status,
                           float scale_factor, float* x3D, int8_t* code, int* nnew, int* status, void* stream);

/* The three-view triangulation of LocalMapping::CreateNewMapLinesConstraint (src/LocalMapping.cc:966-1439, monocular) for the
 * matches of a pl_lsd_search_for_triangulation_dev batch, with the commit, enqueued on `stream`: kernels only, no allocation, copy
 * or synchronisation, so the call can be captured into a CUDA graph together with the search.
 *
 * The geometry of the rows of the PLTriLineKeyframes table (same n_kf and cap): keylines [n_kf][cap] 68 B KeyLine records
 * (KeyFrame::mvKeyLines), line_func [n_kf][cap][3] (mvKeyLineFunctions), Tcw [n_kf][16] (row-major), Ow [n_kf][3]
 * (GetCameraCenter()), K [n_kf][4] (fx fy cx cy), and level_sigma2_line [nlevels] (mvLevelSigma2Line) shared by every keyframe.
 * The caller guarantees 0 <= octave < nlevels for every keyline a triple reads. */
typedef struct PLTriLineGeometry {
  int n_kf, cap;
  const void* keylines; const double* line_func;
  const float* Tcw; const float* Ow; const float* K;
  const float* level_sigma2_line; int nlevels;
} PLTriLineGeometry;
/* Most entries (vpNeighKFs) of one group; the commit keeps its taken state for kf_cur and each entry in shared memory. */
#define PL_TRI_LINE_MAX_ENTRIES 16
/* One group per current keyframe: kf_cur [G], entries entry_start[g] .. entry_start[g] + n_entries[g] - 1 of the entry list, and
 * out_offset [G].  Entry e (TotalvMatchedIndices[e]) names its search problem entry_problem[e] (a problem of the search batch with
 * kf1 = kf_cur), the POSITIONAL keyframe row entry_kf[e] (vpNeighKFs[e], which the reference pairs with entry e even when an
 * earlier neighbour failed the baseline test and the entry holds another neighbour's matches) and entry_median_depth[e]
 * (ComputeSceneMedianDepth(2) of vpNeighKFs[e], INTEGRATION.md).  n_out is the length of the slot outputs. */
typedef struct PLTriLineGroups {
  int G;
  const int* kf_cur; const int* entry_start; const int* n_entries; const int* out_offset;   /* [G] */
  int n_entry_list;
  const int* entry_problem; const int* entry_kf; const float* entry_median_depth;          /* [n_entry_list] */
  int n_out;
} PLTriLineGroups;
/* Group g with E entries and N = n[kf_cur[g]] keylines owns the slots out_offset[g] + pair(i, j) * N + ikl for the E (E - 1) / 2
 * entry pairs i < j in the reference's order (pair(i, j) = i (2E - i - 1) / 2 + j - i - 1) and ikl < N.  code [n_out] gets the
 * first reason in the reference's order: -1 no triple (idx1 or idx2 = -1, idx1 >= n[entry_kf[i]], idx2 >= n[entry_kf[j]], or an
 * entry whose nmatches is 0); 1 one of the three slots (kf_cur: ikl, entry_kf[i]: idx1, entry_kf[j]: idx2) holds a map line at
 * the snapshot has_ml; 2 one of them was taken by a line this call committed at an earlier slot; 3 the epipolar-plane test
 * (|Result| > 0.996); 4 a zero norm; 5 CosSita > 0.0087; 6 vt(3,3) == 0; 7 parallax (>= 0.99998); 8 an end point too close
 * (distance / median depth < 0.3); 9 too long (> 1); 10 behind a camera; 11, 12, 13 reprojection in view 1, 2, 3 (3.84 sigma^2 at
 * the keyline's octave); 14, 15, 16 overlap in view 1, 2, 3 (0.85); 0 committed.  line3D [n_out][6] (start, end; world) is
 * written for every slot whose triple passed all gates (code 0, and code 2 where the slots were taken); other slots keep theirs.
 * Per group: nnew[g] = the number of committed slots; status[g], the first that applies: 2 an entry count negative or over
 * PL_TRI_LINE_MAX_ENTRIES; 1 the entry range or an entry's problem index outside its table; the first nonzero search status of
 * the entries' problems (passed through); 1 kf_cur, an entry's keyframe row or its problem's kf1 / kf2 outside the table; 2 one of
 * their counts negative or over cap; 1 the group's output range outside n_out or a problem's match range outside the search's
 * n_out; 3 an entry's problem has kf1 != kf_cur; 4 a matches entry outside -1 .. n[kf2] - 1 of its problem's kf2; else 0.  A
 * group with a nonzero status writes nothing but status[g].
 * The commit applies a group's slots in slot order (pairs in order, ikl ascending within a pair): a passed slot commits iff none of
 * its three slots is taken, and takes them.  A caller creates the committed lines in slot order (INTEGRATION.md).  Groups are
 * independent; their output ranges must not overlap.
 * PL_ERR_ARG before anything is enqueued: the argument rules of pl_lsd_search_for_triangulation_dev on kfs and problems with
 * (matches, nmatches, search_status) in the places of (matched_pairs, nmatches, status); and a NULL group list, G < 0,
 * n_entry_list < 0 or n_out < 0; and, when G > 0, a NULL group or entry array, geometry, keylines, line_func, Tcw, Ow, K or
 * level_sigma2_line, nlevels < 1, geometry rows other than the table's, a NULL nnew or status, or a NULL code or line3D when
 * n_out > 0.  G = 0 enqueues nothing. */
int pl_lsd_triangulate_dev(const PLTriLineKeyframes* kfs, const PLTriLineGeometry* geom, const PLTriProblems* problems,
                           const int* matches, const int* nmatches, const int* search_status, const PLTriLineGroups* groups,
                           int8_t* code, float* line3D, int* nnew, int* status, void* stream);

/* ------------------------------------------------------------------ redundant keyframes (LocalMapping::KeyFrameCulling)
 * The loop of LocalMapping::KeyFrameCulling (src/LocalMapping.cc:1835-1899, monocular) for G current keyframes at once, on device
 * pointers, enqueued on `stream` (NULL = the legacy default stream): kernels only, no allocation, copy or synchronisation, so the
 * call can be captured into a CUDA graph.
 *
 * Keyframe rows of capacity cap, the layout of PLTriKeyframes.keys_un / n: keys_un [n_kf][cap] (mvKeysUn; only the octave is read),
 * n [n_kf], mp [n_kf][cap] (GetMapPointMatches(): a map-point index or -1 for NULL), origin [n_kf] (mnId == 0) and not_erase [n_kf]
 * (mbNotErase).  Every keyframe that observes a point held by a listed keyframe must be a row; the numbering of the rows is free. */
typedef struct PLCullKeyframes {
  int n_kf, cap;
  const PLKeyPoint* keys_un; const int* n; const int* mp; const uint8_t* origin; const uint8_t* not_erase;
} PLCullKeyframes;
/* Map points: bad [n_mp] (isBad()) and GetObservations() as CSR: point p's observations are (obs_kf[e], obs_idx[e]) for
 * obs_offset[p] <= e < obs_offset[p + 1], one per observing keyframe (monocular: Observations() is their number). */
typedef struct PLCullPoints {
  int n_mp, n_obs;
  const uint8_t* bad; const int* obs_offset /* [n_mp + 1] */; const int* obs_kf; const int* obs_idx;   /* [n_obs] */
} PLCullPoints;
/* Group g walks list[offset[g]] .. list[offset[g] + count[g] - 1] (keyframe rows, GetVectorCovisibleKeyFrames() of its current
 * keyframe, in order).  Groups are independent evaluations of the same snapshot; their list ranges must not overlap. */
typedef struct PLCullGroups {
  int G;
  const int* offset; const int* count;   /* [G] */
  int n_list; const int* list;           /* [n_list] */
} PLCullGroups;
/* Per list entry j: code[j] = -1 skipped (origin), 0 kept, 1 culled (nRedundantObservations > 0.9 * nMPs in double; its
 * observations are erased for the entries after it), 2 redundant but not_erase (SetBadFlag only sets mbToBeErased); n_mps[j],
 * n_redundant[j] = the reference's nMPs and nRedundantObservations (0 for a skipped entry).  An entry is judged on the state the
 * culls of the entries before it leave: a point p with obs observers of which culled(p) were culled earlier has Observations() =
 * obs - culled(p), those observers are gone, and it is bad when it was bad on input or when culled(p) >= 1 and obs - culled(p) <= 2
 * (MapPoint::EraseObservation).  A slot counts in nMPs when its point is not bad; it is redundant when the point's Observations()
 * > 3 and at least 3 other remaining observers see it at an octave <= the slot's octave + 1.  The caller calls SetBadFlag() on
 * the entries with codes 1 and 2 in list order, which reproduces the reference.
 * status[g], the first that applies: 1 the list range outside n_list or a list entry outside the table; 2 a listed keyframe's n
 * negative or over cap; 3 a keyframe listed twice; 4 a slot of a listed keyframe naming a point outside -1 .. n_mp - 1; 5 such a
 * point's obs_offset decreasing or outside 0 .. n_obs; 6 one of its observations naming a keyframe outside the table, an idx
 * outside 0 .. min(n, cap) - 1 of that keyframe, or a slot that does not hold the point; else 0.  A group with a nonzero status
 * writes nothing but status[g].
 * PL_ERR_ARG before anything is enqueued for a NULL groups, G < 0 or n_list < 0; and, when G > 0, for a NULL kfs, points, array or
 * output, n_mp or n_obs < 0, n_kf outside 1 .. 65536 (the culled set is one bit per row in shared memory), cap outside 1 .. 6144
 * or n_kf * cap beyond an int.  G = 0 enqueues nothing. */
int pl_keyframe_culling_dev(const PLCullKeyframes* kfs, const PLCullPoints* points, const PLCullGroups* groups, int8_t* code,
                            int* n_mps, int* n_redundant, int* status, void* stream);

/* ------------------------------------------------------------------ tracking a batch of frames against a fixed map
 * Tracking::TrackLocalMapWithLines (src/Tracking.cc:1491-1562) with SearchLocalPoints (:1751-1801) and SearchLocalLines
 * (:1803-1855), in localisation mode (mbOnlyTracking), for B frames at once; every intermediate stays on the device.
 *
 * The map (pl_map_create, uploaded once): per map point pos = MapPoint::GetWorldPos, normal = GetNormal, the RAW
 * mfMinDistance / mfMaxDistance (see pl_frame_is_in_frustum_points), desc = GetDescriptor; per map line pos = mWorldPos
 * (start, end), normal = GetNormal, the raw distances and desc = GetDescriptor.  Host pointers; the handle owns device copies. */
typedef struct PLMapDesc {
  int n_points;
  const float* pt_pos /*[n][3]*/; const float* pt_normal /*[n][3]*/; const float* pt_min_dist; const float* pt_max_dist;
  const uint8_t* pt_desc /*[n][32]*/;
  int n_lines;
  const double* ln_pos /*[n][6]*/; const double* ln_normal /*[n][3]*/; const float* ln_min_dist; const float* ln_max_dist;
  const uint8_t* ln_desc /*[n][32]*/;
} PLMapDesc;
typedef struct PLMap PLMap;
int pl_map_create(const PLMapDesc* desc, PLMap** out);
void pl_map_destroy(PLMap* m);
/* Sticky flag of the track calls since the last check: PL_ERR_ARG if a local-list entry or a pre-assigned match named an index
 * outside the map (such an entry is treated as absent), else PL_OK; clears the flag.  Synchronises the device.  The host entry
 * point checks it itself; callers of the _dev entry points call it after synchronising their stream. */
int pl_map_check_indices(PLMap* m);

/* The frames ([B][cap] device arrays in the front end's layouts; host arrays with B = 1 for pl_track_local_map):
 *   keys_un = mvKeysUn, desc = mDescriptors, n = N; keylines = mvKeylinesUn (68 B records), line_func = mvKeyLineFunctions,
 *   line_desc = mLdesc, nl = NL; bounds = {mnMinX, mnMinY, mnMaxX, mnMaxY}, one for the batch (the search grid's bounds);
 *   scale_factors / inv_level_sigma2 = mvScaleFactors / mvInvLevelSigma2 ([nlevels]), log_scale_factor = mfLogScaleFactor;
 *   Tcw0 [B][16] = the pose guess (mTcw, row-major), K [B][4] = {fx, fy, cx, cy} of each frame;
 *   point_map_in [B][cap_points] / line_map_in [B][cap_lines] = the matches the frame already holds (mvpMapPoints / mvpMapLines
 *   from TrackWithMotionModel, TrackReferenceKeyFrame or Relocalization) as map indices, -1 for none; NULL = no match held. */
typedef struct PLTrackFrames {
  int B;
  const PLKeyPoint* keys_un; const uint8_t* desc; const int* n; int cap_points;
  const void* keylines; const double* line_func; const uint8_t* line_desc; const int* nl; int cap_lines;
  const float* bounds; const float* scale_factors; const float* inv_level_sigma2; int nlevels; float log_scale_factor;
  const float* Tcw0; const float* K;
  const int* point_map_in; const int* line_map_in;
} PLTrackFrames;
/* The local maps (mvpLocalMapPoints / mvpLocalMapLines, built by the caller's UpdateLocalMap): frame b's list is
 * pt_index[pt_offset[b] .. pt_offset[b] + pt_count[b]) of map-point indices, in the reference's order; frames may share or
 * overlap their ranges.  Offsets, counts and frames_since_reloc are HOST arrays [B] (read during the call); the index arrays
 * (n_pt_index / n_ln_index entries) are on the device (host for pl_track_local_map).  PL_ERR_ARG before anything is enqueued: a
 * count over cap_local_points / cap_local_lines or negative, a negative offset, or a range past the end of its index array.  frames_since_reloc[b] = mCurrentFrame.mnId - mnLastRelocFrameId: th = 5 below 2, else 1
 * (:1793-1798, :1850-1853); max_frames = mMaxFrames: frame b needs 50 inliers while frames_since_reloc[b] < max_frames, else 30
 * (:1555-1561). */
typedef struct PLTrackLocal {
  const int* pt_offset; const int* pt_count; const int* pt_index; int n_pt_index; int cap_local_points;
  const int* ln_offset; const int* ln_count; const int* ln_index; int n_ln_index; int cap_local_lines;
  const int* frames_since_reloc; int max_frames;
} PLTrackLocal;
/* Results (device arrays, host for pl_track_local_map).  Required: Tcw [B][16] = the optimised pose; point_map [B][cap_points] /
 * line_map [B][cap_lines] = mvpMapPoints / mvpMapLines after the searches (map index or -1); point_outlier / line_outlier =
 * mvbOutlier / mvbLineOutlier (0 for features without a match); inliers [B][2] = {mnMatchesInliers, mnLineMatchesInliers};
 * ok [B] = the return value.
 * Optional (NULL = kept in the scratch): the isInFrustum outputs per local-list entry, [B][cap_local_*] (pt_proj [.][2],
 * ln_proj [.][4]; in_view = 0 for entries the frame already holds, :1776-1777), the raw search results pt_match [B][cap_points] /
 * ln_match [B][cap_lines] (local-list position, -1 none, -2 held before the search), and the PoseOptimization problem exactly as
 * pl_pose_optimization_dev reads it ([B][cap_points] / [B][cap_lines] layouts, counts [B]). */
typedef struct PLTrackOut {
  float* Tcw; int* point_map; uint8_t* point_outlier; int* line_map; uint8_t* line_outlier; int* inliers; int* ok;
  uint8_t* pt_in_view; float* pt_proj; int* pt_level; float* pt_view_cos;
  uint8_t* ln_in_view; float* ln_proj; int* ln_level; float* ln_view_cos;
  int* pt_match; int* ln_match;
  int* prob_n_points; float* prob_pt_obs; float* prob_pt_inv_sigma2; float* prob_pt_Xw;
  int* prob_n_lines; double* prob_line_func; double* prob_line_Xw;
} PLTrackOut;
/* Per frame b, in the reference's order: Ow of Frame::UpdatePoseMatrices (Frame.cc:552-558); the local-map entries the frame
 * already holds are skipped (mnLastFrameSeen == mnId, :1754-1779), the others go through isInFrustum(., 0.5); then
 * ORBmatcher(0.8).SearchByProjection(F, mvpLocalMapPoints, th) (ORBmatcher.cc:56-152) and LSDmatcher().SearchByProjection(F,
 * mvpLocalMapLines, th) (LSDmatcher.cpp:221-338, nnratio 0.7), with the features that hold a match pre-assigned; the
 * PoseOptimization problem in feature order, points then lines (Optimizer.cc:640-841: mvKeysUn[i].pt, mvInvLevelSigma2[octave],
 * GetWorldPos; mvKeyLineFunctions[i], mWorldPos), solved by pl_pose_optimization_dev mode 0; then the inlier counts and the
 * return value (:1504-1561, mbOnlyTracking branch).  A frame with fewer than 3 correspondences keeps its pose.
 * The caller applies the map statistics the reference updates on the way: IncreaseVisible for every held match and every local
 * entry with pt_in_view / ln_in_view set, IncreaseFound for every match that is not an outlier.
 * Scratch: pl_track_local_map_scratch_bytes(B, caps) bytes of device memory (16-byte aligned).  Asynchronous on `stream`
 * (NULL = the map's stream); the host arrays of PLTrackLocal are read before the call returns. */
size_t pl_track_local_map_scratch_bytes(int B, int cap_points, int cap_lines, int cap_local_points, int cap_local_lines);
int pl_track_local_map_dev(PLMap* map, const PLTrackFrames* frames, const PLTrackLocal* local, const PLTrackOut* out, void* scratch,
                           void* stream);
/* The same for ONE frame on host pointers (frames->B must be 1; caps = the counts, or larger); synchronous.  Returns ok (0 / 1)
 * or an error. */
int pl_track_local_map(PLMap* map, const PLTrackFrames* frames, const PLTrackLocal* local, const PLTrackOut* out);
/* The same step after pl_track_motion_model_dev: point_seen [B][cap_points] / line_seen [B][cap_lines] (device, may be NULL) are
 * the motion model's outputs of the same names, the map entries it discarded as outliers (-1 none).  Such an entry is skipped by
 * the frustum test exactly like a held match (in_view = 0: the reference stamped it mnLastFrameSeen = mnId, :1384-1390, :1778,
 * :1833) but is not pre-assigned in the search.  With both NULL this is pl_track_local_map_dev, bit for bit. */
int pl_track_local_map_seen_dev(PLMap* map, const PLTrackFrames* frames, const int* point_seen, const int* line_seen,
                                const PLTrackLocal* local, const PLTrackOut* out, void* scratch, void* stream);
/* The step on the features of the front end's LAST step (pl_frontend_run / run_dev / submit): frames 0 .. B-1 of that step
 * (PL_ERR_ARG if B exceeds that step's batch or no step has run), with the
 * handle's bounds and ORB tables; Tcw0 / K / point_map_in / line_map_in are device arrays ([B][capK] / [B][capL] layouts of
 * pl_frontend_capacities).  Asynchronous on `stream` (NULL = the handle's stream). */
int pl_frontend_track_local_map_dev(PLFrontend* h, PLMap* map, int B, const float* Tcw0, const float* K, const int* point_map_in,
                                    const int* line_map_in, const PLTrackLocal* local, const PLTrackOut* out, void* scratch,
                                    void* stream);

/* ------------------------------------------------------------------ the constant-velocity motion model against a fixed map
 * Tracking::TrackWithMotionModel (src/Tracking.cc:1316-1431), monocular, in localisation mode, for B independent frames.
 *
 * The last frames ([B][cap] device arrays, host with B = 1 for pl_track_motion_model), with the caps of the current frames:
 *   keys_un = mLastFrame.mvKeysUn (octave and angle are read), n = N; keylines = mvKeylinesUn (lineLength is read), nl = NL;
 *   point_map / point_outlier = mvpMapPoints (map index, -1 none) / mvbOutlier; line_map / line_outlier likewise for lines;
 *   Tcw [B][16] = mLastFrame.mTcw after the caller's UpdateLastFrame (Tlr * pRef->GetPose(), :1242-1245); velocity [B][16] =
 *   mVelocity.  A -1 or outlier entry is skipped; a non-negative index outside the map sets the map's index flag and is skipped. */
typedef struct PLTrackLast {
  const PLKeyPoint* keys_un; const int* n; const void* keylines; const int* nl;
  const int* point_map; const uint8_t* point_outlier; const int* line_map; const uint8_t* line_outlier;
  const float* Tcw; const float* velocity;
} PLTrackLast;
/* Results (device arrays, host for pl_track_motion_model).  Always written: Tcw [B][16]; point_map [B][cap_points] / line_map
 * [B][cap_lines] = mvpMapPoints / mvpMapLines (map index or -1) after the discard; point_seen / line_seen (same layouts) = the map
 * index of a match discarded as an outlier (mnLastFrameSeen = mnId, mbTrackInView = false; :1384-1390, :1404-1409), else -1 - pass
 * them to pl_track_local_map_seen_dev; nmatches [B][2] = {nmatches, lmatches} after the discard; ok [B] = the return value
 * (nmatches > 20); vo [B] (in / out) = mbVO = nmatchesMap < 10, written only by frames that reach the pose optimisation.  A fixed
 * map's entries all have Observations() > 0, so nmatchesMap counts every match left.  There are no outlier outputs: after the
 * discard every mvbOutlier / mvbLineOutlier is false, and a frame that returned early still has a new Frame's all-false flags.
 * Optional (NULL = kept in the scratch): guess [B][16] = mVelocity * mLastFrame.mTcw; pt_match [B][cap_points] = the search at
 * th = 15 and pt_match_retry = the search at 30 (last-frame keypoint index or -1; written only for frames with retried [B] = 1);
 * ln_match [B][cap_lines] (last-frame line index or -1); the line candidates per LAST-frame line, ln_in_view / ln_proj [.][4] /
 * ln_level / ln_view_cos [B][cap_lines] (isInFrustum at the guess; 0 for skipped lines); and the PoseOptimization problem exactly as
 * pl_pose_optimization_dev reads it (empty for a frame that returned early). */
typedef struct PLTrackMotionOut {
  float* Tcw; int* point_map; int* line_map; int* point_seen; int* line_seen; int* nmatches; int* ok; int* vo;
  float* guess; int* pt_match; int* pt_match_retry; uint8_t* retried; int* ln_match;
  uint8_t* ln_in_view; float* ln_proj; int* ln_level; float* ln_view_cos;
  int* prob_n_points; float* prob_pt_obs; float* prob_pt_inv_sigma2; float* prob_pt_Xw;
  int* prob_n_lines; double* prob_line_func; double* prob_line_Xw;
} PLTrackMotionOut;
/* Per frame b, in the reference's order: the guess mVelocity * mLastFrame.mTcw (cv::Mat's fp32 4x4 product, :1332); ORBmatcher(0.9,
 * true).SearchByProjection(Current, Last, 15, mono) (ORBmatcher.cc:1441-1585) and LSDmatcher().SearchByProjection(Current, Last, 15)
 * (LSDmatcher.cpp:95-190, candidates isInFrustum(pML, 0.5) at the guess with frame b's K); the point search again at 30 if it found
 * under 20 (:1354-1358; lines are not searched again); nmatches < 20 && lmatches < 5: return false with the guess and the search's
 * matches (:1360-1361); PoseOptimization (mode 0, from the guess); the outliers discarded (:1376-1419), mbVO and the return value.
 * frames: PLTrackFrames with Tcw0, point_map_in and line_map_in NULL (PL_ERR_ARG otherwise: the guess is computed and the matches
 * start empty).  PL_ERR_ARG before anything is enqueued for a NULL required pointer, cap_points outside 1..6144 or cap_lines outside
 * 1..32768.  The caller keeps the map statistics and the LOST / no-velocity / mbVO branches (Relocalization, TrackReferenceKeyFrame).
 * Scratch: pl_track_motion_model_scratch_bytes(B, caps) bytes of device memory (16-byte aligned).  Asynchronous on `stream` (NULL =
 * the map's stream); call pl_map_check_indices after synchronising. */
size_t pl_track_motion_model_scratch_bytes(int B, int cap_points, int cap_lines);
int pl_track_motion_model_dev(PLMap* map, const PLTrackFrames* frames, const PLTrackLast* last, const PLTrackMotionOut* out,
                              void* scratch, void* stream);
/* The same for ONE frame on host pointers (B = 1; the counts of both frames within the caps); synchronous.  Returns ok (0 / 1) or
 * an error (PL_ERR_ARG also when the index flag was set). */
int pl_track_motion_model(PLMap* map, const PLTrackFrames* frames, const PLTrackLast* last, const PLTrackMotionOut* out);
/* mVelocity = mCurrentFrame.mTcw * LastTwc (Tracking.cc:492-501), LastTwc = [Rcw^T | Ow] of Tcw_last (Ow as Frame::UpdatePoseMatrices
 * computes it), with the guess's fp32 4x4 product; velocity[b] is written only where ok[b].  Device arrays [B][16], ok [B]. */
int pl_track_velocity_dev(int B, const float* Tcw, const float* Tcw_last, const int* ok, float* velocity, void* stream);

/* ------------------------------------------------------------------ the local map from the keyframe graph
 * Tracking::UpdateLocalMap (src/Tracking.cc:1899-2081) for B frames on the device, so that a localisation-mode frame in state OK
 * runs from UpdateLastFrame to the stored relative pose with no host synchronisation.
 *
 * The keyframe graph of the fixed map (pl_map_set_keyframes, host arrays; the handle keeps device copies, a second call replaces
 * the graph).  NUMBERING: keyframes are 0 .. n_kf-1 in ascending KeyFrame* address, the order in which map<KeyFrame*,int> and
 * set<KeyFrame*> iterate (the reference's keyframeCounter and mspChildrens); numbering by mnId gives other lists wherever the
 * allocator did not hand out increasing addresses.  Per keyframe: Tcw [16] = GetPose(), Twc [16] = GetPoseInverse() (both as
 * stored, row-major), bad (NULL = none bad) = isBad(), parent = GetParent() (-1 none).  CSR rows (offsets [n_kf + 1]):
 * pt_slot = GetMapPointMatches() in feature order (map-point index or -1, also for a bad point), ln_slot = GetMapLineMatches(),
 * cov = mvpOrderedConnectedKeyFrames as stored (the first 10 are read), child = mspChildrens (any order; sorted at upload).  Per
 * map point (offsets [n_points + 1]): obs = the keyframes of GetObservations().
 * Limits, from the kernel's shared memory (4 B per keyframe and 1 bit per keyframe, 1 bit per map point or line): n_kf 1 ..
 * 16384 and the map's n_points, n_lines up to 2^20.  PL_ERR_ARG for a graph over them, an index out of range, or CSR offsets that
 * do not start at 0 or are not monotone; the previous graph is then kept. */
typedef struct PLKeyFrameGraphDesc {
  int n_kf;
  const float* Tcw /*[n_kf][16]*/; const float* Twc /*[n_kf][16]*/; const uint8_t* bad /*[n_kf] or NULL*/; const int* parent;
  const int* pt_slot_offset; const int* pt_slot;
  const int* ln_slot_offset; const int* ln_slot;
  const int* cov_offset; const int* cov;
  const int* child_offset; const int* child;
  const int* obs_offset /*[n_points + 1]*/; const int* obs;
} PLKeyFrameGraphDesc;
int pl_map_set_keyframes(PLMap* m, const PLKeyFrameGraphDesc* graph);
/* Sticky flag of pl_track_update_local_map_dev since the last check: PL_ERR_ARG if a list outgrew its capacity (the counts
 * still hold the true sizes; entries past a capacity were not written), else PL_OK; clears the flag.  Synchronises the device. */
int pl_map_check_capacity(PLMap* m);

/* The local map of B frames (device arrays):
 *   kf [B][cap_kf], n_kf [B] = mvpLocalKeyFrames and ref_kf [B] = mpReferenceKF (keyframe index): IN / OUT, since a frame whose
 *   matches vote for no keyframe keeps both (:1995-1996);
 *   pt_index [B][cap_local_points], pt_count [B] = mvpLocalMapPoints (map-point indices); ln_index / ln_count likewise for lines. */
typedef struct PLLocalMap {
  int* kf; int* n_kf; int cap_kf; int* ref_kf;
  int* pt_index; int* pt_count; int cap_local_points;
  int* ln_index; int* ln_count; int cap_local_lines;
} PLLocalMap;
/* UpdateLocalKeyFrames, UpdateLocalPoints, UpdateLocalLines per frame b on point_map [B][cap_points] (mvpMapPoints as map indices,
 * -1 none; every entry is read, as the motion model writes them): each matched point votes once per keyframe of its observations
 * (lines do not vote); the good voters enter the list in index order and ref_kf = the first strict maximum among them; then, for
 * the original voters only while the list holds at most 80, the first good covisible (of the first 10) not yet in, the first
 * good child not yet in, and the parent if not yet in (not checked for isBad; adding it ends the expansion); no vote at all
 * leaves kf, n_kf and ref_kf as passed.  The points and lines are the first occurrences over the list in list order, then slot
 * order.  A count holds the true size; entries past a capacity are not written and set the flag of pl_map_check_capacity.
 * Gate (device, each may be NULL): frame b runs only if ok[b] && !vo[b] (Tracking.cc:476); a frame that does not run keeps its
 * kf / n_kf / ref_kf and gets pt_count = ln_count = 0.  A point_map entry or stale kf entry outside the map sets the index flag
 * and is skipped.  Needs no scratch; deterministic (integer votes, results independent of the order of atomics).  Asynchronous
 * on `stream` (NULL = the map's stream). */
int pl_track_update_local_map_dev(PLMap* map, int B, const int* point_map, int cap_points, const int* ok, const int* vo,
                                  const PLLocalMap* local, void* stream);
/* pl_track_local_map_seen_dev on the device lists of pl_track_update_local_map_dev: frame b's list is pt_index[b][0 .. pt_count[b])
 * (counts clamped to the capacities), frames_since_reloc [B] is a device array, and the same optional ok / vo gate applies: a
 * frame gated off passes through with Tcw = Tcw0, its held matches as point_map / line_map, outlier flags 0, inliers 0 and
 * ok = ok[b] (1 if ok is NULL); out->ok may be the ok array itself.  Frames that run compute exactly what
 * pl_track_local_map_seen_dev computes on the same lists.  B * cap_local_points and B * cap_local_lines must fit an int.
 * Scratch: pl_track_local_map_lists_scratch_bytes(B, caps) bytes.  Enqueues kernels only. */
size_t pl_track_local_map_lists_scratch_bytes(int B, int cap_points, int cap_lines, int cap_local_points, int cap_local_lines);
int pl_track_local_map_lists_dev(PLMap* map, const PLTrackFrames* frames, const int* point_seen, const int* line_seen,
                                 const PLLocalMap* local, const int* frames_since_reloc, int max_frames, const int* ok, const int* vo,
                                 const PLTrackOut* out, void* scratch, void* stream);
/* The reference-keyframe bookkeeping with cv::Mat's fp32 4x4 product (device arrays [B][16], ref_kf [B]):
 *   relative pose  Tcr = Tcw * Twc[ref_kf]       (mlRelativeFramePoses, Tracking.cc:582)
 *   last pose      Tcw_last = Tcr * Tcw[ref_kf]   (the monocular UpdateLastFrame, :1242-1245)
 * A ref_kf outside the graph sets the index flag and leaves that frame's output unwritten.
 * The OK-state frame is then, on one stream: last pose -> pl_track_motion_model_dev -> pl_track_update_local_map_dev (gated by its
 * ok / vo) -> pl_track_local_map_lists_dev (same gate) -> pl_track_velocity_dev -> relative pose. */
int pl_track_relative_pose_dev(PLMap* map, int B, const float* Tcw, const int* ref_kf, float* Tcr, void* stream);
int pl_track_last_pose_dev(PLMap* map, int B, const float* Tcr, const int* ref_kf, float* Tcw_last, void* stream);

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
