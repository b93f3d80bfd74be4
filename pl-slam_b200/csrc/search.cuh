// Launchers of the batched projection searches (match.cu) with two inputs the public entry points leave NULL:
//   th_frame  [B]       th of each frame (NULL: the scalar th for every frame)
//   desc_row  [B][cap]  row of the descriptor array that entry (b, i) compares with (NULL: row b * cap + i)
// pl_track_local_map_dev (track.cu) uses them to search every frame with its own th against the map's descriptors, read
// through the frame's local-map list instead of a [B][cap_local] gather.  The last-frame search takes last_row the same way
// (position and descriptor of last-frame keypoint (b, i) from row last_row[b][i] of the map's arrays): pl_track_motion_model_dev
// passes the last frame's matches there.
#pragma once
#include "common.cuh"

namespace pl {
// Largest keypoint capacity of the windowed point searches: their grid's 16-bit items and its `fill` area (one rotation bin byte
// per query) hold at most this many keypoints per frame.
constexpr int kMatchMaxKeys = 6144;
// PL_OK if k_search_double's shared memory for line capacities cap1 and cap2 fits the device's opt-in limit per block beside the
// kernel's static shared memory, else PL_ERR_ARG with a message naming the largest equal capacity that fits.
int search_double_fits(int cap1, int cap2);
// The argument and capacity rules of pl_orb_search_for_triangulation_dev (plslam_b200.h), which pl_orb_triangulate_dev applies to
// the same tables: PL_OK or PL_ERR_ARG, nothing enqueued.  `match` is the per-slot array of n_out entries, nmatches / status the
// per-problem outputs.  P = 0 passes without looking at the keyframe table.
int orb_tri_args_ok(const PLTriKeyframes* kfs, const PLTriProblems* problems, const void* match, const void* nmatches,
                    const void* status);
// The same for pl_lsd_search_for_triangulation_dev, which pl_lsd_triangulate_dev applies to its table and problems;
// lsd_tri_table_ok is its part on the keyframe table alone.
int lsd_tri_table_ok(const PLTriLineKeyframes* kfs);
int lsd_tri_args_ok(const PLTriLineKeyframes* kfs, const PLTriProblems* problems, const void* match, const void* nmatches,
                    const void* status);
int search_by_projection_last_launch(const PLKeyPoint* keys_cur, const uint8_t* desc_cur, const int* n_cur, int cap, int B,
                                     const float* bounds, const float* Tcw, const float* K, const float* scale_factors, int nlevels,
                                     const int* n_last, int cap_last, const uint8_t* last_valid, const float* last_pos,
                                     const uint8_t* last_desc, const int* last_row, const int* last_octave, const float* last_angle,
                                     float th, int check_orientation, const uint8_t* cur_preassigned, const int* gate_nmatches,
                                     int gate_min, int* cur_match, int* nmatches, void* stream);
int search_by_projection_points_launch(const PLKeyPoint* keys, const uint8_t* desc, const int* n, int cap, int B,
                                       const float* bounds, const float* scale_factors, const int* n_mp, int cap_mp,
                                       const uint8_t* in_view, const float* proj, const int* level, const float* view_cos,
                                       const uint8_t* mp_desc, float th, const float* th_frame, const int* desc_row, float nnratio,
                                       const uint8_t* preassigned, int* match, int* nmatches, void* stream);
int lsd_search_by_projection_launch(int variant, const void* keylines, const double* linefunc, const uint8_t* desc, const int* n,
                                    int cap, int B, const float* bounds, const int* n_q, int cap_q, const uint8_t* q_valid,
                                    const float* q_proj, const uint8_t* q_desc, const float* q_length_or_view_cos, float th,
                                    const float* th_frame, const int* q_desc_row, float nnratio, const uint8_t* preassigned, int* match,
                                    int* nmatches, void* scratch, void* stream);
}  // namespace pl
