// TOOL — builds tests/golden/refcalls/fuse_protocol.npz with tools/gen_fuse_protocol.py; not part of the library or the tests.
//
// The first loop of LocalMapping::SearchInNeighbors (src/LocalMapping.cc:1535-1546) run by the reference's own code: one point list,
// ORBmatcher::Fuse(pKFi, vpMapPointMatches) for each target in order (src/ORBmatcher.cc:914-1065), with the real map surgery of
// src/MapPoint.cc (AddObservation, Replace, ComputeDistinctiveDescriptors).  Compiled against the mock KeyFrame / Map of
// oracle/shim_slam and the helpers of oracle/ref_match_wrap.cpp, the way oracle/Makefile builds libref_match.so.
#include "ref_match_wrap.cpp"

// Keyframe k holds rows kf_start[k] .. kf_start[k + 1] - 1 of keys / desc, and its camera in row k of Tcw [16], Ow [3], K [4],
// bounds [4].  Map point m starts with the observations (obs_kf[e], obs_idx[e]) of the entries e with obs_mp[e] == m, added in
// entry order; the keyframe's slot then holds the point.  list: the point list (vpMapPointMatches), targets: the keyframes fused
// into, in order.  Outputs: slots [kf_start[n_kf]] = point held by each keyframe slot (-1 none), bad [n_mp], out_desc [n_mp][32]
// (GetDescriptor), nfused [n_targets] (Fuse's return values).
extern "C" void ref_fuse_protocol(int n_kf, const int* kf_start, const void* keys, const uint8_t* desc, const float* Tcw, const float* Ow,
                                  const float* K, const float* bounds, const float* scaleFactors, const float* invLevelSigma2,
                                  float logScaleFactor, int nlevels, int n_mp, const float* pos, const float* normal, const float* minDist,
                                  const float* maxDist, const uint8_t* mp_desc, int n_obs, const int* obs_mp, const int* obs_kf,
                                  const int* obs_idx, int n_list, const int* list, int n_targets, const int* targets, float th, int* slots,
                                  uint8_t* bad, uint8_t* out_desc, int* nfused) {
  std::vector<KeyFrame> kfs((size_t)n_kf);     // one array: address order (std::map<KeyFrame*, size_t>) is index order
  for (int k = 0; k < n_kf; k++) {
    KeyFrame& kf = kfs[k];
    const int n = kf_start[k + 1] - kf_start[k];
    set_view(kf, (const cv::KeyPoint*)keys + kf_start[k], desc + 32 * (size_t)kf_start[k], n, bounds + 4 * k, scaleFactors, nlevels);
    set_K(kf, K + 4 * k);
    kf.mvInvLevelSigma2.assign(invLevelSigma2, invLevelSigma2 + nlevels);
    kf.mfLogScaleFactor = logScaleFactor;
    kf.Tcw = pose44(Tcw + 16 * k);
    kf.Ow = vec3(Ow + 3 * k);
    kf.mnId = (unsigned long)k;
    kf.mvpMapPoints.assign((size_t)n, nullptr);
  }
  World W;
  std::vector<MP*> pts((size_t)n_mp);
  std::map<MapPoint*, int> index;
  for (int m = 0; m < n_mp; m++) {
    pts[m] = W.point(pos + 3 * m, mp_desc + 32 * m, 0);
    pts[m]->set_normal(normal + 3 * m);
    pts[m]->set_dist(minDist[m], maxDist[m]);
    index[pts[m]] = m;
  }
  for (int e = 0; e < n_obs; e++) {
    MP* p = pts[obs_mp[e]];
    p->AddObservation(&kfs[obs_kf[e]], (size_t)obs_idx[e]);
    kfs[obs_kf[e]].mvpMapPoints[obs_idx[e]] = p;
  }
  std::vector<MapPoint*> vpMapPointMatches((size_t)n_list);
  for (int i = 0; i < n_list; i++) vpMapPointMatches[i] = list[i] >= 0 ? pts[list[i]] : nullptr;
  ORBmatcher matcher;
  for (int t = 0; t < n_targets; t++) nfused[t] = matcher.Fuse(&kfs[targets[t]], vpMapPointMatches, th);
  for (int k = 0; k < n_kf; k++)
    for (int i = kf_start[k]; i < kf_start[k + 1]; i++) {
      MapPoint* p = kfs[k].mvpMapPoints[i - kf_start[k]];
      slots[i] = p ? index[p] : -1;
    }
  for (int m = 0; m < n_mp; m++) {
    bad[m] = pts[m]->isBad() ? 1 : 0;
    memcpy(out_desc + 32 * (size_t)m, pts[m]->GetDescriptor().ptr(0), 32);
  }
}
