// TOOL — builds tests/golden/refcalls/keyframe_culling.npz with tools/gen_keyframe_culling.py; not part of the library or the tests.
//
// LocalMapping::KeyFrameCulling (src/LocalMapping.cc:1835-1899, monocular) on one list of keyframes, with every map-point call made
// by the reference's own src/MapPoint.cc: isBad, Observations, GetObservations, AddObservation, EraseObservation and the SetBadFlag
// it cascades into, which clears the mock keyframes' slots (EraseMapPointMatch).  LocalMapping.cc and KeyFrame.cc cannot be
// compiled here, so two pieces are restated from them: the loop, and the part of KeyFrame::SetBadFlag it depends on
// (src/KeyFrame.cc:494-508: mnId == 0 returns, mbNotErase only sets mbToBeErased, otherwise EraseObservation on every slot's point).
// Compiled against the mock KeyFrame / Map of oracle/shim_slam and the helpers of oracle/ref_match_wrap.cpp, the way
// tools/fuse_protocol_ref.cpp is.
#include "ref_match_wrap.cpp"

namespace {
struct CullPoint : MP {       // a map point that can start bad (isBad() on input)
  using MP::MP;
  void set_bad() { mbBad = true; }
};

// KeyFrame::SetBadFlag (src/KeyFrame.cc:490-508) up to the connection and spanning-tree repair, which the loop never reads
int set_bad_flag(KeyFrame* pKF, std::vector<char>& not_erase, std::vector<char>& to_be_erased, int row) {
  if (pKF->mnId == 0) return 0;
  if (not_erase[row]) {
    to_be_erased[row] = 1;
    return 2;
  }
  for (size_t i = 0; i < pKF->mvpMapPoints.size(); i++)
    if (pKF->mvpMapPoints[i]) pKF->mvpMapPoints[i]->EraseObservation(pKF);
  pKF->mbBad = true;
  return 1;
}
}  // namespace

// Keyframe rows [n_kf][cap] (octave of mvKeysUn, mp = map-point index or -1), n [n_kf], origin [n_kf] (mnId == 0), not_erase [n_kf];
// map points bad [n_mp] and observations as CSR (obs_offset [n_mp + 1], obs_kf, obs_idx), added in CSR order.  One group: list
// [n_list] keyframe rows in order.  Outputs per list entry: code (-1 skipped, 0 kept, 1 culled, 2 mbToBeErased), nMPs,
// nRedundantObservations.
extern "C" void ref_keyframe_culling(int n_kf, int cap, const int* octave, const int* n, const int* mp, const uint8_t* origin,
                                     const uint8_t* not_erase_in, int n_mp, const uint8_t* bad, const int* obs_offset, const int* obs_kf,
                                     const int* obs_idx, int n_list, const int* list, int8_t* code, int* n_mps, int* n_redundant) {
  std::vector<KeyFrame> kfs((size_t)n_kf);
  for (int k = 0; k < n_kf; k++) {
    KeyFrame& kf = kfs[k];
    kf.N = n[k];
    kf.mvKeysUn.assign((size_t)n[k], cv::KeyPoint());
    for (int i = 0; i < n[k]; i++) kf.mvKeysUn[i].octave = octave[(size_t)k * cap + i];
    kf.mvuRight.assign((size_t)n[k], -1.f);      // monocular: AddObservation / EraseObservation count one per keyframe
    kf.mnId = origin[k] ? 0 : (unsigned long)k + 1;
    kf.mvpMapPoints.assign((size_t)n[k], nullptr);
  }
  Map map;
  KeyFrame refkf;
  std::vector<std::unique_ptr<CullPoint>> pts((size_t)n_mp);
  for (int m = 0; m < n_mp; m++) {
    static const float zero[3] = {0, 0, 0};
    pts[m].reset(new CullPoint(vec3(zero), &refkf, &map));
    pts[m]->set_obs(0);
    for (int e = obs_offset[m]; e < obs_offset[m + 1]; e++) pts[m]->AddObservation(&kfs[obs_kf[e]], (size_t)obs_idx[e]);
  }
  for (int k = 0; k < n_kf; k++)
    for (int i = 0; i < n[k]; i++) {
      const int m = mp[(size_t)k * cap + i];
      kfs[k].mvpMapPoints[i] = m >= 0 ? pts[m].get() : nullptr;
    }
  for (int m = 0; m < n_mp; m++)
    if (bad[m]) pts[m]->set_bad();
  std::vector<char> not_erase(not_erase_in, not_erase_in + n_kf), to_be_erased((size_t)n_kf, 0);

  // LocalMapping.cc:1841-1898 with mbMonocular
  for (int t = 0; t < n_list; t++) {
    KeyFrame* pKF = &kfs[list[t]];
    code[t] = -1; n_mps[t] = 0; n_redundant[t] = 0;
    if (pKF->mnId == 0) continue;
    const std::vector<MapPoint*> vpMapPoints = pKF->GetMapPointMatches();
    const int thObs = 3;
    int nRedundantObservations = 0, nMPs = 0;
    for (size_t i = 0; i < vpMapPoints.size(); i++) {
      MapPoint* pMP = vpMapPoints[i];
      if (!pMP || pMP->isBad()) continue;
      nMPs++;
      if (pMP->Observations() > thObs) {
        const int scaleLevel = pKF->mvKeysUn[i].octave;
        const std::map<KeyFrame*, size_t> observations = pMP->GetObservations();
        int nObs = 0;
        for (const auto& o : observations) {
          KeyFrame* pKFi = o.first;
          if (pKFi == pKF) continue;
          if (pKFi->mvKeysUn[o.second].octave <= scaleLevel + 1) {
            nObs++;
            if (nObs >= thObs) break;
          }
        }
        if (nObs >= thObs) nRedundantObservations++;
      }
    }
    code[t] = 0;
    if (nRedundantObservations > 0.9 * nMPs) code[t] = (int8_t)set_bad_flag(pKF, not_erase, to_be_erased, list[t]);
    n_mps[t] = nMPs;
    n_redundant[t] = nRedundantObservations;
  }
}
