// ORBmatcher / LSDmatcher / Optimizer of the reference (src/ORBmatcher.cc, src/LSDmatcher.cpp, src/Optimizer.cc), SAME
// signatures, on the plslam_b200 C ABI: every method gathers the members the reference's loop reads into flat arrays,
// calls one pl_* entry point (one kernel launch on the GPU), and writes the members the reference's loop writes.
// In the reference tree: compile with -DPLSLAM_IN_REFERENCE_TREE (real Frame.h ... are included through reference_glue.h)
// IN PLACE of src/ORBmatcher.cc / LSDmatcher.cpp / Optimizer.cc for these methods; here: against reference_mock.h, driven
// by tests/host/glue_track.cpp through TrackWithMotionModel's call sequence (Tracking.cc:1345-1372) and checked against the
// CPU oracle by tests/test_host_cpp.py.
#include "reference_glue.h"
#include <cmath>
#include <stdexcept>
#include <string>
#include "../../include/plslam_b200.h"

namespace ORB_SLAM2 {
#ifndef PLSLAM_IN_REFERENCE_TREE
const int ORBmatcher::TH_HIGH = 100, ORBmatcher::TH_LOW = 50, ORBmatcher::HISTO_LENGTH = 30;
const int LSDmatcher::TH_HIGH = 80, LSDmatcher::TH_LOW = 50, LSDmatcher::HISTO_LENGTH = 30;
float Frame::fx, Frame::fy, Frame::cx, Frame::cy, Frame::mnMinX, Frame::mnMaxX, Frame::mnMinY, Frame::mnMaxY;
std::mutex MapPoint::mGlobalMutex, MapLine::mGlobalMutex;
ORBmatcher::ORBmatcher(float nnratio, bool checkOri) : mfNNratio(nnratio), mbCheckOrientation(checkOri) {}
LSDmatcher::LSDmatcher(float nnratio, bool checkOri) : mfNNratio(nnratio), mbCheckOrientation(checkOri) {}
#endif

namespace {
void fail() { throw std::runtime_error(std::string("plslam_b200: ") + pl_last_error()); }
static_assert(sizeof(cv::KeyPoint) == sizeof(PLKeyPoint), "cv::KeyPoint is the C ABI's 28-byte record");
static_assert(sizeof(KeyLine) == 68, "KeyLine is the C ABI's 68-byte record");
std::vector<uint8_t> rows32(const cv::Mat& m) {
  std::vector<uint8_t> d((size_t)std::max(m.rows, 1) * 32);
  for (int i = 0; i < m.rows; i++) memcpy(&d[(size_t)i * 32], m.ptr(i), 32);
  return d;
}
void pose16(const cv::Mat& Tcw, float out[16]) {
  for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) out[4 * r + c] = Tcw.at<float>(r, c);
}
struct Cam { float K[4], bounds[4]; };
Cam cam_of(const Frame&) {
  return Cam{{Frame::fx, Frame::fy, Frame::cx, Frame::cy}, {Frame::mnMinX, Frame::mnMinY, Frame::mnMaxX, Frame::mnMaxY}};
}
std::vector<double> linefuncs(const std::vector<Eigen::Vector3d>& v) {
  std::vector<double> f(std::max<size_t>(v.size(), 1) * 3);
  for (size_t i = 0; i < v.size(); i++) { f[3 * i] = v[i][0]; f[3 * i + 1] = v[i][1]; f[3 * i + 2] = v[i][2]; }
  return f;
}
}  // namespace

int ORBmatcher::DescriptorDistance(const cv::Mat& a, const cv::Mat& b) {
  int d = 0;
  if (pl_descriptor_distance_batch(a.ptr(0), b.ptr(0), 1, &d) != PL_OK) fail();
  return d;
}
int LSDmatcher::DescriptorDistance(const cv::Mat& a, const cv::Mat& b) { return ORBmatcher::DescriptorDistance(a, b); }

// ---- ORBmatcher::SearchByProjection(CurrentFrame, LastFrame, th, bMono)   src/ORBmatcher.cc:1441-1585
int ORBmatcher::SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, const float th, const bool bMono) {
  if (!bMono) throw std::runtime_error("plslam_b200: the stereo / RGB-D branch (mvuRight) is not on this path");
  const int n = CurrentFrame.N, nl = LastFrame.N;
  if (n == 0 || nl == 0) return 0;
  std::vector<uint8_t> valid(nl, 0), ldesc((size_t)nl * 32, 0), pre(n, 0);
  std::vector<float> pos((size_t)nl * 3, 0.f), ang(nl, 0.f);
  std::vector<int> oct(nl, 0), match(n, -1);
  for (int i = 0; i < nl; i++) {
    MapPoint* pMP = LastFrame.mvpMapPoints[i];
    if (!pMP || LastFrame.mvbOutlier[i]) continue;
    valid[i] = 1;
    const cv::Mat x = pMP->GetWorldPos();
    for (int k = 0; k < 3; k++) pos[3 * i + k] = x.at<float>(k);
    const cv::Mat d = pMP->GetDescriptor();
    memcpy(&ldesc[(size_t)i * 32], d.ptr(0), 32);
    oct[i] = LastFrame.mvKeys[i].octave; ang[i] = LastFrame.mvKeysUn[i].angle;
  }
  for (int i = 0; i < n; i++) pre[i] = CurrentFrame.mvpMapPoints[i] && CurrentFrame.mvpMapPoints[i]->Observations() > 0;
  float T[16];
  pose16(CurrentFrame.mTcw, T);
  const Cam c = cam_of(CurrentFrame);
  const std::vector<uint8_t> desc = rows32(CurrentFrame.mDescriptors);
  const int nm = pl_orb_search_by_projection_last((const PLKeyPoint*)CurrentFrame.mvKeysUn.data(), desc.data(), n, c.bounds, T, c.K,
                                                  CurrentFrame.mvScaleFactors.data(), (int)CurrentFrame.mvScaleFactors.size(), nl, valid.data(),
                                                  pos.data(), ldesc.data(), oct.data(), ang.data(), th, mbCheckOrientation ? 1 : 0, pre.data(),
                                                  match.data());
  if (nm < 0) fail();
  for (int i = 0; i < n; i++) if (match[i] >= 0) CurrentFrame.mvpMapPoints[i] = LastFrame.mvpMapPoints[match[i]];
  return nm;
}

// ---- ORBmatcher::SearchByProjection(F, vpMapPoints, th)   src/ORBmatcher.cc:56-144
int ORBmatcher::SearchByProjection(Frame& F, const std::vector<MapPoint*>& vpMapPoints, const float th) {
  const int n = F.N, nm_ = (int)vpMapPoints.size();
  if (n == 0 || nm_ == 0) return 0;
  std::vector<uint8_t> inview(nm_, 0), mdesc((size_t)nm_ * 32, 0), pre(n, 0);
  std::vector<float> proj((size_t)nm_ * 2, 0.f), vcos(nm_, 0.f);
  std::vector<int> level(nm_, 0), match(n, -1);
  for (int i = 0; i < nm_; i++) {
    MapPoint* pMP = vpMapPoints[i];
    if (!pMP->mbTrackInView || pMP->isBad()) continue;
    inview[i] = 1;
    proj[2 * i] = pMP->mTrackProjX; proj[2 * i + 1] = pMP->mTrackProjY; level[i] = pMP->mnTrackScaleLevel; vcos[i] = pMP->mTrackViewCos;
    const cv::Mat d = pMP->GetDescriptor();
    memcpy(&mdesc[(size_t)i * 32], d.ptr(0), 32);
  }
  for (int i = 0; i < n; i++) pre[i] = F.mvpMapPoints[i] && F.mvpMapPoints[i]->Observations() > 0;
  const Cam c = cam_of(F);
  const std::vector<uint8_t> desc = rows32(F.mDescriptors);
  const int r = pl_orb_search_by_projection_points((const PLKeyPoint*)F.mvKeysUn.data(), desc.data(), n, c.bounds, F.mvScaleFactors.data(),
                                                   (int)F.mvScaleFactors.size(), nm_, inview.data(), proj.data(), level.data(), vcos.data(),
                                                   mdesc.data(), th, mfNNratio, pre.data(), match.data());
  if (r < 0) fail();
  for (int i = 0; i < n; i++) if (match[i] >= 0) F.mvpMapPoints[i] = vpMapPoints[match[i]];
  return r;
}

// ---- ORBmatcher::SearchForInitialization   src/ORBmatcher.cc:455-572
int ORBmatcher::SearchForInitialization(Frame& F1, Frame& F2, std::vector<cv::Point2f>& vbPrevMatched, std::vector<int>& vnMatches12, int windowSize) {
  const int n1 = (int)F1.mvKeysUn.size(), n2 = (int)F2.mvKeysUn.size();
  vnMatches12.assign(n1, -1);
  if (n1 == 0 || n2 == 0) return 0;
  if ((int)vbPrevMatched.size() != n1) throw std::runtime_error("plslam_b200: vbPrevMatched must have F1.N entries");
  const Cam c = cam_of(F2);
  const std::vector<uint8_t> d1 = rows32(F1.mDescriptors), d2 = rows32(F2.mDescriptors);
  static_assert(sizeof(cv::Point2f) == 8, "layout");
  const int nm = pl_orb_search_for_initialization((const PLKeyPoint*)F1.mvKeysUn.data(), d1.data(), n1, (const PLKeyPoint*)F2.mvKeysUn.data(),
                                                  d2.data(), n2, c.bounds, (float*)vbPrevMatched.data(), vnMatches12.data(), windowSize,
                                                  mfNNratio, mbCheckOrientation ? 1 : 0);
  if (nm < 0) fail();
  return nm;
}

// ---- LSDmatcher::SearchByProjection(CurrentFrame, LastFrame, th)   src/LSDmatcher.cpp:72-176
// (the reference also draws every match into a JPEG and writes it per call, :67,:173: debugging output, not reproduced)
int LSDmatcher::SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, const float th) {
  const int n = CurrentFrame.NL, nl = LastFrame.NL;
  if (n == 0 || nl == 0) return 0;
  // Frame::isInFrustum(pML, 0.5) for every candidate of the last frame (it also sets the MapLine's tracking members)
  std::vector<int> cand;
  for (int i = 0; i < nl; i++) if (LastFrame.mvpMapLines[i] && !LastFrame.mvbLineOutlier[i]) cand.push_back(i);
  const int nc = (int)cand.size();
  if (nc == 0) return 0;
  std::vector<double> pos((size_t)nc * 6), nrm((size_t)nc * 3);
  std::vector<float> mind(nc), maxd(nc), proj((size_t)nc * 4), vcos(nc);
  std::vector<uint8_t> inview(nc);
  std::vector<int> level(nc);
  for (int k = 0; k < nc; k++) {
    MapLine* pML = LastFrame.mvpMapLines[cand[k]];
    const Vector6d P = pML->GetWorldPos();
    for (int j = 0; j < 6; j++) pos[6 * k + j] = P[j];
    for (int j = 0; j < 3; j++) nrm[3 * k + j] = pML->mNormalVector[j];
    mind[k] = pML->mfMinDistance; maxd[k] = pML->mfMaxDistance;
  }
  float T[16], Ow[3];
  pose16(CurrentFrame.mTcw, T);
  for (int k = 0; k < 3; k++) Ow[k] = CurrentFrame.mOw.at<float>(k);
  const Cam c = cam_of(CurrentFrame);
  if (pl_frame_is_in_frustum_lines(T, Ow, c.K, c.bounds, CurrentFrame.mfLogScaleFactorLine, 0.5f, nc, pos.data(), nrm.data(), mind.data(),
                                   maxd.data(), inview.data(), proj.data(), level.data(), vcos.data()) != PL_OK) fail();
  std::vector<uint8_t> valid(nl, 0), ldesc((size_t)nl * 32, 0), pre(n, 0);
  std::vector<float> lproj((size_t)nl * 4, 0.f), llen(nl, 0.f);
  std::vector<int> match(n, -1);
  for (int k = 0; k < nc; k++) {
    const int i = cand[k];
    MapLine* pML = LastFrame.mvpMapLines[i];
    pML->mbTrackInView = inview[k] != 0;                            // Frame.cc:625-702 side effects
    if (!inview[k]) continue;
    pML->mTrackProjX1 = proj[4 * k]; pML->mTrackProjY1 = proj[4 * k + 1]; pML->mTrackProjX2 = proj[4 * k + 2]; pML->mTrackProjY2 = proj[4 * k + 3];
    pML->mnTrackScaleLevel = level[k]; pML->mTrackViewCos = vcos[k];
    valid[i] = 1;
    for (int j = 0; j < 4; j++) lproj[4 * i + j] = proj[4 * k + j];
    const cv::Mat d = pML->GetDescriptor();
    memcpy(&ldesc[(size_t)i * 32], d.ptr(0), 32);
    llen[i] = LastFrame.mvKeylinesUn[i].lineLength;
  }
  for (int i = 0; i < n; i++) pre[i] = CurrentFrame.mvpMapLines[i] && CurrentFrame.mvpMapLines[i]->Observations() > 0;
  const std::vector<uint8_t> desc = rows32(CurrentFrame.mLdesc);
  const std::vector<double> lf = linefuncs(CurrentFrame.mvKeyLineFunctions);
  const int nm = pl_lsd_search_by_projection_last(CurrentFrame.mvKeylinesUn.data(), lf.data(), desc.data(), n, c.bounds, nl, valid.data(), lproj.data(),
                                                  ldesc.data(), llen.data(), th, pre.data(), match.data());
  if (nm < 0) fail();
  for (int i = 0; i < n; i++) if (match[i] >= 0) CurrentFrame.mvpMapLines[i] = LastFrame.mvpMapLines[match[i]];
  return nm;
}

// ---- LSDmatcher::SearchByProjection(F, vpMapLines, th)   src/LSDmatcher.cpp:221-338
int LSDmatcher::SearchByProjection(Frame& F, const std::vector<MapLine*>& vpMapLines, const float th) {
  const int n = F.NL, nm_ = (int)vpMapLines.size();
  if (n == 0 || nm_ == 0) return 0;
  std::vector<uint8_t> inview(nm_, 0), mdesc((size_t)nm_ * 32, 0), pre(n, 0);
  std::vector<float> proj((size_t)nm_ * 4, 0.f), vcos(nm_, 0.f);
  std::vector<int> match(n, -1);
  for (int i = 0; i < nm_; i++) {
    MapLine* pML = vpMapLines[i];
    if (!pML->mbTrackInView || pML->isBad()) continue;
    inview[i] = 1;
    proj[4 * i] = pML->mTrackProjX1; proj[4 * i + 1] = pML->mTrackProjY1; proj[4 * i + 2] = pML->mTrackProjX2; proj[4 * i + 3] = pML->mTrackProjY2;
    vcos[i] = pML->mTrackViewCos;
    const cv::Mat d = pML->GetDescriptor();
    memcpy(&mdesc[(size_t)i * 32], d.ptr(0), 32);
  }
  for (int i = 0; i < n; i++) pre[i] = F.mvpMapLines[i] && F.mvpMapLines[i]->Observations() > 0;
  const Cam c = cam_of(F);
  const std::vector<uint8_t> desc = rows32(F.mLdesc);
  const std::vector<double> lf = linefuncs(F.mvKeyLineFunctions);
  const int r = pl_lsd_search_by_projection_lines(F.mvKeylinesUn.data(), lf.data(), desc.data(), n, c.bounds, nm_, inview.data(), proj.data(),
                                                  vcos.data(), mdesc.data(), th, mfNNratio, pre.data(), match.data());
  if (r < 0) fail();
  for (int i = 0; i < n; i++) if (match[i] >= 0) F.mvpMapLines[i] = vpMapLines[match[i]];
  return r;
}

// ---- LSDmatcher::SearchDouble(InitialFrame, CurrentFrame, LineMatches)   src/LSDmatcher.cpp:440-460
int LSDmatcher::SearchDouble(Frame& InitialFrame, Frame& CurrentFrame, std::vector<int>& LineMatches) {
  const int n1 = InitialFrame.mLdesc.rows, n2 = CurrentFrame.mLdesc.rows;
  LineMatches.assign(n1, -1);
  if (n1 == 0 || n2 == 0) return 0;
  const std::vector<uint8_t> d1 = rows32(InitialFrame.mLdesc), d2 = rows32(CurrentFrame.mLdesc);
  const int nm = pl_lsd_search_double(d1.data(), n1, d2.data(), n2, mfNNratio, LineMatches.data());
  if (nm < 0) fail();
  return nm;
}

// ---- Optimizer::PoseOptimization / WithPoints / WithLines   src/Optimizer.cc:640-1284
static int pose_optimization(Frame* pFrame, int mode) {
  // correspondences in the reference's edge order: points i = 0..N-1 with a MapPoint (mono: mvuRight[i] < 0), then lines
  std::vector<int> pidx, lidx;
  std::vector<float> obs, w, Xw;
  std::vector<double> lf, lX;
  {
    std::unique_lock<std::mutex> lock(MapPoint::mGlobalMutex);
    if (mode != 2)
      for (int i = 0; i < pFrame->N; i++) {
        MapPoint* pMP = pFrame->mvpMapPoints[i];
        if (!pMP) continue;
        if (!pFrame->mvuRight.empty() && !(pFrame->mvuRight[i] < 0)) throw std::runtime_error("plslam_b200: stereo observations are not on this path");
        pFrame->mvbOutlier[i] = false;
        const cv::KeyPoint& kpUn = pFrame->mvKeysUn[i];
        pidx.push_back(i);
        obs.push_back(kpUn.pt.x); obs.push_back(kpUn.pt.y);
        w.push_back(pFrame->mvInvLevelSigma2[kpUn.octave]);
        const cv::Mat X = pMP->GetWorldPos();
        for (int k = 0; k < 3; k++) Xw.push_back(X.at<float>(k));
      }
  }
  {
    std::unique_lock<std::mutex> lock(MapLine::mGlobalMutex);
    if (mode != 1)
      for (int i = 0; i < pFrame->NL; i++) {
        MapLine* pML = pFrame->mvpMapLines[i];
        if (!pML) continue;
        pFrame->mvbLineOutlier[i] = false;
        lidx.push_back(i);
        for (int k = 0; k < 3; k++) lf.push_back(pFrame->mvKeyLineFunctions[i][k]);
        const Vector6d P = pML->GetWorldPos();
        for (int k = 0; k < 6; k++) lX.push_back(P[k]);
      }
  }
  const int np = (int)pidx.size(), nl = (int)lidx.size();
  float T[16], Tout[16];
  pose16(pFrame->mTcw, T);
  const float K[4] = {Frame::fx, Frame::fy, Frame::cx, Frame::cy};
  std::vector<uint8_t> po(np + 1), lo(nl + 1);
  static const float zf[3] = {0, 0, 0};
  static const double zd[6] = {0, 0, 0, 0, 0, 0};
  const int n = pl_pose_optimization(mode, T, K, np, np ? obs.data() : zf, np ? w.data() : zf, np ? Xw.data() : zf, nl, nl ? lf.data() : zd,
                                     nl ? lX.data() : zd, Tout, po.data(), lo.data(), nullptr);
  if (n < 0) fail();
  if ((mode == 2 ? nl : np) < 3) return 0;                       // Optimizer.cc:846-847: nothing happened, pose untouched
  for (int k = 0; k < np; k++) pFrame->mvbOutlier[pidx[k]] = po[k] != 0;
  for (int k = 0; k < nl; k++) pFrame->mvbLineOutlier[lidx[k]] = lo[k] != 0;
  cv::Mat pose(4, 4, CV_32F);
  for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) pose.at<float>(r, c) = Tout[4 * r + c];
  pFrame->SetPose(pose);
  return n;
}
int Optimizer::PoseOptimization(Frame* pFrame) { return pose_optimization(pFrame, 0); }
int Optimizer::PoseOptimizationWithPoints(Frame* pFrame) { return pose_optimization(pFrame, 1); }
int Optimizer::PoseOptimizationWithLines(Frame* pFrame) { return pose_optimization(pFrame, 2); }

// ---- Optimizer::LocalBundleAdjustmentWithLine(pKF, pbStopFlag, pMap)   src/Optimizer.cc:1645-2100
void Optimizer::LocalBundleAdjustmentWithLine(KeyFrame* pKF, bool* pbStopFlag, Map* pMap) {
  // :1649-1742  local keyframes, their points and lines, the fixed keyframes that also see them (list orders kept)
  std::list<KeyFrame*> lLocalKeyFrames;
  lLocalKeyFrames.push_back(pKF);
  pKF->mnBALocalForKF = pKF->mnId;
  for (KeyFrame* pKFi : pKF->GetVectorCovisibleKeyFrames()) {
    pKFi->mnBALocalForKF = pKF->mnId;
    if (!pKFi->isBad()) lLocalKeyFrames.push_back(pKFi);
  }
  std::list<MapPoint*> lLocalMapPoints;
  for (KeyFrame* k : lLocalKeyFrames)
    for (MapPoint* pMP : k->GetMapPointMatches())
      if (pMP && !pMP->isBad() && pMP->mnBALocalForKF != pKF->mnId) { lLocalMapPoints.push_back(pMP); pMP->mnBALocalForKF = pKF->mnId; }
  std::list<MapLine*> lLocalMapLines;
  for (KeyFrame* k : lLocalKeyFrames)
    for (MapLine* pML : k->GetMapLineMatches())
      if (pML && !pML->isBad() && pML->mnBALocalForKF != pKF->mnId) { lLocalMapLines.push_back(pML); pML->mnBALocalForKF = pKF->mnId; }
  std::list<KeyFrame*> lFixedCameras;
  auto fixed_of = [&](const std::map<KeyFrame*, size_t>& observations) {
    for (const auto& mit : observations) {
      KeyFrame* pKFi = mit.first;
      if (pKFi->mnBALocalForKF != pKF->mnId && pKFi->mnBAFixedForKF != pKF->mnId) {
        pKFi->mnBAFixedForKF = pKF->mnId;
        if (!pKFi->isBad()) lFixedCameras.push_back(pKFi);
      }
    }
  };
  for (MapPoint* pMP : lLocalMapPoints) fixed_of(pMP->GetObservations());
  for (MapLine* pML : lLocalMapLines) fixed_of(pML->GetObservations());
  if (lLocalMapPoints.empty()) return;        // (the reference indexes MapPointID[size-1] here, :1865: undefined; nothing to optimise)

  // flat problem: keyframes = local then fixed; landmarks in list order; edges in the reference's insertion order
  std::vector<KeyFrame*> kfs(lLocalKeyFrames.begin(), lLocalKeyFrames.end());
  kfs.insert(kfs.end(), lFixedCameras.begin(), lFixedCameras.end());
  std::map<KeyFrame*, int> kfIndex;
  std::vector<float> kfT(kfs.size() * 16), kfK(kfs.size() * 4);
  std::vector<uint8_t> kfFixed(kfs.size(), 0);
  for (size_t i = 0; i < kfs.size(); i++) {
    kfIndex[kfs[i]] = (int)i;
    pose16(kfs[i]->GetPose(), &kfT[16 * i]);
    kfK[4 * i] = kfs[i]->fx; kfK[4 * i + 1] = kfs[i]->fy; kfK[4 * i + 2] = kfs[i]->cx; kfK[4 * i + 3] = kfs[i]->cy;
    kfFixed[i] = (i >= lLocalKeyFrames.size()) || kfs[i]->mnId == 0;
  }
  std::vector<MapPoint*> pts(lLocalMapPoints.begin(), lLocalMapPoints.end());
  std::vector<MapLine*> lns(lLocalMapLines.begin(), lLocalMapLines.end());
  std::vector<float> ptX(pts.size() * 3), peObs, peW;
  std::vector<int> peKf, pePt, leKf, leLn;
  std::vector<KeyFrame*> vpEdgeKFMono; std::vector<MapPoint*> vpMapPointEdgeMono;
  for (size_t i = 0; i < pts.size(); i++) {
    const cv::Mat X = pts[i]->GetWorldPos();
    for (int k = 0; k < 3; k++) ptX[3 * i + k] = X.at<float>(k);
    for (const auto& mit : pts[i]->GetObservations()) {
      KeyFrame* pKFi = mit.first;
      if (pKFi->isBad()) continue;
      const cv::KeyPoint& kpUn = pKFi->mvKeysUn[mit.second];
      peKf.push_back(kfIndex.at(pKFi)); pePt.push_back((int)i);
      peObs.push_back(kpUn.pt.x); peObs.push_back(kpUn.pt.y);
      peW.push_back(pKFi->mvInvLevelSigma2[kpUn.octave]);
      vpEdgeKFMono.push_back(pKFi); vpMapPointEdgeMono.push_back(pts[i]);
    }
  }
  std::vector<double> lnX(std::max<size_t>(lns.size(), 1) * 6), leF;
  std::vector<MapLine*> vpMapLineEdge;
  for (size_t i = 0; i < lns.size(); i++) {
    const Vector6d P = lns[i]->GetWorldPos();
    for (int k = 0; k < 6; k++) lnX[6 * i + k] = P[k];
    for (const auto& mit : lns[i]->GetObservations()) {
      KeyFrame* pKFi = mit.first;
      if (pKFi->isBad()) continue;
      leKf.push_back(kfIndex.at(pKFi)); leLn.push_back((int)i);
      for (int k = 0; k < 3; k++) leF.push_back(pKFi->mvKeyLineFunctions[mit.second][k]);
      vpMapLineEdge.push_back(lns[i]);
    }
  }
  if (pbStopFlag && *pbStopFlag) return;      // :1957-1959
  PLBAProblem Pb;
  memset(&Pb, 0, sizeof(Pb));
  Pb.n_kf = (int)kfs.size(); Pb.kf_Tcw = kfT.data(); Pb.kf_fixed = kfFixed.data(); Pb.kf_K = kfK.data();
  Pb.K_end[0] = pKF->fx; Pb.K_end[1] = pKF->fy; Pb.K_end[2] = pKF->cx; Pb.K_end[3] = pKF->cy;      // the end-point edges' quirk (:1939-1942)
  Pb.n_pt = (int)pts.size(); Pb.pt_Xw = ptX.data(); Pb.n_ln = (int)lns.size(); Pb.ln_Xw = lnX.data();
  Pb.n_pe = (int)pePt.size(); Pb.pe_kf = peKf.data(); Pb.pe_pt = pePt.data(); Pb.pe_obs = peObs.data(); Pb.pe_inv_sigma2 = peW.data();
  Pb.n_le = (int)leLn.size(); Pb.le_kf = leKf.data(); Pb.le_ln = leLn.data(); Pb.le_func = leF.data();
  std::vector<float> Tout(kfs.size() * 16), Xout(std::max<size_t>(pts.size(), 1) * 3);
  std::vector<double> Lout(std::max<size_t>(lns.size(), 1) * 6);
  std::vector<uint8_t> peErase(std::max<size_t>(pePt.size(), 1)), leErase(std::max<size_t>(leLn.size(), 1));
  std::vector<int> leEraseKf(std::max<size_t>(leLn.size(), 1));
  // g2o polls *pbStopFlag between iterations; the device solver polls a device-visible int: the bool is sampled once more
  // here (a LocalMapping that needs mid-solve aborts maps a pinned int and passes it to pl_local_ba directly)
  if (pl_local_ba(&Pb, nullptr, Tout.data(), Xout.data(), Lout.data(), peErase.data(), leErase.data(), leEraseKf.data(), nullptr) != PL_OK) fail();

  std::unique_lock<std::mutex> lock(pMap->mMutexMapUpdate);     // :2044
  for (size_t e = 0; e < pePt.size(); e++)
    if (peErase[e]) { vpEdgeKFMono[e]->EraseMapPointMatch(vpMapPointEdgeMono[e]); vpMapPointEdgeMono[e]->EraseObservation(vpEdgeKFMono[e]); }
  for (size_t e = 0; e < leLn.size(); e++)
    if (leErase[e]) { KeyFrame* k = kfs[leEraseKf[e]]; k->EraseMapLineMatch(vpMapLineEdge[e]); vpMapLineEdge[e]->EraseObservation(k); }
  for (size_t i = 0; i < lLocalKeyFrames.size(); i++) {          // :2069-2076 (local keyframes only)
    cv::Mat pose(4, 4, CV_32F);
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) pose.at<float>(r, c) = Tout[16 * i + 4 * r + c];
    kfs[i]->SetPose(pose);
  }
  for (size_t i = 0; i < pts.size(); i++) {
    cv::Mat X(3, 1, CV_32F);
    for (int k = 0; k < 3; k++) X.at<float>(k) = Xout[3 * i + k];
    pts[i]->SetWorldPos(X);
    pts[i]->UpdateNormalAndDepth();
  }
  for (size_t i = 0; i < lns.size(); i++) {
    Vector6d P;
    for (int k = 0; k < 6; k++) P[k] = (double)(float)Lout[6 * i + k];    // Converter::toCvMat (float) -> toVector3d round trip (:2094)
    lns[i]->SetWorldPos(P);
    lns[i]->UpdateAverageDir();
  }
}

}  // namespace ORB_SLAM2
