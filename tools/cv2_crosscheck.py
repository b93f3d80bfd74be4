"""BASELINE.md §3.2 cross-check of the CPU denominator: the per-frame hot path built from cv2 primitives (single thread,
cv2.setNumThreads(1)) next to the C++ oracle (one thread), stage by stage, on the bench frames.  It needs the cv2 Python
package, which nothing else on the benchmark path does; the result is printed as JSON.
Stages without a cv2 counterpart (LBD: opencv_contrib is not in the wheel; the pose LM: g2o) are timed on the oracle only."""
import json, os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cv2
import bench
import oracle
from plslam_b200 import synth

cv2.setNumThreads(1)
N = 55
frames, problems = bench.make_inputs(N + 1, 1)
K, D = synth.TUM1_K, synth.TUM1_DIST
Kcv = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]], np.float64); Dcv = np.array(D, np.float64)
mapx, mapy = cv2.initUndistortRectifyMap(Kcv, Dcv, np.eye(3), Kcv, (640, 480), cv2.CV_32FC1)
orb = cv2.ORB_create(nfeatures=1000, scaleFactor=1.2, nlevels=8, edgeThreshold=19, fastThreshold=20)
lsd = cv2.createLineSegmentDetector()
bf = cv2.BFMatcher(cv2.NORM_HAMMING)


def med(f, reps=N, warm=5):
    t = []
    for i in range(reps):
        t0 = time.perf_counter(); f(i); t.append(time.perf_counter() - t0)
    return 1000 * float(np.median(t[warm:]))


st = {}
prev = {}
def cv_orb(i): prev["kp"], prev["d"] = orb.detectAndCompute(frames[i], None)
def cv_remap(i): prev["und"] = cv2.remap(frames[i], mapx, mapy, cv2.INTER_LINEAR)
def cv_lsd(i): prev["seg"] = lsd.detect(prev["und"])[0]
def cv_undist(i): cv2.undistortPoints(np.array([k.pt for k in prev["kp"]], np.float32).reshape(-1, 1, 2), Kcv, Dcv, P=Kcv)
d_prev = orb.detectAndCompute(frames[0], None)[1]
def cv_match(i): bf.knnMatch(prev["d"], d_prev, k=2)
st["cv2"] = {"orb_detectAndCompute (cv::ORB, not ORBextractor: no per-cell FAST / quadtree)": med(cv_orb), "remap": med(cv_remap), "lsd_detect": med(cv_lsd),
             "undistortPoints": med(cv_undist), "bf_knn_1000x1000 (upper bound of the windowed search)": med(cv_match)}
o = oracle.OrbOracle(*bench.ORB)
feat = {}
def o_orb(i): feat["k"], feat["d"] = o.extract(frames[i])
def o_remap(i): feat["und"] = oracle.undistort_remap(frames[i], K, D)
def o_lsd(i): feat["seg"] = oracle.lsd_detect(feat["und"])
def o_line(i): feat["kl"], feat["ld"], _ = oracle.line_extract(feat["und"])
def o_undist(i): feat["ku"] = oracle.undistort_keypoints(feat["k"], K, D)
pk, pd = o.extract(frames[0]); pku = oracle.undistort_keypoints(pk, K, D); pld = oracle.line_extract(oracle.undistort_remap(frames[0], K, D))[1]
bnd = oracle.image_bounds(K, D, 640, 480)
def o_match(i):
    pm = np.stack([pku["x"], pku["y"]], 1).astype(np.float32)
    oracle.search_for_initialization(pku, pd, feat["ku"], feat["d"], bnd, pm, 100, 0.9, True); oracle.search_double(pld, feat["ld"], 0.7)
def o_lm(i):
    p = problems[i]
    for _ in range(2):
        oracle.pose_optimization(0, p["Tcw0"], p["K"], p["pt_obs"], p["pt_inv_sigma2"], p["pt_Xw"], p["line_func"], p["line_Xw"])
st["oracle"] = {"orb_extract": med(o_orb), "remap": med(o_remap), "lsd_detect": med(o_lsd), "line_extract (lsd + keylines + lbd)": med(o_line),
                "undistort_keypoints": med(o_undist), "match (SearchForInitialization + SearchDouble)": med(o_match), "2x pose_optimization": med(o_lm)}
cv_sum = sum(st["cv2"].values()); or_sum = sum(v for k, v in st["oracle"].items() if k != "lsd_detect")
lbd = st["oracle"]["line_extract (lsd + keylines + lbd)"] - st["oracle"]["lsd_detect"]
cv_equiv = st["cv2"][next(iter(st["cv2"]))] + st["cv2"]["remap"] + st["cv2"]["lsd_detect"] + st["cv2"]["undistortPoints"] + lbd + \
    st["oracle"]["match (SearchForInitialization + SearchDouble)"] + st["oracle"]["2x pose_optimization"]
out = {"host": f"{os.cpu_count()} cores (build container), one thread, median of {N - 5} frames after 5 warm-up", "cv2_version": cv2.__version__,
       "ms_per_frame": st, "oracle_total_ms": or_sum, "cv2_primitives_plus_oracle_lbd_match_lm_ms": cv_equiv,
       "oracle_over_cv2": or_sum / cv_equiv}
print(json.dumps(out, indent=1))
