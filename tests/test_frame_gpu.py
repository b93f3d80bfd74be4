"""GPU parity tests of the Frame glue (SURVEY.md §8f.1) through the C ABI vs the oracle and the cv2 golden vectors:
undistort remap, UndistortKeyPoints, ComputeImageBounds, isInFrustum (points and lines).  All bit-exact."""
import os
import numpy as np
import pytest
import torch
import oracle
import plslam_b200 as pl
from plslam_b200 import synth
from predict_scale_cases import boundary_set

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "frame_cv2.npz"))
CAMS = {"tum1": (synth.TUM1_K, synth.TUM1_DIST, 640, 480, 1), "euroc": (synth.EUROC_K, synth.EUROC_DIST, 752, 480, 5)}


@pytest.mark.parametrize("cam", ["tum1", "euroc"])
def test_remap_matches_cv2_and_oracle(cam):
    K, D, w, h, seed = CAMS[cam]
    u = pl.Undistorter(K, D, w, h)
    img = synth.synth_frame(w, h, seed)
    got = u.remap(img)
    assert np.array_equal(got, G[f"{cam}_und"])
    img2 = synth.synth_frame(w, h, seed + 10)
    assert np.array_equal(u.remap(img2), oracle.undistort_remap(img2, K, D))


def test_remap_odd_width_and_no_distortion():
    K, D = synth.TUM1_K, synth.TUM1_DIST
    w, h = 321, 243
    img = synth.synth_frame(w, h, 3)
    assert np.array_equal(pl.Undistorter(K, D, w, h).remap(img), oracle.undistort_remap(img, K, D))
    Kc = (300.0, 300.0, 160.0, 120.0)
    assert np.array_equal(pl.Undistorter(Kc, (0, 0, 0, 0, 0), w, h).remap(img), oracle.undistort_remap(img, Kc, (0, 0, 0, 0, 0)))
    with pytest.raises(pl.PLError):
        pl.Undistorter(K, D, w, h).remap(np.zeros((10, 10), np.uint8))


def test_remap_batch_dev():
    K, D, w, h, _ = CAMS["tum1"]
    u = pl.Undistorter(K, D, w, h)
    imgs = np.stack([synth.synth_frame(w, h, s) for s in (1, 2, 3, 4, 5)])
    src = torch.from_numpy(imgs).cuda(); dst = torch.zeros_like(src)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        u.remap_batch_dev(src.data_ptr(), w, w * h, 5, dst.data_ptr(), w, w * h, st.cuda_stream)
    st.synchronize()
    out = dst.cpu().numpy()
    for i in range(5):
        assert np.array_equal(out[i], oracle.undistort_remap(imgs[i], K, D))


@pytest.mark.parametrize("cam", ["tum1", "euroc"])
def test_undistort_keypoints_and_bounds(cam):
    K, D, w, h, _ = CAMS[cam]
    u = pl.Undistorter(K, D, w, h)
    pts, want = G[f"{cam}_pts"], G[f"{cam}_upts"]
    kps = np.zeros(len(pts), pl.KP_DTYPE); kps["x"], kps["y"] = pts[:, 0], pts[:, 1]; kps["octave"] = 2; kps["response"] = 31
    out = u.UndistortKeyPoints(kps)
    assert np.array_equal(np.stack([out["x"], out["y"]], 1), want)
    assert np.array_equal(out.tobytes(), oracle.undistort_keypoints(kps, K, D).tobytes())
    assert np.array_equal(u.ComputeImageBounds(), oracle.image_bounds(K, D, w, h))
    assert len(u.UndistortKeyPoints(kps[:0])) == 0
    z = pl.Undistorter(K, (0, 0, 0, 0, 0), w, h)
    assert np.array_equal(z.UndistortKeyPoints(kps).tobytes(), kps.tobytes())
    assert np.array_equal(z.ComputeImageBounds(), np.array([0, 0, w, h], np.float32))


def test_undistort_extractor_output_batch_dev():
    """UndistortKeyPoints on the ORB extractor's own device output (the Frame constructor order, Frame.cc:215-235)."""
    K, D, w, h, _ = CAMS["tum1"]
    B = 3
    ex = pl.ORBextractor(1000, 1.2, 8, 20, 7, width=w, height=h, max_batch=B)
    imgs = np.stack([synth.synth_frame(w, h, s) for s in (1, 2, 3)])
    kp, _, n = ex.extract_batch(imgs)
    u = pl.Undistorter(K, D, w, h)
    cap = ex.capacity
    assert n.min() > 500
    dk = torch.from_numpy(kp.view(np.uint8).reshape(B, -1)).cuda(); dn = torch.from_numpy(n).cuda(); do = torch.zeros_like(dk)
    u.undistort_keypoints_dev(dk.data_ptr(), dn.data_ptr(), cap, B, do.data_ptr())
    torch.cuda.synchronize()
    out = do.cpu().numpy().view(pl.KP_DTYPE).reshape(B, cap)
    for b in range(B):
        assert np.array_equal(out[b, :n[b]].tobytes(), oracle.undistort_keypoints(kp[b, :n[b]], K, D).tobytes())


@pytest.mark.parametrize("seed,cosl", [(7, 0.5), (8, 0.5), (9, 0.0), (10, 0.9)])
def test_is_in_frustum_points(seed, cosl):
    v = synth.synth_map_view(seed, 6000)
    b = oracle.image_bounds(synth.TUM1_K, synth.TUM1_DIST, 640, 480)
    a = (v["Tcw"], v["Ow"], synth.TUM1_K, b, float(np.float32(np.log(np.float32(1.2)))), 8, cosl, v["pos"], v["normal"], v["min_dist"], v["max_dist"])
    want = oracle.is_in_frustum_points(*a); got = pl.isInFrustum(*a)
    assert want[0].sum() > 100
    for g, w_ in zip(got, want):
        assert np.array_equal(g, w_)
    e = pl.isInFrustum(*a[:7], v["pos"][:0], v["normal"][:0], v["min_dist"][:0], v["max_dist"][:0])
    assert len(e[0]) == 0


@pytest.mark.parametrize("seed,cosl", [(9, 0.5), (11, 0.5), (12, 0.0)])
def test_is_in_frustum_lines(seed, cosl):
    v = synth.synth_map_view(seed, 5000, lines=True)
    if seed == 11:
        v["min_dist"] = (v["max_dist"] / 1.2 ** 12).astype(np.float32)
    b = oracle.image_bounds(synth.TUM1_K, synth.TUM1_DIST, 640, 480)
    a = (v["Tcw"], v["Ow"], synth.TUM1_K, b, float(np.float32(np.log(np.float32(1.2)))), cosl, v["pos"], v["normal"], v["min_dist"], v["max_dist"])
    want = oracle.is_in_frustum_lines(*a); got = pl.isInFrustumLines(*a)
    assert want[0].sum() > 50
    for g, w_ in zip(got, want):
        assert np.array_equal(g, w_)


def test_is_in_frustum_predicted_level_on_boundaries():
    """MapPoint::PredictScale is ceil(logf(ratio) / logScaleFactor) in fp32 (the compiled MapPoint.cc, tests/test_oracle_match_ref.py):
    points whose ratio sits exactly on a level boundary (and its fp32 neighbours) are where the float functions decide."""
    v = synth.synth_map_view(13, 20000)
    PO = (v["pos"] - v["Ow"]).astype(np.float32)
    dist = np.sqrt((PO.astype(np.float64) ** 2).sum(1)).astype(np.float32)
    k = (np.arange(len(dist)) % 9).astype(np.float32)
    mx = (dist * np.float32(1.2) ** k).astype(np.float32)
    sel = np.arange(len(dist)) % 3
    mx = np.where(sel == 0, np.nextafter(mx, np.float32(0)), np.where(sel == 1, np.nextafter(mx, np.float32(1e9)), mx)).astype(np.float32)
    v["max_dist"] = mx; v["min_dist"] = (mx / np.float32(1.2) ** 10).astype(np.float32)
    b = oracle.image_bounds(synth.TUM1_K, synth.TUM1_DIST, 640, 480)
    log_sf = float(np.float32(np.log(np.float32(1.2))))
    a = (v["Tcw"], v["Ow"], synth.TUM1_K, b, log_sf, 8, 0.0, v["pos"], v["normal"], v["min_dist"], v["max_dist"])
    want = oracle.is_in_frustum_points(*a); got = pl.isInFrustum(*a)
    assert want[0].sum() > 2000
    for g, w_ in zip(got, want):
        assert np.array_equal(g, w_)
    ratio = (mx / dist).astype(np.float32)
    f64 = np.clip(np.ceil(np.log(ratio.astype(np.float64)) / np.float64(np.float32(log_sf))), 0, 7).astype(np.int32)
    inv = want[0].astype(bool)
    assert (f64[inv] != want[2][inv]).sum() > 0        # the fp64 formula of round 1 would have failed here


def test_is_in_frustum_lines_predicted_level_on_boundaries():
    """MapLine::PredictScale on the boundary set the reference's own PredictScale is checked on (tests/predict_scale_cases.py):
    segments of 2 mm across the optical axis at depth d, seen from Tcw = I, so the midpoint distance is d exactly.
    MapLine::PredictScale does not clamp (MapLine.cpp:395-404); clamped to the 8 levels, its level must be MapPoint's answer."""
    dist, mx, log_sf = boundary_set()
    n = len(dist)
    pos = np.zeros((n, 6)); pos[:, 0], pos[:, 3] = -1e-3, 1e-3; pos[:, 2] = pos[:, 5] = dist
    normal = np.zeros((n, 3)); normal[:, 2] = 1.0
    mn = (mx / np.float32(1.2) ** 10).astype(np.float32)
    b = oracle.image_bounds(synth.TUM1_K, synth.TUM1_DIST, 640, 480)
    a = (np.eye(4, dtype=np.float32), np.zeros(3, np.float32), synth.TUM1_K, b, float(log_sf), 0.5, pos, normal, mn, mx)
    want = oracle.is_in_frustum_lines(*a); got = pl.isInFrustumLines(*a)
    for name, g, w_ in zip(("in view", "projection", "level", "viewing cosine"), got, want):
        assert np.array_equal(g, w_), f"{name}: {(g != w_).reshape(n, -1).any(1).sum()} of {n} segments differ from the oracle"
    inv = want[0].astype(bool)
    assert inv[:n // 2].all() and inv.sum() > 150000
    level = got[2]
    assert (level[inv] > 7).any(), "raw levels beyond the last one: the clamp is the caller's"
    ref = oracle.ref_predict_scale(dist, mx, log_sf, 8)
    assert np.array_equal(np.clip(level, 0, 7)[inv], ref[inv])
    ratio = (mx / dist).astype(np.float32)
    f64 = np.clip(np.ceil(np.log(ratio.astype(np.float64)) / np.float64(log_sf)), 0, 7).astype(np.int32)
    assert (f64[inv] != ref[inv]).sum() > 0
