"""Tracking::TrackWithMotionModel composed from the CPU oracles (tests/motion_scene.py) on constant-velocity streams of the planar
scene, against motion_scene.shifted_map() (the scene's map with 40 points and 12 lines moved 5 cm, which the pose optimisation rejects).

No GPU: this pins what pl_track_motion_model_dev is compared with in test_track_motion_model_gpu.py.  Over 3 streams x 4 steps of
motion model -> local map (with the motion model's discarded entries) -> velocity, measured with this composite, the local-map
poses reproject the plane within 0.28 px of the true pose and their translations are within 4.4 mm at a plane 3 m away; the
committed bounds are 0.4 px and 6 mm."""
import numpy as np
import pytest

import motion_scene as ms
import track_scene as ts

PX_BOUND = 0.4
T_BOUND = 6e-3
STEPS = 4


def test_mat4_equals_cv2_gemm():
    g = np.load(ms.__file__.replace("motion_scene.py", "golden/mat4_cv2.npz"))
    for a, b, c in zip(g["A"], g["B"], g["C"]):
        assert np.array_equal(ms.mat4(a, b), c)
    # an fp64-accumulated product is a different order: it disagrees on most of the vector
    assert sum(not np.array_equal((a.astype(np.float64) @ b).astype(np.float32), c) for a, b, c in zip(g["A"], g["B"], g["C"])) > 256


def _step(m, f, K, last):
    r = ms.track_motion_model_oracle(m, *f, K, last)
    lp, ll = np.arange(len(m["pt_pos"])), np.arange(len(m["ln_pos"]))
    loc = ms.track_local_map_seen_oracle(m, *f, r["Tcw"], K, lp, ll, 40, 30, r["point_map"], r["line_map"], r["point_seen"], r["line_seen"])
    return r, loc


@pytest.mark.parametrize("s", range(len(ms.STREAMS)))
def test_stream_poses_are_recovered(s):
    m, _, _ = ms.shifted_map()
    K = ms.STREAMS[s][2]
    last = ms.last_frame(m, ms.stream_pose(s, 0), K, seed=s)
    V = ms.STREAMS[s][1]
    for k in range(1, STEPS + 1):
        T = ms.stream_pose(s, k)
        f = ts.features(T, K)
        r, loc = _step(m, f, K, dict(last, velocity=V))
        assert r["ok"] == 1 and r["vo"] == 0 and r["retried"] == 0, (s, k)
        assert loc["ok"] == 1, (s, k)
        assert ts.plane_reprojection_gap(loc["Tcw"], T, K) < PX_BOUND, (s, k)
        assert np.linalg.norm(loc["Tcw"][:3, 3] - T[:3, 3]) < T_BOUND, (s, k)
        V = ms.velocity_oracle(loc["Tcw"], last["Tcw"])
        last = dict(keys=f[0], kl=f[2], point_map=loc["point_map"], point_outlier=loc["point_outlier"], line_map=loc["line_map"],
                    line_outlier=loc["line_outlier"], Tcw=loc["Tcw"])


@pytest.fixture(scope="module")
def cases():
    m, c = ms.motion_cases()
    return m, {k: (T, K, last, ms.track_motion_model_oracle(m, *ts.features(T, K), K, last)) for k, (T, K, last) in c.items()}


def test_plain_frame_discards_outliers_and_skips_last_outliers(cases):
    m, c = cases
    T, K, last, r = c["plain"]
    assert r["ok"] == 1 and r["vo"] == 0 and not r["retried"]
    # the last frame's outliers are never searched: no raw match names one
    out_idx = np.nonzero(last["point_outlier"].astype(bool) & (last["point_map"] >= 0))[0]
    assert len(out_idx) >= 3
    assert not np.isin(r["pt_match"], out_idx).any()
    lout = np.nonzero(last["line_outlier"].astype(bool) & (last["line_map"] >= 0))[0]
    assert len(lout) > 0 and not np.isin(r["ln_match"], lout).any() and not r["ln_in_view"][lout].any()
    # discarded outliers: counted off, named in seen, not in the matches
    ds = int((r["point_seen"] >= 0).sum())
    assert ds > 0 and r["nmatches"][0] == (r["point_map"] >= 0).sum()
    assert not np.isin(np.nonzero(r["point_seen"] >= 0)[0], np.nonzero(r["point_map"] >= 0)[0]).any()


def test_seen_entries_change_the_local_map_frustum(cases):
    m, c = cases
    T, K, last, r = c["plain"]
    f = ts.features(T, K)
    lp, ll = np.arange(len(m["pt_pos"])), np.arange(len(m["ln_pos"]))
    with_seen = ms.track_local_map_seen_oracle(m, *f, r["Tcw"], K, lp, ll, 40, 30, r["point_map"], r["line_map"], r["point_seen"],
                                               r["line_seen"])
    without = ts.track_local_map_oracle(m, *f, r["Tcw"], K, lp, ll, 40, 30, r["point_map"], r["line_map"])
    seen = r["point_seen"][r["point_seen"] >= 0]
    assert without["pt_in_view"][seen].any() and not with_seen["pt_in_view"][seen].any()
    assert not with_seen["pt_match"][r["point_seen"] >= 0].tolist().count(-2)        # not pre-assigned
    # with no seen entries the composite is the plain local-map step
    same = ms.track_local_map_seen_oracle(m, *f, r["Tcw"], K, lp, ll, 40, 30, r["point_map"], r["line_map"])
    for k in ("pt_in_view", "pt_match", "ln_match", "point_map", "Tcw"):
        assert np.array_equal(same[k], without[k]), k


def test_retry_frame(cases):
    _, c = cases
    _, _, _, r = c["retry"]
    n1, n2 = int((r["pt_match"] >= 0).sum()), int((r["pt_match_retry"] >= 0).sum())
    assert r["retried"] == 1 and n1 < 20 and n2 > n1 + 50 and r["ok"] == 1


def test_early_return_frame(cases):
    _, c = cases
    T, K, last, r = c["early"]
    assert not r["solved"] and r["ok"] == 0 and r["vo"] is None
    assert r["nmatches"][0] < 20 and r["nmatches"][1] < 5 and (r["point_map"] >= 0).sum() > 0
    assert np.array_equal(r["Tcw"], r["guess"]) and np.array_equal(r["guess"], ms.mat4(last["velocity"], last["Tcw"]))


def test_few_map_matches_set_vo(cases):
    _, c = cases
    _, _, _, r = c["few"]
    assert r["solved"] and r["retried"] == 1 and r["vo"] == 1 and r["ok"] == 0 and (r["point_map"] >= 0).sum() < 10


def test_velocity_composite():
    T0, T1 = ms.stream_pose(0, 1), ms.stream_pose(0, 2)
    V = ms.velocity_oracle(T1, T0)
    assert np.allclose(V, np.asarray(ms.STREAMS[0][1], np.float64), atol=1e-5)
    assert np.array_equal(ms.mat4(V, T0)[3], [0, 0, 0, 1])
