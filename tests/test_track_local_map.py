"""Tracking::TrackLocalMapWithLines composed from the CPU oracles (tests/track_scene.py) on the planar scene with known poses.

No GPU: this pins what the device step is compared with in test_track_local_map_gpu.py.  The guesses move the plane's
reprojections by 0.9-1.2 px (th = 1 frames) and 5-7 px (th = 5 frames).  Measured with this composite over the frames below, the
recovered poses reproject the plane within 0.21 px of the true pose (largest of 8 cases) and their translations are within 2.5 mm
at a plane 3 m away.  The committed bounds, 0.3 px and 3 mm, keep a margin over those and stay under a third of the smallest guess
error (0.86 px)."""
import numpy as np
import pytest

import track_scene as ts

PX_BOUND = 0.3
T_BOUND = 3e-3


def _run(k, dt, fsr, **kw):
    T, K = ts.TRUE[k]
    kps, desc, kl, ldesc, lf = ts.features(T, K)
    m = ts.scene_map()
    G = ts.perturb(T, dt, k)
    r = ts.track_local_map_oracle(m, kps, desc, kl, ldesc, lf, G, K, np.arange(len(m["pt_pos"])), np.arange(len(m["ln_pos"])), fsr, 30, **kw)
    return r, T, G


@pytest.mark.parametrize("k", range(len(ts.TRUE)))
@pytest.mark.parametrize("dt,fsr", [(0.006, 5), (0.035, 0)])
def test_known_pose_is_recovered(k, dt, fsr):
    r, T, G = _run(k, dt, fsr)
    K = ts.TRUE[k][1]
    err = np.linalg.norm(r["Tcw"][:3, 3] - T[:3, 3])
    gap, guess_gap = ts.plane_reprojection_gap(r["Tcw"], T, K), ts.plane_reprojection_gap(G, T, K)
    assert gap < PX_BOUND and gap < guess_gap / 3, (gap, guess_gap)
    assert err < T_BOUND, err
    assert r["ok"] == 1 and r["inliers"][0] >= 50 and r["inliers"][1] > 100


def test_th_5_is_needed_for_a_6_px_guess():
    """With th = 1 a 6 px guess finds fewer matches than with th = 5 (the relocalisation switch, Tracking.cc:1793-1798)."""
    r5, _, _ = _run(0, 0.035, 0)
    r1, _, _ = _run(0, 0.035, 5)
    assert r5["prob_n_points"] > r1["prob_n_points"] + 20


def test_guess_outside_the_window_is_not_ok():
    for k in range(1, len(ts.TRUE)):
        r, _, _ = _run(k, 0.25, 5)
        assert r["ok"] == 0 and r["inliers"][0] < 30


def test_held_matches_are_not_reprojected_and_enter_the_problem():
    T, K = ts.TRUE[0]
    r0, _, G = _run(0, 0.006, 5)
    pm = np.where(np.arange(len(r0["point_map"])) % 3 == 0, r0["point_map"], -1).astype(np.int32)
    held = np.unique(pm[pm >= 0])
    r, _, _ = _run(0, 0.006, 5, point_map_in=pm)
    lp = np.arange(len(ts.scene_map()["pt_pos"]))
    assert len(held) > 100
    assert not r["pt_in_view"][np.isin(lp, held)].any()               # mnLastFrameSeen == mnId: never projected
    assert (r["pt_match"][pm >= 0] == -2).all()                       # pre-assigned in the search
    assert np.array_equal(r["point_map"][pm >= 0], pm[pm >= 0])       # and kept
    Xw = r["problem"]["pt_Xw"]; pi = np.nonzero(r["point_map"] >= 0)[0]
    assert np.array_equal(Xw, ts.scene_map()["pt_pos"][r["point_map"][pi]])   # in feature order, held ones included
    assert set(np.nonzero(pm >= 0)[0]) <= set(pi)


def test_camera_center_matches_the_pose():
    for T, _ in ts.TRUE:
        Ow = ts.camera_center(T)
        assert np.allclose(Ow, -T[:3, :3].T.astype(np.float64) @ T[:3, 3], atol=1e-6)
