"""GPU parity tests: the CUDA ORB extractor at settings other than the TUM one (level count, scale factor, FAST thresholds,
frame size), against the CPU oracle stage by stage and against the reference's own outputs (tests/golden/orb_ref_set_*.npz,
tools/gen_golden_orb_ref.py SETTINGS).  These settings shape the level sizes and pitches, the resize tables, the FAST cell
grid, the per-level quotas and the quadtree pool, which the TUM setting leaves at one value each."""
import os
import sys
import numpy as np
import pytest
import oracle
import plslam_b200 as pl
from plslam_b200 import synth

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from gen_golden_orb_ref import SETTINGS  # noqa: E402

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
# settings whose densest FAST cells come near the default 128 NMS maxima per cell
SLOT_CAP = {"th5_3": 256, "th12_5": 256, "s20": 256}


def _assert_same(kps, desc, okps, odesc, what=""):
    assert len(kps) == len(okps), what
    for f in ("x", "y", "size", "angle", "response", "octave", "class_id"):
        assert np.array_equal(kps[f], okps[f]), (what, f)
    assert np.array_equal(desc, odesc), what


@pytest.mark.parametrize("name", sorted(SETTINGS))
def test_setting_matches_oracle_and_reference(name):
    w, h, seed, nf, sf, nl, ini, mn = SETTINGS[name]
    frames = np.stack([synth.synth_frame(w, h, seed + k) for k in range(3)])
    ex = pl.ORBextractor(nf, sf, nl, ini, mn, width=w, height=h, max_batch=3, cell_slot_cap=SLOT_CAP.get(name, 0))
    kps, desc, n = ex.extract_batch(frames)
    o = oracle.OrbOracle(nf, sf, nl, ini, mn)
    # constructor tables and level sizes
    t = o.tables()
    assert ex.GetScaleFactors().tobytes() == t["scale"].tobytes()
    assert ex.GetInverseScaleFactors().tobytes() == t["inv_scale"].tobytes()
    assert ex.GetScaleSigmaSquares().tobytes() == t["sigma2"].tobytes()
    assert ex.GetInverseScaleSigmaSquares().tobytes() == t["inv_sigma2"].tobytes()
    assert np.array_equal(ex.mnFeaturesPerLevel, t["per_level"])
    # every frame of the batch (the per-frame offsets of the pyramid and key buffers depend on the setting)
    for b in (1, 2, 0):                       # frame 0 last: the oracle keeps its stage taps
        _assert_same(kps[b, :n[b]], desc[b, :n[b]], *o.extract(frames[b]), what=f"frame {b}")
    assert [(int(a), int(b)) for a, b in zip(ex.level_w, ex.level_h)] == [o.level_dims(l) for l in range(nl)]
    # stage taps of frame 0: every pyramid level, one bordered level, the FAST candidates of every level
    for l in range(nl):
        assert np.array_equal(ex.mvImagePyramid(l, frame=0), o.level(l)), f"pyramid level {l}"
        c, oc = ex.debug_candidates(l, frame=0), o.candidates(l)
        assert len(c) == len(oc), f"candidate count level {l}"
        for f in ("x", "y", "response"):
            assert np.array_equal(c[f], oc[f]), f"candidates {f} level {l}"
    lb = min(2, nl - 1)
    assert np.array_equal(ex.mvImagePyramid(lb, frame=0, with_border=True), o.level(lb, True))
    # the reference's own output on frame 0
    g = np.load(os.path.join(G, f"orb_ref_set_{name}.npz"))
    assert int(frames[0].astype(np.int64).sum()) == int(g["img_sum"])
    assert kps[0, :n[0]].tobytes() == g["kps"].tobytes()
    assert np.array_equal(desc[0, :n[0]], g["desc"])
    assert [tuple(d) for d in g["level_dims"]] == [ex.mvImagePyramid(l).shape[::-1] for l in range(nl)]


@pytest.mark.parametrize("name", sorted(SLOT_CAP))
def test_default_slot_cap_matches_or_is_loud(name):
    """At the default 128 maxima per cell a dense setting either still equals the oracle or fails with the cell_slot_cap
    error: a cell is never truncated silently."""
    w, h, seed, nf, sf, nl, ini, mn = SETTINGS[name]
    frames = np.stack([synth.synth_frame(w, h, seed + k) for k in range(3)])
    ex = pl.ORBextractor(nf, sf, nl, ini, mn, width=w, height=h, max_batch=3)
    try:
        kps, desc, n = ex.extract_batch(frames)
    except pl.PLError as e:
        assert "cell_slot_cap" in str(e)
        return
    o = oracle.OrbOracle(nf, sf, nl, ini, mn)
    for b in range(3):
        _assert_same(kps[b, :n[b]], desc[b, :n[b]], *o.extract(frames[b]), what=f"frame {b}")


def _quadtree_smem(n, n_ini):
    """Shared memory of k_quadtree for a per-level quota n and n_ini root nodes: the node pool (28-byte QNode), the bitonic
    sort region (a power of two of 8-byte keys), the 6-byte free-list and link entries, 64 bytes of counters."""
    pool = (n + 4 * n_ini + 25) & ~1
    p2 = 1
    while p2 < pool:
        p2 <<= 1
    return pool * 28 + p2 * 8 + pool * 6 + 64


def test_quota_over_shared_memory_is_refused():
    """A per-level quota whose quadtree does not fit the device's opt-in shared memory per block is refused at creation with
    PL_ERR_ARG, and the message names the largest quota that fits.  One level of a 640x480 frame has one quadtree root."""
    import torch
    limit = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    assert _quadtree_smem(4800, 1) == 229752 and _quadtree_smem(5000, 1) == 236552
    fit = max(n for n in range(1, 8192) if _quadtree_smem(n, 1) <= limit)
    assert _quadtree_smem(5000, 1) > limit
    with pytest.raises(pl.PLError, match=rf"error -1: .*quota of 5000 .* at most {fit} features"):
        pl.ORBextractor(5000, 1.2, 1, 20, 7)
    with pytest.raises(pl.PLError, match=rf"error -1: .*quota of 5000 .* at most {fit} features"):
        pl.Frontend(640, 480, max_batch=1, orb=(5000, 1.2, 1, 20, 7))
    with pytest.raises(pl.PLError, match=rf"error -1: .*quota of {fit + 1} "):
        pl.ORBextractor(fit + 1, 1.2, 1, 20, 7)
    # the largest quota that fits runs, and equals the oracle
    img = synth.synth_frame(640, 480, 3)
    kps, desc = pl.ORBextractor(fit, 1.2, 1, 20, 7)(img)
    _assert_same(kps, desc, *oracle.OrbOracle(fit, 1.2, 1, 20, 7).extract(img))


def test_matcher_capacities_are_refused_at_creation():
    """A front end whose keypoint capacity (nfeatures + 4 * nlevels) is over the matchers' 6144, or whose line capacity is over
    what the line matcher's shared memory holds, is refused at creation with a message naming the limit; 6144 - 4 * nlevels
    features are accepted."""
    from test_match_batched_gpu import _search_double_limit
    with pytest.raises(pl.PLError, match=r"error -1: .*keypoint capacity of 7032, over the matchers' 6144; at most 6112 features fit at 8 levels"):
        pl.Frontend(640, 480, max_batch=1, orb=(7000, 1.2, 8, 20, 7))
    with pytest.raises(pl.PLError, match=r"error -1: .*at most 6104 features fit at 10 levels"):
        pl.Frontend(640, 480, max_batch=1, orb=(6105, 1.2, 10, 20, 7))
    fe = pl.Frontend(640, 480, max_batch=1, orb=(6112, 1.2, 8, 20, 7))
    del fe
    fit = _search_double_limit()
    with pytest.raises(pl.PLError, match=rf"error -1: .* at most {fit} lines per side"):
        pl.Frontend(640, 480, max_batch=1, lines=(fit, 0.0))


def _frontend_tracking_step(w, h, nf, sfac, nl, ini, mn):
    """One front-end step of 3 frames at a w x h frame with ORB at (nf, sfac, nl, ini, mn), the TUM1 camera scaled to the frame
    (distorting) and the tracking stage; every output equals the oracle's on the same inputs, as in
    test_frontend_gpu.test_tracking_stage_matches_oracle.  Returns the front end's outputs."""
    B = 3
    K, D = synth.TUM1_K, synth.TUM1_DIST
    if (w, h) != (640, 480):
        K = tuple(float(v) for v in np.array(K) * (w / 640, h / 480, w / 640, h / 480))
    # hd: the VGA sequence scaled up, whose smoother texture keeps LSD under the front end's 8192 segments per frame (a native
    # 1920 x 1080 synthetic frame gives over 13000) while ORB still finds its 5000 keypoints
    frames = synth.synth_sequence(B, 640, 480, seed=14)
    if (w, h) != (640, 480):
        frames = np.stack([oracle.resize_linear_u8(f, w, h) for f in frames])
    problems = [synth.synth_pose_problem(130 + k, K=K, w=w, h=h) for k in range(B)]
    for p in problems[1:]:
        p["K"] = problems[0]["K"]
    fe = pl.Frontend(w, h, max_batch=B, orb=(nf, sfac, nl, ini, mn), lm_caps=(320, 88))
    fe.set_camera(K, D)
    fe.set_wrap(True)
    fe.set_pose_problems(problems)
    fe.set_tracking(True)
    out = fe.run(frames)
    ku = fe.fetch_keys_un(B)
    t0, t1 = fe.fetch_tracking(B, 0), fe.fetch_tracking(B, 1)
    o = oracle.OrbOracle(nf, sfac, nl, ini, mn)
    sf = o.tables()["scale"]
    assert len(sf) == nl
    bounds = oracle.image_bounds(K, D, w, h)
    Kp = np.asarray(problems[0]["K"], np.float32)
    for b in range(B):
        okps, odesc = o.extract(frames[b])
        n = out["n"][b]
        _assert_same(out["kps"][b, :n], out["desc"][b, :n], okps, odesc, what=f"frame {b}")
        assert ku[b, :n].tobytes() == oracle.undistort_keypoints(okps, K, D).tobytes()
        okl, oldesc, _ = oracle.line_extract(oracle.undistort_remap(frames[b], K, D))
        nl_b = out["nl"][b]
        assert nl_b == len(okl) and out["keylines"][b, :nl_b].tobytes() == okl.tobytes()
    searched = 0
    for b in range(B):
        a = (b - 1) % B
        n, npv = out["n"][b], out["n"][a]
        ck, cd, pk, pd = ku[b, :n], out["desc"][b, :n], ku[a, :npv], out["desc"][a, :npv]
        T = np.asarray(problems[b]["Tcw0"], np.float32).reshape(4, 4)
        pos = t0["map_pos"][b, :npv]
        valid = np.ones(npv, np.uint8)
        nm, m = oracle.search_by_projection_last(ck, cd, bounds, T, Kp, sf, valid, pos, pd, out["kps"][a, :npv]["octave"],
                                                 pk["angle"], 15.0, True)
        if nm < 20:
            nm, m = oracle.search_by_projection_last(ck, cd, bounds, T, Kp, sf, valid, pos, pd, out["kps"][a, :npv]["octave"],
                                                     pk["angle"], 30.0, True)
        assert t0["n_pt"][b] == nm and np.array_equal(t0["pt_match"][b, :n], m), b
        view = valid.copy(); view[m[m >= 0]] = 0
        assert np.array_equal(t1["pt_in_view"][b, :npv], view)
        nm2, m2 = oracle.search_by_projection_points(ck, cd, bounds, sf, view, np.stack([pk["x"], pk["y"]], 1), pk["octave"],
                                                     np.ones(npv, np.float32), pd, 1.0, 0.8, (m >= 0).astype(np.uint8))
        assert t1["n_pt"][b] == nm2 and np.array_equal(t1["pt_match"][b, :n], m2), b
        searched += nm + nm2
    assert searched > 100
    return out


def test_frontend_tracking_at_a_non_default_orb_setting():
    """ORB at (1500, 1.1, 10, 12, 5): the extractor's level count and scale table reach the projection searches (their window
    radius th * scale[octave])."""
    out = _frontend_tracking_step(640, 480, 1500, 1.1, 10, 12, 5)
    # keypoints on levels past the TUM setting's 8 take part in the matches
    assert any((out["kps"][b, :out["n"][b]]["octave"] >= 8).any() for b in range(3))


def test_frontend_tracking_past_the_packed_grid():
    """1920 x 1080 with 5000 features: over 2048 keypoints per frame, so SearchForInitialization and the tracking searches of
    the front end's batched chain run on the grid whose items are plain keypoint indices."""
    out = _frontend_tracking_step(1920, 1080, 5000, 1.2, 8, 20, 7)
    assert out["n"].min() > 2048
