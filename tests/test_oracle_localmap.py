"""CPU tests of the LocalMapping matcher oracles (SURVEY.md §8f.2): ORBmatcher::SearchForTriangulation
(src/ORBmatcher.cc:720-911) and the search half of ORBmatcher::Fuse (:914-1034).  The reference has no fixtures for these;
the pins are known-answer geometry (matches must join the two views of the same 3-D point) and the literal quirks."""
import numpy as np
import oracle
from plslam_b200 import synth


def _tri(s, ori=True, **over):
    a, b = dict(s["1"]), dict(s["2"])
    a.update(over.get("a", {})); b.update(over.get("b", {}))
    return oracle.search_for_triangulation(a["keys"], a["desc"], a["has_mp"], b["keys"], b["desc"], b["has_mp"], a["fv"], b["fv"],
                                           over.get("F12", s["F12"]), s["Cw1"], b["R"], b["t"], s["K"], s["scale_factors"],
                                           s["level_sigma2"], ori)


def test_triangulation_matches_join_the_same_point():
    s = synth.synth_two_view(5)
    a, b = s["1"], s["2"]
    nm, m = _tri(s, True)
    ok = m >= 0
    assert nm == ok.sum() > 300
    assert (a["pt_id"][ok] == b["pt_id"][m[ok]]).all() and (a["pt_id"][ok] >= 0).all()
    assert not a["has_mp"][ok].any() and not b["has_mp"][m[ok]].any()          # only untracked keypoints are paired
    nm0, m0 = _tri(s, False)
    assert nm0 > nm and ((m == m0) | (m == -1)).all()                            # the rotation histogram only removes


def test_triangulation_respects_the_epipolar_constraint():
    s = synth.synth_two_view(7)
    nm, _ = _tri(s, False)
    F = s["F12"].copy(); F[2, 2] += 0.5                                          # a wrong fundamental matrix kills the matches
    nm_bad, _ = _tri(s, False, F12=F)
    assert nm_bad < nm // 10


def test_triangulation_quirks():
    """vbMatched2 is never set in this reference (ORBmatcher.cc:846-863): two keypoints of KF1 may take the same idx2; and
    among equal distances the LAST candidate of the node wins (dist > bestDist is the rejection test, :819)."""
    s = synth.synth_two_view(9, n_pts=40, n_clutter=0)
    a, b = s["1"], s["2"]
    i1 = int(np.nonzero(a["pt_id"] >= 0)[0][0]); pid = a["pt_id"][i1]
    j = int(np.nonzero(b["pt_id"] == pid)[0][0])
    ka = np.concatenate([a["keys"], a["keys"][i1:i1 + 1]]); da = np.concatenate([a["desc"], a["desc"][i1:i1 + 1]])
    kb = np.concatenate([b["keys"], b["keys"][j:j + 1]]); db = np.concatenate([b["desc"], b["desc"][j:j + 1]])
    fva = {0: [i1, len(ka) - 1]}; fvb = {0: [j, len(kb) - 1]}                    # the copy of j comes last in the node
    nm, m = oracle.search_for_triangulation(ka, da, np.zeros(len(ka), np.uint8), kb, db, np.zeros(len(kb), np.uint8), fva, fvb,
                                            s["F12"], s["Cw1"], b["R"], b["t"], s["K"], s["scale_factors"], s["level_sigma2"], False)
    assert nm == 2 and m[i1] == len(kb) - 1 and m[-1] == len(kb) - 1


def test_fuse_search_known_answers():
    f = synth.synth_fuse_problem(6)
    args = (f["keys"], f["desc"], f["bounds"], f["Tcw"], f["Ow"], f["K"], f["scale_factors"], f["inv_level_sigma2"],
            f["log_scale_factor"], f["skip"], f["pos"], f["normal"], f["min_dist"], f["max_dist"], f["mp_desc"], 3.0)
    bi, bd = oracle.fuse_search(*args)
    assert (bi[f["skip"] > 0] == -1).all() and (bd[f["skip"] > 0] == 256).all()
    good = bd <= 50
    assert good.sum() > 50
    # a fused keypoint lies within the search radius, on the predicted level or the one below, and carries the point's code
    T = f["Tcw"].astype(np.float64); Pc = f["pos"][good].astype(np.float64) @ T[:3, :3].T + T[:3, 3]
    u = f["K"][0] * Pc[:, 0] / Pc[:, 2] + f["K"][2]; v = f["K"][1] * Pc[:, 1] / Pc[:, 2] + f["K"][3]
    kp = f["keys"][bi[good]]
    d3 = np.linalg.norm(f["pos"][good] - f["Ow"], axis=1)
    lvl = np.clip(np.ceil(np.log(f["max_dist"][good] / d3) / np.log(1.2)), 0, 7)
    assert (np.abs(kp["x"] - u) < 3.0 * f["scale_factors"][lvl.astype(int)] + 1e-3).all()
    assert ((kp["octave"] == lvl) | (kp["octave"] == lvl - 1)).mean() > 0.99
    ham = np.unpackbits(f["desc"][bi[good]] ^ f["mp_desc"][good], axis=1).sum(1)
    assert np.array_equal(ham, bd[good])
    # th scales the window: a tiny radius finds (almost) nothing
    bi2, bd2 = oracle.fuse_search(*args[:-1], 0.05)
    assert (bd2 <= 50).sum() < good.sum() // 5


def test_lsd_search_for_triangulation_semantics():
    """= FrameBFMatch both ways at TH_HIGH (80) + mutual check + MapLine filter (LSDmatcher.cpp:744-763)."""
    rng = np.random.default_rng(3)
    base = rng.integers(0, 256, (60, 32), dtype=np.uint8)
    d1 = base.copy(); d2 = base[rng.permutation(60)][:50].copy()
    for d in (d1, d2):
        flips = rng.integers(0, 256, (len(d), 10))
        for j in range(10):
            d[np.arange(len(d)), flips[:, j] // 8] ^= (1 << (flips[:, j] % 8)).astype(np.uint8)
    ml1 = (rng.random(60) < 0.2).astype(np.uint8); ml2 = (rng.random(50) < 0.2).astype(np.uint8)
    f12 = oracle.frame_bf_match(d1, d2, 80.0, 0.8); f21 = oracle.frame_bf_match(d2, d1, 80.0, 0.8)
    nm, m = oracle.lsd_search_for_triangulation(d1, ml1, d2, ml2, 0.8, True)
    want = np.array([j if j >= 0 and f21[j] == i and not ml1[i] and not ml2[j] else -1 for i, j in enumerate(f12)])
    assert nm == (want >= 0).sum() > 10 and np.array_equal(m, want)
    nm1, m1 = oracle.lsd_search_for_triangulation(d1, ml1, d2, ml2, 0.8, False)
    want1 = np.array([j if j >= 0 and not ml1[i] and not ml2[j] else -1 for i, j in enumerate(f12)])
    assert nm1 >= nm and np.array_equal(m1, want1)
    assert oracle.lsd_search_for_triangulation(d1[:0], ml1[:0], d2, ml2)[0] == 0


def test_search_by_bow_known_answers():
    """ORBmatcher::SearchByBoW: matches join the two observations of a point; a frame feature is given away once."""
    s = synth.synth_two_view(5)
    a, b = s["1"], s["2"]
    nm, m = oracle.search_by_bow(a["keys"], a["desc"], a["has_mp"], b["keys"], b["desc"], a["fv"], b["fv"], 0.7, True)
    ok = m >= 0
    assert nm == ok.sum() > 150
    assert (a["pt_id"][m[ok]] == b["pt_id"][ok]).mean() > 0.99 and a["has_mp"][m[ok]].all()
    assert len(np.unique(m[ok])) >= ok.sum() - 2            # (a KF feature may serve two frame features only via duplicates)
    nm0, m0 = oracle.search_by_bow(a["keys"], a["desc"], a["has_mp"], b["keys"], b["desc"], a["fv"], b["fv"], 0.7, False)
    assert nm0 >= nm and ((m == m0) | (m == -1)).all()
    # "already matched" frame features are skipped by later keyframe features of the node: two identical KF features,
    # one frame feature -> the first takes it, the second finds nothing
    k = a["keys"][:2].copy(); d = np.repeat(a["desc"][:1], 2, 0)
    nm2, m2 = oracle.search_by_bow(k, d, [1, 1], k[:1], d[:1], {0: [0, 1]}, {0: [0]}, 0.7, False)
    assert nm2 == 1 and m2[0] == 0


def _reloc_args(seed, th=10.0, dist=100, n_kp=1800):
    f = synth.synth_fuse_problem(seed, n_kp=n_kp)
    rng = np.random.default_rng(seed)
    ang = rng.uniform(0, 360, len(f["pos"])).astype(np.float32)
    k = f["keys"].copy(); k["angle"] = rng.uniform(0, 360, len(k))
    valid = 1 - f["skip"]
    pre = (rng.random(len(k)) < 0.1).astype(np.uint8)
    return (k, f["desc"], f["bounds"], f["Tcw"], f["Ow"], f["K"], f["scale_factors"], f["log_scale_factor"], valid, f["pos"], f["mp_desc"],
            f["min_dist"], f["max_dist"], ang, th, dist), pre


def test_search_by_projection_keyframe_semantics():
    """Relocalisation overload (ORBmatcher.cc:1587-1716): matches respect the preassigned slots, the ORBdist gate and the window."""
    args, pre = _reloc_args(6)
    nm, m = oracle.search_by_projection_keyframe(*args, False, pre)
    assert nm == (m >= 0).sum() > 30 and (m[pre > 0] == -2).all()
    k, desc, mp_desc = args[0], args[1], args[10]
    i2 = np.nonzero(m >= 0)[0]
    ham = np.unpackbits(desc[i2] ^ mp_desc[m[i2]], axis=1).sum(1)
    assert ham.max() <= 100 and len(np.unique(m[i2])) == len(i2)
    nm64, m64 = oracle.search_by_projection_keyframe(*args[:-1], 64, False, pre)
    assert nm64 <= nm
    nmo, mo = oracle.search_by_projection_keyframe(*args, True, pre)
    assert nmo <= nm and ((mo == m) | (mo == -1)).all()


def test_search_by_bow_keyframes_known_answers():
    s = synth.synth_two_view(5)
    a, b = s["1"], s["2"]
    mp1 = 1 - a["has_mp"]; mp2 = 1 - b["has_mp"]                   # most features carry a MapPoint in a loop-closing keyframe
    nm, m = oracle.search_by_bow_keyframes(a["keys"], a["desc"], mp1, b["keys"], b["desc"], mp2, a["fv"], b["fv"], 0.75, True)
    ok = m >= 0
    assert nm == ok.sum() > 150 and (a["pt_id"][ok] == b["pt_id"][m[ok]]).mean() > 0.99
    assert mp1[ok].all() and mp2[m[ok]].all() and len(np.unique(m[ok])) == ok.sum()         # vbMatched2: idx2 used once
