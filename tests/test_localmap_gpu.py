"""GPU parity tests of the LocalMapping matchers (SURVEY.md §8f.2) through the C ABI vs the oracle: bit-exact indices."""
import numpy as np
import pytest
import oracle
import plslam_b200 as pl
from plslam_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed,ori", [(5, True), (5, False), (7, True), (11, True), (12, False)])
def test_search_for_triangulation(seed, ori):
    s = synth.synth_two_view(seed)
    a, b = s["1"], s["2"]
    args = (a["keys"], a["desc"], a["has_mp"], b["keys"], b["desc"], b["has_mp"], a["fv"], b["fv"], s["F12"], s["Cw1"], b["R"], b["t"],
            s["K"], s["scale_factors"], s["level_sigma2"])
    onm, om = oracle.search_for_triangulation(*args, ori)
    nm, m = pl.ORBmatcher(0.6, ori).SearchForTriangulation(*args)
    assert onm > 200 and nm == onm and np.array_equal(m, om)


def test_search_for_triangulation_edge_cases():
    s = synth.synth_two_view(3, n_pts=60, n_clutter=10)
    a, b = s["1"], s["2"]
    base = [a["keys"], a["desc"], a["has_mp"], b["keys"], b["desc"], b["has_mp"], a["fv"], b["fv"], s["F12"], s["Cw1"], b["R"], b["t"],
            s["K"], s["scale_factors"], s["level_sigma2"]]
    M = pl.ORBmatcher(0.6, True)
    # no shared node / empty feature vectors / every keypoint already tracked
    for fv1, fv2 in (({1: [0, 1]}, {2: [0, 1]}), ({}, {}), (a["fv"], {})):
        x = list(base); x[6], x[7] = fv1, fv2
        nm, m = M.SearchForTriangulation(*x)
        assert nm == 0 and (m == -1).all() and oracle.search_for_triangulation(*x, True)[0] == 0
    x = list(base); x[2] = np.ones(len(a["keys"]), np.uint8)
    assert M.SearchForTriangulation(*x)[0] == 0
    # degenerate F (den == 0 for every keypoint): nothing passes CheckDistEpipolarLine
    x = list(base); x[8] = np.zeros((3, 3), np.float32)
    nm, m = M.SearchForTriangulation(*x)
    assert nm == 0 == oracle.search_for_triangulation(*x, True)[0]
    with pytest.raises(pl.PLError):
        y = list(base); y[6] = {0: [len(a["keys"]) + 5]}; y[7] = {0: [0]}
        M.SearchForTriangulation(*y)


FUSE_CASES = [(6, 3.0, 1800), (8, 3.0, 1800), (9, 1.0, 1800), (10, 6.0, 1800), (13, 3.0, 2049), (14, 3.0, 4000), (15, 6.0, 7000)]


# the keypoint count joins a case's id past 1800: up to 2048 the grid keeps each octave beside its keypoint's index, above it not
@pytest.mark.parametrize("seed,th,n_kp", FUSE_CASES, ids=[f"{s}-{t}" + (f"-{n}" if n != 1800 else "") for s, t, n in FUSE_CASES])
def test_fuse_search(seed, th, n_kp):
    f = synth.synth_fuse_problem(seed, n_kp=n_kp)
    args = (f["keys"], f["desc"], f["bounds"], f["Tcw"], f["Ow"], f["K"], f["scale_factors"], f["inv_level_sigma2"],
            f["log_scale_factor"], f["skip"], f["pos"], f["normal"], f["min_dist"], f["max_dist"], f["mp_desc"], th)
    obi, obd = oracle.fuse_search(*args)
    bi, bd = pl.ORBmatcher().FuseSearch(*args)
    assert (obd <= 50).sum() > 20
    assert np.array_equal(bi, obi) and np.array_equal(bd, obd)
    # no skip list; no map points
    a2 = list(args); a2[9] = None
    o2 = oracle.fuse_search(*a2); g2 = pl.ORBmatcher().FuseSearch(*a2)
    assert np.array_equal(g2[0], o2[0]) and np.array_equal(g2[1], o2[1])
    a3 = list(args)
    for k in (9, 10, 11, 12, 13, 14):
        a3[k] = a3[k][:0]
    assert len(pl.ORBmatcher().FuseSearch(*a3)[0]) == 0


@pytest.mark.parametrize("seed,dbl", [(1, True), (2, True), (3, False)])
def test_lsd_search_for_triangulation(seed, dbl):
    f = synth.synth_sequence(2, 640, 480, seed=seed)
    (_, d1, _), (_, d2, _) = oracle.line_extract(f[0]), oracle.line_extract(f[1])
    rng = np.random.default_rng(seed)
    ml1 = (rng.random(len(d1)) < 0.25).astype(np.uint8); ml2 = (rng.random(len(d2)) < 0.25).astype(np.uint8)
    onm, om = oracle.lsd_search_for_triangulation(d1, ml1, d2, ml2, 0.8, dbl)
    nm, m = pl.LSDmatcher(0.8).SearchForTriangulation(d1, ml1, d2, ml2, dbl)
    assert onm > 10 and nm == onm and np.array_equal(m, om)
    onm2, om2 = oracle.lsd_search_for_triangulation(d1, ml1, d2, ml2, 0.8, True, 50.0)     # the pair<> overload: TH_LOW, mutual
    nm2, m2 = pl.LSDmatcher(0.8).SearchForTriangulation(d1, ml1, d2, ml2, True, th=50)
    assert nm2 == onm2 and np.array_equal(m2, om2) and onm2 <= onm + 200
    assert pl.LSDmatcher(0.8).SearchForTriangulation(d1[:0], ml1[:0], d2, ml2)[0] == 0


@pytest.mark.parametrize("seed,ori,ratio", [(5, True, 0.7), (5, False, 0.7), (7, True, 0.9), (11, True, 0.6), (12, False, 0.75)])
def test_search_by_bow(seed, ori, ratio):
    s = synth.synth_two_view(seed)
    a, b = s["1"], s["2"]
    args = (a["keys"], a["desc"], a["has_mp"], b["keys"], b["desc"], a["fv"], b["fv"])
    onm, om = oracle.search_by_bow(*args, ratio, ori)
    nm, m = pl.ORBmatcher(ratio, ori).SearchByBoW(*args)
    assert onm > 100 and nm == onm and np.array_equal(m, om)
    # big nodes (more candidates than lanes) and empty inputs
    fv1 = {0: [i for v in a["fv"].values() for i in v]}; fv2 = {0: [i for v in b["fv"].values() for i in v]}
    onm, om = oracle.search_by_bow(a["keys"], a["desc"], a["has_mp"], b["keys"], b["desc"], fv1, fv2, ratio, ori)
    nm, m = pl.ORBmatcher(ratio, ori).SearchByBoW(a["keys"], a["desc"], a["has_mp"], b["keys"], b["desc"], fv1, fv2)
    assert nm == onm and np.array_equal(m, om)
    assert pl.ORBmatcher(ratio, ori).SearchByBoW(a["keys"], a["desc"], a["has_mp"], b["keys"], b["desc"], {}, b["fv"])[0] == 0


RELOC_CASES = [(6, 10.0, 100, True, 1800), (8, 3.0, 64, True, 1800), (9, 10.0, 100, False, 1800), (10, 3.0, 64, False, 1800),
               (13, 10.0, 100, True, 2049), (14, 3.0, 64, False, 6144)]


@pytest.mark.parametrize("seed,th,dist,ori,n_kp", RELOC_CASES,
                         ids=[f"{s}-{t}-{d}-{o}" + (f"-{n}" if n != 1800 else "") for s, t, d, o, n in RELOC_CASES])
def test_search_by_projection_keyframe(seed, th, dist, ori, n_kp):
    from test_oracle_localmap import _reloc_args
    args, pre = _reloc_args(seed, th, dist, n_kp)
    onm, om = oracle.search_by_projection_keyframe(*args, ori, pre)
    nm, m = pl.ORBmatcher(0.9, ori).SearchByProjectionKeyFrame(*args, pre)
    assert onm > 10 and nm == onm and np.array_equal(m, om)
    onm, om = oracle.search_by_projection_keyframe(*args, ori, None)
    nm, m = pl.ORBmatcher(0.9, ori).SearchByProjectionKeyFrame(*args, None)
    assert nm == onm and np.array_equal(m, om)


@pytest.mark.parametrize("seed,ori,ratio", [(5, True, 0.75), (7, False, 0.75), (11, True, 0.6)])
def test_search_by_bow_keyframes(seed, ori, ratio):
    s = synth.synth_two_view(seed)
    a, b = s["1"], s["2"]
    args = (a["keys"], a["desc"], 1 - a["has_mp"], b["keys"], b["desc"], 1 - b["has_mp"], a["fv"], b["fv"])
    onm, om = oracle.search_by_bow_keyframes(*args, ratio, ori)
    nm, m = pl.ORBmatcher(ratio, ori).SearchByBoWKeyFrames(*args)
    assert onm > 100 and nm == onm and np.array_equal(m, om)
