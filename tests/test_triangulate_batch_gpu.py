"""pl_orb_triangulate_dev on the GPU: the device call equals the oracle (tests/cnmp_oracle.py) bit for bit - codes, x3D bits, nnew
and status - on a mixed batch; pl_orb_search_for_triangulation_dev followed by pl_orb_triangulate_dev on
tests/golden/refcalls/create_new_map_points.npz reproduces the reference's own CreateNewMapPoints loop; a CUDA-graph replay of
search + triangulation equals the eager launches; the call holds no device memory.  DESIGN.md §8f.5 names the mutant each test
catches."""
import numpy as np
import pytest

import plslam_b200 as pl
import cnmp_fixture as cf
import cnmp_oracle as co
from test_triangulate_batch import degenerate_keyframes

pytestmark = pytest.mark.gpu
FILL = co.UNWRITTEN


def _F12(kfs, a, b):
    """LocalMapping::ComputeF12(KF a, KF b) in fp64"""
    Ta, Tb = (np.asarray(kfs[i]["Tcw"], np.float64).reshape(4, 4) for i in (a, b))
    Km = lambda k: np.array([[k[0], 0, k[2]], [0, k[1], k[3]], [0, 0, 1]], np.float64)
    R12 = Ta[:3, :3] @ Tb[:3, :3].T; t12 = -R12 @ Tb[:3, 3] + Ta[:3, 3]
    tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]])
    return np.linalg.inv(Km(kfs[a]["K"])).T @ tx @ R12 @ np.linalg.inv(Km(kfs[b]["K"]))


def _device(b, scale_factor):
    b.run()
    b.triangulate(scale_factor=scale_factor)
    return b.results(), b.triangulated()


def _oracle(b, s, scale_factor):
    """The oracle on the search outputs the device holds"""
    m12 = b.outputs["matches"].cpu().numpy()[:max(b.host["q"]["n_out"], 1)]
    ss = b.outputs["status"].cpu().numpy()[:b.P]
    return co.triangulate(b.host["k"], b.host["q"], m12, ss, scale_factor, s["scale_factors"], s["level_sigma2"])


def _assert_equal(b, oracle_out):
    code, x3D, nnew, status = oracle_out
    n_out = b.host["q"]["n_out"]
    h = {k: v.cpu().numpy() for k, v in b.outputs.items()}
    assert np.array_equal(h["tri_status"][:b.P], status)
    assert np.array_equal(h["code"][:n_out], code)
    assert np.array_equal(h["x3D"][:n_out].view(np.uint32), x3D.view(np.uint32))
    assert np.array_equal(np.where(status == 0, h["nnew"][:b.P], -1), nnew)
    assert (h["nnew"][:b.P][status != 0] == FILL).all()


def test_search_then_triangulate_reproduces_the_reference_loop():
    s = cf.load()
    kfs, probs = cf.keyframes(s), cf.problems(s)
    b = pl.TriangulationProblems(kfs, probs, (s["scale_factors"], s["level_sigma2"]), options=0, out_fill=FILL)
    res, tri = _device(b, s["scale_factor"])
    assert all(r["status"] == 0 for r in res + tri)
    rows, X = [], []
    for (_, j, _), r, t in zip(probs, res, tri):
        i1 = np.nonzero(t["code"] == co.COMMITTED)[0]
        rows += [(j, int(i), int(r["matches"][i])) for i in i1]
        X.append(t["x3D"][i1])
        assert t["nnew"] == len(i1)
    ref_new, ref_X = cf.reference(s)
    assert np.array_equal(np.array(rows, np.int32), ref_new)
    assert np.array_equal(np.concatenate(X).view(np.uint32), ref_X)
    _assert_equal(b, _oracle(b, s, s["scale_factor"]))


def _mixed():
    """Two current keyframes (0 and 1 of the fixture, different intrinsics) against several neighbours, a degenerate pair whose
    x3D[3] is 0, a keyframe without keypoints on either side, a problem the search refused (kf2 outside the table), a problem with
    one matches12 entry past KF2's keypoints, and a problem whose pairs are replaced by arbitrary ones (every gate)."""
    s = cf.load()
    kfs = cf.keyframes(s) + degenerate_keyframes()
    empty = dict(kfs[0], keys=kfs[0]["keys"][:0], desc=kfs[0]["desc"][:0], has_mp=kfs[0]["has_mp"][:0], fv={})
    kfs.append(empty)                                                   # 11
    probs = cf.problems(s)                                              # 0 .. 6: current keyframe 0
    probs += [(1, j, _F12(kfs, 1, j)) for j in (2, 4, 7, 8)]            # 7 .. 10: current keyframe 1
    probs += [(9, 10, np.zeros((3, 3))), (11, 0, _F12(kfs, 0, 1)), (0, 11, _F12(kfs, 0, 1)), (0, 99, _F12(kfs, 0, 1)),
              (0, 2, _F12(kfs, 0, 2)), (0, 3, _F12(kfs, 0, 3))]        # 11 .. 16
    return s, kfs, probs


def _edit_matches(b, kfs):
    """On the device, between the two calls: the degenerate pair, an out-of-range entry in problem 15, arbitrary pairs in 16"""
    q = b.host["q"]
    m = b.outputs["matches"]
    m[int(q["out_offset"][11])] = 0
    m[int(q["out_offset"][15]) + 7] = len(kfs[2]["keys"])
    rng = np.random.default_rng(9)
    a, n1, n2 = int(q["out_offset"][16]), len(kfs[0]["keys"]), len(kfs[3]["keys"])
    r = rng.integers(-1, n2, n1).astype(np.int32)
    import torch
    m[a:a + n1] = torch.from_numpy(r).cuda()


def test_mixed_batch_equals_the_oracle():
    s, kfs, probs = _mixed()
    b = pl.TriangulationProblems(kfs, probs, (s["scale_factors"], s["level_sigma2"]), options=0, out_fill=FILL)
    b.run()
    _edit_matches(b, kfs)
    b.triangulate(scale_factor=s["scale_factor"])
    tri = b.triangulated()
    assert [t["status"] for t in tri[11:]] == [0, 0, 0, 1, 4, 0]
    assert tri[11]["code"].tolist() == [co.W_ZERO]
    assert tri[12]["code"].size == 0 and tri[12]["nnew"] == 0
    assert (tri[13]["code"] == co.NO_PAIR).all() and tri[13]["nnew"] == 0
    assert (tri[15]["code"] == FILL).all() and tri[15]["nnew"] == FILL
    codes = set(np.concatenate([t["code"] for t in tri]).tolist())
    assert set(range(-1, 9)) <= codes, sorted(codes)
    _assert_equal(b, _oracle(b, s, s["scale_factor"]))


def test_reprojection_knife_edge_equals_the_oracle():
    """Every pair that reaches KF1's reprojection gate misses it by less than one rounding of its squared error
    (cnmp_fixture.knife_edge): an error off by one ulp anywhere in the reprojection chain changes codes."""
    s = cf.load()
    kfs, probs, sf, s2, code = cf.knife_edge(s)
    assert (code == co.REPROJ1).sum() > 300
    b = pl.TriangulationProblems(kfs, probs, (sf, s2), options=0, out_fill=FILL)
    b.run()
    b.triangulate(scale_factor=s["scale_factor"])
    b.triangulated()
    _assert_equal(b, _oracle(b, dict(scale_factors=sf, level_sigma2=s2), s["scale_factor"]))
    assert np.array_equal(b.outputs["code"].cpu().numpy()[:len(code)], code)


def test_single_level_table_takes_the_scale_factor_as_an_argument():
    s = cf.load()
    kfs, probs = cf.keyframes(s), cf.problems(s)[:3]
    for k in kfs:
        k["keys"] = k["keys"].copy(); k["keys"]["octave"] = 0
    sf, ls2 = np.ones(1, np.float32), np.ones(1, np.float32)
    b = pl.TriangulationProblems(kfs, probs, (sf, ls2), options=0, out_fill=FILL)
    b.run()
    b.triangulate(scale_factor=1.2)
    b.triangulated()
    m12 = b.outputs["matches"].cpu().numpy()[:b.host["q"]["n_out"]]
    o = co.triangulate(b.host["k"], b.host["q"], m12, b.outputs["status"].cpu().numpy()[:b.P], 1.2, sf, ls2)
    _assert_equal(b, o)
    assert (o[0] == co.COMMITTED).any()


def test_graph_replay_equals_eager():
    import torch
    s, kfs, probs = _mixed()
    probs = probs[:11] + probs[12:15]
    b = pl.TriangulationProblems(kfs, probs, (s["scale_factors"], s["level_sigma2"]), options=0, out_fill=FILL)
    _device(b, s["scale_factor"])
    eager = {k: v.cpu().numpy().copy() for k, v in b.outputs.items()}
    for k, t in b.outputs.items():
        t.fill_(float("nan") if k == "x3D" else FILL)
    st = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        b.run(st)
        b.triangulate(st, scale_factor=s["scale_factor"])
    torch.cuda.synchronize()
    assert (b.outputs["code"] == FILL).all()                # capturing runs nothing
    g.replay()
    torch.cuda.synchronize()
    for k, v in b.outputs.items():
        assert np.array_equal(v.cpu().numpy().view(np.uint8), eager[k].view(np.uint8)), k


def test_call_holds_no_device_memory():
    s = cf.load()
    b = pl.TriangulationProblems(cf.keyframes(s), cf.problems(s), (s["scale_factors"], s["level_sigma2"]), options=0)
    _device(b, s["scale_factor"])
    before = pl.device_bytes()
    for _ in range(3):
        b.run(); b.triangulate(scale_factor=s["scale_factor"])
    b.triangulated()
    assert pl.device_bytes() == before
