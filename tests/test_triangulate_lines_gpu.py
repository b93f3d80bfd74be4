"""pl_lsd_triangulate_dev on the GPU: after pl_lsd_search_for_triangulation_dev, the device call equals the oracle
(tests/cnml_oracle.py) bit for bit - codes, line3D bits, nnew and status - on a mixed batch; a CUDA-graph replay of search +
triangulation equals the eager launches; the call holds no device memory.  DESIGN.md §8f.6 names the mutant each test catches."""
import numpy as np
import pytest

import plslam_b200 as pl
import cnml_oracle as co
import cnml_scene as cs

pytestmark = pytest.mark.gpu
FILL = co.UNWRITTEN
SEARCH = (80.0, 0.8, True)       # TH_HIGH, LSDmatcher's nnratio, isDouble (LocalMapping.cc:961)
N_DUP = 20


def _mixed():
    """kf 0 .. 7 of the scene and kf 8 = kf 0 with its first N_DUP keylines repeated at the end.  Groups: 0 the current keyframe
    with the positional shift and an entry without matches; 1 current keyframe 1 (other intrinsics); 2 an entry whose search
    refused its problem (kf2 outside the table); 3 kf_cur outside the table; 4 17 entries; 5 an entry whose problem has another
    kf1; 6 an entry whose matches hold one index past kf2's keylines; 7 kf 8 with the repeated keylines' matches copied from the
    originals (two ikl of one pair with the same idx1 and idx2)."""
    sc = cs.scene()
    kfs = list(sc["kfs"])
    k0 = kfs[0]
    kfs.append(dict(k0, ldesc=np.concatenate([k0["ldesc"], k0["ldesc"][:N_DUP]]),
                    has_ml=np.concatenate([k0["has_ml"], np.zeros(N_DUP, np.uint8)]),
                    keylines=np.concatenate([k0["keylines"], k0["keylines"][:N_DUP]]),
                    line_func=np.concatenate([k0["line_func"], k0["line_func"][:N_DUP]])))
    probs, at = [], {}

    def prob(a, b):
        probs.append((a, b)); return len(probs) - 1
    p0 = {j: prob(0, j) for j in cs.searched_neighbours()}
    p1 = {j: prob(1, j) for j in (0, 2, 4, 5, 6)}
    bad = prob(0, 99)
    ded = prob(0, 2)
    p8 = {j: prob(8, j) for j in (1, 2, 4, 5)}
    med = sc["medians"]
    g0 = cs.group(sc, p0)
    groups = [g0,
              dict(kf_cur=1, entries=[(p1[j], j, med[j]) for j in (0, 2, 4, 5, 6)]),
              dict(kf_cur=0, entries=[(p0[1], 1, med[1]), (bad, 2, med[2])]),
              dict(kf_cur=99, entries=[(p0[1], 1, med[1]), (p0[2], 2, med[2])]),
              dict(kf_cur=0, entries=[(p0[1], 1, med[1])] * 17),
              dict(kf_cur=1, entries=[(p1[0], 0, med[0]), (p0[2], 2, med[2])]),
              dict(kf_cur=0, entries=[(p0[1], 1, med[1]), (ded, 2, med[2])]),
              dict(kf_cur=8, entries=[(p8[j], j, med[j]) for j in (1, 2, 4, 5)])]
    at.update(ded=ded, p8=p8)
    return sc, kfs, probs, groups, at


def _batch(sc, kfs, probs, groups):
    return pl.TriangulationProblems(kfs, probs, sc["level_sigma2_line"], lines=True, options=SEARCH, out_fill=FILL, groups=groups)


def _edit_matches(b, kfs, at):
    q = b.host["q"]
    m = b.outputs["matches"]
    m[int(q["out_offset"][at["ded"]]) + 3] = len(kfs[2]["keylines"])
    n0 = len(kfs[0]["keylines"])
    for p in at["p8"].values():
        a = int(q["out_offset"][p])
        m[a + n0:a + n0 + N_DUP] = m[a:a + N_DUP].clone()
    import torch
    torch.cuda.synchronize()


def _oracle(b, sc, **kw):
    h = {k: v.cpu().numpy() for k, v in b.outputs.items()}
    q = b.host["q"]
    return co.triangulate_lines(b.host["k"], q, b.host["g"], h["matches"][:max(q["n_out"], 1)], h["nmatches"][:b.P],
                                h["status"][:b.P], sc["level_sigma2_line"], **kw)


def _assert_equal(b, o):
    code, line3D, nnew, status = o
    gr = b.host["g"]
    h = {k: v.cpu().numpy() for k, v in b.outputs.items()}
    assert np.array_equal(h["tri_status"][:gr["G"]], status)
    assert np.array_equal(h["code"][:gr["n_out"]], code)
    assert np.array_equal(h["line3D"][:gr["n_out"]].view(np.uint32), line3D.view(np.uint32))
    assert np.array_equal(np.where(status == 0, h["nnew"][:gr["G"]], -1), nnew)
    assert (h["nnew"][:gr["G"]][status != 0] == FILL).all()


def test_mixed_batch_equals_the_oracle():
    sc, kfs, probs, groups, at = _mixed()
    b = _batch(sc, kfs, probs, groups)
    b.run()
    _edit_matches(b, kfs, at)
    b.triangulate()
    tri = b.triangulated()
    assert [t["status"] for t in tri] == [0, 0, 1, 1, 2, 3, 4, 0]
    res = b.results()
    assert res[len(cs.searched_neighbours()) - 1]["nmatches"] == 0           # neighbour 7 sees nothing
    codes = set(np.concatenate([t["code"].ravel() for t in tri]).tolist())
    assert {-1, 0, 1, 2, 3, 5, 7, 8} <= codes, sorted(codes)
    assert (tri[7]["code"] == co.TAKEN).any()                                 # the repeated keylines lose to their originals
    assert all(t["nnew"] == int((t["code"] == co.COMMITTED).sum()) for t in tri if t["status"] == 0)
    o = _oracle(b, sc)
    _assert_equal(b, o)
    # the oracle's mutants differ from the device on this batch
    for kw in (dict(positional=False), dict(commit_state=False), dict(snapshot=False)):
        assert not np.array_equal(_oracle(b, sc, **kw)[0], o[0]), kw


def test_graph_replay_equals_eager():
    import torch
    sc, kfs, probs, groups, at = _mixed()
    b = _batch(sc, kfs, probs, groups[:2] + groups[7:])
    b.run(); b.triangulate()
    torch.cuda.synchronize()
    eager = {k: v.cpu().numpy().copy() for k, v in b.outputs.items()}
    for k, t in b.outputs.items():
        t.fill_(float("nan") if k == "line3D" else FILL)
    st = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        b.run(st)
        b.triangulate(st)
    torch.cuda.synchronize()
    assert (b.outputs["code"] == FILL).all()                # capturing runs nothing
    g.replay()
    torch.cuda.synchronize()
    for k, v in b.outputs.items():
        assert np.array_equal(v.cpu().numpy().view(np.uint8), eager[k].view(np.uint8)), k


def test_call_holds_no_device_memory():
    sc, kfs, probs, groups, at = _mixed()
    b = _batch(sc, kfs, probs, groups[:2])
    b.run(); b.triangulate(); b.triangulated()
    before = pl.device_bytes()
    for _ in range(3):
        b.run(); b.triangulate()
    b.triangulated()
    assert pl.device_bytes() == before


def test_search_then_triangulate_reproduces_the_reference_loop():
    """tests/golden/refcalls/create_new_map_lines.npz: the reference's searches and its :966-1439 loop (with cv2)"""
    import cnml_fixture as cf
    s = cf.load()
    kfs, probs = cf.keyframes(s), cf.problems(s)
    b = pl.TriangulationProblems(kfs, probs, s["level_sigma2_line"], lines=True, options=SEARCH, out_fill=FILL, groups=[cf.group(s)])
    b.run(); b.triangulate()
    res, tri = b.results(), b.triangulated()
    assert np.array_equal(np.concatenate([r["matches"] for r in res]), s["ref_matches"])
    assert [r["nmatches"] for r in res] == s["ref_nmatches"].tolist()
    assert tri[0]["status"] == 0
    rows, L = cf.created(tri[0]["code"].ravel(), tri[0]["line3D"].reshape(-1, 6), len(kfs[0]["keylines"]), len(probs),
                         lambda e: res[e]["matches"])
    assert np.array_equal(rows, s["ref_new"])
    assert np.array_equal(L.view(np.uint32), s["ref_line3D"].view(np.uint32))
    assert tri[0]["nnew"] == len(rows)
    _assert_equal(b, _oracle(b, dict(level_sigma2_line=s["level_sigma2_line"])))


def _edges():
    """Group 0: the knife-edge triples of cnml_scene.knife_edge (reprojection in view 1 at one rounding of 3.84 sigma^2, |Result|
    at 0.996, a tiny median depth on entry 1); group 1: cnml_scene.degenerate_svd (vt(3,3) == 0); group 2: keyframe 0 with each
    keyline twice in a row and both copies given the same matches, so that equal triples meet inside one 32-slot chunk."""
    sc = cs.scene()
    kk, m, s2 = cs.knife_edge(sc)
    dg = cs.degenerate_svd(sc)
    k0 = sc["kfs"][0]
    dup = dict(k0, ldesc=np.repeat(k0["ldesc"], 2, 0), has_ml=np.repeat(k0["has_ml"], 2), keylines=np.repeat(k0["keylines"], 2),
               line_func=np.repeat(k0["line_func"], 2, 0))
    kfs = kk + dg + [dup]
    probs = [(0, 1), (0, 2), (3, 4), (3, 5), (6, 1), (6, 2)]
    md = sc["medians"]
    groups = [dict(kf_cur=0, entries=[(0, 1, md[1]), (1, 2, np.float32(0.05))]), dict(kf_cur=3, entries=[(2, 4, 5.0), (3, 5, 5.0)]),
              dict(kf_cur=6, entries=[(4, 1, md[1]), (5, 2, md[2])])]
    matches = [m[0], m[1], np.zeros(1), np.zeros(1), np.repeat(m[0], 2), np.repeat(m[1], 2)]
    return kfs, probs, groups, s2, [np.asarray(x, np.int32) for x in matches]


def test_knife_edge_batch_equals_the_oracle():
    import torch
    kfs, probs, groups, s2, matches = _edges()
    b = pl.TriangulationProblems(kfs, probs, s2, lines=True, options=SEARCH, out_fill=FILL, groups=groups)
    b.run()
    b.outputs["matches"][:sum(len(x) for x in matches)] = torch.from_numpy(np.concatenate(matches)).cuda()
    b.outputs["nmatches"][:len(matches)] = torch.tensor([int((x >= 0).sum()) for x in matches], dtype=torch.int32).cuda()
    b.outputs["status"][:len(matches)] = 0
    torch.cuda.synchronize()
    b.triangulate()
    tri = b.triangulated()
    assert [t["status"] for t in tri] == [0, 0, 0]
    c0 = tri[0]["code"]
    assert (c0 == co.REPROJ1).sum() > 10 and (c0 == co.REPROJ2).any() and (c0 == co.REPROJ3).any() and (c0 == co.COMMITTED).sum() > 3
    assert tri[1]["code"].ravel().tolist() == [co.W_ZERO]
    c = tri[2]["code"][0]
    assert ((c[0::2] == co.COMMITTED) & (c[1::2] == co.TAKEN)).any()      # the second copy loses inside its chunk
    _assert_equal(b, _oracle(b, dict(level_sigma2_line=s2)))
