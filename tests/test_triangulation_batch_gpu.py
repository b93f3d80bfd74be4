"""pl_orb_search_for_triangulation_dev / pl_lsd_search_for_triangulation_dev on the GPU: every problem of a mixed batch equals
pl_orb_search_for_triangulation / pl_lsd_search_for_triangulation on its own two keyframes and the oracle, bit for bit; bad problems
write only their status; the snapshot protocol of CreateNewMapPoints replayed through the device call reproduces the reference's own
sequential loop; a CUDA-graph replay equals the eager launch; the calls hold no device memory.  DESIGN.md §8f.4 names the mutant
each test catches."""
import numpy as np
import pytest

import oracle
import plslam_b200 as pl
from plslam_b200 import synth
import triangulation_protocol as tp

pytestmark = pytest.mark.gpu
FILL = -7
LAST_NODE = 1 << 20


def _view(s, name, K):
    v = s[name]
    T = np.eye(4, dtype=np.float32); T[:3, :3] = v["R"]; T[:3, 3] = v["t"]
    Ow = s["Cw1"] if name == "1" else (-v["R"].T @ v["t"]).astype(np.float32)
    return dict(keys=v["keys"], desc=v["desc"], has_mp=v["has_mp"], fv=v["fv"], Tcw=T.reshape(16), Ow=Ow, K=np.asarray(K, np.float32))


def _with_ties(kf, pairs):
    """kf with a copy of keypoint idx2 appended for each pair, listed right after idx2 in its node: the same distance and
    geometry, so the reference's `dist > bestDist` scan takes the copy (the last equal candidate)."""
    n = len(kf["keys"])
    fv = {nd: list(items) for nd, items in kf["fv"].items()}
    node_of = {i: nd for nd, items in fv.items() for i in items}
    copies = []
    for c, (_, i2) in enumerate(pairs):
        items = fv[node_of[int(i2)]]
        items.insert(items.index(int(i2)) + 1, n + c)
        copies.append(int(i2))
    return dict(kf, keys=np.concatenate([kf["keys"], kf["keys"][copies]]), desc=np.concatenate([kf["desc"], kf["desc"][copies]]),
                has_mp=np.concatenate([kf["has_mp"], kf["has_mp"][copies]]), fv=fv)


def _single_args(kfs, problem, sf, ls2):
    k1, k2, F = problem
    a, b = kfs[k1], kfs[k2]
    T = np.asarray(b["Tcw"], np.float32).reshape(4, 4)
    return (a["keys"], a["desc"], a["has_mp"], b["keys"], b["desc"], b["has_mp"], a["fv"], b["fv"], F, a["Ow"],
            np.ascontiguousarray(T[:3, :3]), np.ascontiguousarray(T[:3, 3]), b["K"], sf, ls2)


def _point_batch():
    """Two keyframe pairs with different poses and intrinsics, a keyframe with tied candidates, one without keypoints, and three
    keyframes that become malformed on the device (BAD_START, BAD_ITEM, and an output range past n_out)."""
    A = synth.synth_two_view(5)
    B = synth.synth_two_view(7, K=(600.0, 590.0, 330.0, 250.0))
    kfs = [_view(A, "1", A["K"]), _view(A, "2", A["K"]), _view(B, "1", B["K"]), _view(B, "2", B["K"])]
    _, m = oracle.search_for_triangulation(*_single_args(kfs, (0, 1, A["F12"]), A["scale_factors"], A["level_sigma2"]), False)
    pairs = tp.pairs_of(m)
    for kf, i in zip(kfs[:2], pairs[-1]):         # a matched pair alone in a new last node of both keyframes
        kf["fv"] = {nd: [x for x in items if x != i] for nd, items in kf["fv"].items()}
        kf["fv"][LAST_NODE] = [int(i)]
    kfs.append(_with_ties(kfs[1], pairs[:40]))                                            # 4
    kfs.append(dict(kfs[1], keys=kfs[1]["keys"][:0], desc=kfs[1]["desc"][:0], has_mp=[], fv={}))   # 5: no keypoints
    kfs += [dict(kfs[3]), dict(kfs[3])]                                                    # 6, 7: made malformed below
    FA, FB = A["F12"], B["F12"]
    problems = [(0, 1, FA), (2, 3, FB), (0, 4, FA), (0, 5, FA), (5, 1, FA), (3, 2, FB.T), (9, 1, FA), (2, 6, FB), (2, 7, FB),
                (1, 0, FA.T)]
    bad = {6: 1, 7: 2, 8: 3, 9: 1}
    return kfs, problems, (A["scale_factors"], A["level_sigma2"]), bad


def _break(b):
    """Keyframe 6: fv_start not monotone; keyframe 7: an fv_items entry past n; problem 9: its output range past n_out."""
    b.inputs["k_fv_start"][6, 2] = -1
    b.inputs["k_fv_items"][7, 3] = int(b.host["k"]["n"][7]) + 5
    b.inputs["q_out_offset"][9] = b.host["q"]["n_out"] - 1
    import torch
    torch.cuda.synchronize()


@pytest.mark.parametrize("ori", [False, True])
def test_point_batch_equals_the_single_calls_and_the_oracle(ori):
    kfs, problems, (sf, ls2), bad = _point_batch()
    b = pl.TriangulationProblems(kfs, problems, (sf, ls2), options=int(ori), out_fill=FILL)
    _break(b)
    b.run()
    res = b.results()
    for p, r in enumerate(res):
        if p in bad:
            assert r["status"] == bad[p] and r["nmatches"] == FILL and (r["matches"] == FILL).all(), p
            continue
        args = _single_args(kfs, problems[p], sf, ls2)
        nm, m = pl.ORBmatcher(0.6, ori).SearchForTriangulation(*args)
        onm, om = oracle.search_for_triangulation(*args, ori)
        assert r["status"] == 0 and r["nmatches"] == nm == onm and np.array_equal(r["matches"], m) and np.array_equal(m, om), p
    assert res[0]["nmatches"] > 200 and res[1]["nmatches"] > 200 and res[5]["nmatches"] > 100
    tied = res[2]["matches"] >= len(kfs[1]["keys"])                         # the copies won their ties
    assert tied.sum() >= 25
    assert kfs[4]["keys"][res[2]["matches"][tied]].tobytes() == kfs[1]["keys"][res[0]["matches"][tied]].tobytes()
    assert (res[3]["matches"] == -1).all() and len(res[4]["matches"]) == 0
    assert res[0]["matches"][kfs[0]["fv"][LAST_NODE][0]] == kfs[1]["fv"][LAST_NODE][0]       # the last common node is searched


def _line_batch():
    f = synth.synth_sequence(3, 640, 480, seed=2)
    rng = np.random.default_rng(3)
    kfs = []
    for img in f:
        _, d, _ = oracle.line_extract(img)
        kfs.append(dict(ldesc=d, has_ml=(rng.random(len(d)) < 0.25).astype(np.uint8)))
    kfs.append(dict(ldesc=kfs[0]["ldesc"][:0], has_ml=kfs[0]["has_ml"][:0]))      # 3: no lines
    kfs.append(dict(kfs[1]))                                                      # 4: its n made over the capacity below
    problems = [(0, 1), (1, 0), (0, 2), (2, 1), (0, 3), (3, 0), (6, 0), (4, 0), (1, 4)]
    return kfs, problems, {6: 1, 7: 2, 8: 2}


@pytest.mark.parametrize("dbl", [False, True])
def test_line_batch_equals_the_single_calls_and_the_oracle(dbl):
    import torch
    kfs, problems, bad = _line_batch()
    b = pl.TriangulationProblems(kfs, problems, lines=True, options=(80.0, 0.8, dbl), out_fill=FILL)
    b.inputs["k_n"][4] = b.host["k"]["cap"] + 1
    torch.cuda.synchronize()
    b.run()
    res = b.results()
    for p, r in enumerate(res):
        if p in bad:
            assert r["status"] == bad[p] and r["nmatches"] == FILL and (r["matches"] == FILL).all(), p
            continue
        k1, k2 = problems[p]
        args = (kfs[k1]["ldesc"], kfs[k1]["has_ml"], kfs[k2]["ldesc"], kfs[k2]["has_ml"])
        nm, m = pl.LSDmatcher(0.8).SearchForTriangulation(*args, dbl)
        onm, om = oracle.lsd_search_for_triangulation(*args, 0.8, dbl)
        assert r["status"] == 0 and r["nmatches"] == nm == onm and np.array_equal(r["matches"], m) and np.array_equal(m, om), p
    assert res[0]["nmatches"] > 10 and (res[4]["matches"] == -1).all() and len(res[5]["matches"]) == 0
    # the MapLine filter removed pairs on both sides
    bare = pl.LSDmatcher(0.8).SearchForTriangulation(kfs[0]["ldesc"], kfs[0]["has_ml"] * 0, kfs[1]["ldesc"], kfs[1]["has_ml"] * 0, dbl)[1]
    gone = (bare >= 0) & (res[0]["matches"] < 0)
    assert kfs[0]["has_ml"][gone].any() and kfs[1]["has_ml"][bare[gone]].any()


def test_protocol_through_the_device_call_reproduces_the_reference():
    s = tp.load()
    kfs = [tp.keyframe(s, k) for k in range(len(s["kf_start"]) - 1)]
    problems = [(0, j, s["F12"][j - 1].reshape(3, 3)) for j in range(1, len(kfs))]
    res = pl.ORBmatcher(0.6, False).SearchForTriangulationBatch(kfs, problems, s["scale_factors"], s["level_sigma2"])
    assert all(r["status"] == 0 for r in res)
    snapshot = [r["matches"] for r in res]
    assert tp.same_lists(tp.snapshot_protocol(s, snapshot), tp.reference_lists(s))
    assert not tp.same_lists(tp.snapshot_protocol(s, snapshot, drop=False), tp.reference_lists(s))


@pytest.mark.parametrize("lines", [False, True])
def test_graph_replay_equals_the_eager_launch(lines):
    import torch
    if lines:
        kfs, problems, _ = _line_batch()
        b = pl.TriangulationProblems(kfs, problems[:6], lines=True, options=(80.0, 0.8, True), out_fill=FILL)
    else:
        kfs, problems, scales, _ = _point_batch()
        b = pl.TriangulationProblems(kfs, problems, scales, options=1, out_fill=FILL)
    b.run()
    eager = b.results()
    for t in b.outputs.values():
        t.fill_(FILL)
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        b.run(s)
    torch.cuda.synchronize()
    assert all((t == FILL).all() for t in b.outputs.values())     # capturing runs nothing
    g.replay()
    replay = b.results()
    for e, r in zip(eager, replay):
        assert e.keys() == r.keys() and all(np.array_equal(e[k], r[k]) for k in e)


def test_calls_hold_no_device_memory():
    kfs, problems, scales, _ = _point_batch()
    lkfs, lproblems, _ = _line_batch()
    pb = pl.TriangulationProblems(kfs, problems[:6], scales)
    lb = pl.TriangulationProblems(lkfs, lproblems[:6], lines=True, options=(80.0, 0.8, True))
    pb.run(); lb.run(); pb.results(); lb.results()
    before = pl.device_bytes()
    for _ in range(3):
        pb.run(); lb.run()
        pl.ORBmatcher(0.6, True).SearchForTriangulation(*_single_args(kfs, problems[0], *scales))
        pl.LSDmatcher(0.8).SearchForTriangulation(lkfs[0]["ldesc"], lkfs[0]["has_ml"], lkfs[1]["ldesc"], lkfs[1]["has_ml"], True)
    pb.results(); lb.results()
    assert pl.device_bytes() == before


def test_line_capacity_over_the_shared_memory_is_refused():
    """One line more than k_lsd_search_triangulation's shared memory holds per side is refused with PL_ERR_ARG before any launch."""
    from test_match_batched_gpu import _search_double_limit
    fit = _search_double_limit()
    kfs = [dict(ldesc=np.zeros((fit + 1, 32), np.uint8), has_ml=np.zeros(fit + 1, np.uint8))] * 2
    b = pl.TriangulationProblems(kfs, [(0, 1)], lines=True, options=(80.0, 0.8, True), out_fill=FILL)
    with pytest.raises(pl.PLError, match=rf"error -1: .* at most {fit} lines per side"):
        b.run()
    assert all((t == FILL).all() for t in b.outputs.values())
