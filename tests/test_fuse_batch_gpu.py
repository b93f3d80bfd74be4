"""pl_orb_fuse_search_dev / pl_lsd_fuse_search_dev on the GPU: every problem of a mixed batch equals pl_orb_fuse_search /
pl_lsd_fuse_search on its own inputs and the oracle, bit for bit; bad problems write only their status; the snapshot protocol of
SearchInNeighbors replayed through the device call reproduces the reference's own sequential loop; a CUDA-graph replay equals the
eager launch.  DESIGN.md §8f.3 names the mutant each test catches."""
import numpy as np
import pytest

import oracle
import plslam_b200 as pl
from plslam_b200 import synth
import fuse_protocol as fp
from test_localmap2 import _line_fuse_problem

pytestmark = pytest.mark.gpu
FILL = -7


def _point_batch():
    """Three keyframes with different poses, intrinsics and keypoint counts, one without keypoints; one landmark table; entry lists
    over it in a permuted order, one list reused by two problems, one with the skips of another flipped, one empty."""
    A = synth.synth_fuse_problem(6, n_mp=1500, n_kp=1800)
    B = synth.synth_fuse_problem(8, n_mp=1200, n_kp=2500, K=(600.0, 590.0, 330.0, 250.0))
    kf = lambda f, n=None: dict(keys=f["keys"][:n], desc=f["desc"][:n], Tcw=f["Tcw"], Ow=f["Ow"], K=f["K"], bounds=f["bounds"])
    kfs = [kf(A), kf(B), kf(A, 0)]
    pts = {k: np.concatenate([A[k], B[k]]) for k in ("pos", "normal", "min_dist", "max_dist")}
    pts["desc"] = np.concatenate([A["mp_desc"], B["mp_desc"]])
    nA, nB = len(A["pos"]), len(B["pos"])
    perm = np.random.default_rng(1).permutation(nB)
    lists = [(np.arange(nA), A["skip"]), (nA + perm, B["skip"][perm]), (np.arange(nA), 1 - A["skip"]), ([], []),
             ([0, 1, nA + nB + 3], [0, 0, 0])]
    problems = [(0, 3.0, 0), (1, 3.0, 1), (0, 1.0, 0), (0, 3.0, 2), (2, 3.0, 1), (1, 3.0, 3), (7, 3.0, 0), (1, 3.0, 4), (1, 3.0, 1)]
    scales = dict(scale_factors=A["scale_factors"], inv_level_sigma2=A["inv_level_sigma2"], log_scale_factor=A["log_scale_factor"])
    return kfs, pts, problems, lists, scales, {6: 1, 7: 3}     # problem -> the status it must report


def _point_want(kfs, pts, problems, lists, scales, p):
    k, th, li = problems[p]
    lm, skip = np.asarray(lists[li][0], np.int64), np.asarray(lists[li][1], np.uint8)
    args = (kfs[k]["keys"], kfs[k]["desc"], kfs[k]["bounds"], kfs[k]["Tcw"], kfs[k]["Ow"], kfs[k]["K"], scales["scale_factors"],
            scales["inv_level_sigma2"], scales["log_scale_factor"], skip, pts["pos"][lm], pts["normal"][lm], pts["min_dist"][lm],
            pts["max_dist"][lm], pts["desc"][lm], th)
    return pl.ORBmatcher().FuseSearch(*args), oracle.fuse_search(*args)


def test_point_batch_equals_the_single_calls_and_the_oracle():
    kfs, pts, problems, lists, scales, bad = _point_batch()
    b = pl.FuseProblems(kfs, pts, problems, lists, scales, out_fill=FILL)
    b.run()
    res = b.results()
    for p, r in enumerate(res):
        if p in bad:
            assert r["status"] == bad[p] and (r["best_idx"] == FILL).all() and (r["best_dist"] == FILL).all(), p
            continue
        (bi, bd), (obi, obd) = _point_want(kfs, pts, problems, lists, scales, p)
        assert r["status"] == 0 and np.array_equal(r["best_idx"], bi) and np.array_equal(r["best_dist"], bd), p
        assert np.array_equal(bi, obi) and np.array_equal(bd, obd), p
    assert (res[0]["best_dist"] <= 50).sum() > 20 and (res[1]["best_dist"] <= 50).sum() > 20
    assert not np.array_equal(res[0]["best_idx"], res[2]["best_idx"])        # same keyframe and range, another th
    assert (res[4]["best_idx"] == -1).all() and len(res[5]["best_idx"]) == 0   # a keyframe without keypoints; an empty range


def _line_batch():
    """Three line keyframes (one with a map line behind the camera at entry 37, one with other intrinsics, one without lines or
    point descriptors), each with its own map lines in one table; a list reused by two keyframes; a bad range."""
    fs = [_line_fuse_problem(22, 37), _line_fuse_problem(21), _line_fuse_problem(24)]
    fs[1]["K"] = fs[1]["K"] + np.float32([0.5, 0.5, 0.4, -0.3])
    kfs = [dict(kl=f["kl"], pdesc=f["pdesc"], Tcw=f["Tcw"], Ow=f["Ow"], K=f["K"], bounds=f["bounds"]) for f in fs[:2]]
    kfs.append(dict(kfs[1], kl=fs[2]["kl"][:0], pdesc=fs[2]["pdesc"][:0]))
    lines = {k: np.concatenate([f[k] for f in fs]) for k in ("pos", "normal", "min_dist", "max_dist")}
    lines["desc"] = np.concatenate([f["ml_desc"] for f in fs])
    start = np.cumsum([0] + [len(f["pos"]) for f in fs])
    lists = [(start[i] + np.arange(len(f["pos"])), f["skip"]) for i, f in enumerate(fs[:2])]
    lists.append(([start[3]], [0]))
    problems = [(0, 3.0, 0), (1, 3.0, 1), (1, 8.0, 0), (0, 1.0, 1), (2, 3.0, 1), (3, 3.0, 0), (0, 3.0, 2)]
    scales = dict(scale_line=1.2, log_scale_factor_line=float(np.float32(np.log(np.float32(1.2)))))
    return kfs, lines, problems, lists, scales, {5: 1, 6: 3}


def test_line_batch_equals_the_single_calls_and_the_oracle():
    kfs, lines, problems, lists, scales, bad = _line_batch()
    b = pl.FuseProblems(kfs, lines, problems, lists, scales, lines=True, out_fill=FILL)
    b.run()
    res = b.results()
    for p, r in enumerate(res):
        if p in bad:
            assert r["status"] == bad[p] and r["stop_at"] == FILL and (r["best_idx"] == FILL).all() and (r["best_dist"] == FILL).all(), p
            continue
        k, th, li = problems[p]
        lm, skip = np.asarray(lists[li][0]), np.asarray(lists[li][1], np.uint8)
        args = (kfs[k]["kl"], kfs[k]["pdesc"], kfs[k]["bounds"], kfs[k]["Tcw"], kfs[k]["Ow"], kfs[k]["K"], scales["scale_line"],
                scales["log_scale_factor_line"], skip, lines["pos"][lm], lines["normal"][lm], lines["min_dist"][lm],
                lines["max_dist"][lm], lines["desc"][lm], th)
        bi, bd, stop = pl.LSDmatcher().FuseSearch(*args)
        obi, obd, ostop = oracle.lsd_fuse_search(*args)
        assert r["status"] == 0 and r["stop_at"] == stop == ostop, p
        assert np.array_equal(r["best_idx"], bi) and np.array_equal(r["best_dist"], bd), p
        assert np.array_equal(bi, obi) and np.array_equal(bd, obd), p
    assert res[0]["stop_at"] == 37 and res[1]["stop_at"] == len(lists[1][0])
    assert (res[1]["best_dist"] <= 50).sum() > 10
    assert (res[4]["best_idx"] == -1).all()


def _device_search(s):
    kfs = [fp.keyframe(s, k) for k in range(len(s["Tcw"]))]

    def search(problems, desc):
        pts = dict(pos=s["pos"], normal=s["normal"], min_dist=s["min_dist"], max_dist=s["max_dist"], desc=desc)
        res = pl.ORBmatcher().FuseSearchBatch(kfs, pts, [(t, float(s["th"]), i) for i, (t, _, _) in enumerate(problems)],
                                              [(lm, sk) for _, lm, sk in problems], s["scale_factors"], s["inv_level_sigma2"],
                                              float(s["log_scale_factor"]))
        assert all(r["status"] == 0 for r in res)
        return [(r["best_idx"], r["best_dist"]) for r in res]
    return search


def test_protocol_through_the_device_call_reproduces_the_reference():
    s = fp.load()
    M, nfused = fp.first_loop(s, _device_search(s))
    assert np.array_equal(fp.final_slots(M), s["ref_slots"]) and np.array_equal(M.bad, s["ref_bad"].astype(bool))
    assert np.array_equal(M.desc, s["ref_desc"]) and np.array_equal(nfused, s["ref_nfused"])
    # the snapshot searches themselves equal the oracle's
    snap = fp.MapState(s)
    probs = [(int(t), s["list"], [snap.skip(int(t), m) for m in s["list"]]) for t in s["targets"]]
    for (bi, bd), (obi, obd) in zip(_device_search(s)(probs, snap.desc), fp.oracle_search(s)(probs, snap.desc)):
        assert np.array_equal(bi, obi) and np.array_equal(bd, obd)


@pytest.mark.parametrize("lines", [False, True])
def test_graph_replay_equals_the_eager_launch(lines):
    import torch
    kfs, lms, problems, lists, scales, _ = _line_batch() if lines else _point_batch()
    b = pl.FuseProblems(kfs, lms, problems, lists, scales, lines=lines, out_fill=FILL)
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


@pytest.mark.parametrize("flipped", [(), (37,), (37, 38)])
def test_line_stop_rule_through_the_device_call(flipped):
    """The snapshot from pl_lsd_fuse_search_dev, the rest of the list searched again with pl_lsd_fuse_search when the stop entry
    became skipped: the reference's results (the oracle on the skips at application time)."""
    from test_fuse_batch import _line_stop_case, _live, line_stop_rule, _same_where_reached
    a = _line_stop_case()
    kf = dict(kl=a[0], pdesc=a[1], bounds=a[2], Tcw=a[3], Ow=a[4], K=a[5])
    lines = dict(pos=a[9], normal=a[10], min_dist=a[11], max_dist=a[12], desc=a[13])
    r, = pl.LSDmatcher().FuseSearchBatch([kf], lines, [(0, a[14], 0)], [(np.arange(len(a[9])), a[8])], a[6], a[7])
    assert r["status"] == 0 and r["stop_at"] == 37
    live, got, want = line_stop_rule(a, (r["best_idx"], r["best_dist"], r["stop_at"]), flipped, lambda x: pl.LSDmatcher().FuseSearch(*x))
    assert _same_where_reached(live, got, want) and _same_where_reached(live, got, oracle.lsd_fuse_search(*_live(a, live)))
