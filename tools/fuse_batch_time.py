"""Time the Fuse searches of LocalMapping::SearchInNeighbors as one device call against the loop of host calls.

The workload has the shape of one monocular SearchInNeighbors: a current keyframe with 1,000 map points and 200 map lines, 120 target
keyframes (about 1,000 keypoints and 230 keylines each), and the reverse fuse of 6,000 candidate points and 1,000 candidate lines
into the current keyframe.  Forms timed:
  host:   120 + 1 pl_orb_fuse_search calls and 120 + 1 pl_lsd_fuse_search calls (each stages its inputs and synchronises);
  device: pl_orb_fuse_search_dev with the 120 targets, then with the reverse problem, and the same two for lines (four launches on
          one stream, CUDA events around them);
  batched keyframes: the first loops of --keyframes such keyframes in one pl_orb_fuse_search_dev and one pl_lsd_fuse_search_dev.
After --warmup calls, --rounds rounds alternate the forms; each number is the median over the timed calls.  Prints one JSON line,
with the card's name and power limit read in the same run.

    python tools/fuse_batch_time.py [--rounds 5] [--iters 5] [--warmup 2] [--keyframes 4]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

N_TARGETS, N_POINTS, N_LINES, N_CAND_POINTS, N_CAND_LINES = 120, 1000, 200, 6000, 1000


def workload():
    from plslam_b200 import synth
    from test_localmap2 import _line_fuse_problem
    pt = [synth.synth_fuse_problem(seed, n_mp=N_CAND_POINTS, n_kp=1000) for seed in range(6, 14)]
    ln = [_line_fuse_problem(seed) for seed in range(21, 25)]
    # keyframe 0 is the current keyframe; targets cycle through the generated views
    pkf = [dict(keys=f["keys"], desc=f["desc"], Tcw=f["Tcw"], Ow=f["Ow"], K=f["K"], bounds=f["bounds"]) for f in pt]
    lkf = [dict(kl=f["kl"], pdesc=f["pdesc"], Tcw=f["Tcw"], Ow=f["Ow"], K=f["K"], bounds=f["bounds"]) for f in ln]
    pts = dict(pos=pt[0]["pos"], normal=pt[0]["normal"], min_dist=pt[0]["min_dist"], max_dist=pt[0]["max_dist"], desc=pt[0]["mp_desc"])
    lns = {k: np.concatenate([f[k] for f in ln]) for k in ("pos", "normal", "min_dist", "max_dist")}
    lns["desc"] = np.concatenate([f["ml_desc"] for f in ln])
    ps = dict(scale_factors=pt[0]["scale_factors"], inv_level_sigma2=pt[0]["inv_level_sigma2"], log_scale_factor=pt[0]["log_scale_factor"])
    ls = dict(scale_line=1.2, log_scale_factor_line=float(np.float32(np.log(np.float32(1.2)))))
    return pkf, lkf, pts, lns, ps, ls, pt[0]["skip"], np.concatenate([f["skip"] for f in ln])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--keyframes", type=int, default=4)
    args = ap.parse_args()
    import torch
    import plslam_b200 as pl
    from track_local_map_time import card

    name, plim = card()
    pkf, lkf, pts, lns, ps, ls, pskip, lskip = workload()
    nP, nL = len(pkf), len(lkf)
    tgt_p = [1 + t % (nP - 1) for t in range(N_TARGETS)]
    tgt_l = [1 + t % (nL - 1) for t in range(N_TARGETS)]
    first_p = (np.arange(N_POINTS), pskip[:N_POINTS])
    first_l = (np.arange(N_LINES), lskip[:N_LINES])
    rev_p = (np.arange(N_CAND_POINTS), pskip[:N_CAND_POINTS])
    rev_l = (np.arange(N_CAND_LINES), lskip[:N_CAND_LINES])

    def batch(K):        # K keyframes' first loops: problems (target, th, list), each keyframe its own point list
        p = [(t, 3.0, k) for k in range(K) for t in tgt_p]
        l = [(t, 3.0, k) for k in range(K) for t in tgt_l]
        return p, l

    side = torch.cuda.Stream()
    p1, l1 = batch(1)
    dev = [pl.FuseProblems(pkf, pts, p1, [first_p], ps), pl.FuseProblems(pkf, pts, [(0, 3.0, 0)], [rev_p], ps),
           pl.FuseProblems(lkf, lns, l1, [first_l], ls, lines=True), pl.FuseProblems(lkf, lns, [(0, 3.0, 0)], [rev_l], ls, lines=True)]
    pK, lK = batch(args.keyframes)
    devK = [pl.FuseProblems(pkf, pts, pK, [first_p] * args.keyframes, ps),
            pl.FuseProblems(lkf, lns, lK, [first_l] * args.keyframes, ls, lines=True)]
    M, L = pl.ORBmatcher(), pl.LSDmatcher()

    def host_loop():
        t0 = time.perf_counter()
        for t in tgt_p + [0]:
            lm, sk = (first_p if t else rev_p)
            k = pkf[t]
            M.FuseSearch(k["keys"], k["desc"], k["bounds"], k["Tcw"], k["Ow"], k["K"], ps["scale_factors"], ps["inv_level_sigma2"],
                         ps["log_scale_factor"], sk, pts["pos"][lm], pts["normal"][lm], pts["min_dist"][lm], pts["max_dist"][lm],
                         pts["desc"][lm], 3.0)
        for t in tgt_l + [0]:
            lm, sk = (first_l if t else rev_l)
            k = lkf[t]
            L.FuseSearch(k["kl"], k["pdesc"], k["bounds"], k["Tcw"], k["Ow"], k["K"], ls["scale_line"], ls["log_scale_factor_line"], sk,
                         lns["pos"][lm], lns["normal"][lm], lns["min_dist"][lm], lns["max_dist"][lm], lns["desc"][lm], 3.0)
        return (time.perf_counter() - t0) * 1e3

    def timed(objs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(side)
        for o in objs:
            o.run(side)
        e1.record(side)
        e1.synchronize()
        return e0.elapsed_time(e1)

    # the device call computes what the host calls compute
    dev[0].run(); r = dev[0].results()
    k = pkf[tgt_p[5]]
    bi, bd = M.FuseSearch(k["keys"], k["desc"], k["bounds"], k["Tcw"], k["Ow"], k["K"], ps["scale_factors"], ps["inv_level_sigma2"],
                          ps["log_scale_factor"], first_p[1], pts["pos"][:N_POINTS], pts["normal"][:N_POINTS], pts["min_dist"][:N_POINTS],
                          pts["max_dist"][:N_POINTS], pts["desc"][:N_POINTS], 3.0)
    assert np.array_equal(r[5]["best_idx"], bi) and np.array_equal(r[5]["best_dist"], bd)

    for _ in range(args.warmup):
        host_loop(); timed(dev); timed(devK)
    host, one, many, per = [], [], [], {}
    for _ in range(args.rounds):
        host += [host_loop() for _ in range(args.iters)]
        one += [timed(dev) for _ in range(args.iters)]
        many += [timed(devK) for _ in range(args.iters)]
        for i, nm in enumerate(("points_first", "points_reverse", "lines_first", "lines_reverse")):
            per.setdefault(nm, []).extend(timed([dev[i]]) for _ in range(args.iters))
    med = lambda a: round(float(np.median(a)), 4)
    print(json.dumps(dict(tool="fuse_batch_time", card=name, power_limit=plim, targets=N_TARGETS, points=N_POINTS, lines=N_LINES,
                          reverse_points=N_CAND_POINTS, reverse_lines=N_CAND_LINES, host_loop_ms=med(host), device_ms=med(one),
                          device_launch_ms={k: med(v) for k, v in per.items()}, keyframes=args.keyframes,
                          batched_first_loops_ms=med(many), speedup=round(med(host) / med(one), 1))))


if __name__ == "__main__":
    main()
