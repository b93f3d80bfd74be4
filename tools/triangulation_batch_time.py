"""Time the triangulation searches of LocalMapping as two device calls against the loop of host calls.

The workload has the shape of one monocular keyframe: a current keyframe with about 1,000 keypoints and 230 keylines, searched
against its 20 best covisible neighbours for points (CreateNewMapPoints, ORBmatcher(0.6, false)) and its 10 best for lines
(CreateNewMapLinesConstraint, LSDmatcher(0.8), TH_HIGH, isDouble).  Forms timed:
  host:   20 pl_orb_search_for_triangulation calls and 10 pl_lsd_search_for_triangulation calls (each stages its inputs and
          synchronises);
  device: pl_orb_search_for_triangulation_dev with the 20 problems and pl_lsd_search_for_triangulation_dev with the 10 (two launches
          on one stream, CUDA events around them);
  batched keyframes: the searches of --keyframes such keyframes in one launch per kind;
  point search + triangulation: pl_orb_search_for_triangulation_dev then pl_orb_triangulate_dev (the gates and the neighbour-order
          commit) for one keyframe's 20 problems and for --keyframes keyframes', three launches on one stream, CUDA events around
          them; the triangulation launches alone as well;
  CPU oracle: tests/cnmp_oracle.py's triangulate (numpy, vectorised over the pairs) on the same search outputs, a CPU time;
  line search + triangulation: pl_lsd_search_for_triangulation_dev then pl_lsd_triangulate_dev (CreateNewMapLinesConstraint's
          three-view gates and commit, 45 entry pairs) for one current keyframe of about 230 keylines against 10 neighbours of the
          tests/cnml_scene.py geometry, and for --keyframes such keyframes in one call; the triangulation launches alone as well.
After --warmup calls, --rounds rounds alternate the forms; each number is the median over the timed calls.  Prints one JSON line,
with the card's name and power limit read in the same run.

    python tools/triangulation_batch_time.py [--rounds 5] [--iters 5] [--warmup 2] [--keyframes 4]
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

N_POINT_NEIGH, N_LINE_NEIGH, N_LINES = 20, 10, 230


def workload(n_kf):
    """n_kf + N_POINT_NEIGH point keyframes (keyframes 0 .. n_kf - 1 are current keyframes, the rest their neighbours) and line
    keyframes in the same numbering: correlated descriptors, a quarter of the lines already holding a map line."""
    from gen_triangulation_protocol import scene
    import triangulation_protocol as tp
    s = scene(seed=11, n_neigh=n_kf + N_POINT_NEIGH - 1, n_pts=1100, n_clutter=100)
    pkf = [tp.keyframe(s, k) for k in range(len(s["kf_start"]) - 1)]
    F = lambda j: s["F12"][j - 1].reshape(3, 3)
    rng = np.random.default_rng(12)
    code = rng.integers(0, 256, (N_LINES, 32), dtype=np.uint8)
    lkf = []
    for _ in range(len(pkf)):
        d = code[rng.permutation(N_LINES)].copy()
        for _ in range(8):
            b = rng.integers(0, 256, N_LINES)
            d[np.arange(N_LINES), b // 8] ^= (1 << (b % 8)).astype(np.uint8)
        lkf.append(dict(ldesc=d, has_ml=(rng.random(N_LINES) < 0.25).astype(np.uint8)))
    # current keyframe c searches the neighbours after the current keyframes (F12 of keyframe 0: the timing does not depend on it)
    pprob = lambda c: [(c, n_kf + j, F(n_kf + j)) for j in range(N_POINT_NEIGH)]
    lprob = lambda c: [(c, n_kf + j) for j in range(N_LINE_NEIGH)]
    return s, pkf, lkf, pprob, lprob


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
    s, pkf, lkf, pprob, lprob = workload(args.keyframes)
    scales = (s["scale_factors"], s["level_sigma2"])
    lopt = (80.0, 0.8, True)
    side = torch.cuda.Stream()
    dev = [pl.TriangulationProblems(pkf, pprob(0), scales), pl.TriangulationProblems(lkf, lprob(0), lines=True, options=lopt)]
    devK = [pl.TriangulationProblems(pkf, [p for c in range(args.keyframes) for p in pprob(c)], scales),
            pl.TriangulationProblems(lkf, [p for c in range(args.keyframes) for p in lprob(c)], lines=True, options=lopt)]
    M, L = pl.ORBmatcher(0.6, False), pl.LSDmatcher(0.8)

    def point_args(k1, k2, F):
        a, b = pkf[k1], pkf[k2]
        T = np.asarray(b["Tcw"], np.float32).reshape(4, 4)
        return (a["keys"], a["desc"], a["has_mp"], b["keys"], b["desc"], b["has_mp"], a["fv"], b["fv"], F, a["Ow"],
                np.ascontiguousarray(T[:3, :3]), np.ascontiguousarray(T[:3, 3]), b["K"], *scales)

    def host_loop():
        t0 = time.perf_counter()
        for p in pprob(0):
            M.SearchForTriangulation(*point_args(*p))
        for k1, k2 in lprob(0):
            L.SearchForTriangulation(lkf[k1]["ldesc"], lkf[k1]["has_ml"], lkf[k2]["ldesc"], lkf[k2]["has_ml"], True)
        return (time.perf_counter() - t0) * 1e3

    def timed(objs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(side)
        for o in objs:
            o.run(side)
        e1.record(side)
        e1.synchronize()
        return e0.elapsed_time(e1)

    # the device calls compute what the host calls compute
    dev[0].run(); dev[1].run()
    rp, rl = dev[0].results(), dev[1].results()
    nm, m = M.SearchForTriangulation(*point_args(*pprob(0)[5]))
    assert rp[5]["nmatches"] == nm > 100 and np.array_equal(rp[5]["matches"], m)
    k1, k2 = lprob(0)[3]
    nm, m = L.SearchForTriangulation(lkf[k1]["ldesc"], lkf[k1]["has_ml"], lkf[k2]["ldesc"], lkf[k2]["has_ml"], True)
    assert rl[3]["nmatches"] == nm > 10 and np.array_equal(rl[3]["matches"], m)

    # the triangulation computes what the oracle computes, on the same search outputs
    import cnmp_oracle as co
    sfac = float(s["scale_factors"][1])
    dev[0].triangulate(scale_factor=sfac)
    tri = dev[0].triangulated()
    m12 = dev[0].outputs["matches"].cpu().numpy()[:dev[0].host["q"]["n_out"]]
    st = dev[0].outputs["status"].cpu().numpy()[:dev[0].P]
    oc = co.triangulate(dev[0].host["k"], dev[0].host["q"], m12, st, sfac, *scales)
    assert np.array_equal(np.concatenate([t["code"] for t in tri]), oc[0]) and sum(t["nnew"] for t in tri) == oc[2].sum() > 100

    class SearchTri:                     # search + triangulation of one TriangulationProblems, as one timed object
        def __init__(self, b, only_tri=False):
            self.b, self.only_tri = b, only_tri

        def run(self, stream):
            if not self.only_tri:
                self.b.run(stream)
            self.b.triangulate(stream, scale_factor=sfac)
    st1, stK, tri1, triK = SearchTri(dev[0]), SearchTri(devK[0]), SearchTri(dev[0], True), SearchTri(devK[0], True)

    def oracle_loop():
        t0 = time.perf_counter()
        co.triangulate(dev[0].host["k"], dev[0].host["q"], m12, st, sfac, *scales)
        return (time.perf_counter() - t0) * 1e3

    # lines: current keyframes 0 .. K-1 of a scene with 10 neighbours after them, one group each, entries in neighbour order
    import cnml_oracle as cno
    import cnml_scene as cs
    lsc = cs.scene(seed=7, n_seg=300, n_clutter=30, n_kf=args.keyframes + N_LINE_NEIGH)
    nb = list(range(args.keyframes, args.keyframes + N_LINE_NEIGH))
    lgroup = lambda c, p0: dict(kf_cur=c, entries=[(p0 + e, j, lsc["medians"][j]) for e, j in enumerate(nb)])
    ltri = [pl.TriangulationProblems(lsc["kfs"], [(0, j) for j in nb], lsc["level_sigma2_line"], lines=True, options=lopt,
                                     groups=[lgroup(0, 0)]),
            pl.TriangulationProblems(lsc["kfs"], [(c, j) for c in range(args.keyframes) for j in nb], lsc["level_sigma2_line"],
                                     lines=True, options=lopt, groups=[lgroup(c, c * N_LINE_NEIGH) for c in range(args.keyframes)])]
    ltri[0].run(); ltri[0].triangulate()
    lt = ltri[0].triangulated()
    h = {k: v.cpu().numpy() for k, v in ltri[0].outputs.items()}
    q0 = ltri[0].host["q"]
    lo = cno.triangulate_lines(ltri[0].host["k"], q0, ltri[0].host["g"], h["matches"][:q0["n_out"]], h["nmatches"][:ltri[0].P],
                               h["status"][:ltri[0].P], lsc["level_sigma2_line"])
    assert np.array_equal(lt[0]["code"].ravel(), lo[0]) and lt[0]["nnew"] == lo[2][0]

    class LineTri:
        def __init__(self, b, only_tri=False):
            self.b, self.only_tri = b, only_tri

        def run(self, stream):
            if not self.only_tri:
                self.b.run(stream)
            self.b.triangulate(stream)
    lst1, lstK, ltri1, ltriK = LineTri(ltri[0]), LineTri(ltri[1]), LineTri(ltri[0], True), LineTri(ltri[1], True)

    for _ in range(args.warmup):
        host_loop(); timed(dev); timed(devK); timed([st1]); timed([stK]); oracle_loop()
        timed([lst1]); timed([lstK])
    host, one, many, per = [], [], [], {}
    for _ in range(args.rounds):
        host += [host_loop() for _ in range(args.iters)]
        one += [timed(dev) for _ in range(args.iters)]
        many += [timed(devK) for _ in range(args.iters)]
        for i, nm in enumerate(("points", "lines")):
            per.setdefault(nm, []).extend(timed([dev[i]]) for _ in range(args.iters))
        for nm, o in (("search_triangulate_1kf", st1), ("search_triangulate_kfs", stK), ("triangulate_1kf", tri1), ("triangulate_kfs", triK)):
            per.setdefault(nm, []).extend(timed([o]) for _ in range(args.iters))
        per.setdefault("cpu_oracle_1kf", []).extend(oracle_loop() for _ in range(args.iters))
        for nm, o in (("line_search_triangulate_1kf", lst1), ("line_search_triangulate_kfs", lstK), ("line_triangulate_1kf", ltri1),
                      ("line_triangulate_kfs", ltriK)):
            per.setdefault(nm, []).extend(timed([o]) for _ in range(args.iters))
    med = lambda a: round(float(np.median(a)), 4)
    print(json.dumps(dict(tool="triangulation_batch_time", card=name, power_limit=plim, keypoints=len(pkf[0]["keys"]), keylines=N_LINES,
                          point_neighbours=N_POINT_NEIGH, line_neighbours=N_LINE_NEIGH, host_loop_ms=med(host), device_ms=med(one),
                          device_launch_ms={k: med(per[k]) for k in ("points", "lines")}, keyframes=args.keyframes,
                          batched_keyframes_ms=med(many), speedup=round(med(host) / med(one), 1),
                          point_pairs_1kf=int((m12 >= 0).sum()), new_points_1kf=int(oc[2].sum()),
                          search_triangulate_1kf_ms=med(per["search_triangulate_1kf"]), search_triangulate_kfs_ms=med(per["search_triangulate_kfs"]),
                          triangulate_1kf_ms=med(per["triangulate_1kf"]), triangulate_kfs_ms=med(per["triangulate_kfs"]),
                          cpu_oracle_triangulate_1kf_ms=med(per["cpu_oracle_1kf"]),
                          line_keylines_1kf=len(lsc["kfs"][0]["keylines"]), new_lines_1kf=int(lo[2][0]),
                          line_search_triangulate_1kf_ms=med(per["line_search_triangulate_1kf"]),
                          line_search_triangulate_kfs_ms=med(per["line_search_triangulate_kfs"]),
                          line_triangulate_1kf_ms=med(per["line_triangulate_1kf"]), line_triangulate_kfs_ms=med(per["line_triangulate_kfs"]))))


if __name__ == "__main__":
    main()
