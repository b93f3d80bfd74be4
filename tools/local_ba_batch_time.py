"""Time pl_local_ba_dev (W local windows per launch, one CTA per window) against pl_local_ba, and the KITTI step with its window.

1. batch: W copies of bench.py's KITTI window (synth.synth_ba_problem(seed=4, K=KITTI_K, w=1241, h=376)) for W in --windows:
   one pl_local_ba_dev launch on a side stream against W sequential pl_local_ba calls, each timed with CUDA events.
2. step: bench.py's KITTI step (256 frames of 1241x376 through pl_frontend_run_dev on one stream) followed by its window, once with
   pl_local_ba after the step (as bench.py runs it), once with pl_local_ba_dev on a second stream beside the step; wall time per
   step over --steps steps that end in a device synchronisation.
After --warmup calls, --rounds rounds alternate the two forms; each number is the median over all timed calls, with the
per-round medians.  Prints one JSON line, with the card's name and power limit read in the same run.

    python tools/local_ba_batch_time.py [--windows 1,8,66,132,264] [--rounds 5] [--iters 5] [--steps 10] [--warmup 2]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", default="1,8,66,132,264")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    import bench
    import plslam_b200 as pl
    from plslam_b200 import synth
    from track_local_map_time import card

    name, plim = card()
    res = dict(tool="local_ba_batch_time", card=name, power_limit=plim, batch={}, step={})
    cfg = bench.CONFIGS["kitti"]
    w, h = cfg["W"], cfg["H"]
    p = synth.synth_ba_problem(seed=4, K=bench.KITTI_K, w=w, h=h)
    side = torch.cuda.Stream()
    legacy = torch.cuda.default_stream()

    def events(call, stream, n):
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
        for e0, e1 in ev:
            e0.record(stream); call(); e1.record(stream)
        torch.cuda.synchronize()
        return [e0.elapsed_time(e1) for e0, e1 in ev]

    # 1. one launch of W windows against W sequential pl_local_ba calls
    for W in [int(x) for x in args.windows.split(",")]:
        b = pl.LocalBAWindows([p] * W)
        forms = {"dev": (lambda: b.run(side), side),
                 "sequential": (lambda: [pl.LocalBundleAdjustmentWithLine(p) for _ in range(W)], legacy)}
        for call, s in forms.values():
            for _ in range(args.warmup):
                call()
        torch.cuda.synchronize()
        times = {k: [] for k in forms}
        rounds = {k: [] for k in forms}
        for _ in range(args.rounds):
            for k, (call, s) in forms.items():
                t = events(call, s, args.iters if k == "dev" else max(1, args.iters // max(1, W // 8)))
                times[k] += t; rounds[k].append(float(np.median(t)))
        assert all(r["status"] == 0 for r in b.results())
        res["batch"][W] = {k: dict(ms_per_launch=float(np.median(times[k])), ms_per_window=float(np.median(times[k])) / W,
                                   round_medians_ms=rounds[k], calls=len(times[k])) for k in forms}
        del b
        torch.cuda.empty_cache()

    # 2. the KITTI step with its window after it (pl_local_ba) or beside it (pl_local_ba_dev on a second stream)
    B = cfg["total"]
    K, D = bench.camera_of(cfg)
    frames, problems = bench.make_inputs(B, 1, w, h, K)
    fe = pl.Frontend(w, h, max_batch=B, orb=cfg["orb"], lines=bench.LINES, lm_caps=(bench.N_PTS + 20, bench.N_LINES + 8))
    fe.set_camera(K, D)
    fe.pack_pose_problems(problems, pinned=True)
    fe.upload_pose_problems(None)
    fe.set_tracking(True)
    torch.cuda.synchronize()
    d_frames = torch.from_numpy(frames).cuda()
    fs = torch.cuda.Stream()
    bs = torch.cuda.Stream()
    one = pl.LocalBAWindows([p])

    def after():
        fe.run_dev(d_frames.data_ptr(), w, w * h, B, fs.cuda_stream)
        pl.LocalBundleAdjustmentWithLine(p)

    def beside():
        fe.run_dev(d_frames.data_ptr(), w, w * h, B, fs.cuda_stream)
        one.run(bs)

    forms = {"pl_local_ba after the step": after, "pl_local_ba_dev beside the step": beside,
             "step alone": lambda: fe.run_dev(d_frames.data_ptr(), w, w * h, B, fs.cuda_stream)}
    for f in forms.values():
        for _ in range(args.warmup):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in forms}
    for _ in range(args.rounds):
        for k, f in forms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                f()
            torch.cuda.synchronize()
            times[k].append(1000 * (time.perf_counter() - t0) / args.steps)
    assert one.results()[0]["status"] == 0
    res["step"] = {k: dict(ms_per_step=float(np.median(v)), round_ms=v, frames_per_s=B / float(np.median(v)) * 1e3)
                   for k, v in times.items()}
    res["step_config"] = dict(frames=B, frame=[w, h], steps_per_round=args.steps, rounds=args.rounds)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
