"""Time pl_track_motion_model_dev (Tracking::TrackWithMotionModel on a batch) and pl_track_velocity_dev at B = 4224.

Frames: the first two steps of each constant-velocity stream of tests/motion_scene.py (three streams, two cameras) against the
scene's map; each frame's last frame is the previous step tracked by the local-map composite, with the stream's true velocity.
The three frames are copied to fill the batch.  After --warmup calls, --rounds rounds of --iters calls are timed.  Prints one JSON
line: ms per batch (CUDA events around each call; median over all timed calls, with the spread of the per-round medians) and
frames/s, with the card's name and power limit read in the same run.

    python tools/track_motion_model_time.py [--batch 4224] [--iters 50] [--rounds 3] [--warmup 5]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4224)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    import plslam_b200 as pl
    from plslam_b200 import binding as bd
    import motion_scene as ms
    import track_scene as ts
    from test_track_motion_model_gpu import _batch
    from track_local_map_time import card

    m = ts.scene_map()
    M = pl.Map(**m)
    items = []
    for s in range(len(ms.STREAMS)):
        K = ms.STREAMS[s][2]
        items.append((ms.stream_pose(s, 1), K, dict(ms.last_frame(m, ms.stream_pose(s, 0), K, seed=s), velocity=ms.STREAMS[s][1])))
    fr0, _, last0 = _batch(items)
    B = args.batch
    idx = np.arange(B) % len(items)
    fr = {k: (v[idx] if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == len(items) else v) for k, v in fr0.items()}
    last = {k: v[idx] for k, v in last0.items()}
    cap, capL = fr["keys_un"].shape[1], fr["keylines"].shape[1]
    L = bd._track_lib()
    name, plim = card()
    torch_, keep, to_dev = bd._torch_dev()
    d = {k: to_dev(np.ascontiguousarray(v))[1] for k, v in fr.items() if isinstance(v, np.ndarray)}
    dl = {k: to_dev(np.ascontiguousarray(v))[1] for k, v in last.items()}
    F = bd.PLTrackFrames(B, d["keys_un"], d["desc"], d["n"], cap, d["keylines"], d["line_func"], d["line_desc"], d["nl"], capL,
                         d["bounds"], d["scale_factors"], d["inv_level_sigma2"], len(ts.SF), ts.LOG_SF, None, d["K"], None, None)
    Ls = bd.PLTrackLast(*[dl[k] for k, _ in bd.PLTrackLast._fields_])
    shapes = bd._mm_shapes(B, cap, capL)
    outs = {k: torch.zeros(max(int(np.prod(shapes[k][0])) * np.dtype(shapes[k][1]).itemsize, 16), dtype=torch.uint8, device="cuda")
            for k in bd._MM_OUT[:8]}
    o = bd.PLTrackMotionOut(*[C.c_void_p(outs[k].data_ptr()) if k in outs else None for k in bd._MM_OUT])
    nbytes = int(L.pl_track_motion_model_scratch_bytes(B, cap, capL))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    vel = torch.zeros(B * 16, dtype=torch.float32, device="cuda")
    stream = torch.cuda.Stream()      # a real stream handle: NULL would select the map's own stream, outside the events

    def mm():
        bd.check(L.pl_track_motion_model_dev(M._h, C.byref(F), C.byref(Ls), C.byref(o), C.c_void_p(scratch.data_ptr()),
                                             C.c_void_p(stream.cuda_stream)))

    def velocity():
        bd.check(L.pl_track_velocity_dev(B, C.c_void_p(outs["Tcw"].data_ptr()), dl["Tcw"], C.c_void_p(outs["ok"].data_ptr()),
                                         C.c_void_p(vel.data_ptr()), C.c_void_p(stream.cuda_stream)))

    res = dict(tool="track_motion_model_time", batch=B, card=name, power_limit=plim, cap_points=cap, cap_lines=capL, scratch_bytes=nbytes,
               configs={})
    for label, call in (("motion_model", mm), ("velocity", velocity)):
        for _ in range(args.warmup):
            call()
        torch.cuda.synchronize()
        times, rounds = [], []
        for _ in range(args.rounds):
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
            for e0, e1 in ev:
                e0.record(stream); call(); e1.record(stream)
            torch.cuda.synchronize()
            t = [e0.elapsed_time(e1) for e0, e1 in ev]
            times += t; rounds.append(float(np.median(t)))
        ms = float(np.median(times))
        res["configs"][label] = dict(ms_per_batch=ms, frames_per_s=B / ms * 1e3, round_medians_ms=rounds, calls=len(times))
    M.check_indices()
    ok = outs["ok"][:4 * B].cpu().numpy().view(np.int32)
    res["configs"]["motion_model"]["ok_frames"] = int(ok.sum())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
