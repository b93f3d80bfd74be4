"""Time pl_track_local_map_dev (Tracking::TrackLocalMapWithLines on a batch) at B = 4224 with 2k- and 4k-entry local maps.

Frames: the planar scene of tests/track_scene.py (four rendered frames, two cameras), copied to fill the batch.  Map: the scene's
1004 map points and 201 map lines; the points are tiled 5x (5020 points) with small offsets along the viewing ray so that a
4096-entry list names distinct points (the searches then see up to five candidates per keypoint).  Every frame's list is the first
2048 or 4096 points and all lines.  The two sizes are timed alternately for --rounds rounds of --iters calls each, after --warmup
calls of each.  Prints one JSON line: ms per batch (CUDA events around each call; median over all timed calls, with the spread of
the per-round medians) and frames/s, with the card's name and power limit read in the same run.

    python tools/track_local_map_time.py [--batch 4224] [--iters 50] [--rounds 3] [--warmup 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        name, plim = [s.strip() for s in q.split(",")]
        return name, plim
    except Exception as e:   # the numbers are still printed, with the card unknown
        return f"unknown ({e})", "unknown"


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
    import track_scene as ts

    m = ts.scene_map()
    reps = 5
    off = np.repeat(np.arange(reps, dtype=np.float32), len(m["pt_pos"]))[:, None] * np.float32(0.002)
    big = dict(m, pt_pos=np.tile(m["pt_pos"], (reps, 1)) * (1 + off), pt_normal=np.tile(m["pt_normal"], (reps, 1)),
               pt_min_dist=np.tile(m["pt_min_dist"], reps), pt_max_dist=np.tile(m["pt_max_dist"], reps), pt_desc=np.tile(m["pt_desc"], (reps, 1)))
    M = pl.Map(**big)
    items = [(T, K, ts.perturb(T, 0.006, k), None, None) for k, (T, K) in enumerate(ts.TRUE)]
    fr0, _ = ts.batch_frames(items)
    B = args.batch
    idx = np.arange(B) % len(items)
    fr = {k: (v[idx] if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == len(items) else v) for k, v in fr0.items()}
    L = bd._track_lib()
    name, plim = card()
    res = dict(tool="track_local_map_time", batch=B, card=name, power_limit=plim, configs={})
    runs = {}
    for n_local in (2048, 4096):
        assert n_local <= len(big["pt_pos"]), "the local list must name map points"
        local = dict(pt_index=np.arange(len(big["pt_pos"]), dtype=np.int32), ln_index=np.arange(len(m["ln_pos"]), dtype=np.int32),
                     pt_offset=np.zeros(B, np.int32), pt_count=np.full(B, n_local, np.int32), ln_offset=np.zeros(B, np.int32),
                     ln_count=np.full(B, len(m["ln_pos"]), np.int32), frames_since_reloc=np.full(B, 5, np.int32), max_frames=30)
        torch_, keep, to_dev = bd._torch_dev()
        arr = {k: v for k, v in fr.items() if isinstance(v, np.ndarray)}
        arr["Tcw0"] = arr["Tcw0"].reshape(B, 16)
        d = {k: to_dev(v)[1] for k, v in arr.items()}
        s, cLP, cLL = bd._local_struct(local, B, keep, to_dev)
        cap, capL = fr["keys_un"].shape[1], fr["keylines"].shape[1]
        F = bd.PLTrackFrames(B, d["keys_un"], d["desc"], d["n"], cap, d["keylines"], d["line_func"], d["line_desc"], d["nl"], capL,
                             d["bounds"], d["scale_factors"], d["inv_level_sigma2"], len(ts.SF), ts.LOG_SF, d["Tcw0"], d["K"],
                             d["point_map_in"], d["line_map_in"])
        shapes = bd._out_shapes(B, cap, capL, cLP, cLL)
        outs = {k: torch.zeros(max(int(np.prod(shapes[k][0])) * np.dtype(shapes[k][1]).itemsize, 16), dtype=torch.uint8, device="cuda")
                for k in bd._TRACK_OUT[:7]}
        o = bd.PLTrackOut(*[C.c_void_p(outs[k].data_ptr()) if k in outs else None for k in bd._TRACK_OUT])
        nbytes = int(L.pl_track_local_map_scratch_bytes(B, cap, capL, cLP, cLL))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        runs[n_local] = dict(F=F, s=s, o=o, outs=outs, scratch=scratch, keep=keep, d=d, nbytes=nbytes, times=[], rounds=[])
    stream = torch.cuda.Stream()      # a real stream handle: NULL would select the map's own stream, outside the events

    def call(r):
        bd.check(L.pl_track_local_map_dev(M._h, C.byref(r["F"]), C.byref(r["s"]), C.byref(r["o"]), C.c_void_p(r["scratch"].data_ptr()),
                                          C.c_void_p(stream.cuda_stream)))

    for r in runs.values():
        for _ in range(args.warmup):
            call(r)
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for r in runs.values():
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
            for e0, e1 in ev:
                e0.record(stream); call(r); e1.record(stream)
            torch.cuda.synchronize()
            t = [e0.elapsed_time(e1) for e0, e1 in ev]
            r["times"] += t; r["rounds"].append(float(np.median(t)))
    M.check_indices()
    for n_local, r in runs.items():
        ok = r["outs"]["ok"][:4 * B].cpu().numpy().view(np.int32)
        ms = float(np.median(r["times"]))
        res["configs"][f"local_points_{n_local}"] = dict(ms_per_batch=ms, frames_per_s=B / ms * 1e3, round_medians_ms=r["rounds"],
                                                        calls=len(r["times"]), local_lines=len(m["ln_pos"]), scratch_bytes=r["nbytes"],
                                                        ok_frames=int(ok.sum()))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
