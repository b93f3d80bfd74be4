"""Time pl_track_update_local_map_dev (Tracking::UpdateLocalMap on a batch) and the whole OK-state localisation chain at B = 4224.

update_local_map: a synthetic graph the size of a real map: 300 keyframes x 1000 point slots and 100 line slots over 50 k map
points and 10 k map lines (each point in about 6 keyframes), 20 ordered covisibles per keyframe, a chain of parents.  Each frame
matches 300 of one keyframe's points.
chain: LocalizationChain (last pose -> motion model -> update local map -> local-map step -> velocity -> relative pose) on the
three streams of tests/motion_scene.py against the planar scene's keyframe graph (tests/localmap_scene.py), copied to fill the
batch; every timed step starts from the previous one's state.
After --warmup calls, --rounds rounds of --iters calls are timed with CUDA events.  Prints one JSON line: ms per batch (median
over all timed calls, with the per-round medians) and frames/s, with the card's name and power limit read in the same run.

    python tools/update_local_map_time.py [--batch 4224] [--iters 30] [--rounds 3] [--warmup 3]
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


def synthetic_graph(n_kf=300, slots=1000, n_pts=50000, lslots=100, n_lns=10000, seed=0):
    rng = np.random.default_rng(seed)
    step_p, step_l = n_pts / n_kf, n_lns / n_kf
    pt = np.stack([(int(k * step_p) + rng.choice(5000, slots, replace=False) - 2500) % n_pts for k in range(n_kf)]).astype(np.int32)
    ln = np.stack([(int(k * step_l) + rng.choice(1000, lslots, replace=False) - 500) % n_lns for k in range(n_kf)]).astype(np.int32)
    order = np.argsort(pt.ravel(), kind="stable")
    obs = (order // slots).astype(np.int32)
    obs_off = np.zeros(n_pts + 1, np.int32); obs_off[1:] = np.cumsum(np.bincount(pt.ravel(), minlength=n_pts))
    cov = np.stack([[(k + d) % n_kf for d in sorted([x for x in range(-10, 11) if x], key=abs)] for k in range(n_kf)]).astype(np.int32)
    T = np.tile(np.eye(4, dtype=np.float32), (n_kf, 1, 1))
    g = dict(Tcw=T, Twc=T, parent=np.arange(-1, n_kf - 1, dtype=np.int32), pt_slot=pt.ravel(), ln_slot=ln.ravel(), cov=cov.ravel(),
             child=np.arange(1, n_kf, dtype=np.int32), obs=obs, obs_offset=obs_off,
             pt_slot_offset=np.arange(n_kf + 1, dtype=np.int32) * slots, ln_slot_offset=np.arange(n_kf + 1, dtype=np.int32) * lslots,
             cov_offset=np.arange(n_kf + 1, dtype=np.int32) * 20, child_offset=np.r_[0, np.arange(1, n_kf + 1)].astype(np.int32))
    g["child_offset"][-1] = n_kf - 1
    return g, pt, n_pts, n_lns


def timed(call, stream, args):
    import torch
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
    return float(np.median(times)), rounds, len(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4224)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import plslam_b200 as pl
    from plslam_b200 import binding as bd
    import localmap_scene as ls
    import motion_scene as ms
    import track_scene as ts
    from test_update_local_map_gpu import _frames, _last, _start, CAP_KF
    from track_local_map_time import card

    B = args.batch
    name, plim = card()
    res = dict(tool="update_local_map_time", batch=B, card=name, power_limit=plim, configs={})
    stream = torch.cuda.Stream()      # a real stream handle: NULL would select the map's own stream, outside the events

    # 1. update_local_map alone on a real-size graph
    g, pt, n_pts, n_lns = synthetic_graph()
    M = pl.Map(**ls.quirk_map(dict(n_points=n_pts, n_lines=n_lns)))
    M.set_keyframes(g)
    rng = np.random.default_rng(1)
    cap, cLP, cLL = 1000, 32768, 8192
    pm = np.full((B, cap), -1, np.int32)
    for b in range(B):
        pm[b, :300] = np.unique(pt[rng.integers(len(pt))])[:300]
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
    t = dict(kf=dev(np.zeros((B, 128), np.int32)), n_kf=dev(np.zeros(B, np.int32)), ref_kf=dev(np.zeros(B, np.int32)),
             pt_index=dev(np.zeros((B, cLP), np.int32)), pt_count=dev(np.zeros(B, np.int32)), ln_index=dev(np.zeros((B, cLL), np.int32)),
             ln_count=dev(np.zeros(B, np.int32)))
    s = bd._local_map_struct(t, 128, cLP, cLL)
    pmd = dev(pm)
    L = bd._track_lib()

    def ulm():
        bd.check(L.pl_track_update_local_map_dev(M._h, B, C.c_void_p(pmd.data_ptr()), cap, None, None, C.byref(s),
                                                 C.c_void_p(stream.cuda_stream)))
    ms_, rounds, n = timed(ulm, stream, args)
    M.check_indices(); M.check_capacity()
    res["configs"]["update_local_map"] = dict(ms_per_batch=ms_, frames_per_s=B / ms_ * 1e3, round_medians_ms=rounds, calls=n,
                                              n_kf=300, n_points=n_pts, mean_local_kf=float(t["n_kf"].float().mean()),
                                              mean_local_points=float(t["pt_count"].float().mean()),
                                              mean_local_lines=float(t["ln_count"].float().mean()))

    # 2. the whole chain on the planar scene
    m, _, _ = ms.shifted_map()
    gs = ls.scene_graph(m)
    M2 = pl.Map(**m)
    M2.set_keyframes(ls.to_desc(gs))
    Ks, lasts, kf, n_kf, ref, Tcr, V = _start(m, gs)
    S = len(Ks)
    feats = [ts.features(ms.stream_pose(s_, 1), Ks[s_]) for s_ in range(S)]
    capP = max(max(len(f[0]) for f in feats), max(len(l_["keys"]) for l_ in lasts))
    capL = max(max(len(f[2]) for f in feats), max(len(l_["kl"]) for l_ in lasts))
    idx = np.arange(B) % S
    fr = {k: (v[idx] if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == S else v) for k, v in _frames(feats, Ks, capP, capL).items()}
    la = {k: v[idx] for k, v in _last(lasts, capP, capL).items()}
    ch = pl.LocalizationChain(M2, B, capP, capL, CAP_KF, 2048, 512, ts.BOUNDS, ts.SF, ts.INV_SIGMA2, ts.LOG_SF, max_frames=30)
    ch.set_state(la, Tcr[idx], ref[idx], V[idx], kf[idx], n_kf[idx], frames_since_reloc=np.full(B, 40, np.int32))
    ch.set_frames(fr)
    torch.cuda.synchronize()          # the uploads ran on the default stream
    ms_, rounds, n = timed(lambda: ch.localization_step(stream), stream, args)
    out = ch.fetch()
    M2.check_indices(); M2.check_capacity()
    res["configs"]["chain"] = dict(ms_per_batch=ms_, frames_per_s=B / ms_ * 1e3, round_medians_ms=rounds, calls=n, cap_points=capP,
                                   cap_lines=capL, ok_frames=int(out["lo"]["ok"].sum()),
                                   mean_local_points=float(out["local"]["pt_count"].mean()))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
