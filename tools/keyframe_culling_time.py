"""Time pl_keyframe_culling_dev with CUDA events; prints one JSON line with the card's name and power limit read in the same run.

Two forms on one table of keyframes along a trajectory (tests/kfc_scene.py, bulk: ~1500 slots per keyframe, observers per point
of median ~6, a few of the entries culled):
  single  one current keyframe whose list holds ~60 covisible keyframes: the latency a LocalMapping thread sees;
  batch   --keyframes groups per call (lists of 60 keyframes around their own current keyframe): throughput.
Each time is the median over rounds (the forms alternate round by round) of the mean of --launches launches after warm-up.  The
oracle's (tests/kfc_oracle.py, numpy) CPU time on the single group is reported beside it as a CPU number; the device results are
checked against it first.

Run from the repo root:  python tools/keyframe_culling_time.py [--keyframes 132 528] [--rounds 15] [--launches 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from plslam_b200 import binding as bd  # noqa: E402
import kfc_oracle as ko  # noqa: E402
import kfc_scene as ks  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or [","])[0].split(",")[:2]
    return name.strip(), power.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, nargs="+", default=[132, 528])
    ap.add_argument("--rows", type=int, default=400)
    ap.add_argument("--list", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--seed", type=int, default=3)
    a = ap.parse_args()
    import torch
    rng = np.random.default_rng(a.seed)
    size = rng.integers(1300, 1700, a.rows)
    b, rows = ks.bulk(rng, size)
    keyframes, points, _ = b.scene([])

    def lists(G):
        out = []
        for c in rng.integers(a.list // 2, a.rows - a.list // 2, G):
            near = sorted(range(a.rows), key=lambda k: (abs(k - c), k))
            out.append([rows[k] for k in near[1:a.list + 1]])
        return out

    k = bd.pack_cull_keyframes(keyframes)
    m = bd.pack_cull_points(points)
    forms = {"single": lists(1)}
    forms.update({f"batch_{G}": lists(G) for G in a.keyframes})
    probs = {n: bd.KeyFrameCullingProblems(k, m, bd.pack_cull_groups(g)) for n, g in forms.items()}

    s1 = ks.packed(keyframes, points, forms["single"])
    t0 = time.perf_counter()
    want = ko.cull(s1)
    oracle_ms = (time.perf_counter() - t0) * 1e3
    probs["single"].run()
    got = probs["single"].results()[0]
    assert got["status"] == 0 and np.array_equal(got["code"], want["code"]) and np.array_equal(got["n_mps"], want["n_mps"]) \
        and np.array_equal(got["n_redundant"], want["n_redundant"]), "device differs from the oracle"

    stream = torch.cuda.Stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for p in probs.values():                                  # warm-up
        for _ in range(3):
            p.run(stream)
    stream.synchronize()
    times = {n: [] for n in probs}
    for _ in range(a.rounds):
        for n, p in probs.items():
            ev0.record(stream)
            for _ in range(a.launches):
                p.run(stream)
            ev1.record(stream)
            ev1.synchronize()
            times[n].append(ev0.elapsed_time(ev1) / a.launches)
    name, power = card()
    out = dict(tool="keyframe_culling_time", gpu=name, power_limit=power, rounds=a.rounds, launches=a.launches,
               table_keyframes=a.rows, list_len=a.list, slots_per_keyframe_median=int(np.median(size)),
               observers_per_point_median=float(np.median(np.diff(m["obs_offset"]))),
               single_culled=int((got["code"] == 1).sum()), single_ms=float(np.median(times["single"])),
               oracle_cpu_ms_single=oracle_ms)
    for G in a.keyframes:
        t = float(np.median(times[f"batch_{G}"]))
        out[f"batch_{G}_ms"] = t
        out[f"batch_{G}_groups_per_s"] = G / t * 1e3
    print(json.dumps(out))


if __name__ == "__main__":
    main()
