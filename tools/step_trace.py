"""Kernel timeline of bench steps (torch.profiler / CUPTI): start and end of every kernel relative to the first kernel, per
stream, and how much of each chain's kernel time falls inside the k_lsd_grow_ordered launch.
python tools/step_trace.py [--batch B] [--steps N] [--trace FILE.json] [--list]
PLSLAM_B200_LIB=<path> selects another build of the library (A/B work)."""
import argparse, json, os, sys, tempfile
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
import plslam_b200 as pl

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=4224); ap.add_argument("--steps", type=int, default=2)
ap.add_argument("--trace", default=None, help="keep the Chrome trace here (default: a temporary file)")
ap.add_argument("--list", action="store_true", help="print every kernel with its start and end")
a = ap.parse_args()
B = a.batch
K, D = bench.camera_of(bench.CONFIGS["tum"])
frames, problems = bench.make_inputs(B, 1, bench.W, bench.H, K)
fe = pl.Frontend(bench.W, bench.H, max_batch=B, orb=bench.ORB, lines=bench.LINES, lm_caps=(bench.N_PTS + 20, bench.N_LINES + 8))
fe.set_pose_problems(problems); fe.set_camera(K, D); fe.set_tracking(True)
d = torch.from_numpy(frames).cuda()
st = torch.cuda.Stream()
for _ in range(2):
    fe.run_dev(d.data_ptr(), bench.W, bench.W * bench.H, B, st.cuda_stream)
torch.cuda.synchronize()
from torch.profiler import profile, ProfilerActivity
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(a.steps):
        fe.run_dev(d.data_ptr(), bench.W, bench.W * bench.H, B, st.cuda_stream)
    torch.cuda.synchronize()
path = a.trace or os.path.join(tempfile.mkdtemp(), "trace.json")
prof.export_chrome_trace(path)
ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
ks = sorted(((e["ts"], e["ts"] + e["dur"], e["args"].get("stream"), e["name"].split("(")[0].split("<")[0].split("::")[-1]) for e in ev))
t0 = ks[0][0]
grows = [(s, e) for s, e, _, n in ks if n == "k_lsd_grow_ordered"]
line_st = {k[2] for k in ks if k[3] == "k_lsd_grow_ordered"}
lm_st = {k[2] for k in ks if k[3] == "k_pose_opt"} - line_st
chain = lambda s: "line" if s in line_st else "pose" if s in lm_st else "orb"


def inside(s, e):
    return sum(max(0.0, min(e, ge) - max(s, gs)) for gs, ge in grows)


span = ks[-1][1] - t0
print(f"lib {os.environ.get('PLSLAM_B200_LIB', 'default')}  B={B}  {a.steps} steps  first kernel start to last kernel end "
      f"{span / 1000 / a.steps:.2f} ms/step")
for gs, ge in grows:
    print(f"  k_lsd_grow_ordered  {(gs - t0) / 1000:9.3f} .. {(ge - t0) / 1000:9.3f} ms  ({(ge - gs) / 1000:.3f} ms)")
tot = {}
for s, e, stream, n in ks:
    c = chain(stream)
    t = tot.setdefault(c, [0.0, 0.0])
    t[0] += e - s
    if n != "k_lsd_grow_ordered":
        t[1] += inside(s, e)
sum_all = sum(t[0] for t in tot.values())
for c in ("line", "orb", "pose"):
    if c in tot:
        busy, ov = tot[c]
        print(f"  {c:5s} chain  kernel time {busy / 1000 / a.steps:8.2f} ms/step ({100 * busy / sum_all:4.1f} % of the serialised sum)  "
              f"inside the grow {ov / 1000 / a.steps:8.2f} ms/step")
print(f"  serialised sum {sum_all / 1000 / a.steps:.2f} ms/step, timeline {span / 1000 / a.steps:.2f} ms/step: overlap saves "
      f"{100 * (1 - span / sum_all):.1f} %")
if a.list:
    for s, e, stream, n in ks:
        print(f"  {chain(stream):5s} {n[:40]:40s} {(s - t0) / 1000:9.3f} .. {(e - t0) / 1000:9.3f} ms  {(e - s) / 1000:8.3f}"
              f"  inside grow {inside(s, e) / 1000 if n != 'k_lsd_grow_ordered' else 0.0:8.3f}")
