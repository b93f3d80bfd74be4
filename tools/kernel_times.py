"""Per-kernel CUDA time of one bench step (torch.profiler / CUPTI, no ncu): python tools/kernel_times.py [--batch B]
PLSLAM_B200_LIB=<path> selects another build of the library (A/B work)."""
import argparse, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
import plslam_b200 as pl
from plslam_b200 import synth
ap = argparse.ArgumentParser(); ap.add_argument("--batch", type=int, default=4224); ap.add_argument("--steps", type=int, default=2)
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
rows = [(e.key.split("(")[0][-40:], e.count, e.device_time_total / 1000.0) for e in prof.key_averages() if e.device_time_total > 0]
tot = sum(r[2] for r in rows)
print(f"lib {os.environ.get('PLSLAM_B200_LIB', 'default')}  B={B}  total {tot / a.steps:.2f} ms/step")
for k, n, ms in sorted(rows, key=lambda r: -r[2]):
    print(f"  {k:42s} n/step {n / a.steps:5.1f}  {ms / a.steps:8.3f} ms/step  {100 * ms / tot:5.1f}%")
