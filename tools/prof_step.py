"""N device-resident steps of the bench workload (frames already in HBM), nothing else: the command ncu wraps.
python tools/prof_step.py [--batch B] [--steps N]"""
import argparse, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
import plslam_b200 as pl
from plslam_b200 import synth
ap = argparse.ArgumentParser(); ap.add_argument("--batch", type=int, default=4224); ap.add_argument("--steps", type=int, default=4)
a = ap.parse_args()
B = a.batch
K, D = bench.camera_of(bench.CONFIGS["tum"])
frames, problems = bench.make_inputs(B, 1, bench.W, bench.H, K)
fe = pl.Frontend(bench.W, bench.H, max_batch=B, orb=bench.ORB, lines=bench.LINES, lm_caps=(bench.N_PTS + 20, bench.N_LINES + 8))
fe.set_pose_problems(problems); fe.set_camera(K, D); fe.set_tracking(True)
d = torch.from_numpy(frames).cuda()
st = torch.cuda.Stream()
for _ in range(a.steps):
    fe.run_dev(d.data_ptr(), bench.W, bench.W * bench.H, B, st.cuda_stream)
torch.cuda.synchronize()
print("done", a.steps, "steps of", B, "frames")
