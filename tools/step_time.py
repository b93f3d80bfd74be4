"""Device-resident step time of the bench workload plus a CRC of everything the step returns (A/B of build or
environment variants: the CRC must not move).  python tools/step_time.py [--batch B] [--steps N] [--warmup W] [--tag T]"""
import argparse, os, sys, zlib
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
import plslam_b200 as pl

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=4224); ap.add_argument("--steps", type=int, default=4)
ap.add_argument("--warmup", type=int, default=2); ap.add_argument("--tag", default="")
a = ap.parse_args()
B = a.batch
K, D = bench.camera_of(bench.CONFIGS["tum"])
frames, problems = bench.make_inputs(B, 1, bench.W, bench.H, K)
fe = pl.Frontend(bench.W, bench.H, max_batch=B, orb=bench.ORB, lines=bench.LINES, lm_caps=(bench.N_PTS + 20, bench.N_LINES + 8))
fe.set_pose_problems(problems); fe.set_camera(K, D); fe.set_tracking(True); fe.set_wrap(True); fe.set_timing(True)
d = torch.from_numpy(frames).cuda()
st = torch.cuda.Stream()
with torch.cuda.stream(st):
    for _ in range(a.warmup):
        fe.run_dev(d.data_ptr(), bench.W, bench.W * bench.H, B, st.cuda_stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(st)
    grow = []
    for _ in range(a.steps):
        fe.run_dev(d.data_ptr(), bench.W, bench.W * bench.H, B, st.cuda_stream)
    e1.record(st)
    torch.cuda.synchronize()
    grow.append(fe.grow_ms())
o = fe.fetch(B)
crc = 0
for k in ("kps", "desc", "n", "keylines", "ldesc", "nl", "pt_matches", "line_matches", "inliers"):
    crc = zlib.crc32(np.ascontiguousarray(o[k]).tobytes(), crc)
print(f"{a.tag} B={B} step {e0.elapsed_time(e1) / a.steps:.2f} ms  grow {grow[-1]:.2f} ms  crc {crc:08x}  nl_mean {o['nl'].mean():.1f}")
