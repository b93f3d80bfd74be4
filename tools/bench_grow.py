"""A/B timing of the LSD region-growing kernel across builds of the library: python tools/bench_grow.py lib1.so lib2.so ...
Prints per library the k_lsd_grow time of one launch over B frames (CUDA events inside the library) and a checksum of the
line outputs (must be identical across builds)."""
import ctypes as C, os, sys, zlib
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import plslam_b200 as pl
from plslam_b200 import synth
B = int(os.environ.get("B", 4224)); W, H = 640, 480
base = synth.synth_sequence(64, W, H, seed=1)
rng = np.random.Generator(np.random.PCG64(78))
frames = np.empty((B, H, W), np.uint8)
for r in range(0, B, 64):
    k = min(64, B - r)
    frames[r:r + k] = base[:k] if r == 0 else np.clip(base[:k].astype(np.int16) + rng.integers(-3, 4, (k, H, W), dtype=np.int16), 0, 255).astype(np.uint8)
d = torch.from_numpy(frames).cuda()
vp = C.c_void_p
for path in sys.argv[1:]:
    L = C.CDLL(os.path.abspath(path))
    L.pl_last_error.restype = C.c_char_p
    cfg = pl.binding.PLLineConfig(W, H, 200, 0.0, B, 0, 0)
    h = vp()
    L.pl_line_create.argtypes = [C.POINTER(pl.binding.PLLineConfig), C.POINTER(vp)]
    L.pl_line_extract_batch_dev.argtypes = [vp, vp, C.c_int, C.c_size_t, C.c_int, vp, vp, vp, vp, vp, vp]
    L.pl_line_set_timing.argtypes = [vp, C.c_int]; L.pl_line_grow_ms.argtypes = [vp, vp]; L.pl_line_destroy.argtypes = [vp]
    L.pl_line_capacity.argtypes = [vp]
    assert L.pl_line_create(C.byref(cfg), C.byref(h)) == 0, L.pl_last_error()
    cap = L.pl_line_capacity(h)
    kl = torch.zeros((B, cap, 68), dtype=torch.uint8, device="cuda"); desc = torch.zeros((B, cap, 32), dtype=torch.uint8, device="cuda")
    lf = torch.zeros((B, cap, 3), dtype=torch.float64, device="cuda"); n = torch.zeros(B, dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    L.pl_line_set_timing(h, 1)
    ms = []
    for it in range(4):
        rc = L.pl_line_extract_batch_dev(h, d.data_ptr(), W, W * H, B, None, kl.data_ptr(), desc.data_ptr(), lf.data_ptr(), n.data_ptr(), st.cuda_stream)
        assert rc == 0, L.pl_last_error()
        torch.cuda.synchronize()
        m = C.c_float(0); L.pl_line_grow_ms(h, C.byref(m)); ms.append(m.value)
    nn = n.cpu().numpy()
    crc = zlib.crc32(desc.cpu().numpy()[:256].tobytes()) ^ zlib.crc32(nn.tobytes())
    print(f"{os.path.basename(path):40s} grow_ms {min(ms[1:]):8.2f} (all {['%.1f' % x for x in ms]})  lines/frame {nn.mean():.1f}  crc {crc:08x}", flush=True)
    L.pl_line_destroy(h)
    del kl, desc, lf, n
    torch.cuda.empty_cache()
