"""Generate tests/golden/orb_ref_*.npz from the REFERENCE's own ORBextractor.

oracle/_ref/libref_orb.so is /root/reference/src/ORBextractor.cc compiled unmodified where it lies (oracle/Makefile target
`ref`; the OpenCV primitives behind oracle/shim/ are the oracle's cv2-4.13-pinned restatements, and list nodes get increasing
heap addresses so that the pointer tie-break of ORBextractor.cc:684 is reproducible).  The reference does not travel to the
GPU box, so its outputs on the seeded synthetic frames are committed here: tests/test_oracle_orb_ref.py checks the oracle
against them on CPU, tests/test_orb_gpu.py checks the CUDA path against them on the GPU.
Run from the repo root, in the container that has /root/reference:  python tools/gen_golden_orb_ref.py
"""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import plslam_b200  # noqa  (synth only; no GPU needed)
from plslam_b200 import synth
import oracle

assert oracle.ref_orb_available(), "needs /root/reference (make -C oracle ref)"
out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def frame(kind, w, h, seed):
    if kind == "synth":
        return synth.synth_frame(w, h, seed)
    if kind == "low":      # only the minThFAST fallback fires
        return (synth.synth_frame(w, h, seed) // 16 + 100).astype(np.uint8)
    if kind == "noise":    # maximum candidate density
        return np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)
    if kind == "sparse":   # fewer candidates than the quota
        im = np.full((h, w), 90, np.uint8); im[200:230, 300:340] = 200
        return im
    raise ValueError(kind)


CASES = {"640x480_n1000": ("synth", 640, 480, 1, 1000, 1.2, 8), "640x480_n2000": ("synth", 640, 480, 1, 2000, 1.2, 8),
         "752x480_n1000": ("synth", 752, 480, 5, 1000, 1.2, 8), "1241x376_n2000": ("synth", 1241, 376, 4, 2000, 1.2, 8),
         "640x480_low": ("low", 640, 480, 9, 1000, 1.2, 8), "640x480_noise": ("noise", 640, 480, 5, 1000, 1.2, 8),
         "640x480_sparse": ("sparse", 640, 480, 0, 1000, 1.2, 8), "640x480_n500_s11": ("synth", 640, 480, 11, 500, 1.2, 8)}

# Extractor settings other than the TUM one: level count, scale factor, FAST thresholds and frame size each shape the
# pyramid, the resize tables, the FAST cell grid, the per-level quotas and the quadtree pool.  All on synth frames.
# name: (w, h, seed, nfeatures, scale_factor, nlevels, ini_th, min_th); written to orb_ref_set_<name>.npz
SETTINGS = {"l12": (640, 480, 31, 1000, 1.2, 12, 20, 7),        # 12 levels: the smallest is 86x65, one row of FAST cells
            "l1": (640, 480, 32, 1000, 1.2, 1, 20, 7),          # no resize, one quadtree
            "th12_5": (640, 480, 33, 3000, 1.2, 8, 12, 5),      # low thresholds, large quota
            "th30_15": (640, 480, 34, 1000, 1.2, 8, 30, 15),    # many cells fall back to minThFAST
            "th10_10": (640, 480, 35, 1000, 1.2, 8, 10, 10),    # iniThFAST == minThFAST
            "th5_3": (640, 480, 36, 1000, 1.2, 8, 5, 3),        # ~9000 level-0 candidates
            "s11": (752, 480, 37, 800, 1.1, 10, 20, 7),         # fine pyramid, level widths not multiples of 16
            "s20": (800, 600, 38, 1200, 2.0, 3, 20, 7),         # ratio-2 resize tables
            "s15": (640, 480, 39, 1500, 1.5, 5, 20, 7),
            "kitti10": (1241, 376, 40, 2000, 1.2, 10, 20, 7),   # last level 241x73
            "odd": (333, 251, 41, 300, 1.2, 6, 20, 7),          # odd sizes in both dimensions
            "tiny": (96, 80, 42, 60, 1.2, 1, 20, 7),            # near the smallest frame
            "hd": (1920, 1080, 43, 5000, 1.2, 8, 20, 7),        # ~45k level-0 candidates
            "pool": (1920, 1080, 44, 4800, 1.2, 1, 20, 7)}      # a quadtree pool near an H100's 227 KB of shared memory


def save(path, r, im, params, sf, kind, **extra):
    kps, desc = r.extract(im)
    t = r.tables()
    nl = r.nlevels
    np.savez_compressed(path, kps=kps, desc=desc, img_sum=np.int64(im.astype(np.int64).sum()), params=np.array(params),
                        scale_factor=np.float32(sf), kind=kind,
                        scale=t["scale"], inv_scale=t["inv_scale"], sigma2=t["sigma2"], inv_sigma2=t["inv_sigma2"],
                        level_dims=np.array([r.level(l).shape[::-1] for l in range(nl)]),
                        level_sums=np.array([int(r.level(l).astype(np.int64).sum()) for l in range(nl)]), **extra)
    return len(kps)


if __name__ == "__main__":
    for name, (kind, w, h, seed, nf, sf, nl) in CASES.items():
        im = frame(kind, w, h, seed)
        n = save(os.path.join(out, f"orb_ref_{name}.npz"), oracle.RefOrb(nf, sf, nl, 20, 7), im, [w, h, seed, nf, nl], sf, kind)
        print(name, n)
    for name, (w, h, seed, nf, sf, nl, ini, mn) in SETTINGS.items():
        im = synth.synth_frame(w, h, seed)
        n = save(os.path.join(out, f"orb_ref_set_{name}.npz"), oracle.RefOrb(nf, sf, nl, ini, mn), im,
                 [w, h, seed, nf, nl, ini, mn], sf, "synth")
        print(name, n)
