"""Generate tests/golden/lsd_cv2_scale1.npz: cv2's LSD with scale 1.0 (regions grown on the image itself, no blur or resize) on
small unblurred images, so the whole range of 2x2 gradients reaches region growing: straight step edges at random angles
and contrasts, over a noisy ramp, 96 x 72.  tests/test_oracle_lsd_scale1.py holds the oracle to these segment lists bit for bit.

Usage: python tools/gen_golden_lsd_scale1.py"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "lsd_cv2_scale1.npz")


def images(seed, n, h=72, w=96):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    out = []
    for _ in range(n):
        img = 128 + x * rng.uniform(-1, 1) + y * rng.uniform(-1, 1) + rng.normal(0, rng.uniform(0.5, 4), (h, w))
        for _ in range(rng.integers(3, 7)):      # half-planes: unblurred edges of every direction and height
            t = rng.uniform(0, 2 * np.pi)
            img += rng.uniform(-120, 120) * (np.cos(t) * (x - rng.uniform(0, w)) + np.sin(t) * (y - rng.uniform(0, h)) > 0)
        out.append(np.clip(np.rint(img), 0, 255).astype(np.uint8))
    return np.stack(out)


def cv2_segments(img):
    s = cv2.createLineSegmentDetector(cv2.LSD_REFINE_STD, 1.0).detect(img)[0]
    return np.zeros((0, 4), np.float32) if s is None else s.reshape(-1, 4).astype(np.float32)


def main():
    imgs = images(2026, 24)
    segs = [cv2_segments(im) for im in imgs]
    np.savez_compressed(OUT, imgs=imgs, nseg=np.array([len(s) for s in segs], np.int32), segs=np.concatenate(segs),
                        cv2_version=np.array(cv2.__version__))
    print(f"wrote {OUT}: {len(imgs)} images, {sum(len(s) for s in segs)} segments")


if __name__ == "__main__":
    main()
