"""Which arithmetic cv2's LSD region growing adds to its float sums, pinned on images where it decides the segment list.

lsd.cpp's region_grow adds cos(float(angle)), sin(float(angle)) per pixel.  Three readings are plausible - libm's cosf / sinf,
the fp64 functions rounded to fp32, the fp64 functions added in fp64 to the float sum - and they differ in the last bit on
about 1.3 % of the gradients, which random frames never show.  tests/golden/lsd_cv2_knife_edge.npz (tools/gen_lsd_knife_edge.py)
holds 4 x 2 scale-1 images built so that a candidate lies within a float ulp of 22.5 degrees from the region angle after one
differing addend, with cv2 4.13's segments.  The oracle's three readings must give different segment lists on every image,
cv2 must equal exactly one of them, and that one must be the oracle's default (cosf, what the device gradient table stores)."""
import os

import numpy as np
import pytest

from oracle import binding as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden", "lsd_cv2_knife_edge.npz")


def _golden():
    z = np.load(G)
    off = np.concatenate([[0], np.cumsum(z["nseg"])])
    return z["imgs"], [z["segs"][off[i]:off[i + 1]] for i in range(len(z["imgs"]))]


def _matches(img, ref):
    return [ob.lsd_detect_scale1(img, v).tobytes() == ref.tobytes() for v in ob.LSD_ADDENDS]


def test_cv2_adds_cosf_on_the_knife_edge_images():
    imgs, segs = _golden()
    assert len(imgs) == 48 and imgs.shape[1:] == (2, 4)
    assert any(len(s) == 0 for s in segs) and any(len(s) == 1 for s in segs)     # cosf on either side of the threshold
    for i, (img, ref) in enumerate(zip(imgs, segs)):
        outs = [ob.lsd_detect_scale1(img, v).tobytes() for v in ob.LSD_ADDENDS]
        assert len(set(outs)) > 1, f"image {i}: the three readings agree"
        m = _matches(img, ref)
        assert sum(m) == 1, f"image {i}: cv2 equals the readings {m}"
        assert m[0], f"image {i}: cv2 does not equal the default reading (cosf): {m}"
        assert ob.lsd_detect_scale1(img).tobytes() == ref.tobytes()


def test_live_cv2_on_the_knife_edge_images():
    cv2 = pytest.importorskip("cv2")
    imgs, segs = _golden()
    lsd = cv2.createLineSegmentDetector(cv2.LSD_REFINE_STD, 1.0)
    for i, (img, ref) in enumerate(zip(imgs, segs)):
        s = lsd.detect(img)[0]
        s = np.zeros((0, 4), np.float32) if s is None else s.reshape(-1, 4).astype(np.float32)
        assert s.tobytes() == ref.tobytes(), f"image {i}"
