"""The oracle's LSD with scale 1.0 against cv2.createLineSegmentDetector(LSD_REFINE_STD, 1.0), bit for bit.  At scale 1 regions
grow on the unblurred image, so these images reach the gradients up to |g| = 510 and directions of every kind that the blurred,
0.8x frames of test_oracle_line.py rarely produce.  This pins the scale-1 path as a whole, not the arithmetic of region_grow's
float sums: the three readings of its addend give the same segments on these images (test_oracle_lsd_knife_edge.py pins that on
constructed ones).  Committed cv2 4.13 output (tools/gen_golden_lsd_scale1.py), and live cv2 on fresh images when it is
importable."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from oracle import binding as ob  # noqa: E402

G = os.path.join(ROOT, "tests", "golden", "lsd_cv2_scale1.npz")


def test_lsd_scale1_vs_cv2_golden():
    z = np.load(G)
    imgs, nseg, segs = z["imgs"], z["nseg"], z["segs"]
    assert len(imgs) == 24 and nseg.sum() == len(segs) and len(segs) >= 50
    off = np.concatenate([[0], np.cumsum(nseg)])
    for i, img in enumerate(imgs):
        got = ob.lsd_detect_scale1(img)
        assert got.tobytes() == segs[off[i]:off[i + 1]].tobytes(), f"image {i}: {len(got)} segments vs cv2's {nseg[i]}"


def test_lsd_scale1_vs_live_cv2():
    pytest.importorskip("cv2")
    import gen_golden_lsd_scale1 as gen
    for i, img in enumerate(gen.images(7, 48)):
        assert ob.lsd_detect_scale1(img).tobytes() == gen.cv2_segments(img).tobytes(), f"image {i}"
