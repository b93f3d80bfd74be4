"""Frames and comparisons shared by the line-extraction shape tests (test_line_shapes_gpu.py, test_oracle_line_shapes_ref.py).

SHAPES are the frame sizes past the three camera shapes: the smallest frame the extractor accepts, odd sizes, tiles of
k_lsd_front that end one pixel past or one pixel short of whole tiles (64x32 scaled, 80x40 source), portrait frames (the
KeyLine response divides by the larger side), the two sides of the cluster seed sort's shared-memory limit, 720p and 1080p.
"""
import numpy as np
from plslam_b200 import synth

# (width, height, seed, segment_cap): a textured 1920x1080 frame has ~13,000 segments, over the default cap of 8192
SHAPES = [(64, 64, 3, 0), (81, 121, 3, 0), (321, 243, 3, 0), (641, 481, 3, 0), (719, 439, 3, 0), (480, 640, 3, 0),
          (376, 1241, 3, 0), (800, 600, 3, 0), (1280, 384, 3, 0), (1282, 384, 3, 0), (1280, 720, 3, 0), (1920, 1080, 3, 16384)]
# shapes compared with the reference library itself: portrait, odd tiles, 1080p
REF_SHAPES = [(480, 640, 3), (376, 1241, 3), (641, 481, 3), (719, 439, 3), (1920, 1080, 3)]
# selection edges are taken on this frame (492 segments)
SEL_FRAME = (321, 243, 3)


def flat(w, h):
    return np.full((h, w), 97, np.uint8)            # no gradient anywhere: no seeds, no segments


def one_bin(w, h):
    # triangle wave of slope 8 along x: nearly every pixel lands in the top magnitude bin (test_seed_order_gpu.py)
    x = np.arange(w) % 64
    return np.tile(np.where(x < 32, 8 * x, 8 * (64 - x)).astype(np.uint8), (h, 1))


def corner(w, h, seed):
    """A textured frame whose bottom-right corner holds diagonal stripes: their edges run from the last column to the last row,
    so LSD finds segments with one or both end points clamped onto the frame's border."""
    img = synth.synth_frame(w, h, seed).copy()
    y, x = np.mgrid[0:h, 0:w]
    d = (w - 1 - x) + (h - 1 - y)
    band = d < 120
    img[band] = np.where((d[band] // 15) % 2 == 0, 230, 25).astype(np.uint8)
    return img


def border_mask(w, h):
    """255 everywhere but the last column and the last row"""
    m = np.full((h, w), 255, np.uint8)
    m[:, w - 1] = 0
    m[h - 1, :] = 0
    return m


def patch(w, h, pw, ph, seed):
    """a flat frame with a textured pw x ph patch in its middle: fewer segments than a textured frame of the same size"""
    img = flat(w, h)
    y0, x0 = (h - ph) // 2, (w - pw) // 2
    img[y0:y0 + ph, x0:x0 + pw] = synth.synth_frame(pw, ph, seed)
    return img


def same_line_funcs(a, b):
    """line equations bit for bit; the appended zero KeyLine's equation is 0/0 on both sides (NaN, of either sign)"""
    assert a.shape == b.shape, (a.shape, b.shape)
    fin = np.isfinite(b).all(1)
    assert a[fin].tobytes() == b[fin].tobytes(), "line equations"
    assert np.isnan(a[~fin]).all() and np.isnan(b[~fin]).all(), "line equations of the appended KeyLine"


def same_up_to_equal_response_swaps(k, d, l, rk, rd, rl):
    """LINEextractor's selection against the reference library's.  LineExtractor.cpp:43 sorts with std::sort, which is not
    stable: lines of EQUAL response may come out in either order (this project keeps detection order).  Anything else must match
    bit for bit; such swaps are undone before the comparison."""
    assert len(k) == len(rk), (len(k), len(rk))
    if k.tobytes() != rk.tobytes():
        bad = [i for i in range(len(k)) if k[i].tobytes() != rk[i].tobytes()]
        assert all(k["response"][i] == rk["response"][i] for i in bad) and len(bad) <= 4, bad
        ends = ["startPointX", "startPointY", "endPointX", "endPointY"]
        key = lambda x: [tuple(r) for r in np.sort(x[bad][ends].copy(), order=ends[:2])]
        assert key(k) == key(rk)
        keep = np.setdiff1d(np.arange(len(k)), bad)
        k, d, l, rk, rd, rl = k[keep], d[keep], l[keep], rk[keep], rd[keep], rl[keep]
    assert k.tobytes() == rk.tobytes(), "KeyLine records"
    assert np.array_equal(d, rd), "LBD descriptors"
    assert l.tobytes() == rl.tobytes(), "line equations"
