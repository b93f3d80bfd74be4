"""GPU parity tests of the fused image pass of the line extractor (k_lsd_front): raw frames go in, the extractor reads them
through a bound undistortion map (LINEextractor.set_undistort), and every stage must equal the CPU oracle run on the
oracle's own undistorted frame, byte for byte: scaled image, Sobel pair, LSD segments, KeyLines, LBD descriptors and line
equations.  The shapes cover the camera configurations, tiles cut by the frame edge and batches that do not fill the
frames-per-CTA count."""
import numpy as np
import pytest
import oracle
import plslam_b200 as pl
from plslam_b200 import synth

pytestmark = pytest.mark.gpu


def _small_camera(w, h):
    # a TUM1-like lens scaled to a small frame, so that the map reaches across tile and frame edges
    return np.array([0.8 * w, 0.8 * w, 0.5 * w - 0.3, 0.5 * h + 0.2], np.float32), synth.TUM1_DIST


def _check_batch(w, h, K, D, B, seed):
    frames = synth.synth_sequence(B, w, h, seed=seed) if B > 1 else synth.synth_frame(w, h, seed)[None]
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, width=w, height=h, max_batch=B)
    if K is not None:
        und = pl.Undistorter(K, D, w, h)
        ex.set_undistort(und)
        del und                          # the extractor keeps its map alive
    kl, desc, lf, n = ex.extract_batch(frames)
    for b in range(B):
        img = oracle.undistort_remap(frames[b], K, D) if K is not None else frames[b]
        sc, _, _ = oracle.lsd_stages(img)
        assert np.array_equal(ex.debug_scaled(b), sc), ("scaled image", b)
        dx, dy = ex.debug_sobel(b)
        odx, ody = oracle.lbd_sobel(img)
        assert np.array_equal(dx, odx) and np.array_equal(dy, ody), ("Sobel pair", b)
        seg = ex.debug_segments(b); oseg = oracle.lsd_detect(img)
        assert seg.shape == oseg.shape and seg.tobytes() == oseg.tobytes(), ("segments", b)
        okl, odesc, olf = oracle.line_extract(img)
        assert n[b] == len(okl), ("KeyLine count", b)
        assert kl[b, :n[b]].tobytes() == okl.tobytes(), ("KeyLine records", b)
        assert np.array_equal(desc[b, :n[b]], odesc), ("LBD descriptors", b)
        assert lf[b, :n[b]].tobytes() == olf.tobytes(), ("line equations", b)


@pytest.mark.parametrize("w,h,cam,B,seed", [
    (640, 480, "tum1", 1, 41),
    (640, 480, "tum1", 3, 42),
    (640, 480, "tum1", 11, 43),    # one CTA walks 8 frames: 11 leaves a partial group
    (752, 480, "euroc", 3, 44),
    (1241, 376, None, 3, 45),      # KITTI shape, no map: identity source, scaled width 993 (rows not 16-byte aligned)
    (81, 70, "small", 3, 46),      # scaled width 65 and undistorted width 81: last tile one pixel wide in both
    (64, 64, "small", 2, 47),      # narrower than one tile (51 scaled, 64 undistorted columns)
    (64, 64, None, 1, 48),
])
def test_raw_frames_through_the_map_match_oracle(w, h, cam, B, seed):
    if cam == "tum1":
        K, D = synth.TUM1_K, synth.TUM1_DIST
    elif cam == "euroc":
        K, D = synth.EUROC_K, synth.EUROC_DIST
    elif cam == "small":
        K, D = _small_camera(w, h)
    else:
        K, D = None, None
    _check_batch(w, h, K, D, B, seed)


def test_unbinding_the_map_takes_undistorted_frames_again():
    frames = synth.synth_sequence(2, 640, 480, seed=49)
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, max_batch=2)
    ex.set_undistort(pl.Undistorter(synth.TUM1_K, synth.TUM1_DIST, 640, 480))
    ex.extract_batch(frames)
    ex.set_undistort(None)
    kl, desc, lf, n = ex.extract_batch(frames)
    for b in range(2):
        okl, odesc, _ = oracle.line_extract(frames[b])
        assert kl[b, :n[b]].tobytes() == okl.tobytes() and np.array_equal(desc[b, :n[b]], odesc), b


def test_map_of_another_size_is_an_error():
    ex = pl.LINEextractor(1, 1.2, 200, 0.0)
    with pytest.raises(pl.PLError, match="pl_line_set_undistort"):
        ex.set_undistort(pl.Undistorter(synth.EUROC_K, synth.EUROC_DIST, 752, 480))


def test_full_batch_stages_the_map():
    """From 32 frames per SM on, a CTA stages its tile's camera map in shared memory once for all its frames; the first, a
    middle and the last frame of such a batch against the oracle."""
    import torch
    B = torch.cuda.get_device_properties(0).multi_processor_count * 32
    base = synth.synth_sequence(5, 640, 480, seed=50)
    frames = np.ascontiguousarray(np.tile(base, (B // 5 + 1, 1, 1))[:B])
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, max_batch=B)
    ex.set_undistort(pl.Undistorter(synth.TUM1_K, synth.TUM1_DIST, 640, 480))
    kl, desc, lf, n = ex.extract_batch(frames)
    for b in (0, B // 2 + 3, B - 1):
        img = oracle.undistort_remap(frames[b], synth.TUM1_K, synth.TUM1_DIST)
        assert np.array_equal(ex.debug_scaled(b), oracle.lsd_stages(img)[0]), b
        dx, dy = ex.debug_sobel(b)
        odx, ody = oracle.lbd_sobel(img)
        assert np.array_equal(dx, odx) and np.array_equal(dy, ody), b
        okl, odesc, olf = oracle.line_extract(img)
        assert n[b] == len(okl) and kl[b, :n[b]].tobytes() == okl.tobytes() and np.array_equal(desc[b, :n[b]], odesc), b
