"""GPU parity tests of line extraction past the camera shapes and the default settings, byte for byte against the CPU oracle:
scaled image, seed order, Sobel pair, LSD segment list, KeyLines, LBD descriptors and line equations.

- every shape of line_shapes.SHAPES through both seed sorts (k_lsd_hist/scan/scatter and the cluster kernel k_lsd_seed_order,
  forced with PLSLAM_LSD_SEED_ORDER), one frame alone and three frames of mixed content in one batch;
- a batch of 32 frames per SM at a small odd shape (serial front pass, default cluster sort, k_lsd_grow_ordered<false>), with
  and without an undistortion map, every frame against the same frame extracted alone;
- LINEextractor's selection edges (nfeatures around the line count, min_line_length above every line or equal to a line's
  length, a cut at the first line, masks that drop lines, mask lookups on the clamped last row and column);
- segment_cap: a frame over it raises, keeps the first segment_cap segments and clears the flag; in a batch only that frame is
  cut; a cap whose sort does not fit k_keylines's shared memory, or a negative one, is refused at creation."""
import functools
import numpy as np
import pytest
import oracle
import plslam_b200 as pl
from plslam_b200 import synth
import line_shapes as LS

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

PL_ERR_ARG, PL_ERR_CAPACITY = -1, -3


def _cluster_fits(w, h):
    """pl_line_create's test for k_lsd_seed_order: 8 CTAs share the (sw-1)(sh-1) order positions of the frame, each with
    32 warps x 1024 16-bit bin counters and 2 x 1024 ints beside its slice, 2 KB under the device's opt-in shared memory"""
    sw, sh = round(w * 0.8), round(h * 0.8)
    q = -(-((sh - 1) * sw) // 8)
    s = (-(-((sw - 1) * (sh - 1)) // 8) + 3) // 4 * 4
    smem = s * 4 + 32 * 1024 * 2 + 2 * 1024 * 4
    return q <= 65535 and smem + 2048 <= torch.cuda.get_device_properties(0).shared_memory_per_block_optin


@functools.lru_cache(maxsize=None)
def _frame(w, h, kind, seed):
    img = {"textured": lambda: synth.synth_frame(w, h, seed), "flat": lambda: LS.flat(w, h), "one_bin": lambda: LS.one_bin(w, h)}[kind]()
    img.setflags(write=False)
    return img


@functools.lru_cache(maxsize=None)
def _oracle(w, h, kind, seed):
    img = _frame(w, h, kind, seed)
    sc, mg, an = oracle.lsd_stages(img)
    defined = (an != -1024.0).ravel()
    idx = np.nonzero(defined)[0]
    order = idx[:0]
    if len(idx):      # defined pixels, magnitude bin descending, row-major inside a bin
        mgf = mg.ravel()
        bins = (mgf * (1023.0 / mgf[idx].max())).astype(np.int64)
        order = idx[np.argsort(-bins[idx], kind="stable")]
    return dict(scaled=sc, order=order.astype(np.uint32), sobel=oracle.lbd_sobel(img), segs=oracle.lsd_detect(img),
                lines=oracle.line_extract(img))


def _segments_equal(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert a.tobytes() == b.tobytes(), (what, "first differing segment", int(np.nonzero((a != b).any(1))[0][0]))


def _lines_equal(kl, desc, lf, want, what):
    okl, odesc, olf = want
    assert len(kl) == len(okl), (what, "KeyLine count", len(kl), len(okl))
    assert kl.tobytes() == okl.tobytes(), (what, "KeyLine records")
    assert np.array_equal(desc, odesc), (what, "LBD descriptors")
    LS.same_line_funcs(lf, olf)


def _stages_equal(ex, b, want, kl, desc, lf, what):
    assert np.array_equal(ex.debug_scaled(b), want["scaled"]), (what, "blur + 0.8x resize")
    o = ex.debug_order(b)
    assert len(o) == len(want["order"]) and o.tobytes() == want["order"].tobytes(), (what, "seed order")
    dx, dy = ex.debug_sobel(b)
    assert np.array_equal(dx, want["sobel"][0]) and np.array_equal(dy, want["sobel"][1]), (what, "LBD Sobel pair")
    _segments_equal(ex.debug_segments(b), want["segs"], what)
    _lines_equal(kl, desc, lf, want["lines"], what)


# ---------------------------------------------------------------------------------------------- shapes x seed sorts x batches
@pytest.mark.parametrize("path", ["legacy", "cluster"])
@pytest.mark.parametrize("w,h,seed,cap", LS.SHAPES)
def test_stages_match_oracle(monkeypatch, w, h, seed, cap, path):
    monkeypatch.setenv("PLSLAM_LSD_SEED_ORDER", path)
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, width=w, height=h, max_batch=3, segment_cap=cap)
    if path == "cluster" and not _cluster_fits(w, h):
        with pytest.raises(pl.PLError, match="does not fit k_lsd_seed_order"):
            ex(_frame(w, h, "textured", seed))
        return
    # alone, then between a flat and a one-bin frame: a per-frame stride wrong at this size moves the textured frame's data
    for kinds in ([("textured", seed)], [("flat", 0), ("textured", seed), ("one_bin", 0)]):
        imgs = np.stack([_frame(w, h, k, s) for k, s in kinds])
        ex.debug_fill_order(0xFF)                   # every entry the call reports must be written by this call
        kl, desc, lf, n = ex.extract_batch(imgs)
        assert ex.debug_seed_path() == (path == "cluster")
        for b, (k, s) in enumerate(kinds):
            _stages_equal(ex, b, _oracle(w, h, k, s), kl[b, :n[b]], desc[b, :n[b]], lf[b, :n[b]], (k, b, len(kinds)))


def test_the_two_shapes_straddle_the_cluster_limit():
    if torch.cuda.get_device_properties(0).shared_memory_per_block_optin != 227 * 1024:
        pytest.skip("the 1280x384 / 1282x384 pair brackets the limit of a device with 227 KB of opt-in shared memory (H100)")
    assert _cluster_fits(1280, 384) and not _cluster_fits(1282, 384)


# ---------------------------------------------------------------------------------------------- serial batch at a small shape
def _small_camera(w, h):
    # a TUM1-like lens scaled to the frame: the map moves pixels by several columns near the edges
    return np.array([0.8 * w, 0.8 * w, 0.5 * w - 0.3, 0.5 * h + 0.2], np.float32), synth.TUM1_DIST


@pytest.mark.parametrize("undistort", [False, True])
def test_serial_batch_at_a_small_shape(monkeypatch, undistort):
    """32 frames per SM of 100x77: the serial front pass (with the camera map read inside it when undistorting), the default
    cluster sort and k_lsd_grow_ordered<false>.  Alone, each frame takes k_lsd_front on undistorted frames (k_remap first when
    undistorting), k_lsd_hist/scan/scatter and k_lsd_grow_ordered<true>."""
    monkeypatch.delenv("PLSLAM_LSD_SEED_ORDER", raising=False)
    w, h = 100, 77
    B = torch.cuda.get_device_properties(0).multi_processor_count * 32
    base = synth.synth_sequence(8, w, h, seed=60)
    imgs = np.empty((B, h, w), np.uint8)
    for i in range(B):                       # distinct frames: 8 frames x 100 column shifts x row shifts
        imgs[i] = np.roll(base[i % 8], (i // 800, (i // 8) % 100), axis=(0, 1))
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, width=w, height=h, max_batch=B)
    one = pl.LINEextractor(1, 1.2, 200, 0.0, width=w, height=h)
    K, D = _small_camera(w, h)
    if undistort:
        und = pl.Undistorter(K, D, w, h)
        ex.set_undistort(und)
        one.set_undistort(und)
        assert not np.array_equal(oracle.undistort_remap(imgs[0], K, D), imgs[0])
    kl, desc, lf, n = ex.extract_batch(imgs)
    assert ex.debug_seed_path() == 1
    rng = np.random.default_rng(61)
    for b in sorted(set(rng.choice(B, 48, replace=False).tolist()) | {0, B - 1}):
        img = oracle.undistort_remap(imgs[b], K, D) if undistort else imgs[b]
        assert np.array_equal(ex.debug_scaled(b), oracle.lsd_stages(img)[0]), b
        _segments_equal(ex.debug_segments(b), oracle.lsd_detect(img), b)
        _lines_equal(kl[b, :n[b]], desc[b, :n[b]], lf[b, :n[b]], oracle.line_extract(img), b)
    for b in range(B):
        k1, d1, l1 = one(imgs[b])
        assert one.debug_seed_path() == 0
        assert n[b] == len(k1) and kl[b, :n[b]].tobytes() == k1.tobytes(), b
        assert np.array_equal(desc[b, :n[b]], d1) and lf[b, :n[b]].tobytes() == l1.tobytes(), b


# ---------------------------------------------------------------------------------------------- selection edges
def _select(img, nf, mll, mask=None):
    h, w = img.shape
    kl, desc, lf = pl.LINEextractor(1, 1.2, nf, mll, width=w, height=h)(img, mask)
    _lines_equal(kl, desc, lf, oracle.line_extract(img, mask=mask, nfeatures=nf, min_line_length=mll), (nf, mll))
    return kl


def test_nfeatures_around_the_line_count():
    img = synth.synth_frame(*LS.SEL_FRAME)
    n = len(oracle.lsd_detect(img))
    assert len(_select(img, n - 1, 0.0)) == n                    # nfeatures + 1 kept: every line
    assert len(_select(img, n, 0.0)) == n + 1                    # one zero KeyLine appended
    assert len(_select(img, n + 1, 0.0)) == n + 1
    assert len(_select(img, 1, 0.0)) == 2


def test_min_line_length_edges():
    img = synth.synth_frame(*LS.SEL_FRAME)
    L = oracle.line_extract(img, nfeatures=200)[0]["lineLength"].astype(np.float64)
    assert len(_select(img, 200, 1e6)) == 201                   # above every line: nothing is cut (LineExtractor.cpp quirk)
    k = next(i for i in range(100, 190) if L[i - 1] > L[i] > L[i + 1])
    assert len(_select(img, 200, L[k])) == k + 1                 # a line exactly min_line_length long is kept, the cut after it
    assert len(_select(img, k + 1, L[k])) == k + 2               # ... and when it is the last line kept, nothing is cut
    assert L[0] > L[1]
    assert len(_select(img, 200, (L[0] + L[1]) / 2)) == 1        # the cut at index 0


def test_masks_that_drop_lines():
    w, h, seed = LS.SEL_FRAME
    img = synth.synth_frame(w, h, seed)
    some = np.full((h, w), 255, np.uint8)
    some[40:200, 60:260] = 0
    kept = len(oracle.line_extract(img, mask=some, nfeatures=100000)[0]) - 1
    assert 201 < kept < len(oracle.lsd_detect(img))
    _select(img, 200, 0.0, some)                                 # dropped before the truncation
    assert len(_select(img, kept, 0.0, some)) == kept + 1        # exactly nfeatures left: one zero KeyLine appended
    assert len(_select(img, 200, 0.0, np.zeros((h, w), np.uint8))) == 1


def test_mask_lookups_on_the_clamped_border():
    w, h = 641, 481
    img = LS.corner(w, h, 3)
    m = LS.border_mask(w, h)
    n = len(oracle.lsd_detect(img))
    kept = len(oracle.line_extract(img, mask=m, nfeatures=100000)[0]) - 1
    assert kept < n                                              # lines with both end points on the border are dropped
    _select(img, n + 10, 0.0, m)                                 # every line of the frame


# ---------------------------------------------------------------------------------------------- segment capacity
def _line_dev(ex, imgs):
    B, h, w = imgs.shape
    cap = ex.capacity
    d_img = torch.from_numpy(np.ascontiguousarray(imgs)).cuda()
    kl = torch.zeros(B * cap * pl.KEYLINE_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    desc = torch.zeros(B * cap * 32, dtype=torch.uint8, device="cuda")
    lf = torch.zeros(B * cap * 3, dtype=torch.float64, device="cuda")
    n = torch.zeros(B, dtype=torch.int32, device="cuda")
    ex.extract_batch_dev(d_img.data_ptr(), w, w * h, B, None, kl.data_ptr(), desc.data_ptr(), lf.data_ptr(), n.data_ptr(),
                         torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return (kl.cpu().numpy().view(pl.KEYLINE_DTYPE).reshape(B, cap), desc.cpu().numpy().reshape(B, cap, 32),
            lf.cpu().numpy().reshape(B, cap, 3), n.cpu().numpy())


@pytest.mark.parametrize("w,h,cap,small", [(640, 480, 100, ((96, 96), (120, 90))), (1280, 720, 5000, ((640, 480), (800, 600)))])
def test_segment_cap_overflow(w, h, cap, small):
    big = synth.synth_frame(w, h, 3)
    segs = oracle.lsd_detect(big)
    lo = [LS.patch(w, h, pw, ph, 5) for pw, ph in small]
    assert len(segs) > cap and all(len(oracle.lsd_detect(x)) < cap for x in lo)
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, width=w, height=h, max_batch=3, segment_cap=cap)
    with pytest.raises(pl.PLError, match=f"error {PL_ERR_CAPACITY}: LSD produced more than segment_cap={cap}"):
        ex(big)
    _segments_equal(ex.debug_segments(), segs[:cap], "the first segment_cap segments")
    kl, desc, lf = ex(lo[0])                                     # the check cleared the flag
    _lines_equal(kl, desc, lf, oracle.line_extract(lo[0]), "after the overflow")
    # in a batch only the frame over the cap is cut
    kl, desc, lf, n = _line_dev(ex, np.stack([lo[0], big, lo[1]]))
    assert pl.lib().pl_line_check_overflow(ex._h) == PL_ERR_CAPACITY
    assert pl.lib().pl_line_check_overflow(ex._h) == 0
    _segments_equal(ex.debug_segments(1), segs[:cap], "the frame over the cap")
    for b, img in ((0, lo[0]), (2, lo[1])):
        _segments_equal(ex.debug_segments(b), oracle.lsd_detect(img), b)
        _lines_equal(kl[b, :n[b]], desc[b, :n[b]], lf[b, :n[b]], oracle.line_extract(img), b)


def test_segment_cap_equal_to_the_segment_count():
    img = synth.synth_frame(*LS.SEL_FRAME)
    segs = oracle.lsd_detect(img)
    h, w = img.shape
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, width=w, height=h, segment_cap=len(segs))
    kl, desc, lf = ex(img)
    _segments_equal(ex.debug_segments(), segs, "segment_cap == segments")
    _lines_equal(kl, desc, lf, oracle.line_extract(img), "segment_cap == segments")
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, width=w, height=h, segment_cap=len(segs) - 1)
    with pytest.raises(pl.PLError, match="more than segment_cap"):
        ex(img)
    _segments_equal(ex.debug_segments(), segs[:-1], "segment_cap == segments - 1")


@pytest.mark.parametrize("cap", [16385, 20000, 1 << 20, -1, -8192])
def test_segment_cap_k_keylines_cannot_sort_is_refused(cap):
    # k_keylines sorts pow2(segment_cap) 8-byte keys in one block's shared memory: 16384 (128 KB) is the largest on an H100
    with pytest.raises(pl.PLError, match=f"error {PL_ERR_ARG}: .*segment_cap"):
        pl.LINEextractor(1, 1.2, 200, 0.0, width=1920, height=1080, segment_cap=cap)


def test_textured_1080p_frame_needs_an_explicit_segment_cap():
    img = synth.synth_frame(1920, 1080, 3)
    assert 8192 < len(oracle.lsd_detect(img)) <= 16384
    with pytest.raises(pl.PLError, match="more than segment_cap=8192"):
        pl.LINEextractor(1, 1.2, 200, 0.0, width=1920, height=1080)(img)


# ---------------------------------------------------------------------------------------------- the reference library itself
@pytest.mark.skipif(not oracle.ref_line_available(), reason="neither oracle/_ref/libref_line.so nor its stored outputs exist")
@pytest.mark.parametrize("w,h,seed", LS.REF_SHAPES)
def test_extract_matches_reference_library(w, h, seed):
    img = synth.synth_frame(w, h, seed)
    cap = 16384 if w * h > 1280 * 720 else 0
    kl, desc, lf = pl.LINEextractor(1, 1.2, 200, 0.0, width=w, height=h, segment_cap=cap)(img)
    LS.same_up_to_equal_response_swaps(kl, desc, lf, *oracle.ref_line_extract(img, nfeatures=200, min_line_length=0.0))
