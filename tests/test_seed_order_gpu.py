"""GPU test of the LSD seed order built on chip (k_lsd_seed_order, one 8-CTA cluster per frame, forced at every batch size
by PLSLAM_LSD_SEED_ORDER=cluster) against the three-kernel sort through HBM (k_lsd_hist/scan/scatter,
PLSLAM_LSD_SEED_ORDER=legacy): the order of every frame and its length (ndef)
must be identical, byte for byte, on the three camera shapes (752x480 and 1241x376 have sw % 4 != 0), on a frame without
one defined pixel, on a frame whose pixels nearly all fall into one magnitude bin (that bin straddles several CTAs'
slices of the order), and at batches of 1, 3 and 4224 frames.  The order and its lengths are overwritten with 0xff before
each run, so each run is checked on what it writes itself."""
import numpy as np
import pytest
import plslam_b200 as pl
from plslam_b200 import synth

pytestmark = pytest.mark.gpu


def _flat(w, h):
    return np.full((h, w), 97, np.uint8)            # no gradient anywhere: maxs = 0, ndef = 0


def _one_bin(w, h):
    # triangle wave of slope 8 along x: the blur keeps the ramps and the 0.8x resize maps them to slope exactly 10, so
    # every pixel off the apexes has gx = 20, gy = 0 and lands in bin 1023
    x = np.arange(w) % 64
    row = np.where(x < 32, 8 * x, 8 * (64 - x)).astype(np.uint8)
    return np.tile(row, (h, 1))


def _slice(w, h):
    sw, sh = int(round(w * 0.8)), int(round(h * 0.8))
    return (((sw - 1) * (sh - 1) + 7) // 8 + 3) // 4 * 4     # order positions each CTA of the cluster owns


def _orders(monkeypatch, ex, imgs, legacy):
    monkeypatch.setenv("PLSLAM_LSD_SEED_ORDER", "legacy" if legacy else "cluster")
    ex.debug_fill_order(0xFF)                       # every entry the call reports must be written by this call
    ex.extract_batch(imgs)
    assert ex.debug_seed_path() == (0 if legacy else 1)
    return [ex.debug_order(f) for f in range(len(imgs))]


def _check(monkeypatch, w, h, imgs):
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, width=w, height=h, max_batch=len(imgs))
    old = _orders(monkeypatch, ex, imgs, legacy=True)
    new = _orders(monkeypatch, ex, imgs, legacy=False)
    for f, (a, b) in enumerate(zip(old, new)):
        assert len(a) == len(b), (f, len(a), len(b))
        assert a.tobytes() == b.tobytes(), (f, int(np.nonzero(a != b)[0][0]))
    return [len(a) for a in old]


@pytest.mark.parametrize("w,h,seed", [(640, 480, 1), (752, 480, 5), (1241, 376, 4)])
def test_single_frame(monkeypatch, w, h, seed):
    nd = _check(monkeypatch, w, h, synth.synth_frame(w, h, seed)[None])
    S = _slice(w, h)
    assert nd[0] > S and nd[0] % S != 0          # the order spans several CTAs and ends inside a slice


@pytest.mark.parametrize("w,h,seed", [(640, 480, 2), (752, 480, 6), (1241, 376, 7)])
def test_three_frames_flat_one_bin_textured(monkeypatch, w, h, seed):
    imgs = np.stack([_flat(w, h), _one_bin(w, h), synth.synth_frame(w, h, seed)])
    nd = _check(monkeypatch, w, h, imgs)
    assert nd[0] == 0
    assert nd[1] > 2 * _slice(w, h)
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, width=w, height=h, max_batch=1)
    ex(imgs[1])
    sw = int(round(w * 0.8))
    o = ex.debug_order()
    sc = ex.debug_scaled().astype(np.int32)
    # most of the frame's order is one run of equal gradients: the ramp pixels, in row-major order
    gx = (sc[1:, 1:] - sc[:-1, :-1]) + (sc[:-1, 1:] - sc[1:, :-1])
    gy = (sc[1:, 1:] - sc[:-1, :-1]) - (sc[:-1, 1:] - sc[1:, :-1])
    ramp = np.nonzero(((gx * gx + gy * gy) == 400).ravel())[0]
    ramp = (ramp // (sw - 1)) * sw + ramp % (sw - 1)
    assert len(ramp) > nd[1] // 2
    p = int(np.nonzero(o == ramp[0])[0][0])
    assert np.array_equal(o[p:p + len(ramp)], ramp.astype(np.uint32))


def test_full_batch_4224(monkeypatch):
    w, h, B = 640, 480, 4224
    base = synth.synth_sequence(8, w, h, seed=11)
    imgs = np.empty((B, h, w), np.uint8)
    for i in range(B):                                # distinct frames: the sequence shifted by i pixels
        imgs[i] = np.roll(base[i % 8], i, axis=1)
    imgs[100] = _flat(w, h)
    imgs[2001] = _one_bin(w, h)
    nd = _check(monkeypatch, w, h, imgs)
    assert nd[100] == 0 and min(nd[:100]) > 0


def test_forced_cluster_on_a_frame_it_cannot_sort_is_an_error(monkeypatch):
    # 1920x1080: 863 rows of 1536 scaled pixels over 8 CTAs exceed the 16-bit per-CTA counters
    img = _flat(1920, 1080)
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, width=1920, height=1080)
    monkeypatch.setenv("PLSLAM_LSD_SEED_ORDER", "cluster")
    with pytest.raises(pl.PLError, match="does not fit k_lsd_seed_order"):
        ex(img)
    monkeypatch.delenv("PLSLAM_LSD_SEED_ORDER")
    ex.debug_fill_order(0xFF)
    ex(img)                                           # the default sorts it with k_lsd_hist/scan/scatter
    assert ex.debug_seed_path() == 0 and len(ex.debug_order()) == 0
