"""GPU tests of the frame memory layouts the entry points accept: row stride, frame stride and base address chosen by the
caller.  The device entry points (pl_orb_extract_batch_dev, pl_line_extract_batch_dev, pl_undistort_remap_batch_dev,
pl_frontend_run_dev) read the caller's buffer directly, with its pitch; the host entry points and the front-end's host calls
repack strided frames before the kernels run.  Every byte outside the W x H windows is random, so a kernel that read the
padding (a width used where the stride belongs) changes its result.  Each layout must give, byte for byte, what the packed
frames give, and what the CPU oracle gives."""
import ctypes as C
import numpy as np
import pytest
import oracle
import plslam_b200 as pl
from plslam_b200 import synth
from plslam_b200 import binding as plb

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

LAYOUTS = ["pitch64", "odd", "offset1", "interleaved"]


def _geometry(kind, W, H, B):
    """(row stride, frame stride, base offset, buffer bytes) of a layout."""
    if kind == "pitch64":       # 64-byte aligned rows wider than the frame: the ORB level-0 bulk copies with stride != width
        s = (W + 63) // 64 * 64 + 64
        return s, s * H + 4096, 0, (s * H + 4096) * B
    if kind == "odd":           # rows and frames at odd pitches: plain strided copies
        s = W + 3
        return s, s * H + 1, 0, (s * H + 1) * B
    if kind == "offset1":       # packed rows that start one byte past an aligned address
        return W, W * H, 1, W * H * B + 1
    if kind == "interleaved":   # an [H][B][W] tensor: the frame stride is smaller than stride * H
        return B * W, W, 0, H * B * W
    raise ValueError(kind)


class Frames:
    """B frames [B][H][W] placed in a device buffer of the given layout; all other bytes random."""

    def __init__(self, frames, kind, seed=0):
        B, H, W = frames.shape
        self.stride, self.frame_stride, self.base, nbytes = _geometry(kind, W, H, B)
        rng = np.random.default_rng(seed)
        self.buf = torch.from_numpy(rng.integers(0, 256, nbytes, dtype=np.uint8)).cuda()
        view = torch.as_strided(self.buf, (B, H, W), (self.frame_stride, self.stride, 1), self.base)
        view.copy_(torch.from_numpy(np.ascontiguousarray(frames)).cuda())
        self.ptr = self.buf.data_ptr() + self.base
        torch.cuda.synchronize()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _orb_dev(ex, F, B):
    cap = ex.capacity
    kps = torch.zeros(B * cap * pl.KP_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    desc = torch.zeros(B * cap * 32, dtype=torch.uint8, device="cuda")
    n = torch.zeros(B, dtype=torch.int32, device="cuda")
    ex.extract_batch_dev(F.ptr, F.stride, F.frame_stride, B, kps.data_ptr(), desc.data_ptr(), n.data_ptr(), _stream())
    torch.cuda.synchronize()
    pl.check(pl.lib().pl_orb_check_overflow(ex._h))
    return (kps.cpu().numpy().view(pl.KP_DTYPE).reshape(B, cap), desc.cpu().numpy().reshape(B, cap, 32), n.cpu().numpy())


def _line_dev(ex, F, B):
    cap = ex.capacity
    kl = torch.zeros(B * cap * pl.KEYLINE_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    desc = torch.zeros(B * cap * 32, dtype=torch.uint8, device="cuda")
    lf = torch.zeros(B * cap * 3, dtype=torch.float64, device="cuda")
    n = torch.zeros(B, dtype=torch.int32, device="cuda")
    ex.extract_batch_dev(F.ptr, F.stride, F.frame_stride, B, None, kl.data_ptr(), desc.data_ptr(), lf.data_ptr(), n.data_ptr(),
                         _stream())
    torch.cuda.synchronize()
    pl.check(pl.lib().pl_line_check_overflow(ex._h))
    return (kl.cpu().numpy().view(pl.KEYLINE_DTYPE).reshape(B, cap), desc.cpu().numpy().reshape(B, cap, 32),
            lf.cpu().numpy().reshape(B, cap, 3), n.cpu().numpy())


def _same_batch(a, b, counts):
    for x, y in zip(a, b):
        for f in range(len(counts)):
            assert x[f, :counts[f]].tobytes() == y[f, :counts[f]].tobytes(), f


# ------------------------------------------------------------------------------------------------------------ ORB
@pytest.mark.parametrize("kind", LAYOUTS)
def test_orb_dev_layouts(kind):
    B = 3
    frames = synth.synth_sequence(B, 640, 480, seed=61)
    ex = pl.ORBextractor(1000, 1.2, 8, 20, 7, max_batch=B)
    F = Frames(frames, kind, seed=1)          # kept alive: the handle reads level 0 back from it
    kps, desc, n = _orb_dev(ex, F, B)
    # level 0 is the caller's buffer, read back through its stride
    o = oracle.OrbOracle(1000, 1.2, 8, 20, 7)
    for b in range(B):
        assert np.array_equal(ex.mvImagePyramid(0, frame=b), frames[b]), b
        okps, odesc = o.extract(frames[b])
        assert n[b] == len(okps) and kps[b, :n[b]].tobytes() == okps.tobytes() and np.array_equal(desc[b, :n[b]], odesc), b
        for l in (0, 1):
            c, oc = ex.debug_candidates(l, frame=b), o.candidates(l)
            assert len(c) == len(oc), (b, l)
            for f in ("x", "y", "response"):
                assert np.array_equal(c[f], oc[f]), (b, l, f)
        assert np.array_equal(ex.mvImagePyramid(0, frame=b, with_border=True), o.level(0, True)), b
    pk, pd, pn = ex.extract_batch(frames)              # packed host frames
    assert np.array_equal(pn, n)
    _same_batch((kps, desc), (pk, pd), n)


def test_orb_host_entry_with_explicit_strides():
    """pl_orb_extract_batch with a row stride and frame stride of the caller's (the Python wrapper packs its input first)."""
    B, W, H = 3, 640, 480
    frames = synth.synth_sequence(B, W, H, seed=62)
    stride, fs = W + 3, (W + 3) * H + 1
    host = np.random.default_rng(2).integers(0, 256, fs * B, dtype=np.uint8)
    np.lib.stride_tricks.as_strided(host, (B, H, W), (fs, stride, 1))[:] = frames
    ex = pl.ORBextractor(1000, 1.2, 8, 20, 7, max_batch=B)
    kps = np.zeros((B, ex.capacity), pl.KP_DTYPE); desc = np.zeros((B, ex.capacity, 32), np.uint8); n = np.zeros(B, np.int32)
    pl.check(pl.lib().pl_orb_extract_batch(ex._h, host.ctypes.data_as(C.c_void_p), stride, fs, B, plb._p(kps), plb._p(desc), plb._p(n)))
    pk, pd, pn = ex.extract_batch(frames)
    assert np.array_equal(pn, n)
    _same_batch((kps, desc), (pk, pd), n)


# ------------------------------------------------------------------------------------------------------------ lines
def _check_lines(ex, got, frames, K=None, D=None, which=None):
    kl, desc, lf, n = got
    for b in (range(len(frames)) if which is None else which):
        img = oracle.undistort_remap(frames[b], K, D) if K is not None else frames[b]
        assert np.array_equal(ex.debug_scaled(b), oracle.lsd_stages(img)[0]), ("scaled image", b)
        dx, dy = ex.debug_sobel(b)
        odx, ody = oracle.lbd_sobel(img)
        assert np.array_equal(dx, odx) and np.array_equal(dy, ody), ("Sobel pair", b)
        assert ex.debug_segments(b).tobytes() == oracle.lsd_detect(img).tobytes(), ("segments", b)
        okl, odesc, olf = oracle.line_extract(img)
        assert n[b] == len(okl) and kl[b, :n[b]].tobytes() == okl.tobytes(), ("KeyLines", b)
        assert np.array_equal(desc[b, :n[b]], odesc), ("LBD descriptors", b)
        assert lf[b, :n[b]].tobytes() == olf.tobytes(), ("line equations", b)


@pytest.mark.parametrize("kind", LAYOUTS)
@pytest.mark.parametrize("camera", [False, True])
def test_line_dev_layouts(kind, camera):
    B = 3
    frames = synth.synth_sequence(B, 640, 480, seed=63)
    K, D = (synth.TUM1_K, synth.TUM1_DIST) if camera else (None, None)
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, max_batch=B)
    if camera:                                  # the frames are remapped into the handle's buffer first (B < 32 per SM)
        ex.set_undistort(pl.Undistorter(K, D, 640, 480))
    F = Frames(frames, kind, seed=3)
    got = _line_dev(ex, F, B)
    _check_lines(ex, got, frames, K, D)
    pkl, pdesc, plf, pn = ex.extract_batch(frames)
    assert np.array_equal(pn, got[3])
    _same_batch(got[:3], (pkl, pdesc, plf), pn)


def test_line_dev_pitched_full_batch_stages_the_map():
    """From 32 frames per SM on, the fused pass reads the raw pitched frames through a map staged in shared memory."""
    B = torch.cuda.get_device_properties(0).multi_processor_count * 32
    base = synth.synth_sequence(5, 640, 480, seed=64)
    frames = np.ascontiguousarray(np.tile(base, (B // 5 + 1, 1, 1))[:B])
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, max_batch=B)
    ex.set_undistort(pl.Undistorter(synth.TUM1_K, synth.TUM1_DIST, 640, 480))
    F = Frames(frames, "pitch64", seed=4)
    got = _line_dev(ex, F, B)
    _check_lines(ex, got, frames, synth.TUM1_K, synth.TUM1_DIST, which=(0, B // 2 + 3, B - 1))


def test_line_host_entry_with_explicit_strides():
    B, W, H = 3, 640, 480
    frames = synth.synth_sequence(B, W, H, seed=65)
    stride, fs = W + 3, (W + 3) * H + 1
    host = np.random.default_rng(5).integers(0, 256, fs * B, dtype=np.uint8)
    np.lib.stride_tricks.as_strided(host, (B, H, W), (fs, stride, 1))[:] = frames
    ex = pl.LINEextractor(1, 1.2, 200, 0.0, max_batch=B)
    cap = ex.capacity
    kl = np.zeros((B, cap), pl.KEYLINE_DTYPE); desc = np.zeros((B, cap, 32), np.uint8)
    lf = np.zeros((B, cap, 3), np.float64); n = np.zeros(B, np.int32)
    pl.check(pl.lib().pl_line_extract_batch(ex._h, host.ctypes.data_as(C.c_void_p), stride, fs, B, None, plb._p(kl), plb._p(desc),
                                            plb._p(lf), plb._p(n)))
    pkl, pdesc, plf, pn = ex.extract_batch(frames)
    assert np.array_equal(pn, n)
    _same_batch((kl, desc, lf), (pkl, pdesc, plf), n)


# ------------------------------------------------------------------------------------------------------------ undistortion
def _camera(name):
    if name == "euroc":
        return synth.EUROC_K, synth.EUROC_DIST, 752, 480
    w, h = 321, 243                  # a TUM1-like lens on an odd-sized frame
    return np.array([0.8 * w, 0.8 * w, 0.5 * w - 0.3, 0.5 * h + 0.2], np.float32), synth.TUM1_DIST, w, h


@pytest.mark.parametrize("cam", ["euroc", "odd"])
@pytest.mark.parametrize("dst_off,dframe_pad", [(0, 0), (1, 0), (2, 0), (3, 0), (0, 2), (1, 2)])
def test_undistort_remap_dev_layouts(cam, dst_off, dframe_pad):
    """Pitched source; destination rows of round64(W) bytes starting at any byte offset, and frame strides that are not a
    multiple of 4 (dframe = 2 mod 4): the 4-pixel stores must fall back to bytes where the row is not 4-byte aligned.  Every
    byte outside the destination windows is unchanged."""
    K, D, W, H = _camera(cam)
    B = 3
    frames = np.stack([synth.synth_frame(W, H, 66 + b) for b in range(B)])
    src = Frames(frames, "pitch64", seed=6)
    dstride = (W + 63) // 64 * 64
    dframe = dstride * H + dframe_pad
    assert dframe_pad == 0 or dframe % 4 == 2
    nbytes = dst_off + dframe * B + 64
    init = np.random.default_rng(7).integers(0, 256, nbytes, dtype=np.uint8)
    dst = torch.from_numpy(init.copy()).cuda()
    und = pl.Undistorter(K, D, W, H)
    und.remap_batch_dev(src.ptr, src.stride, src.frame_stride, B, dst.data_ptr() + dst_off, dstride, dframe, _stream())
    torch.cuda.synchronize()
    out = dst.cpu().numpy()
    win = np.lib.stride_tricks.as_strided(out[dst_off:], (B, H, W), (dframe, dstride, 1))
    inside = np.zeros(nbytes, bool)
    np.lib.stride_tricks.as_strided(inside[dst_off:], (B, H, W), (dframe, dstride, 1))[:] = True
    for b in range(B):
        assert np.array_equal(win[b], oracle.undistort_remap(frames[b], K, D)), b
    assert np.array_equal(out[~inside], init[~inside])


# ------------------------------------------------------------------------------------------------------------ front-end
def _frontend(B, problems):
    fe = pl.Frontend(640, 480, max_batch=B, lm_caps=(320, 88))
    fe.set_camera(synth.TUM1_K, synth.TUM1_DIST)
    fe.set_pose_problems(problems)
    fe.set_wrap(True)
    fe.set_tracking(True)
    return fe


@pytest.mark.parametrize("kind", ["pitch64", "offset1"])
def test_frontend_run_dev_layouts(kind):
    """pl_frontend_run_dev on device frames of another layout equals pl_frontend_run on the packed host frames: every field
    of fetch and fetch_tracking, byte for byte."""
    B = 3
    frames = synth.synth_sequence(B, 640, 480, seed=67)
    problems = [synth.synth_pose_problem(140 + k) for k in range(B)]
    ref = _frontend(B, problems)
    want = ref.run(frames)
    want_t = [ref.fetch_tracking(B, w) for w in (0, 1)]
    assert want["n"].min() > 100 and want["nl"].min() > 20
    fe = _frontend(B, problems)
    F = Frames(frames, kind, seed=8)
    fe.run_dev(F.ptr, F.stride, F.frame_stride, B, _stream())
    torch.cuda.synchronize()
    pl.check(pl.lib().pl_frontend_check_overflow(fe._h))
    got = fe.fetch(B)
    for k in pl.Frontend.ORDER:
        if k != "linefunc":                    # fetch does not return the line equations
            assert got[k].tobytes() == want[k].tobytes(), k
    for w in (0, 1):
        t = fe.fetch_tracking(B, w)
        for k in t:
            assert t[k].tobytes() == want_t[w][k].tobytes(), (w, k)
    assert fe.fetch_keys_un(B).tobytes() == ref.fetch_keys_un(B).tobytes()


def test_frontend_run_and_submit_on_strided_host_frames():
    """Frontend.run and .submit on a view a[:, :, :W] of wider host rows (pinned for submit): the per-frame 2D copy."""
    B, W, H, pad = 3, 640, 480, 40
    frames = synth.synth_sequence(B, W, H, seed=68)
    problems = [synth.synth_pose_problem(150 + k) for k in range(B)]
    want = _frontend(B, problems).run(frames)
    wide = np.random.default_rng(9).integers(0, 256, (B, H, W + pad), dtype=np.uint8)
    wide[:, :, :W] = frames
    view = wide[:, :, :W]
    assert view.strides == (H * (W + pad), W + pad, 1)
    got = _frontend(B, problems).run(view)
    for k in pl.Frontend.ORDER:
        assert got[k].tobytes() == want[k].tobytes(), ("run", k)
    pin = torch.empty((B, H, W + pad), dtype=torch.uint8, pin_memory=True)
    pin.numpy()[:] = wide
    fe = _frontend(B, problems)
    out = fe.alloc_outputs(B, pinned=True)
    fe.submit(pin.numpy()[:, :, :W], out)
    fe.wait(0)
    for k in pl.Frontend.ORDER:
        assert out[k].tobytes() == want[k].tobytes(), ("submit", k)
