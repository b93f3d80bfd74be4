"""Every handle owns its device memory: pl_device_bytes() rises when a handle is created and when one of its groups of buffers made
on first use is made, stays put on a repeated call and on the device-pointer entry points, and is back exactly where it was once
the handle is destroyed.  Each cycle runs twice and ends where it started."""
import gc

import pytest

import localmap_scene as ls
import plslam_b200 as pl
from plslam_b200 import synth

pytestmark = pytest.mark.gpu
W, H, B = 640, 480, 2


def _bytes():
    import torch
    torch.cuda.synchronize()
    return pl.device_bytes()


def _twice(cycle):
    gc.collect()
    start = _bytes()
    for _ in range(2):
        cycle()
        assert _bytes() == start


@pytest.fixture(scope="module")
def frames():
    return synth.synth_sequence(B, W, H, seed=4)


def _dev(*shape_dtypes):
    import torch
    return [torch.empty(s, dtype=d, device="cuda") for s, d in shape_dtypes]


def test_orb_handle(frames):
    import torch

    def cycle():
        b0 = _bytes()
        orb = pl.ORBextractor(1000, 1.2, 8, 20, 7, W, H, max_batch=B)
        b1 = _bytes()
        assert b1 > b0
        img = torch.from_numpy(frames).cuda()
        kps, desc, n = _dev(((B * orb.capacity * 28,), torch.uint8), ((B * orb.capacity * 32,), torch.uint8), ((B,), torch.int32))
        orb.extract_batch_dev(img.data_ptr(), W, W * H, B, kps.data_ptr(), desc.data_ptr(), n.data_ptr(),
                              torch.cuda.current_stream().cuda_stream)
        assert _bytes() == b1
        orb.extract_batch(frames)                       # host-pointer staging, made on first use
        b2 = _bytes()
        assert b2 > b1
        orb.extract_batch(frames)
        assert _bytes() == b2
        del orb
        assert _bytes() == b0
    _twice(cycle)


def test_line_handle(frames):
    import torch

    def cycle():
        b0 = _bytes()
        ln = pl.LINEextractor(width=W, height=H, max_batch=B)
        b1 = _bytes()
        assert b1 > b0
        cap = ln.capacity
        img = torch.from_numpy(frames).cuda()
        kl, desc, lf, n = _dev(((B * cap * 68,), torch.uint8), ((B * cap * 32,), torch.uint8), ((B * cap * 3,), torch.float64),
                               ((B,), torch.int32))

        def run():
            ln.extract_batch_dev(img.data_ptr(), W, W * H, B, None, kl.data_ptr(), desc.data_ptr(), lf.data_ptr(), n.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream)
        run()
        assert _bytes() == b1
        ln.set_undistort(pl.Undistorter(synth.TUM1_K, synth.TUM1_DIST, W, H))
        b2 = _bytes()
        run()                                           # below 32 frames per SM: the undistorted frames, made on first use
        b3 = _bytes()
        assert b3 > b2
        run()
        assert _bytes() == b3
        ln.extract_batch(frames)                        # host-pointer staging
        b4 = _bytes()
        assert b4 > b3
        ln.extract_batch(frames)
        assert _bytes() == b4
        del ln                                          # and the undistorter it held
        assert _bytes() == b0
    _twice(cycle)


def test_frontend_handle(frames):
    import torch
    problems = [synth.synth_pose_problem(60 + k) for k in range(B)]
    pinned = torch.empty(frames.shape, dtype=torch.uint8, pin_memory=True)
    pinned.numpy()[:] = frames

    def cycle():
        b0 = _bytes()
        fe = pl.Frontend(W, H, max_batch=B, lm_caps=(320, 88))
        b1 = _bytes()
        assert b1 > b0
        fe.set_pose_problems(problems)
        img = torch.from_numpy(frames).cuda()
        stream = torch.cuda.current_stream().cuda_stream
        fe.run_dev(img.data_ptr(), W, W * H, B, stream)
        assert _bytes() == b1
        fe.set_tracking(True)                           # the tracking stage's buffers
        b2 = _bytes()
        assert b2 > b1
        fe.set_tracking(False)
        fe.set_tracking(True)
        fe.run_dev(img.data_ptr(), W, W * H, B, stream)
        assert _bytes() == b2
        fe.set_camera(synth.TUM1_K, synth.TUM1_DIST)    # the undistortion map and the undistorted keypoints
        b3 = _bytes()
        assert b3 > b2
        fe.set_camera(synth.TUM1_K, synth.TUM1_DIST)
        assert _bytes() == b3
        fe.set_timing(True)
        outs = [fe.alloc_outputs(B, pinned=True) for _ in range(2)]
        fe.submit(pinned.numpy(), outs[0])              # the streaming state (and the line handle's undistorted frames)
        fe.wait(0)
        b4 = _bytes()
        assert b4 > b3
        fe.submit(pinned.numpy(), outs[1])
        fe.wait(0)
        assert _bytes() == b4 and fe.grow_ms() > 0
        del fe
        assert _bytes() == b0
    _twice(cycle)


def test_undistorter_handle(frames):
    def cycle():
        b0 = _bytes()
        u = pl.Undistorter(synth.TUM1_K, synth.TUM1_DIST, W, H)
        b1 = _bytes()
        assert b1 > b0
        u.remap(frames[0])                              # host-pointer staging
        b2 = _bytes()
        assert b2 > b1
        u.remap(frames[0])
        assert _bytes() == b2
        del u
        assert _bytes() == b0
    _twice(cycle)


def test_map_handle():
    g, _ = ls.quirk_cases()
    graph = ls.to_desc(g)

    def cycle():
        b0 = _bytes()
        M = pl.Map(**ls.quirk_map(g))
        b1 = _bytes()
        assert b1 > b0
        M.set_keyframes(graph)
        b2 = _bytes()
        assert b2 > b1
        M.set_keyframes(graph)                          # the new graph replaces the old one
        assert _bytes() == b2
        del M
        assert _bytes() == b0
    _twice(cycle)
