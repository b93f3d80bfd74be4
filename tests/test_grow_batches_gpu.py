"""GPU test of the front-end at the batch sizes the benchmark runs: above 256 frames the region growing takes the full-GPU
form of k_lsd_grow_ordered (no up-front examination of each batch of seeds), and from 32 frames per SM on the three chains
of a step run on one stream.  Copies of a 3-frame cycle must reproduce the 3-frame run bit for bit."""
import numpy as np
import pytest
import torch
import plslam_b200 as pl
from plslam_b200 import synth

pytestmark = pytest.mark.gpu


def _copies_at_32_frames_per_sm():
    return -(-32 * torch.cuda.get_device_properties(0).multi_processor_count // 3)


# 87 copies = 261 frames: three streams.  32 frames per SM (1408 copies on a 132-SM H100): one stream.
@pytest.mark.parametrize("copies", ["261_frames", "32_per_sm"])
def test_frontend_cycle_copies_match_3_frame_run(copies):
    B0, R = 3, (87 if copies == "261_frames" else _copies_at_32_frames_per_sm())
    base = synth.synth_sequence(B0, 640, 480, seed=8)
    problems = [synth.synth_pose_problem(80 + k) for k in range(B0)]
    small = pl.Frontend(640, 480, max_batch=B0, lm_caps=(320, 88)); small.set_wrap(True); small.set_pose_problems(problems)
    small.set_camera(synth.TUM1_K, synth.TUM1_DIST)
    ref = small.run(base)
    del small
    big = pl.Frontend(640, 480, max_batch=B0 * R, lm_caps=(320, 88)); big.set_wrap(True); big.set_pose_problems(problems * R)
    big.set_camera(synth.TUM1_K, synth.TUM1_DIST)
    out = big.run(np.tile(base, (R, 1, 1)))
    for r in range(R):
        for b in range(B0):
            i = r * B0 + b
            n, nl = ref["n"][b], ref["nl"][b]
            assert out["n"][i] == n and out["nl"][i] == nl, i
            assert out["kps"][i, :n].tobytes() == ref["kps"][b, :n].tobytes() and np.array_equal(out["desc"][i, :n], ref["desc"][b, :n])
            assert out["keylines"][i, :nl].tobytes() == ref["keylines"][b, :nl].tobytes(), i
            assert np.array_equal(out["ldesc"][i, :nl], ref["ldesc"][b, :nl]), i
            npv, nlp = ref["n"][(b - 1) % B0], ref["nl"][(b - 1) % B0]
            assert out["n_pt_matches"][i] == ref["n_pt_matches"][b] and np.array_equal(out["pt_matches"][i, :npv], ref["pt_matches"][b, :npv])
            assert out["n_line_matches"][i] == ref["n_line_matches"][b]
            assert np.array_equal(out["line_matches"][i, :nlp], ref["line_matches"][b, :nlp])
            assert np.array_equal(out["poses"][:, i], ref["poses"][:, b]) and np.array_equal(out["inliers"][:, i], ref["inliers"][:, b])
