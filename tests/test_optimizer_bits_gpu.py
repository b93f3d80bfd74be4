"""The pose-only LM and the global BA, byte for byte against tests/golden/optimizer_bits.npz.

Both are deterministic by construction: k_pose_opt has no atomics (a problem's arithmetic does not depend on the batch around
it), and the global BA sums every reduction in a fixed order.  So any change to the order or rounding of one of the g2o formulas
they evaluate (edge errors, Jacobians, Huber weights, the normal-equation blocks, the LM step control) shows up here as a
changed bit, even where the result would still pass the oracle comparisons' tolerances.  The file was recorded with
tools/gen_optimizer_bits.py from the library as built at commit e56e88f, before the optimisers' formulas moved to g2o.cuh.

Local BA windows with free keyframes sum the reduced system with fp64 atomics and vary in the last bits from run to run;
test_local_ba_batch_gpu.py pins the all-fixed window (no atomics) bit for bit instead."""
import os
import numpy as np
import pytest
import plslam_b200 as pl
from test_optimizer_edges_gpu import pose_batch, _pose_dev, gba_camera_map

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "optimizer_bits.npz")
GBA_ITERATIONS = 6


def optimizer_outputs():
    """Every array the file pins, by name: pl_pose_optimization_dev in modes 0, 1, 2 on the 24-problem batch with a camera per
    problem (test_optimizer_edges_gpu.pose_batch), and pl_global_ba with and without Huber kernels on a map with lines and a camera
    per keyframe (gba_camera_map)."""
    out = {}
    probs = pose_batch()
    for mode in (0, 1, 2):
        for k, v in zip(("Tcw", "pt_outlier", "line_outlier", "inliers", "iterations"), _pose_dev(mode, probs)):
            out[f"pose{mode}_{k}"] = v
    p = gba_camera_map()
    for robust in (True, False):
        g = pl.GlobalBundleAdjustemnt(p, GBA_ITERATIONS, robust)
        for k in ("kf_Tcw", "pt_Xw", "ln_Xw"):
            out[f"gba{int(robust)}_{k}"] = g[k]
        out[f"gba{int(robust)}_its"] = np.int32(g["its"])
    return out


def test_optimizers_reproduce_the_recorded_bits():
    want = np.load(GOLDEN)
    got = optimizer_outputs()
    assert sorted(got) == sorted(want.files)
    for k in sorted(got):
        a, b = np.asarray(got[k]), want[k]
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), k
    assert (got["pose0_iterations"] > 0).sum() >= 18 and got["gba1_its"] >= 2 and got["gba0_its"] >= 2
