"""PredictScale arguments on and beside the level boundaries, shared by the check against the reference's own MapPoint.cc
(tests/test_oracle_match_ref.py) and the device check of isInFrustum for map lines (tests/test_frame_gpu.py)."""
import numpy as np


def boundary_set():
    """(dist, max_dist, log_scale_factor) of 200000 PredictScale calls for 8 levels of scale factor 1.2: the second half draws the
    ratio max_dist / dist from 0.5 .. 6; the first half puts dist exactly on max_dist / 1.2^k (k = 0 .. 8) or one fp32 step
    below or above it, where logf and the fp32 quotient decide the level"""
    rng = np.random.default_rng(1)
    n = 200000
    max_dist = rng.uniform(2.0, 12.0, n).astype(np.float32)
    dist = (max_dist / rng.uniform(0.5, 6.0, n)).astype(np.float32)
    k = np.arange(n // 2) % 9
    edge = (max_dist[:n // 2] / (np.float32(1.2) ** k.astype(np.float32))).astype(np.float32)
    dist[:n // 2] = np.nextafter(edge, np.where(np.arange(n // 2) % 3 == 0, np.float32(0), np.where(np.arange(n // 2) % 3 == 1, np.float32(1e9), edge)).astype(np.float32))
    return dist, max_dist, np.float32(np.log(np.float32(1.2)))
