"""GPU: pl_local_ba_dev, several local windows in one launch (one CTA per window), against the fp64 CPU oracle and against
pl_local_ba on each window, at test_ba_gpu._check's bar: 1e-4 relative on translations and points, 1e-3 on line end points,
identical erase masks and iteration counts.  The Schur sum uses fp64 atomics, so two runs of one window differ in the last
bits; every comparison between GPU runs is therefore made at the same bar, not bit for bit."""
import os
import numpy as np
import pytest
import torch
import oracle
import plslam_b200 as pl
from plslam_b200 import synth
from test_optimizer_edges_gpu import (K_END, keyframe_cameras, lba_camera_window, lba_32_free_window, lba_mirrored_point_window,
                                      lba_outlier_keyframe_window, without_points)

pytestmark = pytest.mark.gpu

KITTI_K = (718.856, 718.856, 607.1928, 185.2157)
SENTINEL = 0xA5


def meets_bar(g, o, what="", its=True):
    t, to = g["kf_Tcw"].reshape(-1, 4, 4)[:, :3, 3].astype(np.float64), o["kf_Tcw"].reshape(-1, 4, 4)[:, :3, 3].astype(np.float64)
    assert g["kf_Tcw"].shape == o["kf_Tcw"].shape, what
    assert np.linalg.norm(t - to, axis=1).max() <= 1e-4 * np.linalg.norm(to, axis=1).max(), what
    assert np.abs(g["kf_Tcw"] - o["kf_Tcw"]).max() < 1e-4, what
    assert g["pt_Xw"].shape == o["pt_Xw"].shape and g["ln_Xw"].shape == o["ln_Xw"].shape, what
    if len(o["pt_Xw"]):
        assert np.abs(g["pt_Xw"] - o["pt_Xw"]).max() <= 1e-4 * np.abs(o["pt_Xw"]).max(), what
    if len(o["ln_Xw"]):
        assert np.abs(g["ln_Xw"] - o["ln_Xw"]).max() <= 1e-3 * np.abs(o["ln_Xw"]).max(), what
    if its:
        assert g["its"] == o["its"], (what, g["its"], o["its"])
    assert np.array_equal(g["pe_erase"], o["pe_erase"]) and np.array_equal(g["le_erase"], o["le_erase"]), what
    assert np.array_equal(g["le_erase_kf"], o["le_erase_kf"]), what


def kitti_window():
    """The window bench.py's KITTI configuration runs beside the front end."""
    return synth.synth_ba_problem(seed=4, K=KITTI_K, w=1241, h=376)


def points_only_window():
    p = synth.synth_ba_problem(4, n_free=8, n_fixed=10, n_pt=600, n_ln=80, noise_px=0.0, outlier_frac=0.0)
    q = dict(p)
    q.update(le_kf=p["le_kf"][:0], le_ln=p["le_ln"][:0], le_func=p["le_func"][:0])
    return q


def lines_only_window():
    """Lines only, a camera per keyframe and its own K_end, like test_optimizer_edges_gpu.lba_lines_only_window, on seed 14.  The
    end points of that window's seed 6 slide along their lines far enough that the fp64-atomic summation order alone moves them
    past the 1e-3 bar in about one run in ten, with any build; on seed 14 the largest of 60 runs stayed at 0.06 of the bar."""
    return without_points(synth.synth_ba_problem(14, n_free=8, n_fixed=10, n_pt=50, n_ln=200, Ks=keyframe_cameras(18, 114),
                                                 K_end=K_END))


def all_fixed_window():
    p = synth.synth_ba_problem(35, n_free=6, n_fixed=4, n_pt=500, n_ln=60)
    p["kf_fixed"] = np.ones_like(p["kf_fixed"])
    return p


def no_edge_window():
    p = synth.synth_ba_problem(5, n_free=2, n_fixed=1, n_pt=30, n_ln=5)
    p.update({f: p[f][:0] for f in ("pe_kf", "pe_pt", "pe_obs", "pe_inv_sigma2", "le_kf", "le_ln", "le_func")})
    return p


def mixed_batch():
    return [("cameras", lba_camera_window()), ("lines only", lines_only_window()), ("32 free", lba_32_free_window()),
            ("depth-test point", lba_mirrored_point_window()[0]), ("outlier keyframe", lba_outlier_keyframe_window()[0]),
            ("ba 4", synth.synth_ba_problem(4, n_free=8, n_fixed=10, n_pt=600, n_ln=80)),
            ("ba 6", synth.synth_ba_problem(6, n_free=6, n_fixed=8, n_pt=400, n_ln=60)),
            ("ba 9", synth.synth_ba_problem(9, n_free=12, n_fixed=20, n_pt=1500, n_ln=200)),
            ("full size", synth.synth_ba_problem(11, n_free=20, n_fixed=40, n_pt=3000, n_ln=400)),
            ("points only", points_only_window()), ("every keyframe fixed", all_fixed_window()), ("no edges", no_edge_window())]


def test_mixed_batch_against_the_oracle_and_the_single_window_entry():
    named = mixed_batch()
    res = pl.LocalBundleAdjustmentWithLineBatch([p for _, p in named])
    for (name, p), g in zip(named, res):
        assert g["status"] == 0, name
        single = pl.LocalBundleAdjustmentWithLine(p)
        meets_bar(g, single, name)
        # the oracle counts an optimize() over an empty system as one iteration; the kernel (and pl_local_ba) report none
        meets_bar(g, oracle.local_ba(p), name, its=name != "no edges")
    assert res[-1]["its"] == 0 and res[-2]["its"] > 0 and res[-3]["its"] > 0


def test_one_window_agrees_with_pl_local_ba():
    p = kitti_window()
    g, = pl.LocalBundleAdjustmentWithLineBatch([p])
    assert g["status"] == 0
    meets_bar(g, pl.LocalBundleAdjustmentWithLine(p), "W = 1")


def _device_rows(b):
    return {k: v.cpu().numpy() for k, v in b.outputs.items()}


def test_sentinels_past_the_counts_and_device_side_validation():
    """Windows 1 (an edge naming a point past n_pt), 3 (n_pt over cap_pt) and 5 (a negative n_le) are refused on the device:
    nonzero status, iterations 0, every other output byte still the sentinel.  Windows 0, 2, 4 match a clean batch of the same
    windows, and nothing past their counts is written."""
    a, c, e = (synth.synth_ba_problem(4, n_free=8, n_fixed=10, n_pt=600, n_ln=80), lines_only_window(),
               synth.synth_ba_problem(6, n_free=6, n_fixed=8, n_pt=400, n_ln=60))
    bad_edge = synth.synth_ba_problem(9, n_free=5, n_fixed=3, n_pt=300, n_ln=40)
    bad_edge["pe_pt"] = bad_edge["pe_pt"].copy()
    bad_edge["pe_pt"][17] = len(bad_edge["pt_Xw"])
    bad_count = synth.synth_ba_problem(12, n_free=4, n_fixed=4, n_pt=200, n_ln=30)
    bad_sign = synth.synth_ba_problem(13, n_free=4, n_fixed=4, n_pt=200, n_ln=30)
    probs = [a, bad_edge, c, bad_count, e, bad_sign]
    b = pl.LocalBAWindows(probs, out_fill=SENTINEL)
    b.inputs["n_pt"][3] = b.caps["pt"] + 1
    b.inputs["n_le"][5] = -1
    torch.cuda.synchronize()
    b.run()
    res = b.results()
    raw = _device_rows(b)
    assert [r["status"] for r in res] == [0, 2, 0, 1, 0, 1]
    clean = pl.LocalBundleAdjustmentWithLineBatch([a, c, e])
    for w, ref in zip((0, 2, 4), clean):
        meets_bar(res[w], ref, f"neighbour {w}")
    for w in (1, 3, 5):
        assert res[w]["its"] == 0
        for f in ("kf_Tcw", "pt_Xw", "ln_Xw", "pe_erase", "le_erase", "le_erase_kf"):
            assert (raw[f][w].view(np.uint8) == SENTINEL).all(), (w, f)
    for w in (0, 2, 4):
        n = pl.ba_window_counts(probs[w])
        for f, (k, _, _) in pl.BA_OUTPUTS.items():
            assert (raw[f][w, n[k]:].view(np.uint8) == SENTINEL).all(), (w, f)
            assert n[k] == 0 or not (raw[f][w, :n[k]].view(np.uint8) == SENTINEL).all(), (w, f)


def test_stop_flag_set_before_the_call():
    probs = [synth.synth_ba_problem(4, n_free=8, n_fixed=10, n_pt=600, n_ln=80), lines_only_window(), points_only_window()]
    stop = torch.ones(1, dtype=torch.int32, device="cuda")
    res = pl.LocalBundleAdjustmentWithLineBatch(probs, stop_flag_dev=stop.data_ptr())
    for p, g in zip(probs, res):
        assert g["status"] == 0 and g["its"] == 0
        assert g["kf_Tcw"].tobytes() == p["kf_Tcw"].tobytes() and np.array_equal(g["pt_Xw"], p["pt_Xw"])
        assert not g["pe_erase"].any() and not g["le_erase"].any()
        assert np.array_equal(g["le_erase_kf"], p["le_kf"][np.arange(len(p["le_kf"])) // 2])
        assert np.array_equal(g["ln_Xw"], p["ln_Xw"].astype(np.float32).astype(np.float64))


def test_264_copies_of_the_kitti_window():
    """Two windows per SM: any scratch two windows shared would show as a copy that leaves the bar."""
    p = kitti_window()
    assert oracle.local_ba(p)["gate_gap"] > 1e-5
    single = pl.LocalBundleAdjustmentWithLine(p)
    res = pl.LocalBundleAdjustmentWithLineBatch([p] * 264)
    for w, g in enumerate(res):
        assert g["status"] == 0, w
        meets_bar(g, single, f"copy {w}")


def test_captured_call_replays():
    """pl_local_ba_dev captured on a side stream into a CUDA graph: a device-wide synchronisation or a copy on the legacy stream
    inside the call would invalidate the capture.  The replay, into outputs reset to zero, agrees with the eager run."""
    probs = [kitti_window(), lba_camera_window(), points_only_window()]
    b = pl.LocalBAWindows(probs)
    s = torch.cuda.Stream()
    b.run(s)
    eager = b.results()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        b.run(s)
    for t in b.outputs.values():
        t.zero_()
    torch.cuda.synchronize()
    g.replay()
    replay = b.results()
    for w, (r, e) in enumerate(zip(replay, eager)):
        assert r["status"] == 0 and r["its"] > 0, w
        meets_bar(r, e, f"replay {w}")


def test_repeated_calls_hold_no_device_memory():
    probs = [synth.synth_ba_problem(4, n_free=8, n_fixed=10, n_pt=600, n_ln=80), no_edge_window()]
    b = pl.LocalBAWindows(probs)
    s = torch.cuda.Stream()
    b.run(s)
    b.results()
    before = pl.device_bytes()
    for _ in range(5):
        b.run(s)
    b.results()
    assert pl.device_bytes() == before


def test_csr_lists_keep_insertion_order_bit_for_bit():
    """With every keyframe fixed the kernel runs no atomics: no pose is free, so the Schur sum and the pose blocks are skipped and
    each landmark's blocks are summed by one thread over its CSR list.  The result is then bit-reproducible and depends on the
    order inside each list.  tests/golden/lba_all_fixed_s35.npz holds this window's outputs from the earlier build whose host
    loop made the lists in insertion order; the device-built lists must give the same bits, alone and inside a batch."""
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "lba_all_fixed_s35.npz"))
    p = all_fixed_window()
    single = pl.LocalBundleAdjustmentWithLine(p)
    batch = pl.LocalBundleAdjustmentWithLineBatch([synth.synth_ba_problem(4, n_free=8, n_fixed=10, n_pt=600, n_ln=80), p,
                                                   lines_only_window()])[1]
    assert batch["status"] == 0
    for g in (single, batch):
        assert g["its"] == int(gold["its"]) > 0
        for k in ("kf_Tcw", "pt_Xw", "ln_Xw", "pe_erase", "le_erase", "le_erase_kf"):
            assert np.asarray(g[k]).tobytes() == gold[k].tobytes(), k
