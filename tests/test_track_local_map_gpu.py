"""pl_track_local_map_dev (Tracking::TrackLocalMapWithLines on a batch) against the CPU composite of tests/track_scene.py.

One batch holds two cameras, th = 1 and th = 5 frames, pre-assigned matches, shared and overlapping local lists, an empty local
map and a featureless frame.  In-view flags, projections, levels, view cosines, both match arrays and the pose problem are
bit-exact with the oracle; pose and masks are bit-identical to pl_pose_optimization on the fetched problem and within 1e-4 of the
oracle; masks are compared with the oracle on frames whose outcome is the same under the oracle's rounding variants."""
import numpy as np
import pytest

import oracle
import plslam_b200 as pl
import track_scene as ts
from plslam_b200 import synth
from test_track_local_map import PX_BOUND, T_BOUND

pytestmark = pytest.mark.gpu
MAX_FRAMES = 30


def _close(T, To, tol=1e-4):
    assert np.linalg.norm(T[:3, 3] - To[:3, 3]) <= tol * max(np.linalg.norm(To[:3, 3]), 1e-3), (T, To)
    assert np.abs(T[:3, :3] - To[:3, :3]).max() <= 1e-4


def _scene_batch():
    m = ts.scene_map()
    Np, Nl = len(m["pt_pos"]), len(m["ln_pos"])
    T2, K2 = ts.TRUE[2]
    k2 = ts.features(T2, K2)
    # pre-assigned matches for frame 2: every third match of a search without them
    r = ts.track_local_map_oracle(m, *k2, ts.perturb(T2, 0.006, 2), K2, np.arange(Np), np.arange(Nl), 5, MAX_FRAMES)
    pm = np.where(np.arange(len(r["point_map"])) % 3 == 0, r["point_map"], -1).astype(np.int32)
    lm = np.where(np.arange(len(r["line_map"])) % 4 == 0, r["line_map"], -1).astype(np.int32)
    items = [(*ts.TRUE[0], ts.perturb(ts.TRUE[0][0], 0.006, 0), None, None),
             (*ts.TRUE[1], ts.perturb(ts.TRUE[1][0], 0.035, 1), None, None),
             (T2, K2, ts.perturb(T2, 0.006, 2), pm, lm),
             (*ts.TRUE[3], ts.perturb(ts.TRUE[3][0], 0.006, 3), None, None),
             (*ts.TRUE[0], ts.perturb(ts.TRUE[0][0], 0.006, 4), None, None),     # empty local map
             (*ts.TRUE[1], ts.perturb(ts.TRUE[1][0], 0.006, 5), None, None)]     # featureless
    fr, feats = ts.batch_frames(items)
    fr["n"][5] = 0; fr["nl"][5] = 0
    B = len(items)
    local = dict(pt_index=np.arange(Np, dtype=np.int32), ln_index=np.arange(Nl, dtype=np.int32),
                 pt_offset=np.array([0, 0, 200, 0, 0, 0], np.int32), pt_count=np.array([Np, Np, Np - 300, Np, 0, Np], np.int32),
                 ln_offset=np.array([0, 0, 20, 0, 0, 0], np.int32), ln_count=np.array([Nl, Nl, Nl - 40, Nl, 0, Nl], np.int32),
                 frames_since_reloc=np.array([5, 0, 40, 1, 7, 9], np.int32), max_frames=MAX_FRAMES)
    assert B == len(local["pt_offset"])
    return m, fr, feats, local


@pytest.fixture(scope="module")
def batch():
    m, fr, feats, local = _scene_batch()
    M = pl.Map(**m)
    out = pl.track_local_map(M, fr, local, taps=True)
    return m, M, fr, feats, local, out


def test_batch_matches_the_oracle_composite(batch):
    m, M, fr, feats, local, out = batch
    stable = 0
    for b in range(len(fr["n"])):
        n, nl = int(fr["n"][b]), int(fr["nl"][b])
        kps, desc, kl, ldesc, lf = feats[b]
        kps, desc, kl, ldesc, lf = kps[:n], desc[:n], kl[:nl], ldesc[:nl], np.asarray(lf).reshape(-1, 3)[:nl]
        o0, c0 = local["pt_offset"][b], local["pt_count"][b]
        l0, lc = local["ln_offset"][b], local["ln_count"][b]
        lp, ll = local["pt_index"][o0:o0 + c0], local["ln_index"][l0:l0 + lc]
        T0, K = fr["Tcw0"][b], fr["K"][b]
        pm = fr["point_map_in"][b, :n] if n else None
        lm = fr["line_map_in"][b, :nl] if nl else None
        if n == 0:   # featureless: frustum outputs only; nothing matched, pose kept, not ok
            iv, pr, lv, vc = oracle.is_in_frustum_points(T0, ts.camera_center(T0), K, ts.BOUNDS, ts.LOG_SF, ts.NLEV, 0.5, m["pt_pos"][lp],
                                                         m["pt_normal"][lp], m["pt_min_dist"][lp], m["pt_max_dist"][lp])
            assert np.array_equal(out["pt_in_view"][b, :c0], iv) and np.array_equal(out["pt_proj"][b, :c0], pr)
            assert np.array_equal(out["Tcw"][b], T0) and out["ok"][b] == 0 and (out["inliers"][b] == 0).all()
            continue
        r = ts.track_local_map_oracle(m, kps, desc, kl, ldesc, lf, T0, K, lp, ll, local["frames_since_reloc"][b], MAX_FRAMES, pm, lm)
        for k in ("pt_in_view", "pt_proj", "pt_level", "pt_view_cos"):
            assert np.array_equal(out[k][b, :c0], r[k]), (b, k)
        for k in ("ln_in_view", "ln_proj", "ln_level", "ln_view_cos"):
            assert np.array_equal(out[k][b, :lc], r[k]), (b, k)
        assert np.array_equal(out["pt_match"][b, :n], r["pt_match"]), b
        assert np.array_equal(out["ln_match"][b, :nl], r["ln_match"]), b
        assert np.array_equal(out["point_map"][b, :n], r["point_map"]) and np.array_equal(out["line_map"][b, :nl], r["line_map"]), b
        P = r["problem"]; npp, nlp = out["prob_n_points"][b], out["prob_n_lines"][b]
        assert (npp, nlp) == (r["prob_n_points"], r["prob_n_lines"]), b
        assert np.array_equal(out["prob_pt_obs"][b, :npp], P["pt_obs"]) and np.array_equal(out["prob_pt_inv_sigma2"][b, :npp], P["pt_inv_sigma2"])
        assert np.array_equal(out["prob_pt_Xw"][b, :npp], P["pt_Xw"]), b
        assert np.array_equal(out["prob_line_func"][b, :nlp], P["line_func"]) and np.array_equal(out["prob_line_Xw"][b, :nlp], P["line_Xw"])
        # the device's own pose LM on the fetched problem: bit-identical pose and masks
        gn, gT, gpo, glo, _ = pl.Optimizer.PoseOptimization(T0, K, out["prob_pt_obs"][b, :npp], out["prob_pt_inv_sigma2"][b, :npp],
                                                            out["prob_pt_Xw"][b, :npp], out["prob_line_func"][b, :nlp], out["prob_line_Xw"][b, :nlp])
        assert np.array_equal(out["Tcw"][b], gT), b
        pi = np.nonzero(out["point_map"][b, :n] >= 0)[0]; li = np.nonzero(out["line_map"][b, :nl] >= 0)[0]
        assert np.array_equal(out["point_outlier"][b, pi].astype(bool), gpo) and np.array_equal(out["line_outlier"][b, li].astype(bool), glo)
        assert not out["point_outlier"][b, :n][out["point_map"][b, :n] < 0].any()
        _close(out["Tcw"][b], r["Tcw"])
        if ts.outcome_is_rounding_stable(P, T0, K):
            stable += 1
            assert np.array_equal(out["point_outlier"][b, :n], r["point_outlier"]) and np.array_equal(out["line_outlier"][b, :nl], r["line_outlier"])
            assert np.array_equal(out["inliers"][b], r["inliers"]) and out["ok"][b] == r["ok"], b
    assert stable >= 4
    # frame 1: th = 5 with a 6 px guess; frame 3: th = 5 and the 50-inlier rule; frame 4: empty local map
    assert out["ok"][1] == 1 and out["ok"][3] == (out["inliers"][3, 0] >= 50)
    assert out["prob_n_points"][4] == 0 and out["ok"][4] == 0 and np.array_equal(out["Tcw"][4], fr["Tcw0"][4])
    # frame 2's held matches are kept and never projected
    held = fr["point_map_in"][2][fr["point_map_in"][2] >= 0]
    lp2 = local["pt_index"][200:200 + local["pt_count"][2]]
    assert len(held) > 50 and not out["pt_in_view"][2, :len(lp2)][np.isin(lp2, held)].any()


def test_host_entry_equals_the_batched_entry(batch):
    m, M, fr, feats, local, out = batch
    b = 2
    one = {k: (v[b:b + 1] if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == len(fr["n"]) else v) for k, v in fr.items()}
    loc = dict(local, pt_offset=local["pt_offset"][b:b + 1], pt_count=local["pt_count"][b:b + 1], ln_offset=local["ln_offset"][b:b + 1],
               ln_count=local["ln_count"][b:b + 1], frames_since_reloc=local["frames_since_reloc"][b:b + 1])
    h = pl.track_local_map(M, one, loc, taps=True, host=True)
    n, nl = int(fr["n"][b]), int(fr["nl"][b]); c0, lc = local["pt_count"][b], local["ln_count"][b]
    assert np.array_equal(h["Tcw"][0], out["Tcw"][b]) and np.array_equal(h["inliers"][0], out["inliers"][b]) and h["ok"][0] == out["ok"][b]
    for k in ("point_map", "point_outlier", "pt_match"):
        assert np.array_equal(h[k][0, :n], out[k][b, :n]), k
    for k in ("line_map", "line_outlier", "ln_match"):
        assert np.array_equal(h[k][0, :nl], out[k][b, :nl]), k
    assert np.array_equal(h["pt_proj"][0, :c0], out["pt_proj"][b, :c0]) and np.array_equal(h["ln_proj"][0, :lc], out["ln_proj"][b, :lc])


def test_capacity_refusal_and_out_of_range_index(batch):
    m, M, fr, feats, local, out = batch
    with pytest.raises(pl.PLError):
        pl.track_local_map(M, fr, dict(local, cap_local_points=100))
    with pytest.raises(pl.PLError):
        pl.track_local_map(M, fr, dict(local, ln_count=np.where(np.arange(len(fr["n"])) == 1, -1, local["ln_count"]).astype(np.int32)))
    B = len(fr["n"])
    # a list range past the end of its index array, or a negative offset: refused before anything runs
    with pytest.raises(pl.PLError):
        pl.track_local_map(M, fr, dict(local, pt_offset=np.where(np.arange(B) == 2, 400, local["pt_offset"]).astype(np.int32)))
    with pytest.raises(pl.PLError):
        pl.track_local_map(M, fr, dict(local, ln_offset=np.where(np.arange(B) == 3, -1, local["ln_offset"]).astype(np.int32)))
    with pytest.raises(pl.PLError):
        pl.track_local_map(M, fr, dict(local, pt_index=local["pt_index"][:-1]))
    bad = dict(local, pt_index=local["pt_index"].copy())
    bad["pt_index"][7] = len(m["pt_pos"]) + 5
    with pytest.raises(pl.PLError):
        pl.track_local_map(M, fr, bad)
    M.check_indices()                                   # the flag was reported and cleared
    good = pl.track_local_map(M, fr, local)             # and the map still works
    assert np.array_equal(good["Tcw"], out["Tcw"])


def test_4224_copies_are_bit_identical(batch):
    m, M, fr, feats, local, out = batch
    B0 = len(fr["n"]); reps = 4224 // B0
    big = {k: (np.concatenate([v] * reps) if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == B0 else v) for k, v in fr.items()}
    loc = dict(local, **{k: np.tile(local[k], reps) for k in ("pt_offset", "pt_count", "ln_offset", "ln_count", "frames_since_reloc")})
    got = pl.track_local_map(M, big, loc)
    for k, v in got.items():
        assert np.array_equal(v, np.concatenate([out[k]] * reps)), k


def test_frontend_track_local_map_equals_the_standalone_call():
    """Frames rendered on the plane, run through the front end, then tracked on the step's own features."""
    import ctypes
    libm = ctypes.CDLL("libm.so.6"); libm.logf.restype = ctypes.c_float; libm.logf.argtypes = [ctypes.c_float]
    m = ts.scene_map()
    M = pl.Map(**m)
    items = [ts.TRUE[0], ts.TRUE[1], ts.TRUE[2]]
    imgs = np.stack([ts.render(T, K) for T, K in items])
    B = len(items)
    fe = pl.Frontend(ts.W, ts.H, max_batch=B, lm_caps=(320, 88))
    fe.set_pose_problems([synth.synth_pose_problem(60 + k) for k in range(B)])
    Tcw0 = np.stack([ts.perturb(T, 0.006, 10 + b) for b, (T, _) in enumerate(items)])
    K = np.stack([Kb for _, Kb in items])
    Np, Nl = len(m["pt_pos"]), len(m["ln_pos"])
    local = dict(pt_index=np.arange(Np, dtype=np.int32), ln_index=np.arange(Nl, dtype=np.int32), pt_offset=np.zeros(B, np.int32),
                 pt_count=np.full(B, Np, np.int32), ln_offset=np.zeros(B, np.int32), ln_count=np.full(B, Nl, np.int32),
                 frames_since_reloc=np.array([3, 0, 50], np.int32), max_frames=MAX_FRAMES)
    pm = np.full((B, fe.capK), -1, np.int32); pm[0, :40] = np.arange(40)
    with pytest.raises(pl.PLError):      # no step has run yet: there are no features to track
        fe.track_local_map(M, Tcw0, K, local)
    fe.run(imgs[:2])
    with pytest.raises(pl.PLError):      # more frames than the last step produced
        fe.track_local_map(M, Tcw0, K, local)
    res = fe.run(imgs)
    got = fe.track_local_map(M, Tcw0, K, local, point_map_in=pm, taps=True)
    fr = dict(keys_un=fe.fetch_keys_un(B), desc=res["desc"], n=res["n"], keylines=res["keylines"], line_func=res["linefunc"],
              line_desc=res["ldesc"], nl=res["nl"], bounds=ts.BOUNDS, scale_factors=ts.SF, inv_level_sigma2=ts.INV_SIGMA2,
              log_scale_factor=float(libm.logf(np.float32(ts.SCALE))), Tcw0=Tcw0, K=K, point_map_in=pm)
    ref = pl.track_local_map(M, fr, local, taps=True)
    for k, v in ref.items():
        assert np.array_equal(got[k], v), k
    assert got["ok"].all() and got["inliers"][:, 0].min() > 100
    for b, (T, Kb) in enumerate(items):
        assert np.linalg.norm(got["Tcw"][b][:3, 3] - T[:3, 3]) < T_BOUND, b
        assert ts.plane_reprojection_gap(got["Tcw"][b], T, Kb) < PX_BOUND, b
