"""pl_track_motion_model_dev (Tracking::TrackWithMotionModel on a batch), pl_track_local_map_seen_dev and pl_track_velocity_dev
against the CPU composites of tests/motion_scene.py.

One batch holds the named cases of motion_scene.motion_cases() (a plain frame with last-frame outliers and discards, a retry frame,
a frame under 10 map matches, an early-return frame), a frame of a third stream, a featureless frame and an empty last frame, with
two cameras.  The guess, the line candidates, both raw point searches, the line search, the retried flags, the pose problem, the
matches before the discard and nmatches are bit-exact with the composite; the pose and the discard are bit-identical to
pl_pose_optimization on the fetched problem and within 1e-4 of the composite, whose masks are compared on rounding-stable frames."""
import numpy as np
import pytest

import plslam_b200 as pl
import motion_scene as ms
import track_scene as ts

pytestmark = pytest.mark.gpu
NAMES = ["plain", "retry", "few", "early", "stream2", "featureless", "empty_last"]


def _close(T, To, tol=1e-4):
    assert np.linalg.norm(T[:3, 3] - To[:3, 3]) <= tol * max(np.linalg.norm(To[:3, 3]), 1e-3), (T, To)
    assert np.abs(T[:3, :3] - To[:3, :3]).max() <= 1e-4


def _batch(items):
    """items: list of (T_true, K, last) -> (frames, feats, last dict of the batch)."""
    feats = [ts.features(T, K) for T, K, _ in items]
    cap = max(max(len(f[0]) for f in feats), max(len(l["keys"]) for _, _, l in items), 1)
    capL = max(max(len(f[2]) for f in feats), max(len(l["kl"]) for _, _, l in items), 1)
    fr, _ = ts.batch_frames([(T, K, np.eye(4, dtype=np.float32), None, None) for T, K, _ in items], cap, capL)
    for k in ("Tcw0", "point_map_in", "line_map_in"):
        fr.pop(k)
    B = len(items)
    import oracle
    last = dict(keys_un=np.zeros((B, cap), oracle.KP_DTYPE), n=np.zeros(B, np.int32), keylines=np.zeros((B, capL), oracle.KEYLINE_DTYPE),
                nl=np.zeros(B, np.int32), point_map=np.full((B, cap), -1, np.int32), point_outlier=np.zeros((B, cap), np.uint8),
                line_map=np.full((B, capL), -1, np.int32), line_outlier=np.zeros((B, capL), np.uint8), Tcw=np.zeros((B, 4, 4), np.float32),
                velocity=np.zeros((B, 4, 4), np.float32), vo=np.full(B, 7, np.int32))
    for b, (_, _, l) in enumerate(items):
        n0, nl0 = len(l["keys"]), len(l["kl"])
        last["keys_un"][b, :n0] = l["keys"]; last["n"][b] = n0; last["keylines"][b, :nl0] = l["kl"]; last["nl"][b] = nl0
        last["point_map"][b, :n0] = l["point_map"]; last["point_outlier"][b, :n0] = l["point_outlier"]
        last["line_map"][b, :nl0] = l["line_map"]; last["line_outlier"][b, :nl0] = l["line_outlier"]
        last["Tcw"][b] = l["Tcw"]; last["velocity"][b] = l["velocity"]
    return fr, feats, last


def _items():
    m, c = ms.motion_cases()
    items = [c["plain"], c["retry"], c["few"], c["early"]]
    T1, K2 = ms.stream_pose(2, 1), ms.STREAMS[2][2]
    items.append((ms.stream_pose(2, 2), K2, dict(ms.last_frame(m, T1, K2, seed=2), velocity=ms.STREAMS[2][1])))
    items.append((c["plain"][0], c["plain"][1], c["plain"][2]))                     # featureless: counts set to 0 below
    empty = dict(keys=c["few"][2]["keys"][:0], kl=c["few"][2]["kl"][:0], point_map=np.zeros(0, np.int32), point_outlier=np.zeros(0, np.uint8),
                 line_map=np.zeros(0, np.int32), line_outlier=np.zeros(0, np.uint8), Tcw=c["few"][2]["Tcw"], velocity=c["few"][2]["velocity"])
    items.append((c["few"][0], c["few"][1], empty))
    return m, items


@pytest.fixture(scope="module")
def batch():
    m, items = _items()
    fr, feats, last = _batch(items)
    fr["n"][5] = 0; fr["nl"][5] = 0
    M = pl.Map(**m)
    out = pl.track_motion_model(M, fr, last, taps=True)
    return m, M, items, fr, feats, last, out


def _oracle(m, items, feats, fr, b):
    n, nl = int(fr["n"][b]), int(fr["nl"][b])
    kps, desc, kl, ldesc, lf = feats[b]
    T, K, l = items[b]
    return ms.track_motion_model_oracle(m, kps[:n], desc[:n], kl[:nl], ldesc[:nl], np.asarray(lf).reshape(-1, 3)[:nl], K, l)


def test_batch_matches_the_oracle_composite(batch):
    m, M, items, fr, feats, last, out = batch
    stable = 0
    for b in range(len(items)):
        n, nl, nl0 = int(fr["n"][b]), int(fr["nl"][b]), int(last["nl"][b])
        r = _oracle(m, items, feats, fr, b)
        assert np.array_equal(out["guess"][b], r["guess"]), b
        for k in ("ln_in_view", "ln_proj", "ln_level", "ln_view_cos"):
            assert np.array_equal(out[k][b, :nl0], r[k]), (b, k)
        assert np.array_equal(out["pt_match"][b, :n], r["pt_match"]) and out["retried"][b] == r["retried"], b
        if r["retried"]:
            assert np.array_equal(out["pt_match_retry"][b, :n], r["pt_match_retry"]), b
        assert np.array_equal(out["ln_match"][b, :nl], r["ln_match"]), b
        P = r["problem"]; npp, nlp = out["prob_n_points"][b], out["prob_n_lines"][b]
        assert (npp, nlp) == (r["prob_n_points"], r["prob_n_lines"]), b
        assert np.array_equal(out["prob_pt_obs"][b, :npp], P["pt_obs"]) and np.array_equal(out["prob_pt_Xw"][b, :npp], P["pt_Xw"]), b
        assert np.array_equal(out["prob_pt_inv_sigma2"][b, :npp], P["pt_inv_sigma2"]), b
        assert np.array_equal(out["prob_line_func"][b, :nlp], P["line_func"]) and np.array_equal(out["prob_line_Xw"][b, :nlp], P["line_Xw"])
        # the matches before the discard are bit-exact
        pre = np.where(out["point_seen"][b, :n] >= 0, out["point_seen"][b, :n], out["point_map"][b, :n])
        rpre = np.where(r["point_seen"] >= 0, r["point_seen"], r["point_map"])
        lpre = np.where(out["line_seen"][b, :nl] >= 0, out["line_seen"][b, :nl], out["line_map"][b, :nl])
        rlpre = np.where(r["line_seen"] >= 0, r["line_seen"], r["line_map"])
        assert np.array_equal(pre, rpre) and np.array_equal(lpre, rlpre), b
        if not r["solved"]:
            assert np.array_equal(out["Tcw"][b], r["guess"]) and out["ok"][b] == 0 and out["vo"][b] == 7, b
            assert np.array_equal(out["nmatches"][b], r["nmatches"]) and (out["point_seen"][b] == -1).all(), b
            continue
        # the device's own pose LM on the fetched problem decides the discard bit for bit
        _, gT, gpo, glo, _ = pl.Optimizer.PoseOptimization(r["guess"], items[b][1], out["prob_pt_obs"][b, :npp],
                                                           out["prob_pt_inv_sigma2"][b, :npp], out["prob_pt_Xw"][b, :npp],
                                                           out["prob_line_func"][b, :nlp], out["prob_line_Xw"][b, :nlp])
        assert np.array_equal(out["Tcw"][b], gT), b
        pi = np.nonzero(pre >= 0)[0]; li = np.nonzero(lpre >= 0)[0]
        assert np.array_equal(out["point_seen"][b, pi] >= 0, gpo) and np.array_equal(out["line_seen"][b, li] >= 0, glo), b
        nm = int((pre >= 0).sum()) - int(gpo.sum())
        assert out["nmatches"][b, 0] == (r["nmatches"][0] + int((r["point_seen"] >= 0).sum()) - int(gpo.sum())), b
        assert out["ok"][b] == int(nm > 20) and out["vo"][b] == int(nm < 10), b
        _close(out["Tcw"][b], r["Tcw"])
        if ts.outcome_is_rounding_stable(P, r["guess"], items[b][1]):
            stable += 1
            for k in ("point_map", "line_map", "point_seen", "line_seen"):
                assert np.array_equal(out[k][b, :(n if k.startswith("point") else nl)], r[k]), (b, k)
            assert np.array_equal(out["nmatches"][b], r["nmatches"]) and out["ok"][b] == r["ok"] and out["vo"][b] == r["vo"], b
    assert stable >= 3
    # the named branches are reached on the device
    assert out["retried"][1] == 1 and out["ok"][1] == 1
    assert out["vo"][2] == 1 and out["ok"][2] == 0
    assert out["vo"][3] == 7 and np.array_equal(out["Tcw"][3], out["guess"][3]) and (out["point_map"][3] >= 0).sum() > 0
    assert (out["point_seen"][0] >= 0).any() and out["ok"][0] == 1 and out["ok"][4] == 1
    assert out["ok"][5] == 0 and (out["point_map"][5] == -1).all() and out["ok"][6] == 0 and out["nmatches"][6].sum() == 0


def test_local_map_with_seen(batch):
    m, M, items, fr, feats, last, out = batch
    b = 0
    T, K, _ = items[b]
    n, nl = int(fr["n"][b]), int(fr["nl"][b])
    Np, Nl = len(m["pt_pos"]), len(m["ln_pos"])
    one = {k: (v[b:b + 1] if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == len(items) else v) for k, v in fr.items()}
    one = dict(one, Tcw0=out["Tcw"][b:b + 1], point_map_in=out["point_map"][b:b + 1], line_map_in=out["line_map"][b:b + 1])
    local = dict(pt_index=np.arange(Np, dtype=np.int32), ln_index=np.arange(Nl, dtype=np.int32), pt_offset=np.zeros(1, np.int32),
                 pt_count=np.full(1, Np, np.int32), ln_offset=np.zeros(1, np.int32), ln_count=np.full(1, Nl, np.int32),
                 frames_since_reloc=np.full(1, 40, np.int32), max_frames=30)
    plain = pl.track_local_map(M, one, local, taps=True)
    none = pl.track_local_map(M, one, local, taps=True, seen=dict(point_seen=np.full_like(out["point_seen"][b:b + 1], -1),
                                                                  line_seen=np.full_like(out["line_seen"][b:b + 1], -1)))
    for k, v in plain.items():
        assert np.array_equal(none[k], v), k
    got = pl.track_local_map(M, one, local, taps=True, seen=dict(point_seen=out["point_seen"][b:b + 1], line_seen=out["line_seen"][b:b + 1]))
    kps, desc, kl, ldesc, lf = feats[b]
    r = ms.track_local_map_seen_oracle(m, kps[:n], desc[:n], kl[:nl], ldesc[:nl], np.asarray(lf).reshape(-1, 3)[:nl], out["Tcw"][b], K,
                                       np.arange(Np), np.arange(Nl), 40, 30, out["point_map"][b, :n], out["line_map"][b, :nl],
                                       out["point_seen"][b, :n], out["line_seen"][b, :nl])
    for k in ("pt_in_view", "pt_proj", "ln_in_view", "ln_proj"):
        assert np.array_equal(got[k][0], r[k]), k
    assert np.array_equal(got["pt_match"][0, :n], r["pt_match"]) and np.array_equal(got["point_map"][0, :n], r["point_map"])
    seen = out["point_seen"][b][out["point_seen"][b] >= 0]
    assert len(seen) and plain["pt_in_view"][0, seen].any() and not got["pt_in_view"][0, seen].any()
    _close(got["Tcw"][0], r["Tcw"])


def test_chain_of_three_streams(batch):
    """motion model -> local map with seen -> velocity, 3 streams x 5 steps; the composite starts each step from the GPU's pose
    and velocity."""
    m, M = batch[0], batch[1]
    S, steps = len(ms.STREAMS), 5
    Ks = [ms.STREAMS[s][2] for s in range(S)]
    lasts = [dict(ms.last_frame(m, ms.stream_pose(s, 0), Ks[s], seed=s), velocity=np.asarray(ms.STREAMS[s][1], np.float32)) for s in range(S)]
    Np, Nl = len(m["pt_pos"]), len(m["ln_pos"])
    for k in range(1, steps + 1):
        items = [(ms.stream_pose(s, k), Ks[s], lasts[s]) for s in range(S)]
        fr, feats, last = _batch(items)
        mm = pl.track_motion_model(M, fr, last, taps=True)
        cap, capL = fr["keys_un"].shape[1], fr["keylines"].shape[1]
        fl = dict(fr, Tcw0=mm["Tcw"], point_map_in=mm["point_map"], line_map_in=mm["line_map"])
        local = dict(pt_index=np.arange(Np, dtype=np.int32), ln_index=np.arange(Nl, dtype=np.int32), pt_offset=np.zeros(S, np.int32),
                     pt_count=np.full(S, Np, np.int32), ln_offset=np.zeros(S, np.int32), ln_count=np.full(S, Nl, np.int32),
                     frames_since_reloc=np.full(S, 40, np.int32), max_frames=30)
        lo = pl.track_local_map(M, fl, local, taps=True, seen=mm)
        V = pl.track_velocity(lo["Tcw"], last["Tcw"], lo["ok"], last["velocity"])
        for s in range(S):
            n, nl = int(fr["n"][s]), int(fr["nl"][s])
            kps, desc, kl, ldesc, lf = feats[s]
            r = ms.track_motion_model_oracle(m, kps, desc, kl, ldesc, lf, Ks[s], lasts[s])
            assert np.array_equal(mm["guess"][s], r["guess"]) and np.array_equal(mm["pt_match"][s, :n], r["pt_match"]), (k, s)
            _close(mm["Tcw"][s], r["Tcw"])
            rl = ms.track_local_map_seen_oracle(m, kps, desc, kl, ldesc, lf, mm["Tcw"][s], Ks[s], np.arange(Np), np.arange(Nl), 40, 30,
                                                mm["point_map"][s, :n], mm["line_map"][s, :nl], mm["point_seen"][s, :n], mm["line_seen"][s, :nl])
            assert np.array_equal(lo["pt_in_view"][s], rl["pt_in_view"]) and np.array_equal(lo["pt_match"][s, :n], rl["pt_match"]), (k, s)
            _close(lo["Tcw"][s], rl["Tcw"])
            assert lo["ok"][s] == 1 and mm["ok"][s] == 1, (k, s)
            assert np.array_equal(V[s], ms.velocity_oracle(lo["Tcw"][s], last["Tcw"][s])), (k, s)
            lasts[s] = dict(keys=kps, kl=kl, point_map=lo["point_map"][s, :n], point_outlier=lo["point_outlier"][s, :n],
                            line_map=lo["line_map"][s, :nl], line_outlier=lo["line_outlier"][s, :nl], Tcw=lo["Tcw"][s], velocity=V[s])
    # velocity is written only where ok
    V0 = np.full((2, 4, 4), 3.0, np.float32)
    got = pl.track_velocity(np.stack([ms.stream_pose(0, 1)] * 2), np.stack([ms.stream_pose(0, 0)] * 2), np.array([0, 1]), V0)
    assert (got[0] == 3.0).all() and np.array_equal(got[1], ms.velocity_oracle(ms.stream_pose(0, 1), ms.stream_pose(0, 0)))


def test_host_entry_equals_the_batched_entry(batch):
    m, M, items, fr, feats, last, out = batch
    for b in (0, 3):
        one = {k: (v[b:b + 1] if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == len(items) else v) for k, v in fr.items()}
        l1 = {k: v[b:b + 1] for k, v in last.items()}
        h = pl.track_motion_model(M, one, l1, taps=True, host=True)
        n, nl = int(fr["n"][b]), int(fr["nl"][b])
        for k in ("Tcw", "nmatches", "ok", "vo", "guess", "retried"):
            assert np.array_equal(h[k][0], out[k][b]), (b, k)
        for k in ("point_map", "point_seen", "pt_match"):
            assert np.array_equal(h[k][0, :n], out[k][b, :n]), (b, k)
        for k in ("line_map", "line_seen", "ln_match"):
            assert np.array_equal(h[k][0, :nl], out[k][b, :nl]), (b, k)


def test_refusals_and_out_of_range_index(batch):
    m, M, items, fr, feats, last, out = batch
    L = pl.binding._track_lib()
    with pytest.raises(pl.PLError):      # Tcw0 must be NULL: the guess is computed
        F = pl.binding.PLTrackFrames(); F.B = 1; F.cap_points = 8; F.cap_lines = 8; F.nlevels = 8
        import ctypes as C
        F.Tcw0 = C.c_void_p(16)
        pl.binding.check(L.pl_track_motion_model_dev(M._h, C.byref(F), C.byref(pl.binding.PLTrackLast()),
                                                     C.byref(pl.binding.PLTrackMotionOut()), C.c_void_p(16), None))
    with pytest.raises(pl.PLError):      # cap_points over 6144
        big = dict(fr, keys_un=np.zeros((len(items), 6200), fr["keys_un"].dtype), desc=np.zeros((len(items), 6200, 32), np.uint8))
        pl.track_motion_model(M, big, dict(last, keys_un=np.zeros((len(items), 6200), fr["keys_un"].dtype),
                                           point_map=np.full((len(items), 6200), -1, np.int32), point_outlier=np.zeros((len(items), 6200), np.uint8)))
    bad = {k: v.copy() if isinstance(v, np.ndarray) else v for k, v in last.items()}
    i = int(np.nonzero((bad["point_map"][0] >= 0) & (bad["point_outlier"][0] == 0))[0][0])
    bad["point_map"][0, i] = len(m["pt_pos"]) + 3
    with pytest.raises(pl.PLError):
        pl.track_motion_model(M, fr, bad)
    M.check_indices()                                   # reported and cleared
    # an outlier entry outside the map is skipped without a look at the map
    bad["point_outlier"][0, i] = 1
    pl.track_motion_model(M, fr, bad)
    M.check_indices()
    good = pl.track_motion_model(M, fr, last)
    assert np.array_equal(good["Tcw"], out["Tcw"])


def test_4224_copies_are_bit_identical(batch):
    m, M, items, fr, feats, last, out = batch
    B0 = len(items); reps = 4224 // B0
    big = {k: (np.concatenate([v] * reps) if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == B0 else v) for k, v in fr.items()}
    bl = {k: np.concatenate([v] * reps) for k, v in last.items()}
    got = pl.track_motion_model(M, big, bl)
    for k, v in got.items():
        assert np.array_equal(v, np.concatenate([out[k]] * reps)), k
