"""pl_track_update_local_map_dev, pl_track_local_map_lists_dev and the reference-keyframe poses against the restatement of
tests/localmap_scene.py, and the whole localisation chain (LocalizationChain) against the separate calls, eagerly and replayed
from one CUDA graph."""
import gc

import numpy as np
import pytest

import oracle
import plslam_b200 as pl
import localmap_scene as ls
import motion_scene as ms
import track_scene as ts

pytestmark = pytest.mark.gpu
CAP, CAP_KF, CLP, CLL = 128, 96, 160, 64


def _quirk_batch(cases, names):
    B = len(names)
    pm = np.full((B, CAP), -1, np.int32); kf = np.full((B, CAP_KF), -1, np.int32)
    n_kf = np.zeros(B, np.int32); ref = np.zeros(B, np.int32)
    for b, nm in enumerate(names):
        c = cases[nm]
        pm[b, :len(c["point_map"])] = c["point_map"]; kf[b, :len(c["kf_prev"])] = c["kf_prev"]
        n_kf[b] = len(c["kf_prev"]); ref[b] = c["ref_prev"]
    return pm, kf, n_kf, ref


@pytest.fixture(scope="module")
def quirk():
    g, cases = ls.quirk_cases()
    M = pl.Map(**ls.quirk_map(g))
    M.set_keyframes(ls.to_desc(g))
    names = list(cases)
    pm, kf, n_kf, ref = _quirk_batch(cases, names)
    out = pl.update_local_map(M, pm, kf, n_kf, ref, CLP, CLL)
    M.check_capacity()
    return g, cases, names, M, (pm, kf, n_kf, ref), out


def _assert_frame(out, b, r):
    n = len(r["kf"])
    assert out["n_kf"][b] == n and out["kf"][b, :n].tolist() == r["kf"] and out["ref_kf"][b] == r["ref_kf"], b
    assert out["pt_count"][b] == len(r["points"]) and out["pt_index"][b, :len(r["points"])].tolist() == r["points"], b
    assert out["ln_count"][b] == len(r["lines"]) and out["ln_index"][b, :len(r["lines"])].tolist() == r["lines"], b


def test_every_named_case_is_bit_exact(quirk):
    g, cases, names, M, _, out = quirk
    for b, nm in enumerate(names):
        c = cases[nm]
        _assert_frame(out, b, ls.update_local_map_ref(g, c["point_map"], c["kf_prev"], c["ref_prev"]))
    # the cases reach their branches on the device
    k = cases["limit_80"]["kfs"]; b = names.index("limit_80")
    assert out["n_kf"][b] == 82 and out["kf"][b, 80:82].tolist() == [k["x0"], k["x1"]]
    b = names.index("stale")
    assert out["kf"][b, :3].tolist() == cases["stale"]["kf_prev"] and out["ref_kf"][b] == cases["stale"]["ref_prev"]
    assert out["pt_index"][names.index("dedup"), :4].tolist() == cases["dedup"]["P"]


def test_gate_and_determinism(quirk):
    g, cases, names, M, (pm, kf, n_kf, ref), out = quirk
    B = len(names)
    ok = np.ones(B, np.int32); vo = np.zeros(B, np.int32)
    ok[0] = 0; vo[1] = 1
    got = pl.update_local_map(M, pm, kf, n_kf, ref, CLP, CLL, ok=ok, vo=vo)
    for b in (0, 1):
        assert np.array_equal(got["kf"][b], kf[b]) and got["n_kf"][b] == n_kf[b] and got["ref_kf"][b] == ref[b]
        assert got["pt_count"][b] == 0 and got["ln_count"][b] == 0
    for k, v in out.items():
        assert np.array_equal(got[k][2:], v[2:]), k
    again = pl.update_local_map(M, pm, kf, n_kf, ref, CLP, CLL)
    for k, v in out.items():
        assert np.array_equal(again[k], v), k


def test_capacity_overflow_reports_true_counts(quirk):
    g, cases, names, M, (pm, kf, n_kf, ref), out = quirk
    b = names.index("limit_80")
    got = pl.update_local_map(M, pm[b:b + 1], kf[b:b + 1, :8], n_kf[b:b + 1] * 0, ref[b:b + 1], 5, 1)
    assert got["n_kf"][0] == 82 and got["kf"][0].tolist() == out["kf"][b, :8].tolist()
    assert got["pt_count"][0] == out["pt_count"][b] and got["pt_index"][0].tolist() == out["pt_index"][b, :5].tolist()
    with pytest.raises(pl.PLError):
        M.check_capacity()
    M.check_capacity()                                          # reported and cleared


def test_upload_refuses_bad_graphs(quirk):
    g, cases, names, M, (pm, kf, n_kf, ref), out = quirk
    d = ls.to_desc(g)
    gc.collect()
    held = pl.device_bytes()
    M.set_keyframes(d)                                              # the same graph again: replaced, not added
    assert pl.device_bytes() == held
    for key, edit in (("pt_slot", lambda a: a.__setitem__(0, g["n_points"])), ("cov", lambda a: a.__setitem__(0, len(g["bad"]))),
                      ("obs", lambda a: a.__setitem__(0, -1)), ("child_offset", lambda a: a.__setitem__(3, a[4] + 1)),
                      ("parent", lambda a: a.__setitem__(0, -2))):
        bad = {k: v.copy() for k, v in d.items()}
        edit(bad[key])
        with pytest.raises(pl.PLError):
            M.set_keyframes(bad)
    big = dict(d, Tcw=np.zeros((16385, 4, 4), np.float32), Twc=np.zeros((16385, 4, 4), np.float32))
    with pytest.raises(pl.PLError):
        M.set_keyframes(big)
    assert pl.device_bytes() == held
    again = pl.update_local_map(M, pm, kf, n_kf, ref, CLP, CLL)       # the graph in place is kept
    for k, v in out.items():
        assert np.array_equal(again[k], v), k


def test_4224_copies_equal_the_single_result(quirk):
    g, cases, names, M, (pm, kf, n_kf, ref), out = quirk
    reps = 4224 // len(names) + 1
    tile = lambda a: np.concatenate([a] * reps)[:4224]   # noqa: E731
    got = pl.update_local_map(M, tile(pm), tile(kf), tile(n_kf), tile(ref), CLP, CLL)
    for k, v in out.items():
        assert np.array_equal(got[k], tile(v)), k


def test_relative_and_last_pose_are_bit_exact(quirk):
    g, cases, names, M, _, _ = quirk
    rng = np.random.default_rng(3)
    B = 64
    T = np.stack([ts.pose(rng.uniform(-0.1, 0.1, 3), rng.uniform(-0.5, 0.5, 3)) for _ in range(B)])
    ref = rng.integers(0, len(g["bad"]), B).astype(np.int32)
    Tcr = pl.relative_pose(M, T, ref)
    Tl = pl.last_pose(M, Tcr, ref)
    for b in range(B):
        assert np.array_equal(Tcr[b], ms.mat4(T[b], g["Twc"][ref[b]])), b
        assert np.array_equal(Tl[b], ms.mat4(Tcr[b], g["Tcw"][ref[b]])), b
    ref[5] = len(g["bad"])
    keep = np.full((B, 4, 4), 7.0, np.float32)
    got = pl.relative_pose(M, T, ref, out=keep)
    assert (got[5] == 7.0).all() and np.array_equal(got[4], Tcr[4])
    with pytest.raises(pl.PLError):
        M.check_indices()


# ---------------------------------------------------------------------------------------------------- the planar scene
@pytest.fixture(scope="module")
def scene():
    m, _, _ = ms.shifted_map()
    g = ls.scene_graph(m)
    M = pl.Map(**m)
    M.set_keyframes(ls.to_desc(g))
    feats = {(s, k): ts.features(ms.stream_pose(s, k), ms.STREAMS[s][2]) for s in range(3) for k in range(6)}
    cap = max(len(f[0]) for f in feats.values()); capL = max(len(f[2]) for f in feats.values())
    return m, g, M, cap, capL


def _frames(feats, Ks, cap, capL):
    B = len(feats)
    fr = dict(keys_un=np.zeros((B, cap), oracle.KP_DTYPE), desc=np.zeros((B, cap, 32), np.uint8), n=np.zeros(B, np.int32),
              keylines=np.zeros((B, capL), oracle.KEYLINE_DTYPE), line_func=np.zeros((B, capL, 3)), line_desc=np.zeros((B, capL, 32), np.uint8),
              nl=np.zeros(B, np.int32), bounds=ts.BOUNDS, scale_factors=ts.SF, inv_level_sigma2=ts.INV_SIGMA2, log_scale_factor=ts.LOG_SF,
              K=np.asarray(Ks, np.float32))
    for b, (kps, desc, kl, ldesc, lf) in enumerate(feats):
        n, nl = len(kps), len(kl)
        fr["keys_un"][b, :n] = kps; fr["desc"][b, :n] = desc; fr["n"][b] = n
        fr["keylines"][b, :nl] = kl; fr["line_func"][b, :nl] = np.asarray(lf).reshape(-1, 3); fr["line_desc"][b, :nl] = ldesc; fr["nl"][b] = nl
    return fr


def _last(lasts, cap, capL):
    B = len(lasts)
    la = dict(keys_un=np.zeros((B, cap), oracle.KP_DTYPE), n=np.zeros(B, np.int32), keylines=np.zeros((B, capL), oracle.KEYLINE_DTYPE),
              nl=np.zeros(B, np.int32), point_map=np.full((B, cap), -1, np.int32), point_outlier=np.zeros((B, cap), np.uint8),
              line_map=np.full((B, capL), -1, np.int32), line_outlier=np.zeros((B, capL), np.uint8))
    for b, l in enumerate(lasts):
        n0, nl0 = len(l["keys"]), len(l["kl"])
        la["keys_un"][b, :n0] = l["keys"]; la["n"][b] = n0; la["keylines"][b, :nl0] = l["kl"]; la["nl"][b] = nl0
        la["point_map"][b, :n0] = l["point_map"]; la["point_outlier"][b, :n0] = l["point_outlier"]
        la["line_map"][b, :nl0] = l["line_map"]; la["line_outlier"][b, :nl0] = l["line_outlier"]
    return la


def _start(m, g, S=3):
    Ks = [ms.STREAMS[s][2] for s in range(S)]
    lasts = [ms.last_frame(m, ms.stream_pose(s, 0), Ks[s], seed=s) for s in range(S)]
    rs = [ls.update_local_map_ref(g, l["point_map"], [], -1) for l in lasts]
    kf = np.full((S, CAP_KF), -1, np.int32)
    for s, r in enumerate(rs):
        kf[s, :len(r["kf"])] = r["kf"]
    ref = np.array([r["ref_kf"] for r in rs], np.int32)
    Tcr = np.stack([ms.mat4(l["Tcw"], g["Twc"][r]) for l, r in zip(lasts, ref)])
    V = np.stack([np.asarray(ms.STREAMS[s][1], np.float32) for s in range(S)])
    return Ks, lasts, kf, np.array([len(r["kf"]) for r in rs], np.int32), ref, Tcr, V


def _chain(M, cap, capL):
    return pl.LocalizationChain(M, 3, cap, capL, CAP_KF, 2048, 512, ts.BOUNDS, ts.SF, ts.INV_SIGMA2, ts.LOG_SF, max_frames=30)


def test_lists_step_equals_the_host_offset_step(scene):
    m, g, M, cap, capL = scene
    Ks, lasts, kf, n_kf, ref, Tcr, V = _start(m, g)
    S = 3
    fr = _frames([ts.features(ms.stream_pose(s, 1), Ks[s]) for s in range(S)], Ks, cap, capL)
    Tl = pl.last_pose(M, Tcr, ref)
    mm = pl.track_motion_model(M, fr, dict(_last(lasts, cap, capL), Tcw=Tl, velocity=V))
    loc = pl.update_local_map(M, mm["point_map"], kf, n_kf, ref, 2048, 512, ok=mm["ok"], vo=mm["vo"])
    assert (loc["pt_count"] > 100).all()
    fl = dict(fr, Tcw0=mm["Tcw"], point_map_in=mm["point_map"], line_map_in=mm["line_map"])
    since = np.full(S, 40, np.int32)
    got = pl.track_local_map_lists(M, fl, loc, since, 30, taps=True, seen=mm)
    host = dict(pt_index=loc["pt_index"].ravel(), ln_index=loc["ln_index"].ravel(), pt_offset=np.arange(S, dtype=np.int32) * 2048,
                pt_count=loc["pt_count"], ln_offset=np.arange(S, dtype=np.int32) * 512, ln_count=loc["ln_count"], frames_since_reloc=since,
                max_frames=30, cap_local_points=2048, cap_local_lines=512)
    want = pl.track_local_map(M, fl, host, taps=True, seen=mm)
    for k, v in want.items():
        assert np.array_equal(got[k], v), k
    # gated off: ok = 0 or vo = 1 pass through
    ok = mm["ok"].copy(); ok[0] = 0
    vo = mm["vo"].copy(); vo[1] = 1
    gated = pl.track_local_map_lists(M, fl, loc, since, 30, taps=True, seen=mm, ok=ok, vo=vo)
    for b in (0, 1):
        assert np.array_equal(gated["Tcw"][b], mm["Tcw"][b]) and np.array_equal(gated["point_map"][b], mm["point_map"][b])
        assert np.array_equal(gated["line_map"][b], mm["line_map"][b]) and not gated["point_outlier"][b].any()
        assert not gated["line_outlier"][b].any() and gated["ok"][b] == ok[b] and gated["prob_n_points"][b] == 0
    for k, v in want.items():
        assert np.array_equal(gated[k][2], v[2]), k


def _run_chain(scene, steps, graph_replay=False):
    """Run the chain; at every step check each stage tap against the separate calls and the restatement."""
    import torch
    m, g, M, cap, capL = scene
    Ks, lasts, kf, n_kf, ref, Tcr, V = _start(m, g)
    S = 3
    ch = _chain(M, cap, capL)
    ch.set_state(_last(lasts, cap, capL), Tcr, ref, V, kf, n_kf, frames_since_reloc=np.full(S, 40, np.int32))
    taps = []
    for k in range(1, steps + 1):
        feats = [ts.features(ms.stream_pose(s, k), Ks[s]) for s in range(S)]
        fr = _frames(feats, Ks, cap, capL)
        ch.set_frames(fr)
        ch.localization_step()
        out = ch.fetch()
        taps.append(out)
        # last pose
        Tl = np.stack([ms.mat4(Tcr[s], g["Tcw"][ref[s]]) for s in range(S)])
        assert np.array_equal(out["Tlast"], Tl), k
        # motion model: the separate call on the same last frames
        mm = pl.track_motion_model(M, fr, dict(_last(lasts, cap, capL), Tcw=Tl, velocity=V))
        for key in ("Tcw", "point_map", "line_map", "point_seen", "line_seen", "nmatches", "ok", "vo"):
            assert np.array_equal(out["mm"][key], mm[key]), (k, key)
        # update local map: the restatement
        for s in range(S):
            r = ls.update_local_map_ref(g, mm["point_map"][s], kf[s, :n_kf[s]].tolist(), int(ref[s]))
            _assert_frame(out["local"], s, r)
        loc = out["local"]
        # the local-map step on host offsets
        fl = dict(fr, Tcw0=mm["Tcw"], point_map_in=mm["point_map"], line_map_in=mm["line_map"])
        host = dict(pt_index=loc["pt_index"].ravel(), ln_index=loc["ln_index"].ravel(), pt_offset=np.arange(S, dtype=np.int32) * 2048,
                    pt_count=loc["pt_count"], ln_offset=np.arange(S, dtype=np.int32) * 512, ln_count=loc["ln_count"],
                    frames_since_reloc=np.full(S, 40, np.int32), max_frames=30, cap_local_points=2048, cap_local_lines=512)
        lo = pl.track_local_map(M, fl, host, seen=mm)
        for key, v in lo.items():
            assert np.array_equal(out["lo"][key], v), (k, key)
        for s in range(S):
            T = ms.stream_pose(s, k)
            assert lo["ok"][s] == 1 and ts.plane_reprojection_gap(lo["Tcw"][s], T, Ks[s]) < 0.4, (k, s)
            assert np.linalg.norm(lo["Tcw"][s][:3, 3] - T[:3, 3]) < 6e-3, (k, s)
            assert np.array_equal(out["velocity"][s], ms.velocity_oracle(lo["Tcw"][s], Tl[s])), (k, s)
            assert np.array_equal(out["Tcr"][s], ms.mat4(lo["Tcw"][s], g["Twc"][loc["ref_kf"][s]])), (k, s)
        kf, n_kf, ref, Tcr, V = loc["kf"], loc["n_kf"], loc["ref_kf"], out["Tcr"], out["velocity"]
        lasts = [dict(keys=feats[s][0], kl=feats[s][2], point_map=lo["point_map"][s, :len(feats[s][0])],
                      point_outlier=lo["point_outlier"][s, :len(feats[s][0])], line_map=lo["line_map"][s, :len(feats[s][2])],
                      line_outlier=lo["line_outlier"][s, :len(feats[s][2])]) for s in range(S)]
    M.check_indices(); M.check_capacity()
    torch.cuda.synchronize()
    return taps


def test_chain_of_three_streams_matches_every_stage(scene):
    _run_chain(scene, 5)


def test_chain_replays_from_one_cuda_graph(scene):
    """The chain enqueues no host synchronisation and no host copy: captured into a CUDA graph and replayed, it gives the eager
    run's outputs."""
    import torch
    m, g, M, cap, capL = scene
    Ks, lasts, kf, n_kf, ref, Tcr, V = _start(m, g)
    S = 3
    fr = _frames([ts.features(ms.stream_pose(s, 1), Ks[s]) for s in range(S)], Ks, cap, capL)
    ch = _chain(M, cap, capL)

    def reset():
        ch.set_state(_last(lasts, cap, capL), Tcr, ref, V, kf, n_kf, frames_since_reloc=np.full(S, 40, np.int32))
        ch.set_frames(fr)
        torch.cuda.synchronize()
    reset()
    ch.localization_step()
    eager = ch.fetch()
    reset()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode="relaxed"):
        ch.localization_step()
    reset()
    graph.replay()
    replayed = ch.fetch()
    for stage in ("Tlast", "velocity", "Tcr"):
        assert np.array_equal(replayed[stage], eager[stage]), stage
    for stage in ("mm", "local", "lo"):
        for k, v in eager[stage].items():
            assert np.array_equal(replayed[stage][k], v), (stage, k)
    assert eager["lo"]["ok"].all()
