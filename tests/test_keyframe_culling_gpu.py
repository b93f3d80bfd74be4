"""pl_keyframe_culling_dev on the device against the oracle (tests/kfc_oracle.py), which equals the reference's own culling loop on
the golden scene (tests/test_keyframe_culling.py): the golden scene, a mixed batch with one malformed group per status code, a
large group (200 entries, cap 6144, points with 500 observers), G = 0, a CUDA-graph replay and the library's device memory."""
import numpy as np
import pytest

import plslam_b200 as pl
from plslam_b200 import binding as bd
import kfc_oracle as ko
import kfc_scene as ks
from test_keyframe_culling import load

pytestmark = pytest.mark.gpu
OUTS = ("code", "n_mps", "n_redundant")


def run(s, stream=None):
    b = bd.KeyFrameCullingProblems(*ks.split(s))
    b.run(stream)
    return b.results()


def assert_matches_oracle(s, res):
    r = ko.cull(s)
    for g, got in enumerate(res):
        assert got["status"] == r["status"][g], g
        a, c = int(s["offset"][g]), int(s["count"][g])
        for n in OUTS:
            want = r[n][a:a + c] if a >= 0 and c >= 0 and a + c <= len(s["list"]) else got[n]
            assert np.array_equal(got[n], want), (g, n)
    return r


def test_golden_scene():
    s = load()
    res = run(s)
    assert_matches_oracle(s, res)
    for n in OUTS:
        assert np.array_equal(np.concatenate([r[n] for r in res]), s[f"ref_{n}"]), n


def with_malformed_groups(s):
    """s plus, per status code, four private keyframes and twelve private points, and a group over three of them broken in one
    place; the golden groups and the broken ones alternate"""
    s = {n: v.copy() for n, v in s.items() if not n.startswith("ref_")}
    n_kf, cap = s["mp"].shape
    groups = [list(s["list"][a:a + c]) for a, c in zip(s["offset"], s["count"])]
    bad_groups = {}
    for st in range(1, 7):
        r0, p0 = len(s["n"]), len(s["bad"])
        rows = np.zeros((4, cap), np.int32) - 1
        keys = np.zeros((4, cap), s["keys_un"].dtype)
        obs = []
        for i in range(12):
            for j, r in enumerate(range(i % 2, i % 2 + 3)):
                rows[r, i] = p0 + i
                keys["octave"][r, i] = (i + j) % 3
                obs.append((r0 + r, i))
        s["mp"] = np.concatenate([s["mp"], rows]); s["keys_un"] = np.concatenate([s["keys_un"], keys])
        s["n"] = np.concatenate([s["n"], np.full(4, 12, np.int32)])
        s["origin"] = np.concatenate([s["origin"], np.zeros(4, np.uint8)]); s["not_erase"] = np.concatenate([s["not_erase"], np.zeros(4, np.uint8)])
        s["bad"] = np.concatenate([s["bad"], np.zeros(12, np.uint8)])
        per = {p0 + i: [(r, idx) for r, idx in obs if idx == i] for i in range(12)}
        base = len(s["obs_kf"])
        flat = [e for i in range(12) for e in per[p0 + i]]
        s["obs_kf"] = np.concatenate([s["obs_kf"], np.array([e[0] for e in flat], np.int32)])
        s["obs_idx"] = np.concatenate([s["obs_idx"], np.array([e[1] for e in flat], np.int32)])
        s["obs_offset"] = np.concatenate([s["obs_offset"], base + np.cumsum([len(per[p0 + i]) for i in range(12)]).astype(np.int32)])
        lst = [r0, r0 + 1, r0 + 2]
        if st == 1:
            lst[1] = -3
        elif st == 2:
            s["n"][r0 + 1] = cap + 1
        elif st == 3:
            lst[2] = r0
        elif st == 4:
            s["mp"][r0 + 1, 0] = 1 << 30
        elif st == 5:
            s["obs_offset"][p0 + 3] = s["obs_offset"][p0 + 4] + 1
        elif st == 6:
            s["obs_idx"][s["obs_offset"][p0 + 5]] = 6     # a slot of that keyframe that holds another point
        bad_groups[st] = lst
    mixed = [g for good, st in zip(groups, range(1, 7)) for g in (good, bad_groups[st])]
    s.update(bd.pack_cull_groups(mixed))
    return s, mixed


def test_mixed_batch_with_one_malformed_group_per_status():
    gold = load()
    s, mixed = with_malformed_groups(gold)
    res = run(s)
    r = assert_matches_oracle(s, res)
    assert sorted(set(r["status"].tolist()) - {0}) == [1, 2, 3, 4, 5, 6]
    good = [x for x, st in zip(res, r["status"]) if st == 0]
    for n in OUTS:      # the good groups' results do not depend on their neighbours
        assert np.array_equal(np.concatenate([x[n] for x in good]), gold[f"ref_{n}"]), n


def test_large_group_multi_warp():
    rng = np.random.default_rng(5)
    size = np.concatenate([rng.integers(1000, 6144 - 16, 200), np.full(320, 64)])
    size[[3, 50, 120]] = 6144 - 16
    b, rows = ks.bulk(rng, size, heavy=16, heavy_obs=500)
    s = ks.packed(*b.scene([rows[:200]]), cap=6144)
    assert s["mp"].shape[1] == 6144 and np.diff(s["obs_offset"]).max() == 500
    r = assert_matches_oracle(s, run(s))
    assert (r["code"] == 1).sum() >= 2 and r["n_mps"].max() > 4096


def test_no_groups_enqueue_nothing():
    import torch
    s = load()
    k, m, _ = ks.split(s)
    b = bd.KeyFrameCullingProblems(k, m, bd.pack_cull_groups([]))
    n0 = pl.launch_count()
    b.run()
    assert pl.launch_count() == n0
    assert all((t.cpu() == -7).all() for t in b.outputs.values())
    torch.cuda.synchronize()


def test_graph_replay_equals_eager():
    import torch
    s = load()
    eager = run(s)
    b = bd.KeyFrameCullingProblems(*ks.split(s), out_fill=-5)
    stream = torch.cuda.Stream()
    b.run(stream)                        # warm-up outside the capture
    stream.synchronize()
    for t in b.outputs.values():
        t.fill_(-5)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        b.run(stream)
    for t in b.outputs.values():
        t.fill_(-5)
    torch.cuda.synchronize()
    graph.replay()
    got = b.results()
    for e, g in zip(eager, got):
        assert e["status"] == g["status"]
        for n in OUTS:
            assert np.array_equal(e[n], g[n])


def test_device_bytes_unchanged():
    s = load()
    b = bd.KeyFrameCullingProblems(*ks.split(s))
    before = pl.device_bytes()
    b.run()
    b.results()
    assert pl.device_bytes() == before
