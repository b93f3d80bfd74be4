"""Tracking::UpdateLocalMap restated on the CPU (tests/localmap_scene.py): one named test per behaviour of the reference that the
device must reproduce, and the localisation chain over the planar scene's keyframe graph.

No GPU: this pins what pl_track_update_local_map_dev is compared with in test_update_local_map_gpu.py.  Over 3 streams x 4 steps
of last pose -> motion model -> update local map -> local-map step -> velocity -> relative pose, measured with these composites,
the local-map poses stay within the bounds test_track_motion_model.py uses (0.4 px, 6 mm)."""
import numpy as np
import pytest

import localmap_scene as ls
import motion_scene as ms
import track_scene as ts


@pytest.fixture(scope="module")
def quirks():
    g, cases = ls.quirk_cases()
    return g, cases, {n: ls.update_local_map_ref(g, c["point_map"], c["kf_prev"], c["ref_prev"], c["line_map"]) for n, c in cases.items()}


def test_voter_order_is_index_order(quirks):
    g, c, r = quirks
    k = c["voter_order"]["kfs"]
    assert r["voter_order"]["kf"] == [k["a"], k["b"], k["c"]] and r["voter_order"]["ref_kf"] == k["b"]


def test_reference_keyframe_is_the_first_max_over_good_voters(quirks):
    g, c, r = quirks
    k = c["first_max"]["kfs"]
    assert r["first_max"]["ref_kf"] == k["e"]                    # e and f tie at 3, the bad g has 5
    assert r["first_max"]["kf"] == [k["d"], k["e"], k["f"]]


def test_only_the_original_voters_are_expanded(quirks):
    g, c, r = quirks
    k = c["only_voters"]["kfs"]
    assert r["only_voters"]["kf"] == [k["h"], k["i"]]


def test_size_over_80_is_checked_at_the_top_of_each_visit(quirks):
    g, c, r = quirks
    k = c["limit_80"]["kfs"]
    lst = r["limit_80"]["kf"]
    assert len(lst) == 82 and lst[80:] == [k["x0"], k["x1"]] and k["x2"] not in lst


def test_parent_break_ends_the_whole_expansion(quirks):
    g, c, r = quirks
    k = c["parent_break"]["kfs"]
    assert r["parent_break"]["kf"] == [k["k1"], k["k2"], k["q"]]


def test_bad_skipped_for_covisibles_and_children_but_not_the_parent(quirks):
    g, c, r = quirks
    k = c["bad_skips"]["kfs"]
    assert r["bad_skips"]["kf"] == [k["v"], k["cg"], k["hg"], k["pb"]]
    assert g["pt"][k["pb"]][0] in r["bad_skips"]["points"]       # the bad parent's points are in the local map


def test_empty_vote_keeps_the_stale_list_and_reference(quirks):
    g, c, r = quirks
    s = c["stale"]
    assert r["stale"]["kf"] == s["kf_prev"] and r["stale"]["ref_kf"] == s["ref_prev"]
    want = ls.update_local_map_ref(g, [], [], -1)
    y, h, a = s["kf_prev"]
    assert want["points"] == [] and r["stale"]["points"] == c["dedup"]["P"][:3] + g["pt"][h] + g["pt"][a]
    assert r["stale"]["lines"] == c["dedup"]["L"][:2]


def test_bad_voters_only_empty_the_list_and_keep_the_reference(quirks):
    g, c, r = quirks
    assert r["bad_voters"]["kf"] == [] and r["bad_voters"]["ref_kf"] == c["bad_voters"]["ref_prev"] and r["bad_voters"]["points"] == []


def test_lines_do_not_vote(quirks):
    g, c, r = quirks
    k, cs = c["lines_no_vote"]["kfs"], c["lines_no_vote"]
    assert r["lines_no_vote"]["kf"] == [k["t"]]
    voted = ls.update_local_map_ref(g, cs["point_map"], [], -1, cs["line_map"], variant="lines_vote")
    assert voted["kf"] == [k["t"], k["u"]]


def test_first_occurrence_dedup_across_and_within_keyframes(quirks):
    g, c, r = quirks
    cs = c["dedup"]
    assert r["dedup"]["kf"] == [cs["kfs"]["y"], cs["kfs"]["z"]]
    assert r["dedup"]["points"] == cs["P"] and r["dedup"]["lines"] == cs["L"]


@pytest.fixture(scope="module")
def scene():
    m, _, _ = ms.shifted_map()
    return m, ls.scene_graph(m)


def test_scene_graph_follows_the_reference_rules(scene):
    m, g = scene
    K = len(g["bad"])
    obs = ls.observations(g)
    roots = [k for k in range(K) if g["parent"][k] < 0]
    assert len(roots) == 1
    for k in range(K):
        w = {}
        for p in g["pt"][k]:
            for o in obs[p]:
                if o != k:
                    w[o] = w.get(o, 0) + 1
        cov = g["cov"][k]
        assert all(w[o] >= 15 for o in cov) or len(cov) == 1
        assert [(w[o], o) for o in cov] == sorted([(w[o], o) for o in cov], reverse=True)
        assert len(cov) >= 2
    # creation order differs from index order, so "earlier" is not "lower index"
    assert any(g["parent"][k] > k for k in range(K))


def _local_lists(m, g, point_map, kf_prev, ref_prev):
    r = ls.update_local_map_ref(g, point_map, kf_prev, ref_prev)
    return r, np.asarray(r["points"], np.int64), np.asarray(r["lines"], np.int64)


@pytest.mark.parametrize("s", range(len(ms.STREAMS)))
def test_chain_recovers_the_stream_poses(scene, s):
    m, g = scene
    K = ms.STREAMS[s][2]
    last = ms.last_frame(m, ms.stream_pose(s, 0), K, seed=s)
    r, _, _ = _local_lists(m, g, last["point_map"], [], -1)
    kf, ref = r["kf"], r["ref_kf"]
    Tcr = ms.mat4(last["Tcw"], g["Twc"][ref])
    V = ms.STREAMS[s][1]
    for k in range(1, 5):
        T = ms.stream_pose(s, k)
        f = ts.features(T, K)
        Tlast = ms.mat4(Tcr, g["Tcw"][ref])                       # UpdateLastFrame
        assert np.abs(Tlast - last["Tcw"]).max() < 1e-5
        mm = ms.track_motion_model_oracle(m, *f, K, dict(last, Tcw=Tlast, velocity=V))
        assert mm["ok"] == 1 and mm["vo"] == 0, (s, k)
        r, lp, ll = _local_lists(m, g, mm["point_map"], kf, ref)
        kf, ref = r["kf"], r["ref_kf"]
        assert len(lp) > 100 and len(ll) > 10
        lo = ms.track_local_map_seen_oracle(m, *f, mm["Tcw"], K, lp, ll, 40, 30, mm["point_map"], mm["line_map"], mm["point_seen"],
                                            mm["line_seen"])
        assert lo["ok"] == 1, (s, k)
        assert ts.plane_reprojection_gap(lo["Tcw"], T, K) < 0.4, (s, k)
        assert np.linalg.norm(lo["Tcw"][:3, 3] - T[:3, 3]) < 6e-3, (s, k)
        V = ms.velocity_oracle(lo["Tcw"], Tlast)
        Tcr = ms.mat4(lo["Tcw"], g["Twc"][ref])
        last = dict(keys=f[0], kl=f[2], point_map=lo["point_map"], point_outlier=lo["point_outlier"], line_map=lo["line_map"],
                    line_outlier=lo["line_outlier"], Tcw=lo["Tcw"])
