"""pl_orb_search_for_triangulation_dev / pl_lsd_search_for_triangulation_dev without a GPU: the exported symbols, the argument
refusals that come before the device check, the packers of the Python binding, and the snapshot protocol of
LocalMapping::CreateNewMapPoints against the reference's own sequential loop (tests/golden/refcalls/triangulation_protocol.npz, made by
tools/gen_triangulation_protocol.py)."""
import ctypes as C

import numpy as np
import pytest

import oracle
import plslam_b200 as pl
from plslam_b200 import binding as bd
import triangulation_protocol as tp

FAKE = 4096          # a non-NULL address: every call below is refused before anything could read it


def test_symbols_are_exported():
    L = pl.lib()
    for name in ("pl_orb_search_for_triangulation", "pl_lsd_search_for_triangulation", "pl_orb_search_for_triangulation_dev",
                 "pl_lsd_search_for_triangulation_dev"):
        assert hasattr(L, name), name


def _tables(lines, P=3):
    q = bd.PLTriProblems(P, FAKE, FAKE, None if lines else FAKE, FAKE, 100)
    if lines:
        k = bd.PLTriLineKeyframes(4, 300, FAKE, FAKE, FAKE)
    else:
        k = bd.PLTriKeyframes(4, 2000, 120, *([FAKE] * 13), 8)
    return k, q


def _call(lines, k, q, use=(True, True), out=FAKE, nmatches=FAKE, status=FAKE):
    L = bd._tri_lib()
    a = [C.byref(x) if u else None for x, u in zip((k, q), use)]
    if lines:
        return L.pl_lsd_search_for_triangulation_dev(*a, 80.0, 0.8, 1, out, nmatches, status, None)
    return L.pl_orb_search_for_triangulation_dev(*a, 0, out, nmatches, status, None)


CASES = ["no keyframes", "no problems", "P < 0", "n_out < 0", "n_kf 0", "cap 0", "cap over", "n_kf * cap over an int", "kf1 NULL",
         "kf2 NULL", "out_offset NULL", "matches NULL", "nmatches NULL", "status NULL", "keyframe n NULL"]
POINT_CASES = CASES + ["F12 NULL", "cap_nodes 0", "n_kf * cap_nodes over an int", "nlevels 0", "keys_un NULL", "desc NULL",
                       "has_mp NULL", "fv_nodes NULL", "fv_start NULL", "fv_items NULL", "nn NULL", "Tcw NULL", "Ow NULL", "K NULL",
                       "scale_factors NULL", "level_sigma2 NULL"]
LINE_CASES = CASES + ["ldesc NULL", "has_ml NULL"]


def _refused(lines, case):
    k, q = _tables(lines)
    kw = {}
    if case.startswith("no "):
        kw["use"] = (case != "no keyframes", case != "no problems")
    elif case == "P < 0":
        q.P = -1
    elif case == "n_out < 0":
        q.n_out = -1
    elif case == "n_kf 0":
        k.n_kf = 0
    elif case in ("cap 0", "cap_nodes 0", "nlevels 0"):
        setattr(k, case.split(" ")[0], 0)
    elif case == "cap over":
        k.cap = 32000 if lines else 6145
    elif case == "n_kf * cap over an int":
        k.n_kf, k.cap = 1 << 20, 4096
    elif case == "n_kf * cap_nodes over an int":
        k.n_kf, k.cap_nodes = 1 << 20, 4096
    elif case in ("matches NULL", "nmatches NULL", "status NULL"):
        kw[{"matches NULL": "out", "nmatches NULL": "nmatches", "status NULL": "status"}[case]] = None
    elif case == "keyframe n NULL":
        k.n = None
    else:
        name = case.split(" ")[0]
        setattr(q if name in ("kf1", "kf2", "F12", "out_offset") else k, name, None)
    return _call(lines, k, q, **kw)


@pytest.mark.parametrize("case", POINT_CASES)
def test_point_refusals_before_the_device_check(case):
    assert _refused(False, case) == -1, case


@pytest.mark.parametrize("case", LINE_CASES)
def test_line_refusals_before_the_device_check(case):
    assert _refused(True, case) == -1, case


@pytest.mark.parametrize("lines", [False, True])
def test_no_problems_enqueue_nothing(lines):
    k, q = _tables(lines, P=0)
    assert _call(lines, k, q, use=(False, True), out=None, nmatches=None, status=None) == 0


def _keyframes():
    s = tp.load()
    return [tp.keyframe(s, k) for k in (0, 1)] + [dict(tp.keyframe(s, 2), keys=s["keys"][:0], desc=s["desc"][:0], has_mp=[], fv={})]


def test_point_keyframe_packer_layout():
    kfs = _keyframes()
    h = bd.pack_tri_keyframes(kfs)
    n = [len(k["keys"]) for k in kfs]
    nn = [len(k["fv"]) for k in kfs]
    assert h["n"].tolist() == n and h["cap"] == max(n) and h["keys_un"].shape == (3, max(n)) and h["desc"].shape == (3, max(n), 32)
    assert h["nn"].tolist() == nn and h["cap_nodes"] == max(nn) and h["fv_start"].shape == (3, max(nn) + 1)
    for i, k in enumerate(kfs):
        assert h["keys_un"][i, :n[i]].tobytes() == np.asarray(k["keys"]).tobytes() and not h["keys_un"][i, n[i]:].view(np.uint8).any()
        assert np.array_equal(h["desc"][i, :n[i]], k["desc"]) and np.array_equal(h["has_mp"][i, :n[i]], k["has_mp"])
        nodes, start, items = bd._fv_csr(k["fv"])
        assert np.array_equal(h["fv_nodes"][i, :nn[i]], nodes) and np.array_equal(h["fv_start"][i, :nn[i] + 1], start)
        assert np.array_equal(h["fv_items"][i, :len(items)], items) and h["fv_start"][i, nn[i]] == len(items)
        assert np.array_equal(h["Tcw"][i], np.asarray(k["Tcw"], np.float32)) and np.array_equal(h["K"][i], k["K"])
    big = bd.pack_tri_keyframes(kfs, cap=4000, cap_nodes=300)
    assert big["cap"] == 4000 and big["cap_nodes"] == 300 and big["fv_items"].shape == (3, 4000) and big["fv_start"].shape == (3, 301)
    with pytest.raises(ValueError):
        bd.pack_tri_keyframes(kfs, cap=5)


def test_line_keyframe_packer_layout():
    rng = np.random.default_rng(1)
    kfs = [dict(ldesc=rng.integers(0, 256, (n, 32), dtype=np.uint8), has_ml=rng.integers(0, 2, n)) for n in (5, 0, 9)]
    h = bd.pack_tri_keyframes(kfs, lines=True)
    assert h["n"].tolist() == [5, 0, 9] and h["cap"] == 9 and h["ldesc"].shape == (3, 9, 32) and h["has_ml"].shape == (3, 9)
    assert np.array_equal(h["ldesc"][2], kfs[2]["ldesc"]) and np.array_equal(h["has_ml"][0, :5], kfs[0]["has_ml"])
    assert not h["ldesc"][0, 5:].any() and not h["has_ml"][1].any()


def test_problem_packer_lays_outputs_end_to_end():
    F = np.arange(9, dtype=np.float32).reshape(3, 3)
    q = bd.pack_tri_problems([(0, 1, F), (2, 0, F + 1), (0, 2, F), (5, 1, F)], [7, 3, 0])
    assert q["P"] == 4 and q["kf1"].tolist() == [0, 2, 0, 5] and q["kf2"].tolist() == [1, 0, 2, 1]
    assert q["out_offset"].tolist() == [0, 7, 7, 14] and q["n_out"] == 14 and q["count"].tolist() == [7, 0, 7, 0]
    assert np.array_equal(q["F12"][1], F.reshape(9) + 1)
    lq = bd.pack_tri_problems([(1, 0), (0, 1)], [4, 6])
    assert lq["out_offset"].tolist() == [0, 6] and lq["n_out"] == 10 and not lq["F12"].any()
    assert bd.pack_tri_problems([], [1])["n_out"] == 0


@pytest.fixture(scope="module")
def protocol():
    return tp.load()


def _oracle_snapshot(s):
    has = [tp.keyframe(s, k)["has_mp"] for k in range(len(s["kf_start"]) - 1)]
    return [oracle.search_for_triangulation(*tp.search_args(s, j, has[0], has[j]), False)[1] for j in range(1, len(has))]


def test_fixture_exercises_the_protocol(protocol):
    ref = tp.reference_lists(protocol)
    assert len(ref) == 6 and all(len(r) > 10 for r in ref)


def test_reference_loop_restated_on_the_oracle(protocol):
    s = protocol
    lists = tp.create_new_map_points(s, lambda j, has: oracle.search_for_triangulation(*tp.search_args(s, j, has[0], has[j]), False)[1])
    assert tp.same_lists(lists, tp.reference_lists(s))


def test_snapshot_and_drop_reproduce_the_reference(protocol):
    assert tp.same_lists(tp.snapshot_protocol(protocol, _oracle_snapshot(protocol)), tp.reference_lists(protocol))


def test_snapshot_without_the_drop_rule_differs(protocol):
    ref = tp.reference_lists(protocol)
    lists = tp.snapshot_protocol(protocol, _oracle_snapshot(protocol), drop=False)
    assert np.array_equal(lists[0], ref[0])                       # the first neighbour sees the snapshot itself
    assert all(len(a) > len(b) for a, b in zip(lists[1:], ref[1:]))     # each later one keeps pairs the reference skipped
