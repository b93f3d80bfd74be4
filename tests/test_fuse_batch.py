"""pl_orb_fuse_search_dev / pl_lsd_fuse_search_dev without a GPU: the exported symbols, the argument refusals that come before the
device check, the packers of the Python binding, and the snapshot protocol of LocalMapping::SearchInNeighbors against the
reference's own sequential Fuse loop (tests/golden/refcalls/fuse_protocol.npz, made by tools/gen_fuse_protocol.py)."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as pl
from plslam_b200 import binding as bd
from plslam_b200 import synth
import fuse_protocol as fp
import oracle

FAKE = 4096          # a non-NULL address: every call below is refused before anything could read it


def test_symbols_are_exported():
    L = pl.lib()
    for name in ("pl_orb_fuse_search", "pl_lsd_fuse_search", "pl_orb_fuse_search_dev", "pl_lsd_fuse_search_dev"):
        assert hasattr(L, name), name


def _tables(lines, P=3):
    q = bd.PLFuseProblems(P, *([FAKE] * 5), 10, FAKE, FAKE, 10)
    m = bd.PLFuseLandmarks(20, *([FAKE] * 5))
    if lines:
        k = bd.PLFuseLineKeyframes(4, 300, 500, *([FAKE] * 8), 1.2, 0.18)
    else:
        k = bd.PLFuseKeyframes(4, 2000, *([FAKE] * 9), 8, 0.18)
    return k, m, q


def _call(lines, k, m, q, use=(True, True, True), stop=FAKE, status=FAKE, out=FAKE):
    L = bd._fuse_lib()
    a = [C.byref(x) if u else None for x, u in zip((k, m, q), use)]
    if lines:
        return L.pl_lsd_fuse_search_dev(*a, out, out, stop, status, None)
    return L.pl_orb_fuse_search_dev(*a, out, out, status, None)


CASES = ["no keyframes", "no landmarks", "no problems", "P < 0", "n_entries < 0", "n_out < 0", "landmarks < 0", "n_kf 0", "cap 0",
         "cap over", "n_kf * cap over an int", "kf NULL", "th NULL", "offset NULL", "count NULL", "out_offset NULL", "entry_lm NULL",
         "entry_skip NULL", "status NULL", "best_idx NULL", "keyframe n NULL", "Tcw NULL", "bounds NULL", "landmark desc NULL"]
POINT_CASES = CASES + ["nlevels 0", "scale_factors NULL", "inv_level_sigma2 NULL"]
LINE_CASES = CASES + ["cap_pdesc 0", "cap_pdesc over", "pdesc NULL", "n_pdesc NULL", "stop_at NULL"]


def _refused(lines, case):
    k, m, q = _tables(lines)
    kw = {}
    if case.startswith("no "):
        kw["use"] = tuple(case != f"no {x}" for x in ("keyframes", "landmarks", "problems"))
    elif case == "P < 0":
        q.P = -1
    elif case in ("n_entries < 0", "n_out < 0"):
        setattr(q, case.split(" ")[0], -1)
    elif case == "landmarks < 0":
        m.n = -1
    elif case == "n_kf 0":
        k.n_kf = 0
    elif case in ("cap 0", "cap_pdesc 0"):
        setattr(k, case.split(" ")[0], 0)
    elif case == "cap over":
        k.cap = 32769 if lines else 6145
    elif case == "cap_pdesc over":
        k.cap_pdesc = 32769
    elif case == "n_kf * cap over an int":
        k.n_kf, k.cap = 1 << 20, 4096
    elif case == "nlevels 0":
        k.nlevels = 0
    elif case in ("status NULL", "stop_at NULL", "best_idx NULL"):
        kw[{"status NULL": "status", "stop_at NULL": "stop", "best_idx NULL": "out"}[case]] = None
    elif case == "keyframe n NULL":
        k.n = None
    elif case == "landmark desc NULL":
        m.desc = None
    else:
        name = case.split(" ")[0]
        setattr(q if hasattr(q, name) and name not in ("n",) else k, name, None)
    return _call(lines, k, m, q, **kw)


@pytest.mark.parametrize("case", POINT_CASES)
def test_point_refusals_before_the_device_check(case):
    assert _refused(False, case) == -1, case


@pytest.mark.parametrize("case", LINE_CASES)
def test_line_refusals_before_the_device_check(case):
    assert _refused(True, case) == -1, case


@pytest.mark.parametrize("lines", [False, True])
def test_no_problems_enqueue_nothing(lines):
    k, m, q = _tables(lines, P=0)
    assert _call(lines, k, m, q, use=(False, True, True), stop=None, status=None, out=None) == 0


def _keyframes(lines):
    if lines:
        return [dict(kl=np.zeros(n, pl.KEYLINE_DTYPE), pdesc=np.full((n // 2, 32), n, np.uint8), Tcw=np.eye(4) * (n + 1),
                     Ow=[n, 0, 0], K=[500, 500, 320, 240 + n], bounds=[0, 0, 640, 480]) for n in (3, 0, 7)]
    f = synth.synth_fuse_problem(6, n_mp=10, n_kp=40)
    return [dict(keys=f["keys"][:n], desc=f["desc"][:n], Tcw=np.eye(4) * (n + 1), Ow=[n, 0, 0], K=[500, 500, 320, 240 + n],
                 bounds=[0, 0, 640, 480]) for n in (25, 0, 40)]


@pytest.mark.parametrize("lines", [False, True])
def test_keyframe_packer_layouts(lines):
    kfs = _keyframes(lines)
    h = bd.pack_fuse_keyframes(kfs, lines)
    name, rows = ("keylines", "kl") if lines else ("keys_un", "keys")
    n = [len(k[rows]) for k in kfs]
    assert h["n"].tolist() == n and h["cap"] == max(n) and h[name].shape == (3, max(n))
    for i, k in enumerate(kfs):
        assert h[name][i, :n[i]].tobytes() == np.asarray(k[rows]).tobytes() and not h[name][i, n[i]:].view(np.uint8).any()
        assert np.array_equal(h["Tcw"][i], np.asarray(k["Tcw"], np.float32).reshape(16)) and h["K"][i, 3] == 240 + n[i]
    if lines:
        assert h["n_pdesc"].tolist() == [1, 0, 3] and h["cap_pdesc"] == 3 and h["pdesc"].shape == (3, 3, 32)
        assert (h["pdesc"][2, :3] == 7).all() and not h["pdesc"][0, 1:].any()
    else:
        assert h["desc"].shape == (3, 40, 32) and np.array_equal(h["desc"][0, :25], kfs[0]["desc"])
    big = bd.pack_fuse_keyframes(kfs, lines, cap=64)
    assert big["cap"] == 64 and big[name].shape == (3, 64)
    with pytest.raises(ValueError):
        bd.pack_fuse_keyframes(kfs, lines, cap=5)


def test_problem_packer_shares_entry_lists_and_lays_outputs_end_to_end():
    lists = [(np.arange(5), [0, 1, 0, 0, 1]), ([], []), ([7, 3], [1, 0])]
    q = bd.pack_fuse_problems([(0, 3.0, 0), (2, 1.0, 0), (1, 3.0, 1), (0, 6.0, 2)], lists)
    assert q["P"] == 4 and q["kf"].tolist() == [0, 2, 1, 0] and q["th"].tolist() == [3, 1, 3, 6]
    assert q["offset"].tolist() == [0, 0, 5, 5] and q["count"].tolist() == [5, 5, 0, 2]
    assert q["out_offset"].tolist() == [0, 5, 10, 10] and q["n_out"] == 12
    assert q["entry_lm"].tolist() == [0, 1, 2, 3, 4, 7, 3] and q["entry_skip"].tolist() == [0, 1, 0, 0, 1, 1, 0]
    assert bd.pack_fuse_problems([], [])["n_out"] == 0
    with pytest.raises(ValueError):
        bd.pack_fuse_problems([(0, 3.0, 0)], [([1, 2], [0])])


@pytest.fixture(scope="module")
def protocol():
    return fp.load()


def test_fixture_exercises_the_protocol(protocol):
    s = protocol
    assert (s["ref_nfused"] > 20).all() and s["ref_bad"].sum() > 20
    # point 0 is fused into a keypoint of target 2 that its original descriptor does not pick
    a, b = s["kf_start"][2], s["kf_start"][3]
    assert (s["ref_slots"][a:b] == 0).sum() == 1


def test_reference_loop_restated_on_the_oracle(protocol):
    M, nfused = fp.first_loop(protocol, fp.oracle_search(protocol), snapshot=False)
    assert np.array_equal(fp.final_slots(M), protocol["ref_slots"]) and np.array_equal(M.bad, protocol["ref_bad"].astype(bool))
    assert np.array_equal(M.desc, protocol["ref_desc"]) and np.array_equal(nfused, protocol["ref_nfused"])


def test_snapshot_protocol_reproduces_the_reference(protocol):
    M, nfused = fp.first_loop(protocol, fp.oracle_search(protocol))
    assert np.array_equal(fp.final_slots(M), protocol["ref_slots"]) and np.array_equal(M.bad, protocol["ref_bad"].astype(bool))
    assert np.array_equal(M.desc, protocol["ref_desc"]) and np.array_equal(nfused, protocol["ref_nfused"])


def test_snapshot_protocol_needs_the_research_rule(protocol):
    M, _ = fp.first_loop(protocol, fp.oracle_search(protocol), research=False)
    slots = fp.final_slots(M)
    a, b = protocol["kf_start"][2], protocol["kf_start"][3]
    assert not np.array_equal(slots, protocol["ref_slots"])
    assert not np.array_equal(slots[a:b] == 0, protocol["ref_slots"][a:b] == 0)     # point 0 lands on the other keypoint


def _line_stop_case():
    """A line problem whose map lines at entries 37 and 38 are behind the camera (the second is the first one again)."""
    from test_localmap2 import _line_fuse_problem, _args
    a = list(_args(_line_fuse_problem(22, 37)))
    idx = np.concatenate([np.arange(38), [37], np.arange(38, len(a[9]))])
    for k in range(8, 14):
        a[k] = np.asarray(a[k])[idx]
    return a


def _live(a, skip):
    b = list(a)
    b[8] = skip
    return b


def line_stop_rule(a, snapshot, flipped, search):
    """The results the line protocol acts on when the entries `flipped` became skipped after the snapshot, and the reference's."""
    live = np.array(a[8]); live[list(flipped)] = 1
    bi, bd, stop = snapshot
    rest = lambda j0: search([x[j0:] if k in range(8, 14) else x for k, x in enumerate(_live(a, live))])
    got = fp.line_results_at_application(bi, bd, stop, live, rest)
    want = search(_live(a, live))
    return live, got, want


def _same_where_reached(live, got, want):
    bi, bd, stop = got
    wbi, wbd, wstop = want
    reach = (np.arange(len(live)) < stop) & (live == 0)      # the entries the reference acts on
    return stop == wstop and np.array_equal(bi[reach], wbi[reach]) and np.array_equal(bd[reach], wbd[reach])


@pytest.mark.parametrize("flipped,stop", [((), 37), ((37,), 38), ((37, 38), None)])
def test_line_stop_entry_that_becomes_skipped_is_searched_past(flipped, stop):
    a = _line_stop_case()
    search = lambda x: oracle.lsd_fuse_search(*x)
    snapshot = search(a)
    assert snapshot[2] == 37
    live, got, want = line_stop_rule(a, snapshot, flipped, search)
    assert got[2] == (len(live) if stop is None else stop)
    assert _same_where_reached(live, got, want)
    if flipped:     # without the rule the target stops at the snapshot's stop and misses the reference's fusions after it
        assert not _same_where_reached(live, snapshot, want)
    if stop is None:
        assert (want[1][39:] <= 50).sum() > 10
