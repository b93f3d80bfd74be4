"""pl_orb_triangulate_dev without a GPU: the exported symbol, the argument refusals that come before the device check, and the
oracle (tests/cnmp_oracle.py) against the reference's own CreateNewMapPoints loop on tests/golden/refcalls/create_new_map_points.npz
(tools/gen_create_new_map_points.py): the snapshot searches, the gates and the neighbour-order commit reproduce the reference's new
points, in creation order and bit for bit; without the commit rule they do not; every gate code occurs."""
import ctypes as C

import numpy as np
import pytest

import oracle
import plslam_b200 as pl
from plslam_b200 import binding as bd
import cnmp_fixture as cf
import cnmp_oracle as co
import triangulation_protocol as tp

PL_ERR_ARG = -1
FAKE = 4096          # a non-NULL address: every call below is refused before anything could read it


def test_symbol_is_exported():
    assert hasattr(pl.lib(), "pl_orb_triangulate_dev")


def _call(case):
    q = bd.PLTriProblems(3, FAKE, FAKE, FAKE, FAKE, 100)
    k = bd.PLTriKeyframes(4, 2000, 120, *([FAKE] * 13), 8)
    a = dict(kfs=C.byref(k), problems=C.byref(q), matches12=FAKE, search_status=FAKE, x3D=FAKE, code=FAKE, nnew=FAKE, status=FAKE)
    if case in a:
        a[case] = None
    elif case == "P < 0":
        q.P = -1
    elif case == "n_out < 0":
        q.n_out = -1
    elif case == "cap over":
        k.cap = 6145
    elif case == "n_kf * cap over an int":
        k.n_kf, k.cap = 1 << 20, 4096
    elif case == "nlevels 0":
        k.nlevels = 0
    else:
        setattr(k, case.split(" ")[0], None)
    L = bd._tri_lib()
    return L.pl_orb_triangulate_dev(a["kfs"], a["problems"], a["matches12"], a["search_status"], 1.2, a["x3D"], a["code"], a["nnew"],
                                    a["status"], None)


# the search's rules (the shared validation) and this call's own outputs
CASES = ["kfs", "problems", "matches12", "search_status", "x3D", "code", "nnew", "status", "P < 0", "n_out < 0", "cap over",
         "n_kf * cap over an int", "nlevels 0", "keys_un NULL", "desc NULL", "n NULL", "Tcw NULL", "Ow NULL", "K NULL", "fv_items NULL",
         "scale_factors NULL", "level_sigma2 NULL"]


@pytest.mark.parametrize("case", CASES)
def test_refusals_before_the_device_check(case):
    assert _call(case) == PL_ERR_ARG


def test_no_problems_enqueue_nothing():
    q = bd.PLTriProblems(0, None, None, None, None, 0)
    assert bd._tri_lib().pl_orb_triangulate_dev(None, C.byref(q), None, None, 1.2, None, None, None, None, None) == 0


def _snapshot(s):
    """The oracle's searches of every searched neighbour against the map-point state before the loop, packed as the device call
    takes them: (k, q, matches12)."""
    kfs, probs = cf.keyframes(s), cf.problems(s)
    k = bd.pack_tri_keyframes(kfs)
    q = bd.pack_tri_problems(probs, k["n"])
    m12 = np.full(q["n_out"], -1, np.int32)
    for p, (_, j, _) in enumerate(probs):
        _, m = oracle.search_for_triangulation(*tp.search_args(s, j, kfs[0]["has_mp"], kfs[j]["has_mp"]), False)
        m12[q["out_offset"][p]:q["out_offset"][p] + len(m)] = m
    return k, q, m12, probs


def _replay(s, drop=True):
    k, q, m12, probs = _snapshot(s)
    code, x3D, nnew, status = co.triangulate(k, q, m12, np.zeros(q["P"], np.int32), s["scale_factor"], s["scale_factors"],
                                             s["level_sigma2"], drop=drop)
    rows, X = cf.new_points(code, x3D, probs, q["out_offset"], int(k["n"][0]))
    idx2 = np.array([m12[q["out_offset"][[p for p, pr in enumerate(probs) if pr[1] == j][0]] + i] for j, i in rows], np.int32)
    return np.column_stack([rows, idx2]).astype(np.int32).reshape(-1, 3), X, code, nnew, status


def test_oracle_reproduces_the_reference_loop():
    s = cf.load()
    new, X, code, nnew, status = _replay(s)
    ref_new, ref_X = cf.reference(s)
    assert (status == 0).all()
    assert np.array_equal(new, ref_new), "new points (neighbour, idx1, idx2) in creation order"
    assert np.array_equal(X, ref_X), "x3D bits"
    assert nnew.sum() == len(ref_new)
    assert not s["searched"].all(), "the fixture has a neighbour the baseline test skips"


def test_without_the_commit_rule_the_result_differs():
    s = cf.load()
    new, _, code, _, _ = _replay(s, drop=False)
    assert len(new) > len(s["ref_new"])
    assert (_replay(s)[2] == co.DROPPED).sum() == len(new) - len(s["ref_new"])


def test_two_idx1_share_an_idx2():
    new = cf.load()["ref_new"]
    _, counts = np.unique(new[:, [0, 2]], axis=0, return_counts=True)
    assert (counts > 1).any(), "the reference creates both points (SearchForTriangulation never marks KF2's keypoints)"


def degenerate_keyframes():
    """Two keyframes whose rotations have rank 1 (rows proportional to one vector, the first row a power of two times the third):
    the rays are not parallel, but the first three columns of A vanish exactly, so vt.row(3) = (1, 0, 0, 0) and x3D[3] == 0."""
    def kf(r, x, y):
        T = np.zeros((4, 4), np.float32)
        T[2, :3] = r; T[0, :3] = x * r; T[1, :3] = y * r; T[:3, 3] = (0.5, -0.25, 2.0); T[3, 3] = 1
        keys = np.zeros(1, bd.KP_DTYPE); keys["x"], keys["y"] = x, y
        return dict(keys=keys, desc=np.zeros((1, 32), np.uint8), has_mp=np.zeros(1, np.uint8), fv={1: [0]}, Tcw=T.reshape(16),
                    Ow=np.zeros(3, np.float32), K=np.array([1, 1, 0, 0], np.float32))
    return [kf(np.array([1, 0, 1], np.float32), 0.5, 0.25), kf(np.array([0, 1, 1], np.float32), 0.25, -0.5)]


def test_degenerate_pose_gives_w_zero():
    kfs = degenerate_keyframes()
    k = bd.pack_tri_keyframes(kfs)
    q = bd.pack_tri_problems([(0, 1)], k["n"])
    sf = np.array([1, 1.2], np.float32)
    code, *_ = co.triangulate(k, q, np.zeros(1, np.int32), np.zeros(1, np.int32), 1.2, sf, sf * sf)
    assert code.tolist() == [co.W_ZERO]


def random_pairs(s, seed=3):
    """matches12 for every neighbour that pairs each current-keyframe keypoint with an arbitrary neighbour keypoint (a third of
    them with -1): pairs the search would not choose, which reach every gate"""
    rng = np.random.default_rng(seed)
    k, q, m12, probs = _snapshot(s)
    for p, (_, j, _) in enumerate(probs):
        a, n1, n2 = q["out_offset"][p], int(k["n"][0]), int(k["n"][j])
        m = rng.integers(0, n2, n1).astype(np.int32)
        m[rng.random(n1) < 0.33] = -1
        keep = rng.random(n1) < 0.5
        m12[a:a + n1] = np.where(keep, m12[a:a + n1], m)
    return k, q, m12


def test_every_gate_code_occurs():
    s = cf.load()
    _, _, code, _, _ = _replay(s)
    seen = set(code.tolist())
    assert {co.NO_PAIR, co.COMMITTED, co.DROPPED, co.PARALLAX, co.BEHIND1, co.BEHIND2, co.SCALE} <= seen, seen
    k, q, m12 = random_pairs(s)
    c, *_ = co.triangulate(k, q, m12, np.zeros(q["P"], np.int32), s["scale_factor"], s["scale_factors"], s["level_sigma2"])
    assert set(range(-1, 9)) - {co.W_ZERO} <= set(c.tolist()), sorted(set(c.tolist()))


def test_bad_problems_write_only_their_status():
    s = cf.load()
    k, q, m12, probs = _snapshot(s)
    q = dict(q, kf1=q["kf1"].copy(), kf2=q["kf2"].copy())
    ss = np.zeros(q["P"], np.int32)
    ss[1] = 3                                           # the search's own status passes through
    q["kf2"][2] = 99                                    # outside the table
    a, n1 = q["out_offset"][3], int(k["n"][0])
    m12[a + 5] = int(k["n"][q["kf2"][3]])               # one past KF2's keypoints
    code, x3D, nnew, status = co.triangulate(k, q, m12, ss, s["scale_factor"], s["scale_factors"], s["level_sigma2"])
    assert status.tolist()[:4] == [0, 3, 1, 4]
    for p in (1, 2, 3):
        a = q["out_offset"][p]
        assert (code[a:a + n1] == co.UNWRITTEN).all() and nnew[p] == -1



def test_knife_edge_rejects_every_pair_that_reaches_the_kf1_reprojection_gate():
    """cnmp_fixture.knife_edge (the device's knife-edge test): no pair gets past KF1's reprojection gate, and many reach it"""
    kfs, probs, sf, s2, code = cf.knife_edge(cf.load())
    assert (code == co.REPROJ1).sum() > 300
    assert not np.isin(code, [co.COMMITTED, co.DROPPED, co.REPROJ2, co.SCALE]).any()
