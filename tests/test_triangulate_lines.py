"""pl_lsd_triangulate_dev without a GPU: the exported and declared symbol, the argument refusals that come before the device check,
the cv2 pins of the arithmetic the line triangulation adds to the point triangulation's (cv::invert and cv::solve of 3x3 CV_32F
matrices, cv::gemm with and without GEMM_1_T, cv::norm), and the oracle (tests/cnml_oracle.py) on the scene of tests/cnml_scene.py
with matches taken from the segment ids: its mutants change the result, and the crafted variants reach the gate codes."""
import ctypes as C
import os

import numpy as np
import pytest

import plslam_b200 as pl
from plslam_b200 import binding as bd
import cnml_oracle as co
import cnml_scene as cs

PL_ERR_ARG = -1
FAKE = 4096          # a non-NULL address: every call below is refused before anything could read it
f32, f64 = np.float32, np.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_symbol_is_exported_and_declared():
    assert hasattr(pl.lib(), "pl_lsd_triangulate_dev")
    with open(os.path.join(ROOT, "include", "plslam_b200.h")) as f:
        h = f.read()
    assert "int pl_lsd_triangulate_dev(" in h and "#define PL_TRI_LINE_MAX_ENTRIES 16" in h


def _call(case):
    q = bd.PLTriProblems(3, FAKE, FAKE, None, FAKE, 100)
    k = bd.PLTriLineKeyframes(4, 300, FAKE, FAKE, FAKE)
    gm = bd.PLTriLineGeometry(4, 300, *([FAKE] * 6), 2)
    g = bd.PLTriLineGroups(2, FAKE, FAKE, FAKE, FAKE, 6, FAKE, FAKE, FAKE, 500)
    a = dict(kfs=C.byref(k), geom=C.byref(gm), problems=C.byref(q), matches=FAKE, nmatches=FAKE, search_status=FAKE, groups=C.byref(g),
             code=FAKE, line3D=FAKE, nnew=FAKE, status=FAKE)
    if case in a:
        a[case] = None
    elif case == "P < 0":
        q.P = -1
    elif case == "n_out < 0":
        q.n_out = -1
    elif case == "cap over":
        k.cap = gm.cap = 32000
    elif case == "G < 0":
        g.G = -1
    elif case == "n_entry_list < 0":
        g.n_entry_list = -1
    elif case == "groups n_out < 0":
        g.n_out = -1
    elif case == "nlevels 0":
        gm.nlevels = 0
    elif case == "geometry rows":
        gm.cap = 299
    elif case == "geometry n_kf":
        gm.n_kf = 5
    elif case.startswith("group "):
        setattr(g, case.split(" ")[1], None)
    else:
        setattr(k if case.split(" ")[0] in ("ldesc", "has_ml", "n") else gm, case.split(" ")[0], None)
    return bd._tri_lib().pl_lsd_triangulate_dev(a["kfs"], a["geom"], a["problems"], a["matches"], a["nmatches"], a["search_status"],
                                                a["groups"], a["code"], a["line3D"], a["nnew"], a["status"], None)


# the line search's rules (the shared validation) and this call's own inputs and outputs
CASES = ["kfs", "problems", "matches", "nmatches", "search_status", "groups", "geom", "code", "line3D", "nnew", "status", "P < 0",
         "n_out < 0", "cap over", "G < 0", "n_entry_list < 0", "groups n_out < 0", "nlevels 0", "geometry rows", "geometry n_kf",
         "ldesc NULL", "has_ml NULL", "n NULL", "keylines NULL", "line_func NULL", "Tcw NULL", "Ow NULL", "K NULL",
         "level_sigma2_line NULL", "group kf_cur", "group entry_start", "group n_entries", "group out_offset", "group entry_problem",
         "group entry_kf", "group entry_median_depth"]


@pytest.mark.parametrize("case", CASES)
def test_refusals_before_the_device_check(case):
    assert _call(case) == PL_ERR_ARG


def test_no_groups_enqueue_nothing():
    q = bd.PLTriProblems(0, None, None, None, None, 0)
    g = bd.PLTriLineGroups(0, None, None, None, None, 0, None, None, None, 0)
    assert bd._tri_lib().pl_lsd_triangulate_dev(None, None, C.byref(q), None, None, None, C.byref(g), None, None, None, None, None) == 0


# ------------------------------------------------------------------------------------------------------------ cv2 pins
def _cv2():
    return pytest.importorskip("cv2")


def _kmat(rng):
    return np.array([[rng.uniform(300, 900), 0, rng.uniform(200, 400)], [0, rng.uniform(300, 900), rng.uniform(150, 300)], [0, 0, 1]], f32)


def test_invert_3x3_is_the_fp64_adjugate():
    cv2 = _cv2()
    rng = np.random.default_rng(1)
    for S in [_kmat(rng) for _ in range(500)] + [rng.normal(size=(3, 3)).astype(f32) for _ in range(500)]:
        _, D = cv2.invert(S, flags=cv2.DECOMP_LU)
        assert np.array_equal(D.view(np.uint32), co.inv3(S).view(np.uint32))


def test_solve_one_column_is_cramer_in_fp64_with_one_fp32_product():
    """cv::solve's n = 3 path rounds bf(1) * Sf(2,2) in fp32; the all-fp64 form differs on most random matrices"""
    cv2 = _cv2()
    rng = np.random.default_rng(2)
    S = np.concatenate([np.stack([_kmat(rng) for _ in range(300)]), rng.normal(size=(2000, 3, 3)).astype(f32)])
    b = np.concatenate([np.stack([rng.uniform(0, 640, 300), rng.uniform(0, 480, 300), np.ones(300)], 1),
                        rng.normal(size=(2000, 3))]).astype(f32)
    got = co.solve3(S, b)
    ref = np.stack([cv2.solve(S[i], b[i].reshape(3, 1), flags=cv2.DECOMP_LU)[1].ravel() for i in range(len(S))])
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    d = S[300:]
    m = lambda i, j: d[:, i, j].astype(f64)
    r = 1.0 / co.det3(d)
    B = b[300:].astype(f64)
    t1 = (r * (m(0, 0) * (B[:, 1] * m(2, 2) - m(1, 2) * B[:, 2]) - B[:, 0] * (m(1, 0) * m(2, 2) - m(1, 2) * m(2, 0))
               + m(0, 2) * (m(1, 0) * B[:, 2] - B[:, 1] * m(2, 0)))).astype(f32)
    assert (t1 != ref[300:, 1]).mean() > 0.05


def test_solve_three_columns_is_fp32_lu():
    cv2 = _cv2()
    rng = np.random.default_rng(3)
    for i in range(600):
        A = np.ascontiguousarray(_kmat(rng).T) if i % 2 else rng.normal(size=(3, 3)).astype(f32)
        B = rng.normal(size=(3, 3)).astype(f32)
        assert np.array_equal(cv2.solve(A, B, flags=cv2.DECOMP_LU)[1].view(np.uint32), co.lu_solve3(A, B).view(np.uint32))


def test_gemm_orders():
    """A * B (3x3 and 3x4) in fp32 order; klF.t() * M (GEMM_1_T) in fp64; the two differ"""
    cv2 = _cv2()
    rng = np.random.default_rng(4)
    diff = 0
    for _ in range(500):
        A, K = rng.normal(size=(3, 3)).astype(f32), _kmat(rng)
        R, T = rng.normal(size=(3, 3)).astype(f32), rng.normal(size=(3, 4)).astype(f32)
        assert np.array_equal(cv2.gemm(A, R, 1, None, 0), co.gemm33(A, R))
        assert np.array_equal(cv2.gemm(K, T, 1, None, 0), co.gemm33(K, T))
        f = rng.normal(size=(1, 3))
        v = f.astype(f32).reshape(3, 1)
        got = co._klf_row(f, T[None])[0]
        assert np.array_equal(cv2.gemm(v, T, 1, None, 0, flags=cv2.GEMM_1_T).ravel(), got)
        diff += not np.array_equal(got, ((v[0] * T[0] + v[1] * T[1]) + v[2] * T[2]))
    assert diff > 250


def test_norm_of_short_vectors():
    cv2 = _cv2()
    rng = np.random.default_rng(5)
    for n in (2, 3):
        v = rng.normal(size=(300, n)).astype(f32)
        assert all(cv2.norm(v[i].reshape(n, 1)) == np.sqrt(co._dot(v[i:i + 1], v[i:i + 1]))[0] for i in range(300))


# ------------------------------------------------------------------------------------------------------------ the oracle
def _scene_batch(sc=None, kfs=None, sigma=None, median=None):
    sc = sc or cs.scene()
    kfs = kfs or sc["kfs"]
    neigh = cs.searched_neighbours()
    probs = [(0, j) for j in neigh]
    k = bd.pack_tri_keyframes(kfs, lines=True)
    q = bd.pack_tri_problems(probs, k["n"])
    ms = [cs.truth_matches(sc, 0, j) for j in neigh]
    nm = np.array([(m >= 0).sum() for m in ms], np.int32)
    g = cs.group(sc, {j: p for p, j in enumerate(neigh)})
    if median is not None:
        g["entries"] = [(p, r, median) for p, r, _ in g["entries"]]
    gr = bd.pack_tri_line_groups([g], k["n"])
    return k, q, gr, np.concatenate(ms), nm, np.zeros(q["P"], np.int32), sc["level_sigma2_line"] if sigma is None else sigma


def test_oracle_on_the_scene_and_its_mutants():
    a = _scene_batch()
    code, L, nnew, st = co.triangulate_lines(*a)
    assert st.tolist() == [0] and nnew[0] == (code == co.COMMITTED).sum() > 10
    assert np.isfinite(L[code == co.COMMITTED]).all()
    assert {-1, 0, 1, 2, 3, 5, 7, 8} <= set(code.tolist())
    for kw in (dict(positional=False), dict(commit_state=False), dict(snapshot=False)):
        assert not np.array_equal(co.triangulate_lines(*a, **kw)[0], code), kw


def test_crafted_variants_reach_the_later_gates():
    sc = cs.scene()
    codes = set(co.triangulate_lines(*_scene_batch(sc))[0].tolist())
    # a small median depth: segments too long (9)
    codes |= set(co.triangulate_lines(*_scene_batch(sc, median=0.4))[0].tolist())
    # the triples of entries 0 and 1 (neighbours 1 and 2, whose matches and positional keyframes agree) reach the last gates.  Octave 1 with a tiny sigma in one of them (12, 13); its keylines shortened along
    # themselves, line functions kept (15, 16)
    for v in (1, 2):
        kfs = [dict(k, keylines=k["keylines"].copy()) for k in sc["kfs"]]
        for i, k in enumerate(kfs):
            k["keylines"]["octave"] = 1 if i == v else 0
        codes |= set(co.triangulate_lines(*_scene_batch(sc, kfs, sigma=np.array([1.0, 1e-9], f32)))[0].tolist())
        kfs = [dict(k, keylines=k["keylines"].copy()) for k in sc["kfs"]]
        kl = kfs[v]["keylines"]
        for a, b in (("startPointX", "endPointX"), ("startPointY", "endPointY")):
            kl[a] = kl[a] + f32(0.45) * (kl[b] - kl[a])
        codes |= set(co.triangulate_lines(*_scene_batch(sc, kfs))[0].tolist())
    # the current keyframe's angle field turned to the other axis (14)
    kfs = [dict(k, keylines=k["keylines"].copy()) for k in sc["kfs"]]
    kl0 = kfs[0]["keylines"]
    kl0["angle"] = np.where(np.abs(kl0["angle"]) > np.pi / 4, f32(0), f32(1.2))
    codes |= set(co.triangulate_lines(*_scene_batch(sc, kfs))[0].tolist())
    # a current keyframe keyline with equal end points: L1 = 0 (4)
    kfs = [dict(k, keylines=k["keylines"].copy()) for k in sc["kfs"]]
    kl0 = kfs[0]["keylines"]
    kl0["endPointX"], kl0["endPointY"] = kl0["startPointX"], kl0["startPointY"]
    codes |= set(co.triangulate_lines(*_scene_batch(sc, kfs))[0].tolist())
    assert {4, 9, 10, 11, 12, 13, 14, 15, 16} <= codes, sorted(codes)


# ------------------------------------------------------------------------------------------------------------ the reference's loop
def _fixture_oracle(**kw):
    import cnml_fixture as cf
    s = cf.load()
    kfs = cf.keyframes(s)
    k = bd.pack_tri_keyframes(kfs, lines=True)
    q = bd.pack_tri_problems(cf.problems(s), k["n"])
    gr = bd.pack_tri_line_groups([cf.group(s)], k["n"])
    code, L, nnew, st = co.triangulate_lines(k, q, gr, s["ref_matches"], s["ref_nmatches"], np.zeros(q["P"], np.int32),
                                             s["level_sigma2_line"], **kw)
    n = int(k["n"][0])
    rows, L = cf.created(code, L, n, q["P"], lambda e: s["ref_matches"][q["out_offset"][e]:q["out_offset"][e] + n])
    return s, rows, L, code


def test_oracle_reproduces_the_reference_loop():
    """tools/gen_create_new_map_lines.py ran the reference's searches and its :966-1439 loop with cv2"""
    s, rows, L, code = _fixture_oracle()
    assert len(s["ref_new"]) > 20
    assert np.array_equal(rows, s["ref_new"])
    assert np.array_equal(L.view(np.uint32), s["ref_line3D"].view(np.uint32))
    assert (code == co.TAKEN).any()


@pytest.mark.parametrize("mutant", [dict(positional=False), dict(commit_state=False)])
def test_oracle_mutants_miss_the_reference_loop(mutant):
    s, rows, L, _ = _fixture_oracle(**mutant)
    assert not (np.array_equal(rows, s["ref_new"]) and np.array_equal(L.view(np.uint32), s["ref_line3D"].view(np.uint32)))


def test_knife_edge_and_degenerate_batches_reach_their_codes():
    """the batches of tests/test_triangulate_lines_gpu.py: view-1 reprojection at one rounding of 3.84 sigma^2 (11 and 0), and a
    triangulation matrix whose vt.row(3) has a zero fourth component (6)"""
    sc = cs.scene()
    kfs, m, s2 = cs.knife_edge(sc)
    k = bd.pack_tri_keyframes(kfs, lines=True)
    q = bd.pack_tri_problems([(0, 1), (0, 2)], k["n"])
    gr = bd.pack_tri_line_groups([dict(kf_cur=0, entries=[(0, 1, sc["medians"][1]), (1, 2, f32(0.05))])], k["n"])
    nm = (m >= 0).sum(1).astype(np.int32)
    c = co.triangulate_lines(k, q, gr, m.reshape(-1), nm, np.zeros(2, np.int32), s2)[0]
    assert (c == co.REPROJ1).sum() > 10 and (c == co.REPROJ2).any() and (c == co.REPROJ3).any() and (c == co.COMMITTED).sum() > 3 and (c == co.EPIPOLAR).any()
    d = cs.degenerate_svd(sc)
    k = bd.pack_tri_keyframes(d, lines=True)
    q = bd.pack_tri_problems([(0, 1), (0, 2)], k["n"])
    gr = bd.pack_tri_line_groups([dict(kf_cur=0, entries=[(0, 1, 5.0), (1, 2, 5.0)])], k["n"])
    c = co.triangulate_lines(k, q, gr, np.zeros(2, np.int32), np.ones(2, np.int32), np.zeros(2, np.int32), np.ones(1, f32))[0]
    assert c.tolist() == [co.W_ZERO]


def test_no_float_angle_lies_between_the_pi_and_m_pi_bounds():
    """The overlap axis compares fabs(angle), a float, with 3.0*PI/4.0 and 1.0*PI/4.0 in double, PI = 3.1415926.  No float lies
    between those bounds and the M_PI ones, so writing M_PI there changes no decision: the mutant is equivalent."""
    for k in (1.0, 3.0):
        a, b = sorted((k * 3.1415926 / 4.0, k * np.pi / 4.0))
        lo = f32(a)
        for x in (np.nextafter(lo, f32(-1)), lo, np.nextafter(lo, f32(9))):
            assert not (a < float(x) < b) and float(x) not in (a, b)
