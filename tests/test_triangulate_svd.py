"""The arithmetic of pl_orb_triangulate_dev against cv2, without a GPU: cv::SVD::compute for 4x4 CV_32F matrices as the oracle
(tests/cnmp_oracle.py) and the device header (pl-slam_b200/csrc/svd4.cuh, compiled here for the host) restate it, bit for bit in w
and the whole of vt, on tests/golden/orb_cv2_svd4.npz (tools/gen_svd4_cv2.py) and live on fresh matrices where cv2 imports, including matrices
on which OpenCV's own hypot and the C library's give different results; and the fp64 form of MatExpr's  s * M1 - M2."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cnmp_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "orb_cv2_svd4.npz")


def _fixture():
    with np.load(FIXTURE) as z:
        return z["A"], z["w"], z["vt"]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def host_svd4(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("svd4") / "libsvd4.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++",
                           os.path.join(ROOT, "tests", "host", "svd4_host.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.svd4_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]

    def run(A):
        A = np.ascontiguousarray(A, np.float32).reshape(-1, 4, 4)
        w = np.zeros((len(A), 4), np.float32); vt = np.zeros((len(A), 4, 4), np.float32)
        lib.svd4_batch(A.ctypes.data, len(A), w.ctypes.data, vt.ctypes.data)
        return w, vt
    return run


def test_fixture_families():
    A, w, vt = _fixture()
    assert len(A) >= 3000
    assert (w[:, 3] == 0).any() and (np.abs(A).max((1, 2)) == 0).any(), "rank-deficient and zero matrices"


def test_oracle_svd_equals_cv2_on_the_fixture():
    A, w, vt = _fixture()
    ow, ovt = co.svd4(A)
    assert np.array_equal(_bits(ow), _bits(w))
    assert np.array_equal(_bits(ovt), _bits(vt))


def test_device_header_svd_equals_cv2_on_the_fixture(host_svd4):
    A, w, vt = _fixture()
    hw, hvt = host_svd4(A)
    assert np.array_equal(_bits(hw), _bits(w))
    assert np.array_equal(_bits(hvt), _bits(vt))


def test_svd_equals_live_cv2(host_svd4):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(2024)
    n = 100000
    A = np.concatenate([co.triangulation_matrices(rng, n // 2),
                        (rng.normal(size=(n // 2, 4, 4)) * 10.0 ** rng.uniform(-4, 4, (n // 2, 1, 1))).astype(np.float32)])
    w = np.zeros((n, 4), np.float32); vt = np.zeros((n, 4, 4), np.float32)
    for i in range(n):
        a, _, v = cv2.SVDecomp(A[i].copy(), flags=cv2.SVD_MODIFY_A | cv2.SVD_FULL_UV)
        w[i], vt[i] = a.ravel(), v
    ow, ovt = co.svd4(A)
    hw, hvt = host_svd4(A)
    for x, y in ((ow, w), (ovt, vt), (hw, w), (hvt, vt)):
        assert np.array_equal(_bits(x), _bits(y))


def test_u_is_not_needed():
    """FULL_UV's completion of zero singular values touches U only: w and vt of a rank-deficient matrix are the same with and
    without FULL_UV, so a restatement that never forms U loses nothing the reference reads."""
    cv2 = pytest.importorskip("cv2")
    A, _, _ = _fixture()
    for M in A[-500:]:
        w1, _, vt1 = cv2.SVDecomp(M.copy(), flags=cv2.SVD_MODIFY_A | cv2.SVD_FULL_UV)
        w2, _, vt2 = cv2.SVDecomp(M.copy(), flags=cv2.SVD_MODIFY_A)
        assert np.array_equal(_bits(w1), _bits(w2)) and np.array_equal(_bits(vt1), _bits(vt2))


def test_addweighted_is_fp64_with_one_rounding():
    """cv::MatExpr  s * M1 - M2  on CV_32F rows (the rows of A) goes through addWeighted, which forms s * a - b + 0 in fp64 and
    rounds once: (1 + 2^-12)^2 + 2^-60 rounds to even in fp32 after fp64 (an FMA would round up), and random rows differ from
    the separately rounded fp32 form."""
    cv2 = pytest.importorskip("cv2")
    x = np.float32(1 + 2 ** -12)
    r = cv2.addWeighted(np.full((1, 4), x, np.float32), float(x), np.full((1, 4), -2.0 ** -60, np.float32), -1.0, 0.0)
    assert (r == np.float32(1 + 2 ** -11)).all()
    rng = np.random.default_rng(5)
    s = rng.normal(size=3000).astype(np.float32); a = rng.normal(size=(3000, 4)).astype(np.float32); b = rng.normal(size=(3000, 4)).astype(np.float32)
    cv = np.concatenate([cv2.addWeighted(a[i:i + 1], float(s[i]), b[i:i + 1], -1.0, 0.0) for i in range(3000)])
    assert np.array_equal(_bits(cv), _bits(co._addw(s, a, b)))
    assert not np.array_equal(_bits(cv), _bits(s[:, None] * a - b))


def test_fixture_tells_the_two_hypots_apart():
    """cv::SVD's Jacobi takes gamma from OpenCV's own hypot template, not from the C library's hypot.  The fixture's last matrices
    (tools/svd4_hypot_search.cpp) are ones on which the two give different vt: with the C library's hypot the oracle's SVD
    differs from cv2 on every one of them, with OpenCV's it equals cv2."""
    with np.load(FIXTURE) as z:
        h = int(z["n_hypot"]); A, vt = z["A"][-h:], z["vt"][-h:]
    assert h >= 5
    assert np.array_equal(_bits(co.svd4(A)[1]), _bits(vt))
    libm = co.cv_hypot
    try:
        co.cv_hypot = np.hypot
        other = co.svd4(A)[1]
    finally:
        co.cv_hypot = libm
    assert (_bits(other) != _bits(vt)).reshape(h, -1).any(1).all()
    assert (_bits(other[:, 3]) != _bits(vt[:, 3])).any(1).sum() >= 3, "vt.row(3), the row the triangulation reads"


def test_hypot_is_opencvs_formula():
    """cv_hypot against the formula on values where it and the C library's hypot disagree in the last bit"""
    rng = np.random.default_rng(7)
    a, b = rng.normal(size=200000) * 10.0 ** rng.uniform(-3, 3, 200000), rng.normal(size=200000)
    h = co.cv_hypot(a, b)
    x, y = np.abs(a), np.abs(b)
    ref = np.where(x > y, x * np.sqrt(1 + (y / x) ** 2), y * np.sqrt(1 + (x / y) ** 2))
    assert np.array_equal(h, ref) and (h != np.hypot(a, b)).any()
    assert co.cv_hypot(np.zeros(1), np.zeros(1))[0] == 0
