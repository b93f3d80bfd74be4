"""The library's own device build of the float libm restatements (pl-slam_b200/csrc/libm_glibc.cuh) and of the 4x4 SVD
(svd4.cuh), through the test-only entry points pl_debug_float_math_dev and pl_debug_svd4_dev, bit for bit against the host build
of the same headers, the C library and cv2.

The host tests (tests/test_libm_glibc.py, tests/test_triangulate_svd.py) prove the headers compiled by g++; the device objects are
another compilation whose exactness rests on the library's flags (-fmad=false keeps atanf_'s fp32 products and sums apart) and on
the device intrinsics svd4 is written in.  A frame reaches a few thousand angles and triangulations, too few to meet the
arguments that decide a last bit, so these tests take the host check's 2e7 libm arguments (tests/host/libm_args.h) and the SVD
fixture's zero, rank-deficient and hypot-discriminating matrices, plus 1e6 fresh triangulation-shaped and Gaussian matrices."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import plslam_b200 as pl
import cnmp_oracle as co
from cnml_oracle import _klf_row
from test_libm_glibc import _glibc
from test_triangulate_svd import FIXTURE, _bits, host_svd4  # noqa: F401  (host_svd4: the host build of svd4.cuh, a fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32

N_LIBM = 20_000_000           # the host check's count (tests/test_libm_glibc.py)
CHUNK = 2_000_000             # cases per round trip: 64 MB of host records
LIBM_CASE = np.dtype([(k, "<f4") for k in ("y", "x", "atan2", "t", "sin", "cos", "q", "log")])   # LibmCase
FNS = {"atan2f": 0, "sincosf": 1, "logf": 2}


@pytest.fixture(scope="module")
def host_libm(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("libm") / "liblibm_args.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-mfma", "-fPIC", "-shared", "-x", "c++",
                           os.path.join(ROOT, "tests", "host", "libm_args.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.libm_cases.restype = C.c_long
    lib.libm_cases.argtypes = [C.POINTER(C.c_uint64), C.c_long, C.c_long, C.c_void_p]
    lib.libm_header.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_void_p]
    return lib


def _libm_chunks(lib):
    """the 2e7 cases of the host check, CHUNK at a time"""
    st = C.c_uint64(0)
    buf = np.zeros(CHUNK, LIBM_CASE)
    for i0 in range(0, N_LIBM, CHUNK):
        m = lib.libm_cases(C.byref(st), i0, min(CHUNK, N_LIBM - i0), buf.ctypes.data)
        yield buf[:m]


def _dev_math(fn, a, b=None):
    L = pl.lib()
    L.pl_debug_float_math_dev.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    da = torch.from_numpy(a).cuda()
    db = torch.from_numpy(b).cuda() if b is not None else None
    o0 = torch.empty_like(da)
    o1 = torch.empty_like(da) if fn == 1 else None
    pl.check(L.pl_debug_float_math_dev(fn, da.data_ptr(), db.data_ptr() if db is not None else None, len(a), o0.data_ptr(),
                                       o1.data_ptr() if o1 is not None else None, torch.cuda.current_stream().cuda_stream))
    return [o.cpu().numpy() for o in (o0, o1) if o is not None]


def _host_math(lib, fn, a, b=None):
    out = [np.zeros(len(a), f32) for _ in range(2 if fn == 1 else 1)]
    lib.libm_header(fn, a.ctypes.data, b.ctypes.data if b is not None else None, len(a), out[0].ctypes.data,
                    out[1].ctypes.data if fn == 1 else None)
    return out


def _dev_svd4(A):
    L = pl.lib()
    L.pl_debug_svd4_dev.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    dA = torch.from_numpy(np.ascontiguousarray(A, f32).reshape(-1, 16)).cuda()
    w = torch.empty((len(dA), 4), dtype=torch.float32, device="cuda")
    vt = torch.empty((len(dA), 4, 4), dtype=torch.float32, device="cuda")
    pl.check(L.pl_debug_svd4_dev(dA.data_ptr(), len(dA), w.data_ptr(), vt.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return w.cpu().numpy(), vt.cpu().numpy()


def _differing(x, y):
    """number of matrices (rows of the leading axis) whose bits differ anywhere"""
    return int((_bits(x) != _bits(y)).reshape(len(x), -1).any(1).sum())


@pytest.mark.parametrize("name", list(FNS))
def test_libm_device_equals_host_header_and_c_library(host_libm, name):
    fn = FNS[name]
    bytes0, launches0 = pl.device_bytes(), pl.launch_count()
    n = vs_header = vs_libm = 0
    for c in _libm_chunks(host_libm):
        n += len(c)
        if fn == 0:
            args, libm = (c["y"].copy(), c["x"].copy()), (c["atan2"],)
        elif fn == 1:
            args, libm = (c["t"].copy(),), (c["sin"], c["cos"])
            assert (np.abs(args[0]) < 120).all()
        else:
            args, libm = (c["q"].copy(),), (c["log"],)
            assert (np.isfinite(args[0]) & (args[0] >= np.finfo(f32).tiny)).all(), "positive normals only"
        dev, host = _dev_math(fn, *args), _host_math(host_libm, fn, *args)
        vs_header += sum(int((_bits(d) != _bits(h)).sum()) for d, h in zip(dev, host))
        vs_libm += sum(int((_bits(d) != _bits(r)).sum()) for d, r in zip(dev, libm))
    assert n == N_LIBM
    assert pl.launch_count() - launches0 == N_LIBM // CHUNK and pl.device_bytes() == bytes0
    assert vs_header == 0, f"{name}: the device build differs from the host build of libm_glibc.cuh on {vs_header} of {n} results"
    if vs_libm and not _glibc().startswith("2.39"):
        pytest.skip(f"glibc {_glibc()} computes {name} differently from the 2.39 the restatement follows ({vs_libm} results)")
    assert vs_libm == 0, f"{name}: the device build differs from the C library on {vs_libm} of {n} results"


def test_svd4_device_equals_cv2_on_the_fixture():
    """all of tests/golden/orb_cv2_svd4.npz: w and the whole of vt equal cv2.SVDecomp's bits, on the zero and rank-deficient
    matrices and on the last n_hypot, where OpenCV's hypot and the C library's give different vt"""
    with np.load(FIXTURE) as z:
        A, w, vt, h = z["A"], z["w"], z["vt"], int(z["n_hypot"])
    assert len(A) == 4005 and h >= 5
    bytes0 = pl.device_bytes()
    dw, dvt = _dev_svd4(A)
    assert pl.device_bytes() == bytes0
    bad = (_bits(dw) != _bits(w)).any(1) | (_bits(dvt) != _bits(vt)).reshape(len(A), -1).any(1)
    assert not bad.any(), f"{bad.sum()} of {len(A)} matrices differ from cv2, {bad[-h:].sum()} of the {h} hypot-discriminating ones"


def _rot(a):
    """R = Rz Ry Rx for angles a [n][3] (fp64)"""
    c, s = np.cos(a), np.sin(a)
    o, z = np.ones(len(a)), np.zeros(len(a))
    Rx = np.stack([o, z, z, z, c[:, 0], -s[:, 0], z, s[:, 0], c[:, 0]], 1).reshape(-1, 3, 3)
    Ry = np.stack([c[:, 1], z, s[:, 1], z, o, z, -s[:, 1], z, c[:, 1]], 1).reshape(-1, 3, 3)
    Rz = np.stack([c[:, 2], -s[:, 2], z, s[:, 2], c[:, 2], z, z, z, o], 1).reshape(-1, 3, 3)
    return Rz @ Ry @ Rx


def line_triangulation_matrices(rng, n):
    """n end-point matrices A of LocalMapping::CreateNewMapLinesConstraint, built as cnml_oracle.gates builds them: the rows
    klF.t() * M3, klF.t() * M2 of the segment's keylines in two other keyframes (line functions as Frame forms them), then
    x * M1.row(2) - M1.row(0), y * M1.row(2) - M1.row(1) of its start point in the first.  TUM-like intrinsics, baselines of
    about 0.3 m, segments 3-8 m away, 0.4 px of noise"""
    K = np.array([517.3, 516.5, 318.6, 255.3])
    Kf = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]], f32)
    mid = np.stack([rng.uniform(-2.5, 2.5, n), rng.uniform(-1.8, 1.8, n), rng.uniform(3, 8, n)], 1)
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1)[:, None]
    half = rng.uniform(0.2, 0.8, n)[:, None]
    P = (mid - half * d, mid + half * d)
    M, f, start = [], [], None
    for v in range(3):
        R = _rot(rng.normal(0, 0.04, (n, 3)))
        c = np.zeros((n, 3)) if v == 0 else rng.normal(0, 0.3 / np.sqrt(3), (n, 3))
        t = -np.einsum("nij,nj->ni", R, c)
        ends = []
        for X in P:
            Xc = np.einsum("nij,nj->ni", R, X) + t
            ends.append((K[:2] * Xc[:, :2] / Xc[:, 2:] + K[2:] + rng.normal(0, 0.4, (n, 2))).astype(f32))
        T = np.concatenate([R, t[:, :, None]], 2).astype(f32)
        # K * Tcw.rowRange(0, 3) in cv::gemm's fp32 order
        M.append((Kf[None, :, 0, None] * T[:, None, 0] + Kf[None, :, 1, None] * T[:, None, 1]) + Kf[None, :, 2, None] * T[:, None, 2])
        sp, ep = (np.concatenate([e.astype(np.float64), np.ones((n, 1))], 1) for e in ends)
        lf = np.cross(sp, ep)
        f.append(lf / np.sqrt(lf[:, 0] ** 2 + lf[:, 1] ** 2)[:, None])
        if v == 0:
            start = ends[0]
    return np.stack([_klf_row(f[2], M[2]), _klf_row(f[1], M[1]), co._addw(start[:, 0], M[0][:, 2], M[0][:, 0]),
                     co._addw(start[:, 1], M[0][:, 2], M[0][:, 1])], 1)


def test_svd4_device_equals_host_header_on_fresh_matrices(host_svd4):
    """1e6 matrices the fixture does not hold: point and line triangulation matrices and Gaussian matrices scaled by 1e-4 .. 1e4;
    the device build must equal the host build of svd4.cuh bit for bit"""
    rng = np.random.default_rng(2026)
    families = {"point triangulation": co.triangulation_matrices(rng, 250_000),
                "line triangulation": line_triangulation_matrices(rng, 250_000),
                "scaled Gaussian": (rng.normal(size=(500_000, 4, 4)) * 10.0 ** rng.uniform(-4, 4, (500_000, 1, 1))).astype(f32)}
    bad = {}
    for name, A in families.items():
        assert A.shape[1:] == (4, 4) and np.isfinite(A).all()
        dw, dvt = _dev_svd4(A)
        hw, hvt = host_svd4(A)
        bad[name] = _differing(np.concatenate([dw, dvt.reshape(-1, 16)], 1), np.concatenate([hw, hvt.reshape(-1, 16)], 1))
    assert not any(bad.values()), f"matrices whose device w / vt differ from the host build: {bad}"
