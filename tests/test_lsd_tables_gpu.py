"""What LSD region growing reads that no input changes, read back from a line handle and checked on every argument, and the
sure / maybe alignment shortcut of region_grow checked against its own exact test.

A frame reaches a few thousand gradients and a few hundred thousand alignment decisions, and a last-bit error in either almost
never moves a segment, so the frame tests (test_line_gpu.py, test_lsd_front_gpu.py) cannot see one.  Here:
  - the gradient table: all 1021 x 1021 records {fastAtan2 degrees, cosf, sinf} and seed (cos, sin), bit for bit against a host
    reference (the oracle's fastAtan2, pinned to cv2; the C library's cosf / sinf of float(angle) and fp64 cos / sin of the
    angle, lsd.cpp's arithmetic);
  - the weight table sqrt(i / 4) on all its 520,201 entries;
  - the shortcut (pl_debug_lsd_align_dev runs region_grow's own decision code with the handle's constants and table): never
    "surely aligned" where the exact test says not aligned, never "surely not" where it says aligned, on 1e8 sums in the
    +-0.05 degree band around 22.5 degrees from the candidate (and from its opposite), every reachable gradient among them;
  - the exact test's prec_hi fold against the generic isAligned on the float angle pairs whose difference is near 2 pi."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import plslam_b200 as pl
from oracle import binding as ob
from test_libm_glibc import _glibc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R, N = 510, 1021
NW = 2 * R * R + 1
f32 = np.float32
PREC_DEG = 22.5
BAND_DEG = 0.05                  # the shortcut's margin M: the band it must leave to the exact test
RHO2 = 4 * (2.0 / np.sin(np.pi * PREC_DEG / 180)) ** 2     # a gradient is defined iff gx^2 + gy^2 > RHO2


@pytest.fixture(scope="module")
def line():
    return pl.LINEextractor(width=640, height=480)


@pytest.fixture(scope="module")
def host_ref(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lsdtab") / "liblsd_tables_ref.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++",
                           os.path.join(ROOT, "tests", "host", "lsd_tables_ref.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.lsd_table_ref.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_void_p]
    return lib


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _tables(line):
    L = pl.lib()
    L.pl_line_debug_tables.argtypes = [C.c_void_p] * 4
    g = np.zeros((N * N, 4), f32); s = np.zeros((N * N, 2), f32); w = np.zeros(NW, np.float64)
    pl.check(L.pl_line_debug_tables(line._h, g.ctypes.data, s.ctypes.data, w.ctypes.data))
    return g, s, w


def _grid():
    """gx, gy of every table index (gx + 510) * 1021 + gy + 510"""
    i = np.arange(N * N)
    return i // N - R, i % N - R


def test_gradient_table_equals_reference_arithmetic(line, host_ref):
    g, s, _ = _tables(line)
    gx, gy = _grid()
    fa = ob.lib().oracle_fast_atan2
    deg = np.array([fa(float(x), float(-y)) for x, y in zip(gx, gy)], f32)
    rec = np.zeros((N * N, 4), f32); seed = np.zeros((N * N, 2), f32)
    host_ref.lsd_table_ref(deg.ctypes.data, N * N, rec.ctypes.data, seed.ctypes.data)
    reach = ((gx - gy) % 2 == 0) & (gx * gx + gy * gy > RHO2)      # the gradients a 2x2 window can have, defined
    assert reach.sum() == 521_044
    bad = {"deg": _bits(g[:, 0]) != _bits(rec[:, 0]), "cos": _bits(g[:, 1]) != _bits(rec[:, 1]),
           "sin": _bits(g[:, 2]) != _bits(rec[:, 2]), "pad": _bits(g[:, 3]) != 0,
           "seed cos": _bits(s[:, 0]) != _bits(seed[:, 0]), "seed sin": _bits(s[:, 1]) != _bits(seed[:, 1])}
    counts = {k: (int(v.sum()), int((v & reach).sum())) for k, v in bad.items() if v.any()}
    # only the cos / sin columns come from the glibc 2.39 restatement; the angle, the pad and the seed do not depend on the C library
    if counts and not _glibc().startswith("2.39") and set(counts) <= {"cos", "sin"}:
        pytest.skip(f"glibc {_glibc()} computes cosf / sinf differently from the 2.39 the device restatement follows: {counts}")
    assert not counts, f"table entries that differ from the reference (all, reachable) of {N * N}: {counts}"


def test_weight_table_is_sqrt_of_quarter(line):
    _, _, w = _tables(line)
    ref = np.sqrt(np.arange(NW) / 4.0)
    assert (w.view(np.uint64) != ref.view(np.uint64)).sum() == 0


def _align(line, sx, sy, gx, gy):
    L = pl.lib()
    L.pl_debug_lsd_align_dev.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 6
    out = torch.empty(len(sx), dtype=torch.uint8, device="cuda")
    _launch(L.pl_debug_lsd_align_dev, line._h, len(sx), sx.data_ptr(), sy.data_ptr(), gx.data_ptr(), gy.data_ptr(), out.data_ptr())
    return out


def _launch(fn, *args):
    """an entry point on the handle's own stream (non-blocking: it does not order itself after torch's default stream), so the
    inputs are complete before it and its output after it"""
    torch.cuda.synchronize()
    pl.check(fn(*args, None))
    torch.cuda.synchronize()


def _violations(out):
    """(sure but not aligned, aligned but not maybe, fold != generic, aligned cases, cases in the band: maybe and not sure);
    every case must name a gradient of the table"""
    sure, maybe, exact, generic, outside = ((out >> k) & 1 for k in range(5))
    assert int(outside.sum()) == 0
    return torch.stack([(sure & (1 - exact)).sum(), (exact & (1 - maybe)).sum(), (exact != generic).sum(), exact.sum(),
                        (maybe & (1 - sure)).sum()]).cpu().numpy()


def _reachable(gen, n):
    """n random gradients a 2x2 window can have (gx = gy mod 2), defined (gx^2 + gy^2 > rho^2 * 4)"""
    gx = torch.randint(-R, R + 1, (2 * n,), device="cuda", generator=gen)
    gy = torch.randint(-R, R + 1, (2 * n,), device="cuda", generator=gen)
    gy = torch.where((gx - gy) % 2 == 0, gy, torch.where(gy < R, gy + 1, gy - 1))
    ok = (gx * gx + gy * gy).double() > RHO2
    return gx[ok][:n].int(), gy[ok][:n].int()


def _sums_around(gen, gx, gy, mag_lo=1.0, mag_hi=1e5):
    """float sums at 22.5 +- 0.05 degrees from the candidate's direction, either side, a quarter of them around its opposite,
    |sum| log-uniform in [mag_lo, mag_hi]"""
    n = len(gx)
    a = torch.atan2(gx.double(), -gy.double())         # the candidate's level-line direction (-gy, gx): the record's cos / sin
    side = torch.where(torch.rand(n, device="cuda", generator=gen, dtype=torch.float64) < 0.5, -1.0, 1.0)
    d = PREC_DEG + BAND_DEG * (2 * torch.rand(n, device="cuda", generator=gen, dtype=torch.float64) - 1)
    flip = torch.rand(n, device="cuda", generator=gen, dtype=torch.float64) < 0.25
    th = a + side * torch.deg2rad(d) + torch.where(flip, np.pi, 0.0)
    m = torch.exp(np.log(mag_lo) + (np.log(mag_hi) - np.log(mag_lo)) * torch.rand(n, device="cuda", generator=gen, dtype=torch.float64))
    return (m * torch.cos(th)).float(), (m * torch.sin(th)).float()


def test_alignment_shortcut_never_contradicts_the_exact_test(line):
    """1e8 decisions: every reachable gradient at 16 sums around it, then random gradients and sums; the band is where the
    shortcut must defer to the exact test"""
    gen = torch.Generator(device="cuda"); gen.manual_seed(2026)
    tot = np.zeros(5, np.int64)
    n = 0
    # every reachable gradient, 16 sums each
    gx0, gy0 = (torch.from_numpy(v) for v in _grid())
    ok = ((gx0 - gy0) % 2 == 0) & ((gx0 * gx0 + gy0 * gy0).double() > RHO2)
    gx0, gy0 = gx0[ok].int().cuda().repeat(16), gy0[ok].int().cuda().repeat(16)
    assert len(gx0) == 16 * 521_044
    sx, sy = _sums_around(gen, gx0, gy0)
    tot += _violations(_align(line, sx, sy, gx0, gy0)); n += len(sx)
    chunk = 10_000_000
    while n < 100_000_000:
        gx, gy = _reachable(gen, chunk)
        sx, sy = _sums_around(gen, gx, gy)
        tot += _violations(_align(line, sx, sy, gx, gy)); n += len(sx)
    sure_bad, maybe_bad, fold_bad, aligned, band = tot.tolist()
    # the sums sit uniformly within +-0.05 degrees of the threshold, so with the margin M = 0.05 degrees about 3/4 of them (all but
    # the opposite-facing quarter) must fall in the band the shortcut leaves to the exact test: a narrower margin fails here
    assert n >= 100_000_000 and 0.1 * n < aligned < 0.9 * n, (n, aligned)
    assert band > 0.2 * n, f"only {band} of {n} sums within 0.05 degrees of the threshold are left to the exact test: the margin is not 0.05 degrees"
    assert sure_bad == 0 and maybe_bad == 0, f"of {n}: {sure_bad} 'surely aligned' that are not, {maybe_bad} aligned not 'maybe'"
    assert fold_bad == 0


def test_alignment_shortcut_on_accumulated_sums(line, host_ref):
    """sums built as region_grow builds them: a seed's unit vector plus up to 255 table records of gradients within 22.5
    degrees of it, added in fp32; candidates near 22.5 degrees from the sum, on either side and opposite"""
    rng = np.random.default_rng(7)
    g, s, _ = _tables(line)
    gx0, gy0 = _grid()
    reach = np.flatnonzero(((gx0 - gy0) % 2 == 0) & (gx0 * gx0 + gy0 * gy0 > RHO2))
    n, steps = 1 << 20, 255
    seed = rng.choice(reach, n)
    sx, sy = s[seed, 0].copy(), s[seed, 1].copy()
    base = np.arctan2(gx0[seed], -gy0[seed])
    k = rng.integers(0, steps + 1, n)
    for t in range(steps):
        # a gradient whose level line is within 20 degrees of the seed's, magnitude 6 .. 360
        th = base + np.deg2rad(rng.uniform(-20, 20, n))
        r = rng.uniform(6, 360, n)
        ax, ay = np.rint(r * np.sin(th)).astype(np.int64), np.rint(-r * np.cos(th)).astype(np.int64)
        ay += (ax - ay) % 2
        idx = (np.clip(ax, -R, R) + R) * N + np.clip(ay, -R, R) + R
        on = t < k
        sx = np.where(on, sx + g[idx, 1], sx).astype(f32)
        sy = np.where(on, sy + g[idx, 2], sy).astype(f32)
    mag = np.hypot(sx.astype(np.float64), sy.astype(np.float64))
    assert mag.min() > 0.999 and mag.max() > 100
    phi = np.arctan2(sy.astype(np.float64), sx.astype(np.float64))
    cases = []
    for off in (PREC_DEG, -PREC_DEG, 180 - PREC_DEG, 180 + PREC_DEG):
        for r in (120.0, 250.0, 505.0):
            th = phi + np.deg2rad(off + rng.uniform(-BAND_DEG, BAND_DEG, n))
            cx, cy = np.rint(r * np.sin(th)).astype(np.int64), np.rint(-r * np.cos(th)).astype(np.int64)
            cx = np.clip(cx + (cx - cy) % 2, -R, R)
            cases.append((cx, cy))
    cx = np.concatenate([c[0] for c in cases]); cy = np.concatenate([c[1] for c in cases])
    reps = len(cases)
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).astype(dt)).cuda()
    out = _align(line, t(np.tile(sx, reps), np.float32), t(np.tile(sy, reps), np.float32), t(cx, np.int32), t(cy, np.int32))
    sure_bad, maybe_bad, fold_bad, aligned, band = _violations(out).tolist()
    assert band > 0.05 * len(cx) and aligned > 0.1 * len(cx), (aligned, band)
    assert sure_bad == 0 and maybe_bad == 0 and fold_bad == 0, (sure_bad, maybe_bad, fold_bad)


def test_prec_hi_fold_equals_generic_is_aligned_near_two_pi(line):
    """the exact test folds isAligned's  n > 3pi/2 ? |n - 2pi| : n  <= prec  into  n <= prec || n >= prec_hi; for every table
    angle within 22.5 degrees of 0 / 360 and the 64 float region angles either side of it + / - 337.5 degrees, both forms agree"""
    g, _, _ = _tables(line)
    deg = np.unique(g[:, 0])
    lo, hi = deg[deg <= 23.0], deg[deg >= 337.0]
    a = np.concatenate([lo, hi])
    centre = np.concatenate([(lo.astype(np.float64) + 337.5), (hi.astype(np.float64) - 337.5)]).astype(f32)
    k = np.arange(-64, 65)
    bits = centre.view(np.int32)[:, None] + k[None, :]
    reg = bits.astype(np.int32).view(f32).ravel()
    cand = np.repeat(a, len(k))
    L = pl.lib()
    L.pl_debug_lsd_fold_dev.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 4
    dr, dc = torch.from_numpy(reg).cuda(), torch.from_numpy(cand).cuda()
    out = torch.empty(len(reg), dtype=torch.uint8, device="cuda")
    _launch(L.pl_debug_lsd_fold_dev, line._h, len(reg), dr.data_ptr(), dc.data_ptr(), out.data_ptr())
    o = out.cpu().numpy()
    fold, generic = o & 1, (o >> 1) & 1
    assert len(reg) > 1_000_000 and 0 < fold.sum() < len(reg)
    assert (fold != generic).sum() == 0, f"{(fold != generic).sum()} of {len(reg)} angle pairs"


def test_alignment_entry_flags_gradients_outside_the_table(line):
    """a gradient outside [-510, 510]^2 reads the clamped table entry and is flagged, never read past the table"""
    gx = torch.tensor([511, -511, 0, 510, 4000], dtype=torch.int32, device="cuda")
    gy = torch.tensor([0, 0, -600, 510, -4000], dtype=torch.int32, device="cuda")
    one = torch.ones(5, dtype=torch.float32, device="cuda")
    out = _align(line, one, one, gx, gy).cpu().numpy()
    assert ((out >> 4) & 1).tolist() == [1, 1, 1, 0, 1]
