"""GPU parity: line grid (Frame::AssignFeaturesToGridForLine) and the two LSDmatcher::SearchByProjection variants."""
import numpy as np
import pytest
import oracle
import plslam_b200 as pl
from plslam_b200 import synth

pytestmark = pytest.mark.gpu
BOUNDS = [0.0, 0.0, 640.0, 480.0]


@pytest.fixture(scope="module")
def lines():
    f0 = synth.synth_frame(640, 480, 1); f1 = synth.warp_frame(f0, 1001)
    return [oracle.line_extract(f, nfeatures=400) for f in (f0, f1)]


def test_line_grid(lines):
    kl = lines[0][0][:-1]
    s, it = pl.frame_assign_grid_lines(kl, BOUNDS)
    os_, oit = oracle.assign_grid_lines(kl, BOUNDS)
    assert np.array_equal(s, os_) and np.array_equal(it, oit) and len(it) > len(kl)


def _queries(lines, rng, jitter):
    (kl0, d0, lf0), (kl1, d1, lf1) = lines
    kl0, d0 = kl0[:-1], d0[:-1]
    n = len(kl0)
    proj = np.stack([kl0["startPointX"], kl0["startPointY"], kl0["endPointX"], kl0["endPointY"]], 1).astype(np.float32)
    proj += rng.normal(0, jitter, proj.shape).astype(np.float32)
    valid = rng.random(n) < 0.85
    return kl0, d0, proj, valid


@pytest.mark.parametrize("th", [15.0, 40.0])
def test_search_by_projection_last(lines, th):
    rng = np.random.default_rng(3)
    kl0, d0, proj, valid = _queries(lines, rng, 1.5)
    kl1, d1, lf1 = lines[1]
    kl1, d1, lf1 = kl1[:-1], d1[:-1], lf1[:-1]
    pre = (rng.random(len(kl1)) < 0.05).astype(np.uint8)
    a = (kl1, lf1, d1, BOUNDS, valid, proj, d0, kl0["lineLength"], th)
    nm, m = pl.LSDmatcher(0.7).SearchByProjectionLast(*a, preassigned=pre)
    onm, om = oracle.line_search_by_projection_last(*a, preassigned=pre)
    assert onm > 30 and nm == onm and np.array_equal(m, om)


@pytest.mark.parametrize("th", [1.0, 3.0])
def test_search_by_projection_lines(lines, th):
    rng = np.random.default_rng(5)
    kl0, d0, proj, valid = _queries(lines, rng, 1.0)
    kl1, d1, lf1 = lines[1]
    kl1, d1, lf1 = kl1[:-1], d1[:-1], lf1[:-1]
    vc = rng.uniform(0.99, 1.0, len(kl0)).astype(np.float32)
    a = (kl1, lf1, d1, BOUNDS, valid, proj, vc, d0)
    nm, m = pl.LSDmatcher(0.7).SearchByProjectionLines(*a, th=th)
    onm, om = oracle.line_search_by_projection_lines(*a, th, 0.7)
    assert onm > 20 and nm == onm and np.array_equal(m, om)


@pytest.mark.skipif(not oracle.ref_match_available(), reason="oracle/_ref/libref_match.so did not travel")
def test_line_matchers_equal_the_reference_matcher_code(lines):
    """The CUDA line matchers against the REFERENCE's own LSDmatcher.cpp (compiled into oracle/_ref/libref_match.so, run on this box's
    CPU): SearchDouble and the two projection searches, same inputs, identical match lists."""
    d0, d1 = lines[0][1][:-1], lines[1][1][:-1]
    nm, m = pl.LSDmatcher(0.7).SearchDouble(d0, d1)
    rnm, rm = oracle.search_double(d0, d1, 0.7, impl="ref")
    assert rnm > 30 and nm == rnm and np.array_equal(m, rm)
    rng = np.random.default_rng(13)
    kl0, dd0, proj, valid = _queries(lines, rng, 1.5)
    kl1, dd1, lf1 = (x[:-1] for x in lines[1])
    pre = (rng.random(len(kl1)) < 0.05).astype(np.uint8)
    a = (kl1, lf1, dd1, BOUNDS, valid, proj, dd0, kl0["lineLength"], 15.0)
    nm, m = pl.LSDmatcher(0.7).SearchByProjectionLast(*a, preassigned=pre)
    rnm, rm = oracle.line_search_by_projection_last(*a, preassigned=pre, impl="ref")
    assert rnm > 30 and nm == rnm and np.array_equal(m, rm)
    vc = rng.uniform(0.99, 1.0, len(kl0)).astype(np.float32)
    a = (kl1, lf1, dd1, BOUNDS, valid, proj, vc, dd0)
    nm, m = pl.LSDmatcher(0.7).SearchByProjectionLines(*a, th=3.0)
    rnm, rm = oracle.line_search_by_projection_lines(*a, 3.0, 0.7, impl="ref")
    assert rnm > 20 and nm == rnm and np.array_equal(m, rm)


def _crowded_cell_lines(rng):
    """1100 short vertical lines inside grid cell (30, 20) of a 640 x 480 frame, then line X (id 1100, slot 1100 of that cell)
    and line Y (id 1101, slot 0 of cell (30, 21)), both horizontal, 3.5 px either side of the query's y = 208.5 and at the same
    descriptor distance from it.  The query's windows span cells iy 20-22, so (30, 20) and (30, 21) are consecutive in the
    traversal: the reference reaches X first and keeps it on the tie."""
    nf = 1100
    kl = np.zeros(nf + 2, pl.KEYLINE_DTYPE)
    xs = 300.5 + (np.arange(nf) % 9)
    kl["startPointX"][:nf], kl["endPointX"][:nf] = xs, xs
    kl["startPointY"][:nf], kl["endPointY"][:nf] = 201.0, 208.0
    kl["startPointX"][nf:], kl["endPointX"][nf:] = 301.0, 309.0
    kl["startPointY"][nf:], kl["endPointY"][nf:] = (205.0, 212.0), (205.0, 212.0)
    kl["octave"][nf:] = (0, 1)
    dx, dy = kl["endPointX"] - kl["startPointX"], kl["endPointY"] - kl["startPointY"]
    kl["lineLength"] = np.sqrt(dx * dx + dy * dy)
    kl["angle"] = np.arctan2(dy, dx)
    kl["ptx"], kl["pty"] = (kl["startPointX"] + kl["endPointX"]) / 2, (kl["startPointY"] + kl["endPointY"]) / 2
    sp = np.stack([kl["startPointX"], kl["startPointY"], np.ones(nf + 2)], 1).astype(np.float64)
    ep = np.stack([kl["endPointX"], kl["endPointY"], np.ones(nf + 2)], 1).astype(np.float64)
    lf = np.cross(sp, ep)
    lf /= np.sqrt(lf[:, 0] ** 2 + lf[:, 1] ** 2)[:, None]
    q = rng.integers(0, 256, (1, 32), dtype=np.uint8)
    desc = rng.integers(0, 256, (nf + 2, 32), dtype=np.uint8)
    desc[nf:] = q
    desc[nf, 0] ^= 0x0f; desc[nf + 1, 5] ^= 0xf0              # distance 4 each
    proj = np.array([[296.0, 208.5, 314.0, 208.5]], np.float32)
    return kl, lf, desc, q, proj


@pytest.mark.parametrize("variant", ["last", "lines"])
def test_line_search_through_a_cell_of_more_than_1024_lines(variant):
    """The line searches order candidates by (probe, cell rank, slot in cell); a cell crossed by more than 1024 lines must not
    let its later slots sort after the next cell's first ones.  Two equally distant candidates, one at slot 1100 of a cell and
    one at slot 0 of the next: the GPU must pick the reference's, the first one reached."""
    kl, lf, desc, q, proj = _crowded_cell_lines(np.random.default_rng(21))
    s, _ = oracle.assign_grid_lines(kl, BOUNDS)
    assert s[30 * 48 + 21] - s[30 * 48 + 20] == 1101
    valid = np.ones(1, np.uint8)
    if variant == "last":
        a = (kl, lf, desc, BOUNDS, valid, proj, q, np.array([8.0], np.float32), 5.0)
        nm, m = pl.LSDmatcher(0.7).SearchByProjectionLast(*a)
        onm, om = oracle.line_search_by_projection_last(*a)
    else:
        a = (kl, lf, desc, BOUNDS, valid, proj, np.ones(1, np.float32), q)
        nm, m = pl.LSDmatcher(0.7).SearchByProjectionLines(*a, th=1.0)
        onm, om = oracle.line_search_by_projection_lines(*a, 1.0, 0.7)
    assert onm == 1 and om[1100] == 0 and om[1101] == -1
    assert nm == onm and np.array_equal(m, om)
