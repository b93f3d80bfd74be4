"""GPU parity tests: matching through the C ABI vs the CPU oracle — indices and Hamming distances bit-exact."""
import numpy as np
import pytest
import oracle
import plslam_b200 as pl
from plslam_b200 import synth

pytestmark = pytest.mark.gpu
BOUNDS = [0.0, 0.0, 640.0, 480.0]


@pytest.fixture(scope="module")
def frames():
    seq = synth.synth_sequence(3, 640, 480, seed=2)
    out = {}
    for nf in (1000, 2000):
        o = oracle.OrbOracle(nf, 1.2, 8, 20, 7)
        out[nf] = [o.extract(f) for f in seq]
    return out


def test_descriptor_distance(frames):
    rng = np.random.default_rng(0)
    a = rng.integers(0, 256, (500, 32), dtype=np.uint8); b = rng.integers(0, 256, (500, 32), dtype=np.uint8)
    b[:50] = a[:50]; b[50:60] = ~a[50:60]
    got = pl.ORBmatcher.DescriptorDistance(a, b)
    assert list(got) == [oracle.descriptor_distance(a[i], b[i]) for i in range(500)]
    assert got[0] == 0 and got[55] == 256


@pytest.mark.parametrize("nf", [1000, 2000])
def test_assign_grid(frames, nf):
    k, d = frames[nf][0]
    s, it = pl.frame_assign_grid(k, BOUNDS)
    os_, oit = oracle.assign_grid(k, BOUNDS)
    assert np.array_equal(s, os_) and np.array_equal(it, oit)
    # keypoints outside the bounds are dropped (Frame::PosInGrid)
    k2 = k.copy(); k2["x"][:50] += 700
    s, it = pl.frame_assign_grid(k2, BOUNDS)
    os_, oit = oracle.assign_grid(k2, BOUNDS)
    assert np.array_equal(s, os_) and np.array_equal(it, oit)


@pytest.mark.parametrize("nf,win,ratio,ori", [(1000, 100, 0.9, True), (2000, 100, 0.9, True), (2000, 30, 0.7, False)])
def test_search_for_initialization(frames, nf, win, ratio, ori):
    (k1, d1), (k2, d2) = frames[nf][0], frames[nf][1]
    prev = np.stack([k1["x"], k1["y"]], 1).astype(np.float32)
    nm, m, pm = pl.ORBmatcher(ratio, ori).SearchForInitialization(k1, d1, k2, d2, BOUNDS, prev, win)
    onm, om, opm = oracle.search_for_initialization(k1, d1, k2, d2, BOUNDS, prev, win, ratio, ori)
    assert onm > 50
    assert nm == onm and np.array_equal(m, om) and np.array_equal(pm, opm)
    # second call re-uses the updated vbPrevMatched like Tracking::MonocularInitialization does
    nm2, m2, _ = pl.ORBmatcher(ratio, ori).SearchForInitialization(k1, d1, frames[nf][2][0], frames[nf][2][1], BOUNDS, pm, win)
    onm2, om2, _ = oracle.search_for_initialization(k1, d1, frames[nf][2][0], frames[nf][2][1], BOUNDS, opm, win, ratio, ori)
    assert nm2 == onm2 and np.array_equal(m2, om2)


def _fake_map(k_last, rng, K):
    """3-D points whose projection with identity pose is the last frame's keypoint."""
    z = rng.uniform(1.5, 6.0, len(k_last)).astype(np.float32)
    X = np.stack([(k_last["x"] - K[2]) / K[0] * z, (k_last["y"] - K[3]) / K[1] * z, z], 1).astype(np.float32)
    return X


@pytest.mark.parametrize("nf,th", [(1000, 15.0), (2000, 7.0)])
def test_search_by_projection_last(frames, nf, th):
    rng = np.random.default_rng(4)
    (kl, dl), (kc, dc) = frames[nf][0], frames[nf][1]
    K = np.array(synth.TUM1_K, np.float32)
    X = _fake_map(kl, rng, K)
    valid = rng.random(len(kl)) < 0.8
    T = np.eye(4, dtype=np.float32); T[:3, 3] = [0.004, -0.003, 0.002]
    sf = oracle.OrbOracle(nf, 1.2, 8, 20, 7).tables()["scale"]
    pre = (rng.random(len(kc)) < 0.05).astype(np.uint8)
    args = (kc, dc, BOUNDS, T, K, sf, valid, X, dl, kl["octave"], kl["angle"], th)
    for ori in (True, False):
        nm, m = pl.ORBmatcher(0.9, ori).SearchByProjectionLast(*args, preassigned=pre)
        onm, om = oracle.search_by_projection_last(*args, check_ori=ori, preassigned=pre)
        assert onm > 100
        assert nm == onm and np.array_equal(m, om)


def test_search_by_projection_points(frames):
    rng = np.random.default_rng(6)
    k, d = frames[1000][1]
    kl, dl = frames[1000][0]
    n_mp = 1500
    src = rng.integers(0, len(kl), n_mp)
    proj = np.stack([kl["x"][src], kl["y"][src]], 1).astype(np.float32) + rng.normal(0, 2.0, (n_mp, 2)).astype(np.float32)
    level = np.clip(kl["octave"][src] + rng.integers(-1, 2, n_mp), 0, 7).astype(np.int32)
    in_view = rng.random(n_mp) < 0.85
    view_cos = rng.uniform(0.99, 1.0, n_mp).astype(np.float32)
    sf = oracle.OrbOracle(1000, 1.2, 8, 20, 7).tables()["scale"]
    for th in (1.0, 3.0, 5.0):
        a = (k, d, BOUNDS, sf, in_view, proj, level, view_cos, dl[src])
        nm, m = pl.ORBmatcher(0.8).SearchByProjectionPoints(*a, th=th)
        onm, om = oracle.search_by_projection_points(*a, th, 0.8)
        assert onm > 100
        assert nm == onm and np.array_equal(m, om)


def test_bf_knn_and_line_matching():
    rng = np.random.default_rng(8)
    # tie-heavy descriptors (bytes are 0x00/0xff) exercise "lower train index first"
    d1 = rng.integers(0, 2, (201, 32), dtype=np.uint8) * 255
    d2 = rng.integers(0, 2, (187, 32), dtype=np.uint8) * 255
    idx, dist = pl.LSDmatcher.knnMatch(d1, d2)
    oi, od = oracle.bf_knn2(d1, d2)
    assert np.array_equal(idx, oi) and np.array_equal(dist, od)
    # realistic: second set = noisy permutation of the first
    base = rng.integers(0, 256, (201, 32), dtype=np.uint8)
    perm = rng.permutation(201)[:180]
    d2 = base[perm].copy()
    for i in range(len(d2)):
        bits = rng.integers(0, 256, rng.integers(0, 30))
        for b in bits:
            d2[i, b // 8] ^= np.uint8(1 << (b % 8))
    for th, ratio in ((50.0, 0.7), (80.0, 0.9)):
        m = pl.LSDmatcher(ratio).FrameBFMatch(base, d2, th)
        assert np.array_equal(m, oracle.frame_bf_match(base, d2, th, ratio))
    nm, m = pl.LSDmatcher(0.7).SearchDouble(base, d2)
    onm, om = oracle.search_double(base, d2, 0.7)
    assert onm > 100 and nm == onm and np.array_equal(m, om)
    # degenerate sizes (reference reads out of bounds for <2 rows; defined as "no matches")
    for a, b in ((base[:0], d2), (base, d2[:0]), (base, d2[:1]), (base[:1], d2), (base[:2], d2[:2])):
        nm, m = pl.LSDmatcher(0.7).SearchDouble(a, b)
        onm, om = oracle.search_double(a, b, 0.7)
        assert nm == onm and np.array_equal(m, om)


# ---------------------------------------------------------------------------------------------- past the packed grid
# Up to 2048 keypoints the windowed searches keep each grid item's octave beside its index; above, the level filter reads the
# keypoint.  Synthetic sets hit exact counts on both sides of that line and up to the matchers' 6144 capacity.
HD_BOUNDS = [0.0, 0.0, 1920.0, 1080.0]
HD_K = np.array([1000.0, 1000.0, 960.0, 540.0], np.float32)


def _grid_ties(lo, hi, cells, count, rng):
    """`count` float32 coordinates c in [lo, hi] with (c - lo) * (cells / (hi - lo)) exactly k + 0.5 in float32: roundf's tie."""
    inv = np.float32(cells) / np.float32(np.float32(hi) - np.float32(lo))
    out = []
    for k in rng.permutation(cells - 1)[:4 * count]:
        c = np.float32(np.float32(lo) + np.float32(k + 0.5) / inv)
        for _ in range(8):
            v = (c - np.float32(lo)) * inv
            if v == np.float32(k + 0.5):
                out.append(c)
                break
            c = np.nextafter(c, np.float32(np.inf) if v < k + 0.5 else np.float32(-np.inf), dtype=np.float32)
        if len(out) == count:
            break
    return np.array(out, np.float32)


def synth_keypoint_pair(n, seed, bounds, ties=False, n_cur=None):
    """A previous and a current set of synthetic keypoints (n and n_cur, default n) over `bounds` and a little past it.
    The previous set holds a cell of 48 keypoints, keypoints on the grid's rounding ties and on all four borders, octaves 0-7
    (a third on 0) and random angles.  In the current set 60 % are moved copies (1.5 px, octave +-1, angle +-5 degrees) whose
    descriptors differ in a few bits, 10 % are closer decoys two octaves up that the level filters must reject, the rest random.
    ties: descriptor bytes are 0x00 / 0xff, so distances come in steps of 8 and the traversal order decides between equals."""
    rng = np.random.default_rng(seed)
    n_cur = n if n_cur is None else n_cur
    x0, y0, x1, y1 = [float(v) for v in bounds]
    W, H = x1 - x0, y1 - y0

    def desc(m):
        return (rng.integers(0, 2, (m, 32), dtype=np.uint8) * 255) if ties else rng.integers(0, 256, (m, 32), dtype=np.uint8)

    def flip(d, lo, hi):
        d = d.copy()
        for r in range(len(d)):
            if ties:
                bytes_ = rng.choice(32, rng.integers(lo, hi + 1) // 8 + 1, replace=False)
                d[r, bytes_] ^= 0xff
            else:
                for b in rng.choice(256, rng.integers(lo, hi + 1), replace=False):
                    d[r, b // 8] ^= np.uint8(1 << (b % 8))
        return d

    prev = np.zeros(n, pl.KP_DTYPE)
    prev["x"] = rng.uniform(x0 - 0.02 * W, x1 + 0.02 * W, n)
    prev["y"] = rng.uniform(y0 - 0.02 * H, y1 + 0.02 * H, n)
    cw, ch = W / 64, H / 48
    k = 0
    cx, cy = x0 + 31 * cw, y0 + 23 * ch                      # one cell of 48 keypoints
    m = min(48, n); prev["x"][k:k + m] = cx + rng.uniform(-0.4, 0.4, m) * cw; prev["y"][k:k + m] = cy + rng.uniform(-0.4, 0.4, m) * ch
    k += m
    tx, ty = _grid_ties(x0, x1, 64, 12, rng), _grid_ties(y0, y1, 48, 12, rng)
    m = min(len(tx), len(ty), n - k); prev["x"][k:k + m] = tx[:m]; prev["y"][k:k + m] = ty[:m]
    k += m
    border = [(x0, None), (x1, None), (None, y0), (None, y1), (x0, y0), (x1, y1), (x0, y1), (x1, y0)]
    for bx, by in border[:max(0, n - k)]:
        if bx is not None:
            prev["x"][k] = bx
        if by is not None:
            prev["y"][k] = by
        k += 1
    prev["octave"] = rng.choice(8, n, p=[0.34] + [0.66 / 7] * 7)
    prev["angle"] = rng.uniform(0, 360, n)
    prev["size"] = 31.0; prev["response"] = rng.uniform(0, 100, n)
    dprev = desc(n)

    cur = np.zeros(n_cur, pl.KP_DTYPE)
    dcur = desc(n_cur)
    cur["x"] = rng.uniform(x0 - 0.02 * W, x1 + 0.02 * W, n_cur); cur["y"] = rng.uniform(y0 - 0.02 * H, y1 + 0.02 * H, n_cur)
    cur["octave"] = rng.integers(0, 8, n_cur); cur["angle"] = rng.uniform(0, 360, n_cur)
    cur["size"] = 31.0; cur["response"] = rng.uniform(0, 100, n_cur)
    if n:
        n_copy, n_decoy = min(int(0.6 * n_cur), n), min(int(0.1 * n_cur), n)
        src = rng.permutation(n)
        s = src[:n_copy]
        cur[:n_copy]["x"] = prev["x"][s] + rng.normal(0, 1.5, n_copy); cur[:n_copy]["y"] = prev["y"][s] + rng.normal(0, 1.5, n_copy)
        cur[:n_copy]["octave"] = np.clip(prev["octave"][s] + rng.choice([-1, 0, 0, 0, 1], n_copy), 0, 7)
        cur[:n_copy]["angle"] = np.mod(prev["angle"][s] + rng.normal(0, 5, n_copy), 360)
        dcur[:n_copy] = flip(dprev[s], 0, 24)
        s = src[:n_decoy]
        e = slice(n_copy, n_copy + n_decoy)
        cur["x"][e] = prev["x"][s] + rng.normal(0, 1.5, n_decoy); cur["y"][e] = prev["y"][s] + rng.normal(0, 1.5, n_decoy)
        cur["octave"][e] = np.where(prev["octave"][s] <= 5, prev["octave"][s] + 2, prev["octave"][s] - 2)
        cur["angle"][e] = prev["angle"][s]
        dcur[e] = flip(dprev[s], 0, 3)
        perm = rng.permutation(n_cur)
        cur, dcur = cur[perm], dcur[perm]
    return prev, dprev, cur, dcur


# keypoint count, bounds (None: the TUM1 camera's undistorted bounds at 640 x 480), tie-heavy descriptors
PAST_PACKED = [(2048, HD_BOUNDS, False), (2048, None, True), (2049, None, False), (2049, HD_BOUNDS, True),
               (4000, HD_BOUNDS, False), (4000, None, True), (6144, None, False), (6144, HD_BOUNDS, True)]


def _bounds(b):
    return oracle.image_bounds(synth.TUM1_K, synth.TUM1_DIST, 640, 480) if b is None else np.asarray(b, np.float32)


def _case_id(c):
    return f"{c[0]}-{'hd' if c[1] else 'tum'}-{'ties' if c[2] else 'rand'}"


@pytest.mark.parametrize("n,bounds,ties", PAST_PACKED + [(2100, BOUNDS, False)],
                         ids=[_case_id(c) for c in PAST_PACKED] + ["2100-vga-window250"])
def test_search_for_initialization_past_the_packed_grid(n, bounds, ties):
    b = _bounds(bounds)
    k1, d1, k2, d2 = synth_keypoint_pair(n, 100 + n, b, ties)
    prev = np.stack([k1["x"], k1["y"]], 1).astype(np.float32)
    # a 250 px window spans more than 32 of the 48 rows of cells at 480 px: the cell walk's q32 = 0 branch
    wins = [(250, 0.9, True)] if bounds is BOUNDS else [(100, 0.9, True), (30, 0.7, False)]
    for win, ratio, ori in wins:
        nm, m, pm = pl.ORBmatcher(ratio, ori).SearchForInitialization(k1, d1, k2, d2, b, prev, win)
        onm, om, opm = oracle.search_for_initialization(k1, d1, k2, d2, b, prev, win, ratio, ori)
        assert onm > 50
        assert nm == onm and np.array_equal(m, om) and pm.tobytes() == opm.tobytes(), (win, ratio, ori)


def _last_frame_map(k_last, rng, K):
    """_fake_map with a pose that moves the camera a little; some points behind it."""
    X = _fake_map(k_last, rng, K)
    X[rng.random(len(X)) < 0.02, 2] *= -1
    T = np.eye(4, dtype=np.float32); T[:3, 3] = [0.004, -0.003, 0.002]
    return X, T


@pytest.mark.parametrize("n,bounds,ties", PAST_PACKED, ids=[_case_id(c) for c in PAST_PACKED])
def test_search_by_projection_last_past_the_packed_grid(n, bounds, ties):
    rng = np.random.default_rng(200 + n)
    b = _bounds(bounds)
    kl, dl, kc, dc = synth_keypoint_pair(n, 200 + n, b, ties)
    K = HD_K if bounds else np.array(synth.TUM1_K, np.float32)
    X, T = _last_frame_map(kl, rng, K)
    valid = rng.random(n) < 0.85
    sf = oracle.OrbOracle(1000, 1.2, 8, 20, 7).tables()["scale"]
    pre = (rng.random(n) < 0.05).astype(np.uint8)
    for th, ori in ((15.0, True), (7.0, False)):
        args = (kc, dc, b, T, K, sf, valid, X, dl, kl["octave"], kl["angle"], th)
        nm, m = pl.ORBmatcher(0.9, ori).SearchByProjectionLast(*args, preassigned=pre)
        onm, om = oracle.search_by_projection_last(*args, check_ori=ori, preassigned=pre)
        assert onm > 100
        assert nm == onm and np.array_equal(m, om), (th, ori)


@pytest.mark.parametrize("n,bounds,ties", PAST_PACKED, ids=[_case_id(c) for c in PAST_PACKED])
def test_search_by_projection_points_past_the_packed_grid(n, bounds, ties):
    rng = np.random.default_rng(300 + n)
    b = _bounds(bounds)
    kl, dl, k, d = synth_keypoint_pair(n, 300 + n, b, ties)
    n_mp = n + 500
    src = rng.integers(0, n, n_mp)
    proj = np.stack([kl["x"][src], kl["y"][src]], 1).astype(np.float32) + rng.normal(0, 1.0, (n_mp, 2)).astype(np.float32)
    level = kl["octave"][src].astype(np.int32)
    in_view = rng.random(n_mp) < 0.85
    view_cos = rng.uniform(0.997, 1.0, n_mp).astype(np.float32)
    sf = oracle.OrbOracle(1000, 1.2, 8, 20, 7).tables()["scale"]
    pre = (rng.random(n) < 0.05).astype(np.uint8)
    for th in (1.0, 3.0):
        a = (k, d, b, sf, in_view, proj, level, view_cos, dl[src])
        nm, m = pl.ORBmatcher(0.8).SearchByProjectionPoints(*a, th=th, preassigned=pre)
        onm, om = oracle.search_by_projection_points(*a, th, 0.8, preassigned=pre)
        assert onm > 100
        assert nm == onm and np.array_equal(m, om), th


@pytest.mark.parametrize("n", [2048, 2049, 6144])
def test_assign_grid_past_the_packed_grid(n):
    k, _, _, _ = synth_keypoint_pair(n, 400 + n, HD_BOUNDS)
    s, it = pl.frame_assign_grid(k, HD_BOUNDS)
    os_, oit = oracle.assign_grid(k, HD_BOUNDS)
    assert np.array_equal(s, os_) and np.array_equal(it, oit) and (np.diff(os_) > 32).any()


@pytest.mark.skipif(not oracle.ref_match_available(), reason="oracle/_ref/libref_match.so did not travel")
def test_matchers_equal_the_reference_matcher_code(frames):
    """The CUDA matchers against the REFERENCE's own ORBmatcher.cc (compiled into oracle/_ref/libref_match.so, run on this box's CPU):
    SearchForInitialization and the two tracking searches, same inputs, identical match lists."""
    (k1, d1), (k2, d2) = frames[1000][0], frames[1000][1]
    prev = np.stack([k1["x"], k1["y"]], 1).astype(np.float32)
    nm, m, pm = pl.ORBmatcher(0.9, True).SearchForInitialization(k1, d1, k2, d2, BOUNDS, prev, 100)
    rnm, rm, rpm = oracle.search_for_initialization(k1, d1, k2, d2, BOUNDS, prev, 100, 0.9, True, impl="ref")
    assert rnm > 50 and nm == rnm and np.array_equal(m, rm) and pm.tobytes() == rpm.tobytes()
    rng = np.random.default_rng(14)
    K = np.array(synth.TUM1_K, np.float32)
    X = _fake_map(k1, rng, K)
    valid = rng.random(len(k1)) < 0.8
    T = np.eye(4, dtype=np.float32); T[:3, 3] = [0.004, -0.003, 0.002]
    sf = oracle.OrbOracle(1000, 1.2, 8, 20, 7).tables()["scale"]
    pre = (rng.random(len(k2)) < 0.05).astype(np.uint8)
    args = (k2, d2, BOUNDS, T, K, sf, valid, X, d1, k1["octave"], k1["angle"], 15.0)
    nm, m = pl.ORBmatcher(0.9, True).SearchByProjectionLast(*args, preassigned=pre)
    rnm, rm = oracle.search_by_projection_last(*args, check_ori=True, preassigned=pre, impl="ref")
    assert rnm > 100 and nm == rnm and np.array_equal(m, rm)
    n_mp = 1500
    src = rng.integers(0, len(k1), n_mp)
    proj = np.stack([k1["x"][src], k1["y"][src]], 1).astype(np.float32) + rng.normal(0, 2.0, (n_mp, 2)).astype(np.float32)
    level = np.clip(k1["octave"][src] + rng.integers(-1, 2, n_mp), 0, 7).astype(np.int32)
    a = (k2, d2, BOUNDS, sf, rng.random(n_mp) < 0.85, proj, level, rng.uniform(0.99, 1.0, n_mp).astype(np.float32), d1[src])
    nm, m = pl.ORBmatcher(0.8).SearchByProjectionPoints(*a, th=3.0)
    rnm, rm = oracle.search_by_projection_points(*a, 3.0, 0.8, impl="ref")
    assert rnm > 100 and nm == rnm and np.array_equal(m, rm)
