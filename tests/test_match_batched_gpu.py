"""GPU parity of the matchers' batched C entry points, called directly on torch CUDA buffers: one launch over frames that each
hold a different problem (counts from 0 to the capacity and past 2048, a capacity per side, a pose, camera, pre-assignment and
gate per frame), every input row past a frame's count filled with random bytes and every output with a sentinel.  Each frame
must equal the oracle's single-frame call on its own slice, and nothing past a frame's count may be written.  The host-pointer
wrappers and the front end reach these launches only with B = 1 or with the same capacity on both sides, where a per-frame
offset taken from the wrong capacity or the wrong frame cannot show."""
import ctypes as C
import numpy as np
import pytest
import oracle
import plslam_b200 as pl
from plslam_b200 import synth
from test_match_gpu import HD_BOUNDS, HD_K, _fake_map, synth_keypoint_pair

pytestmark = pytest.mark.gpu
SENTINEL = -0x5a5a5a5b
SF = None


def _scale():
    global SF
    if SF is None:
        SF = oracle.OrbOracle(1000, 1.2, 8, 20, 7).tables()["scale"]
    return SF


def _noise(shape, dtype, rng):
    """An array of random bytes viewed as `dtype` (NaNs and huge values included)."""
    dtype = np.dtype(dtype)
    return rng.integers(0, 256, int(np.prod(shape)) * dtype.itemsize, dtype=np.uint8).view(dtype).reshape(shape)


def _pack(rows, cap, dtype, rng, inner=()):
    """[B][cap](+inner) array of random bytes with frame b's first len(rows[b]) rows replaced by rows[b]."""
    out = _noise((len(rows), cap) + tuple(inner), dtype, rng)
    for b, r in enumerate(rows):
        out[b, :len(r)] = r
    return out


def _dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).cuda()


def _host(t, like):
    return t.cpu().numpy().view(like.dtype).reshape(like.shape)


def _sentinel(shape):
    import torch
    return torch.full(shape, SENTINEL, dtype=torch.int32, device="cuda")


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _call(name, argtypes, *args, restype=C.c_int):
    import torch
    f = getattr(pl.lib(), name)
    f.argtypes, f.restype = argtypes, restype
    torch.cuda.synchronize()
    rc = f(*args)
    torch.cuda.synchronize()
    return rc


# ---------------------------------------------------------------------------------------------- ORB point searches
CAP = 2400
# per frame: previous / current keypoint counts (an empty side, a frame at the capacity, frames past 2048, tiny frames)
N_PREV = [0, 700, CAP, 2100, 5, 1500]
N_CUR = [40, 0, CAP, 2300, 1, 1600]


def _point_frames():
    out = []
    for b, (n1, n2) in enumerate(zip(N_PREV, N_CUR)):
        k1, d1, k2, d2 = synth_keypoint_pair(max(n1, 1), 900 + b, HD_BOUNDS, ties=b % 2 == 1, n_cur=n2)
        out.append((k1[:n1], d1[:n1], k2, d2))
    return out


def test_assign_grid_dev():
    rng = np.random.default_rng(1)
    fr = _point_frames()
    keys = _pack([f[2] for f in fr], CAP, pl.KP_DTYPE, rng)
    n = np.array([len(f[2]) for f in fr], np.int32)
    B = len(fr)
    start, items = _sentinel((B, 3073)), _sentinel((B, CAP))
    dk, dn, db = _dev(keys), _dev(n), _dev(np.asarray(HD_BOUNDS, np.float32))
    pl.check(_call("pl_frame_assign_grid_dev", [C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 4,
                   _ptr(dk), _ptr(dn), CAP, B, _ptr(db), _ptr(start), _ptr(items), None))
    s, it = start.cpu().numpy(), items.cpu().numpy()
    for b, f in enumerate(fr):
        os_, oit = oracle.assign_grid(f[2], HD_BOUNDS)
        assert np.array_equal(s[b], os_) and np.array_equal(it[b, :len(oit)], oit), b
        assert (it[b, len(oit):] == SENTINEL).all(), b


def test_search_for_initialization_dev():
    rng = np.random.default_rng(2)
    fr = _point_frames()
    B = len(fr)
    k1 = _pack([f[0] for f in fr], CAP, pl.KP_DTYPE, rng); d1 = _pack([f[1] for f in fr], CAP, np.uint8, rng, (32,))
    k2 = _pack([f[2] for f in fr], CAP, pl.KP_DTYPE, rng); d2 = _pack([f[3] for f in fr], CAP, np.uint8, rng, (32,))
    pm0 = [np.stack([f[0]["x"], f[0]["y"]], 1).astype(np.float32) + rng.normal(0, 1, (len(f[0]), 2)).astype(np.float32) for f in fr]
    pm = _pack(pm0, CAP, np.float32, rng, (2,))
    n1, n2 = np.array(N_PREV, np.int32), np.array(N_CUR, np.int32)
    t = {k: _dev(v) for k, v in dict(k1=k1, d1=d1, k2=k2, d2=d2, n1=n1, n2=n2, pm=pm, b=np.asarray(HD_BOUNDS, np.float32)).items()}
    m, nm, scr = _sentinel((B, CAP)), _sentinel((B,)), _sentinel((B, 2 * CAP))
    pl.check(_call("pl_orb_search_for_initialization_dev", [C.c_void_p] * 6 + [C.c_int, C.c_int] + [C.c_void_p] * 4 +
                   [C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_void_p],
                   _ptr(t["k1"]), _ptr(t["d1"]), _ptr(t["n1"]), _ptr(t["k2"]), _ptr(t["d2"]), _ptr(t["n2"]), CAP, B, _ptr(t["b"]),
                   _ptr(t["pm"]), _ptr(m), _ptr(nm), 100, 0.9, 1, _ptr(scr), None))
    gm, gnm, gpm = m.cpu().numpy(), nm.cpu().numpy(), _host(t["pm"], pm)
    total = 0
    for b, f in enumerate(fr):
        onm, om, opm = oracle.search_for_initialization(f[0], f[1], f[2], f[3], HD_BOUNDS, pm0[b], 100, 0.9, True)
        a = N_PREV[b]
        assert gnm[b] == onm and np.array_equal(gm[b, :a], om), b
        assert gpm[b, :a].tobytes() == opm.tobytes(), b
        assert (gm[b, a:] == SENTINEL).all() and gpm[b, a:].tobytes() == pm[b, a:].tobytes(), b
        total += onm
    assert total > 500


def _last_side(fr, rng):
    """Per frame: the previous keypoints as the last frame (3-D points, valid flags), a pose and a camera of its own."""
    out = []
    for b, f in enumerate(fr):
        K = (HD_K * (1 + 0.02 * b, 1 - 0.01 * b, 1, 1) + (0, 0, 3 * b, -2 * b)).astype(np.float32)
        X = _fake_map(f[0], rng, K)
        T = np.eye(4, dtype=np.float32); T[:3, 3] = [0.003 * b, -0.002, 0.001 * (b % 3)]
        valid = (rng.random(len(f[0])) < 0.85).astype(np.uint8)
        pre = (rng.random(len(f[2])) < 0.05 * (b % 3)).astype(np.uint8)
        out.append(dict(K=K, X=X, T=T, valid=valid, pre=pre))
    return out


def test_search_by_projection_last_dev_with_gate():
    """Two passes as the front end makes them: th 15, then th 30 for the frames under 20 matches, the first pass's counts
    passed as both gate and outputs.  Frames 0, 1 and 4 (an empty side, five and one keypoints) stay under 20 and take the
    second pass; the others are gated."""
    rng = np.random.default_rng(3)
    fr = _point_frames()
    B = len(fr)
    cap_last = CAP + 37
    ls = _last_side(fr, rng)
    k = _pack([f[2] for f in fr], CAP, pl.KP_DTYPE, rng); d = _pack([f[3] for f in fr], CAP, np.uint8, rng, (32,))
    lv = _pack([s["valid"] for s in ls], cap_last, np.uint8, rng)
    lp = _pack([s["X"] for s in ls], cap_last, np.float32, rng, (3,))
    ld = _pack([f[1] for f in fr], cap_last, np.uint8, rng, (32,))
    lo = _pack([f[0]["octave"].astype(np.int32) for f in fr], cap_last, np.int32, rng)
    la = _pack([f[0]["angle"] for f in fr], cap_last, np.float32, rng)
    pre = _pack([s["pre"] for s in ls], CAP, np.uint8, rng)
    T = np.stack([s["T"].reshape(16) for s in ls]); K = np.stack([s["K"] for s in ls])
    n, nl = np.array(N_CUR, np.int32), np.array(N_PREV, np.int32)
    t = {k_: _dev(v) for k_, v in dict(k=k, d=d, n=n, b=np.asarray(HD_BOUNDS, np.float32), T=T, K=K, sf=_scale(), nl=nl, lv=lv, lp=lp,
                                       ld=ld, lo=lo, la=la, pre=pre).items()}
    m, nm = _sentinel((B, CAP)), _sentinel((B,))
    argt = [C.c_void_p] * 3 + [C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 5 + \
        [C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    res = []
    for th, gate in ((15.0, None), (30.0, nm)):
        pl.check(_call("pl_orb_search_by_projection_last_dev", argt, _ptr(t["k"]), _ptr(t["d"]), _ptr(t["n"]), CAP, B, _ptr(t["b"]),
                       _ptr(t["T"]), _ptr(t["K"]), _ptr(t["sf"]), 8, _ptr(t["nl"]), cap_last, _ptr(t["lv"]), _ptr(t["lp"]), _ptr(t["ld"]),
                       _ptr(t["lo"]), _ptr(t["la"]), th, 1, _ptr(t["pre"]), _ptr(gate), 20, _ptr(m), _ptr(nm), None))
        res.append((m.cpu().numpy(), nm.cpu().numpy()))
    gated = 0
    for b, f in enumerate(fr):
        s = ls[b]
        a = (f[2], f[3], HD_BOUNDS, s["T"], s["K"], _scale(), s["valid"], s["X"], f[1], f[0]["octave"], f[0]["angle"])
        onm, om = oracle.search_by_projection_last(*a, 15.0, check_ori=True, preassigned=s["pre"])
        nc = N_CUR[b]
        assert res[0][1][b] == onm and np.array_equal(res[0][0][b, :nc], om), b
        if onm >= 20:                     # gated: the second pass leaves the row and the count exactly as they were
            gated += 1
            assert res[1][1][b] == onm and res[1][0][b].tobytes() == res[0][0][b].tobytes(), b
        else:
            onm, om = oracle.search_by_projection_last(*a, 30.0, check_ori=True, preassigned=s["pre"])
            assert res[1][1][b] == onm and np.array_equal(res[1][0][b, :nc], om), b
        assert (res[1][0][b, nc:] == SENTINEL).all(), b
    assert 2 <= gated < B


def test_search_by_projection_points_dev():
    rng = np.random.default_rng(4)
    fr = _point_frames()
    B = len(fr)
    cap_mp = CAP + 101
    mp = []
    for b, f in enumerate(fr):
        nm_ = len(f[0]) + 300 * (b % 2) if len(f[0]) else 0
        src = rng.integers(0, max(len(f[0]), 1), nm_)
        proj = (np.stack([f[0]["x"][src], f[0]["y"][src]], 1) + rng.normal(0, 1.0, (nm_, 2))).astype(np.float32) if nm_ else np.zeros((0, 2), np.float32)
        mp.append(dict(in_view=(rng.random(nm_) < 0.85).astype(np.uint8), proj=proj,
                       level=f[0]["octave"][src].astype(np.int32) if nm_ else np.zeros(0, np.int32),
                       view_cos=rng.uniform(0.997, 1.0, nm_).astype(np.float32), desc=f[1][src] if nm_ else np.zeros((0, 32), np.uint8),
                       pre=(rng.random(len(f[2])) < 0.05).astype(np.uint8)))
    n_mp = np.array([len(x["in_view"]) for x in mp], np.int32)
    assert n_mp.max() <= cap_mp
    t = {k_: _dev(v) for k_, v in dict(
        k=_pack([f[2] for f in fr], CAP, pl.KP_DTYPE, rng), d=_pack([f[3] for f in fr], CAP, np.uint8, rng, (32,)),
        n=np.array(N_CUR, np.int32), b=np.asarray(HD_BOUNDS, np.float32), sf=_scale(), nmp=n_mp,
        iv=_pack([x["in_view"] for x in mp], cap_mp, np.uint8, rng), pr=_pack([x["proj"] for x in mp], cap_mp, np.float32, rng, (2,)),
        lv=_pack([x["level"] for x in mp], cap_mp, np.int32, rng), vc=_pack([x["view_cos"] for x in mp], cap_mp, np.float32, rng),
        md=_pack([x["desc"] for x in mp], cap_mp, np.uint8, rng, (32,)), pre=_pack([x["pre"] for x in mp], CAP, np.uint8, rng)).items()}
    m, nm = _sentinel((B, CAP)), _sentinel((B,))
    pl.check(_call("pl_orb_search_by_projection_points_dev", [C.c_void_p] * 3 + [C.c_int, C.c_int] + [C.c_void_p] * 3 + [C.c_int] +
                   [C.c_void_p] * 5 + [C.c_float, C.c_float] + [C.c_void_p] * 4,
                   _ptr(t["k"]), _ptr(t["d"]), _ptr(t["n"]), CAP, B, _ptr(t["b"]), _ptr(t["sf"]), _ptr(t["nmp"]), cap_mp, _ptr(t["iv"]),
                   _ptr(t["pr"]), _ptr(t["lv"]), _ptr(t["vc"]), _ptr(t["md"]), 3.0, 0.8, _ptr(t["pre"]), _ptr(m), _ptr(nm), None))
    gm, gnm = m.cpu().numpy(), nm.cpu().numpy()
    total = 0
    for b, f in enumerate(fr):
        x = mp[b]
        onm, om = oracle.search_by_projection_points(f[2], f[3], HD_BOUNDS, _scale(), x["in_view"], x["proj"], x["level"], x["view_cos"],
                                                     x["desc"], 3.0, 0.8, preassigned=x["pre"])
        nc = N_CUR[b]
        assert gnm[b] == onm and np.array_equal(gm[b, :nc], om), b
        assert (gm[b, nc:] == SENTINEL).all(), b
        total += onm
    assert total > 500


# ---------------------------------------------------------------------------------------------- line matching
def _line_descs(rng):
    """Per frame (d1, d2): line descriptor sets of 0, 1 and 2 rows on either side, and larger ones where the second set is a
    noisy permutation of the first."""
    def noisy(base, m):
        d = base[rng.permutation(len(base))[:m]].copy()
        for r in range(len(d)):
            for bit in rng.integers(0, 256, rng.integers(0, 30)):
                d[r, bit // 8] ^= np.uint8(1 << (bit % 8))
        return d
    out = []
    for n1, n2 in ((0, 5), (7, 0), (1, 3), (2, 2), (3, 1), (260, 240), (300, 300), (120, 180)):
        base = rng.integers(0, 256, (max(n1, n2, 1), 32), dtype=np.uint8)
        out.append((base[:n1], noisy(base, n2)))
    return out


@pytest.mark.parametrize("mutual", [1, 0])
def test_lsd_search_double_dev(mutual):
    rng = np.random.default_rng(5 + mutual)
    fr = _line_descs(rng)
    B, cap1, cap2 = len(fr), 300, 331
    t = {k_: _dev(v) for k_, v in dict(d1=_pack([f[0] for f in fr], cap1, np.uint8, rng, (32,)), n1=np.array([len(f[0]) for f in fr], np.int32),
                                       d2=_pack([f[1] for f in fr], cap2, np.uint8, rng, (32,)),
                                       n2=np.array([len(f[1]) for f in fr], np.int32)).items()}
    m, nm = _sentinel((B, cap1)), _sentinel((B,))
    th, ratio = (50.0, 0.7) if mutual else (80.0, 0.9)
    pl.check(_call("pl_lsd_search_double_dev", [C.c_void_p] * 4 + [C.c_int] * 3 + [C.c_float, C.c_float, C.c_int] + [C.c_void_p] * 3,
                   _ptr(t["d1"]), _ptr(t["n1"]), _ptr(t["d2"]), _ptr(t["n2"]), cap1, cap2, B, th, ratio, mutual, _ptr(m), _ptr(nm), None))
    gm, gnm = m.cpu().numpy(), nm.cpu().numpy()
    total = 0
    for b, (d1, d2) in enumerate(fr):
        if mutual:
            onm, om = oracle.search_double(d1, d2, ratio)
        else:
            om = oracle.frame_bf_match(d1, d2, th, ratio) if len(d1) and len(d2) else np.full(len(d1), -1, np.int32)
            onm = int((om >= 0).sum())
        assert gnm[b] == onm and np.array_equal(gm[b, :len(d1)], om), b
        assert (gm[b, len(d1):] == SENTINEL).all(), b
        total += onm
    assert total > 100


def _search_double_limit():
    """Largest equal line capacity whose k_search_double shared memory (8 B per line, beside its 1040 static B: hist[257] and
    three counters) fits the device's opt-in shared memory per block."""
    import torch
    return (torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 1040) // 8


def test_lsd_search_double_at_the_shared_memory_limit():
    """The largest capacity that fits equals the oracle; one line more is refused with PL_ERR_ARG before any launch, through
    the batched form and through the host form."""
    import torch
    fit = _search_double_limit()
    rng = np.random.default_rng(9)
    base = rng.integers(0, 256, (fit, 32), dtype=np.uint8)
    d2 = base[rng.permutation(fit)].copy()
    flips = rng.integers(0, 256, (fit, 12))
    for r in range(fit):
        for bit in flips[r]:
            d2[r, bit // 8] ^= np.uint8(1 << (bit % 8))
    m = pl.LSDmatcher(0.7).FrameBFMatch(base, d2, 50.0)
    om = oracle.frame_bf_match(base, d2, 50.0, 0.7)
    assert (om >= 0).sum() > 100 and np.array_equal(m, om)
    over = np.zeros((fit + 1, 32), np.uint8)
    with pytest.raises(pl.PLError, match=rf"error -1: .* at most {fit} lines per side"):
        pl.LSDmatcher(0.7).SearchDouble(over, over)
    d = torch.zeros((fit + 1) * 32, dtype=torch.uint8, device="cuda"); n = torch.ones(1, dtype=torch.int32, device="cuda")
    m, nm = _sentinel((fit + 1,)), _sentinel((1,))
    before = pl.launch_count()
    rc = _call("pl_lsd_search_double_dev", [C.c_void_p] * 4 + [C.c_int] * 3 + [C.c_float, C.c_float, C.c_int] + [C.c_void_p] * 3,
               _ptr(d), _ptr(n), _ptr(d), _ptr(n), fit + 1, fit + 1, 1, 50.0, 0.7, 1, _ptr(m), _ptr(nm), None)
    assert rc == -1 and pl.launch_count() == before and (m.cpu().numpy() == SENTINEL).all()
    assert _call("pl_lsd_search_double_dev", [C.c_void_p] * 4 + [C.c_int] * 3 + [C.c_float, C.c_float, C.c_int] + [C.c_void_p] * 3,
                 _ptr(d), _ptr(n), _ptr(d), _ptr(n), fit, fit + 1, 1, 50.0, 0.7, 1, _ptr(m), _ptr(nm), None) == -1


@pytest.fixture(scope="module")
def line_frames():
    """Lines of consecutive synthetic frames, each with its warped successor (keylines, line functions, descriptors)."""
    out = []
    for s in (1, 2, 3):
        f0 = synth.synth_frame(640, 480, s); f1 = synth.warp_frame(f0, 1000 + s)
        out.append([oracle.line_extract(f, nfeatures=300) for f in (f0, f1)])
    return out


@pytest.mark.parametrize("variant", [0, 1])
def test_lsd_search_by_projection_dev(line_frames, variant):
    """Both line searches over frames of 0 to cap lines (the last at cap, so its rows end the scratch), queries with their own
    capacity, per-frame pre-assignment; the scratch of exactly pl_lsd_search_scratch_bytes(cap, B) bytes sits in a larger
    buffer whose guard bytes after it must stay unchanged."""
    import torch
    rng = np.random.default_rng(10 + variant)
    bounds = [0.0, 0.0, 640.0, 480.0]
    frames = []
    for (kl0, d0, _), (kl1, d1, lf1) in line_frames:
        frames.append((kl0, d0, kl1, d1, lf1))
    cap = max(len(f[2]) for f in frames) + 4
    # frame counts: empty, a few lines, three full frames, the last one padded to the capacity with short extra lines
    sel = [(0, 0), (0, 3), (0, None), (1, None), (2, None), (1, cap)]
    probs = []
    for i, cnt in sel:
        kl0, d0, kl1, d1, lf1 = frames[i]
        if cnt == cap:
            extra = cap - len(kl1)
            idx = rng.integers(0, len(kl1), extra)
            kl1, lf1 = np.concatenate([kl1, kl1[idx]]), np.concatenate([lf1, lf1[idx]])
            d1 = np.concatenate([d1, rng.integers(0, 256, (extra, 32), dtype=np.uint8)])
        elif cnt is not None:
            kl1, d1, lf1 = kl1[:cnt], d1[:cnt], lf1[:cnt]
        proj = np.stack([kl0["startPointX"], kl0["startPointY"], kl0["endPointX"], kl0["endPointY"]], 1).astype(np.float32)
        proj += rng.normal(0, 1.2, proj.shape).astype(np.float32)
        q_valid = (rng.random(len(kl0)) < 0.85).astype(np.uint8)
        aux = kl0["lineLength"].astype(np.float32) if variant == 0 else rng.uniform(0.99, 1.0, len(kl0)).astype(np.float32)
        pre = (rng.random(len(kl1)) < 0.05).astype(np.uint8)
        probs.append(dict(kl=kl1, d=d1, lf=lf1, proj=proj, q_valid=q_valid, q_desc=d0, aux=aux, pre=pre))
    B = len(probs)
    assert len(probs[-1]["kl"]) == cap
    cap_q = max(len(p["proj"]) for p in probs) + 19
    t = {k_: _dev(v) for k_, v in dict(
        kl=_pack([p["kl"] for p in probs], cap, pl.KEYLINE_DTYPE, rng), lf=_pack([p["lf"] for p in probs], cap, np.float64, rng, (3,)),
        d=_pack([p["d"] for p in probs], cap, np.uint8, rng, (32,)), n=np.array([len(p["kl"]) for p in probs], np.int32),
        b=np.asarray(bounds, np.float32), nq=np.array([len(p["proj"]) for p in probs], np.int32),
        qv=_pack([p["q_valid"] for p in probs], cap_q, np.uint8, rng), qp=_pack([p["proj"] for p in probs], cap_q, np.float32, rng, (4,)),
        qd=_pack([p["q_desc"] for p in probs], cap_q, np.uint8, rng, (32,)), qa=_pack([p["aux"] for p in probs], cap_q, np.float32, rng),
        pre=_pack([p["pre"] for p in probs], cap, np.uint8, rng)).items()}
    nbytes = _call("pl_lsd_search_scratch_bytes", [C.c_int, C.c_int], cap, B, restype=C.c_size_t)
    guard = 4 * cap * B + 4096
    scratch = torch.full((nbytes + guard,), 0xA5, dtype=torch.uint8, device="cuda")
    m, nm = _sentinel((B, cap)), _sentinel((B,))
    th = 15.0 if variant == 0 else 3.0
    pl.check(_call("pl_lsd_search_by_projection_dev", [C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_int] + [C.c_void_p] * 2 + [C.c_int] +
                   [C.c_void_p] * 4 + [C.c_float, C.c_float] + [C.c_void_p] * 5,
                   variant, _ptr(t["kl"]), _ptr(t["lf"]), _ptr(t["d"]), _ptr(t["n"]), cap, B, _ptr(t["b"]), _ptr(t["nq"]), cap_q, _ptr(t["qv"]),
                   _ptr(t["qp"]), _ptr(t["qd"]), _ptr(t["qa"]), th, 0.7, _ptr(t["pre"]), _ptr(m), _ptr(nm), _ptr(scratch), None))
    gm, gnm = m.cpu().numpy(), nm.cpu().numpy()
    assert (scratch[nbytes:].cpu().numpy() == 0xA5).all()
    total = 0
    for b, p in enumerate(probs):
        if variant == 0:
            onm, om = oracle.line_search_by_projection_last(p["kl"], p["lf"], p["d"], bounds, p["q_valid"], p["proj"], p["q_desc"], p["aux"],
                                                            th, preassigned=p["pre"])
        else:
            onm, om = oracle.line_search_by_projection_lines(p["kl"], p["lf"], p["d"], bounds, p["q_valid"], p["proj"], p["aux"], p["q_desc"],
                                                             th, 0.7, preassigned=p["pre"])
        nc = len(p["kl"])
        assert gnm[b] == onm and np.array_equal(gm[b, :nc], om), b
        assert (gm[b, nc:] == SENTINEL).all(), b
        total += onm
    assert total > 60
