"""The host-pointer entry points refuse a NULL input array whose count is > 0.

Each call below gets a NULL for one required host array with a count > 0: it returns PL_ERR_ARG and launches nothing.  The same
call with the array supplied then succeeds and returns exactly what the binding's own call returns on those inputs, so no error
state is left behind."""
import ctypes as C

import numpy as np
import pytest

import oracle
import plslam_b200 as pl
import track_scene as ts
from plslam_b200 import binding as B
from plslam_b200 import synth

pytestmark = pytest.mark.gpu
PL_ERR_ARG = -1
W, H = 640, 480


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _refused_then_run(f, args, i):
    """f(*args) with argument i NULL must return PL_ERR_ARG without a launch; returns f(*args)."""
    bad = list(args)
    bad[i] = None
    n0 = B.launch_count()
    assert f(*bad) == PL_ERR_ARG
    assert B.launch_count() == n0
    rc = f(*args)
    assert rc >= 0, B.lib().pl_last_error().decode()
    return rc


@pytest.fixture(scope="module")
def frame():
    """1000 keypoints with random descriptors and, for each, a point at 2-5 m on its viewing ray (identity pose)."""
    rng = np.random.default_rng(11)
    n = 1000
    kp = np.zeros(n, B.KP_DTYPE)
    kp["x"] = rng.uniform(20, W - 20, n); kp["y"] = rng.uniform(20, H - 20, n); kp["size"] = 31
    kp["angle"] = rng.uniform(0, 360, n); kp["octave"] = rng.integers(0, 8, n)
    K = np.array([500, 500, W / 2, H / 2], np.float32)
    z = rng.uniform(2, 5, n)
    pos = np.stack([(kp["x"] - K[2]) / K[0] * z, (kp["y"] - K[3]) / K[1] * z, z], 1).astype(np.float32)
    return dict(keys=kp, desc=rng.integers(0, 256, (n, 32), dtype=np.uint8), K=K, pos=pos, Tcw=np.eye(4, dtype=np.float32),
                bounds=np.array([0, 0, W, H], np.float32), sf=(1.2 ** np.arange(8)).astype(np.float32))


def test_orb_search_by_projection_last(frame):
    f, n = frame, len(frame["keys"])
    valid = np.ones(n, np.uint8); octave = f["keys"]["octave"].astype(np.int32); angle = f["keys"]["angle"].astype(np.float32)
    nm, match = pl.ORBmatcher(0.9, True).SearchByProjectionLast(f["keys"], f["desc"], f["bounds"], f["Tcw"], f["K"], f["sf"], valid,
                                                                  f["pos"], f["desc"], octave, angle, 7.0)
    assert nm > 0
    out = np.zeros(n, np.int32)
    args = [_p(f["keys"]), _p(f["desc"]), n, _p(f["bounds"]), _p(f["Tcw"]), _p(f["K"]), _p(f["sf"]), len(f["sf"]), n, _p(valid),
            _p(f["pos"]), _p(f["desc"]), _p(octave), _p(angle), 7.0, 1, None, _p(out)]
    assert _refused_then_run(B.lib().pl_orb_search_by_projection_last, args, 12) == nm      # last_octave
    assert np.array_equal(out, match)


def test_orb_search_by_projection_points(frame):
    f, n = frame, len(frame["keys"])
    idx = np.arange(0, n, 3)
    kp = f["keys"][idx]
    in_view = np.ones(len(idx), np.uint8); proj = np.stack([kp["x"], kp["y"]], 1).astype(np.float32)
    level = kp["octave"].astype(np.int32); view_cos = np.ones(len(idx), np.float32); mp_desc = np.ascontiguousarray(f["desc"][idx])
    matcher = pl.ORBmatcher(0.8)
    nm, match = matcher.SearchByProjectionPoints(f["keys"], f["desc"], f["bounds"], f["sf"], in_view, proj, level, view_cos, mp_desc, th=3)
    assert nm > 0
    out = np.zeros(n, np.int32)
    args = [_p(f["keys"]), _p(f["desc"]), n, _p(f["bounds"]), _p(f["sf"]), len(f["sf"]), len(idx), _p(in_view), _p(proj), _p(level),
            _p(view_cos), _p(mp_desc), 3.0, matcher.mfNNratio, None, _p(out)]
    assert _refused_then_run(B.lib().pl_orb_search_by_projection_points, args, 9) == nm    # level
    assert np.array_equal(out, match)


def test_lsd_search_by_projection_last():
    f0 = synth.synth_frame(W, H, 1); f1 = synth.warp_frame(f0, 1001)
    (kl0, d0, _), (kl1, d1, lf1) = [[x[:-1] for x in oracle.line_extract(f, nfeatures=400)] for f in (f0, f1)]
    rng = np.random.default_rng(3)
    proj = np.stack([kl0["startPointX"], kl0["startPointY"], kl0["endPointX"], kl0["endPointY"]], 1).astype(np.float32)
    proj += rng.normal(0, 1.5, proj.shape).astype(np.float32)
    valid = (rng.random(len(kl0)) < 0.85).astype(np.uint8)
    kl1, lf1, d1, d0 = (np.ascontiguousarray(a) for a in (kl1, np.asarray(lf1, np.float64), d1, d0))
    length = np.ascontiguousarray(kl0["lineLength"], np.float32); bounds = np.array([0, 0, W, H], np.float32)
    nm, match = pl.LSDmatcher(0.7).SearchByProjectionLast(kl1, lf1, d1, bounds, valid, proj, d0, length, 15.0)
    assert nm > 0
    out = np.zeros(len(kl1), np.int32)
    args = [_p(kl1), _p(lf1), _p(d1), len(kl1), _p(bounds), len(kl0), _p(valid), _p(proj), _p(d0), _p(length), 15.0, None, _p(out)]
    assert _refused_then_run(B.lib().pl_lsd_search_by_projection_last, args, 6) == nm      # last_valid
    assert np.array_equal(out, match)


def test_pose_optimization():
    p = synth.synth_pose_problem(4, n_points=300, n_lines=80)
    want = pl.Optimizer.PoseOptimization(p["Tcw0"], p["K"], p["pt_obs"], p["pt_inv_sigma2"], p["pt_Xw"], p["line_func"], p["line_Xw"])
    T0, K = np.ascontiguousarray(p["Tcw0"], np.float32), np.ascontiguousarray(p["K"], np.float32)
    po, pw, px = (np.ascontiguousarray(p[k], np.float32) for k in ("pt_obs", "pt_inv_sigma2", "pt_Xw"))
    lf, lx = (np.ascontiguousarray(p[k], np.float64) for k in ("line_func", "line_Xw"))
    Tout = np.zeros((4, 4), np.float32); pout = np.zeros(len(pw), np.uint8); lout = np.zeros(len(lf), np.uint8); its = C.c_int(0)
    args = [0, _p(T0), _p(K), len(pw), _p(po), _p(pw), _p(px), len(lf), _p(lf), _p(lx), _p(Tout), _p(pout), _p(lout), C.byref(its)]
    assert _refused_then_run(B.lib().pl_pose_optimization, args, 4) == want[0]              # pt_obs
    assert np.array_equal(Tout, want[1]) and np.array_equal(pout.astype(bool), want[2]) and np.array_equal(lout.astype(bool), want[3])
    assert its.value == want[4]


def test_frame_is_in_frustum_points(frame):
    f, n = frame, len(frame["pos"])
    Ow = np.zeros(3, np.float32)
    dist = np.linalg.norm(f["pos"], axis=1)
    normal = (f["pos"] / dist[:, None]).astype(np.float32)
    dmin, dmax = (0.5 * dist).astype(np.float32), (2.0 * dist).astype(np.float32)
    logsf = float(np.log(np.float32(1.2)))
    want = pl.isInFrustum(f["Tcw"], Ow, f["K"], f["bounds"], logsf, 8, 0.5, f["pos"], normal, dmin, dmax)
    assert want[0].sum() > 0
    got = [np.zeros(n, np.uint8), np.zeros((n, 2), np.float32), np.zeros(n, np.int32), np.zeros(n, np.float32)]
    args = [_p(f["Tcw"]), _p(Ow), _p(f["K"]), _p(f["bounds"]), C.c_float(logsf), C.c_int(8), C.c_float(0.5), C.c_int(n), _p(f["pos"]),
            _p(normal), _p(dmin), _p(dmax), *[_p(a) for a in got]]
    assert _refused_then_run(B.lib().pl_frame_is_in_frustum_points, args, 8) == 0           # pos
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


def test_track_local_map():
    m = ts.scene_map()
    T, K = ts.TRUE[0]
    fr, _ = ts.batch_frames([(T, K, ts.perturb(T, 0.006, 0), None, None)])
    Np, Nl = len(m["pt_pos"]), len(m["ln_pos"])
    local = dict(pt_index=np.arange(Np, dtype=np.int32), ln_index=np.arange(Nl, dtype=np.int32), pt_offset=[0], pt_count=[Np],
                 ln_offset=[0], ln_count=[Nl], frames_since_reloc=[5], max_frames=30)
    M = pl.Map(**m)
    want = pl.track_local_map(M, fr, local, host=True)
    keep = []
    loc, cLP, cLL = B._local_struct(local, 1, keep, lambda a: (a, B._p(a)))
    a = {k: np.ascontiguousarray(fr[k], dt) for k, dt in (
        ("keys_un", B.KP_DTYPE), ("desc", np.uint8), ("n", np.int32), ("keylines", B.KEYLINE_DTYPE), ("line_func", np.float64),
        ("line_desc", np.uint8), ("nl", np.int32), ("bounds", np.float32), ("scale_factors", np.float32),
        ("inv_level_sigma2", np.float32), ("Tcw0", np.float32), ("K", np.float32), ("point_map_in", np.int32), ("line_map_in", np.int32))}
    assert a["n"][0] > 0
    cap, capL = a["keys_un"].shape[1], a["keylines"].shape[1]
    shapes = B._out_shapes(1, cap, capL, cLP, cLL)
    names = B._TRACK_OUT[:6]
    out = {k: np.zeros(*shapes[k]) for k in names}
    o = B.PLTrackOut(*[_p(out[k]) if k in out else None for k in B._TRACK_OUT])
    fields = [1, _p(a["keys_un"]), _p(a["desc"]), _p(a["n"]), cap, _p(a["keylines"]), _p(a["line_func"]), _p(a["line_desc"]), _p(a["nl"]),
              capL, _p(a["bounds"]), _p(a["scale_factors"]), _p(a["inv_level_sigma2"]), len(a["scale_factors"]),
              float(fr["log_scale_factor"]), _p(a["Tcw0"]), _p(a["K"]), _p(a["point_map_in"]), _p(a["line_map_in"])]
    bad = B.PLTrackFrames(*fields[:1], None, *fields[2:])                                    # keys_un
    good = B.PLTrackFrames(*fields)
    f = B._track_lib().pl_track_local_map
    n0 = B.launch_count()
    assert f(M._h, C.byref(bad), C.byref(loc), C.byref(o)) == PL_ERR_ARG
    assert B.launch_count() == n0
    assert f(M._h, C.byref(good), C.byref(loc), C.byref(o)) == want["ok"][0]
    for k in names:
        assert np.array_equal(out[k], want[k]), k
