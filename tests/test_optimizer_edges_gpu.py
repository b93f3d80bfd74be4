"""GPU parity of the optimisers where an indexing slip would still give a plausible pose: a camera per problem, keyframe or
frame; solver sizes on the kernels' thread strides and Cholesky tile edges; windows with gated, unobserved or fixed parts.
Every case is compared with the fp64 CPU oracle at the tolerances of test_lm_gpu.py and test_ba_gpu.py: 1e-4 relative on
translations and structure, 1e-3 on line end points, identical outlier / erase masks, inlier and iteration counts.
test_optimizer_cameras.py shows, without a GPU, that the oracle's answer for each camera case is far (over 100 x these
tolerances) from the answer of the plausible wrong camera model, so these comparisons can tell the two apart."""
import ctypes as C
import numpy as np
import pytest
import oracle
import plslam_b200 as pl
from plslam_b200 import synth
from test_ba_gpu import _check as check_local, _check_global as check_global
from test_lm_gpu import _close

pytestmark = pytest.mark.gpu

# ---------------------------------------------------------------------------------------------- problem builders (also used on the CPU)
TUM1, EUROC = np.array(synth.TUM1_K), np.array(synth.EUROC_K)
CAMERAS = [TUM1, EUROC, TUM1 * (1.03, 0.97, 1, 1) + (0, 0, 9, -7), EUROC * (0.97, 1.02, 1, 1) + (0, 0, -8, 6)]
CAP_P, CAP_L = 320, 160
# correspondence counts at k_pose_opt's edges: 0..3 (the "< 3: untouched" rule), 9 / 10 (one round below 10 edges), the 32-lane
# and 128-thread strides, the capacity, and one problem over it (b = 13) that the kernel clamps to its first CAP_P / CAP_L
POSE_NP = [0, 2, 3, 9, 10, 31, 32, 33, 127, 128, 129, 300, CAP_P, 400, 60, 80, 100, 200, 3, 10, 40, 250, 128, 33]
POSE_NL = [40, 0, 1, 2, 0, 1, 2, 150, 0, 40, 2, 80, CAP_L, 200, 129, 128, 127, 3, 9, 33, 32, 31, 10, 60]
# Once chi2 has reached rounding noise, g2o's stop rule (rho == 0, or ten rejected trials) is decided by the last bits of the
# chi2 and H sums, so the iteration count depends on the summation order and on the line Jacobians' central-difference scale
# (g2o's 1 / (2 * 1e-9) in the oracle, the literal 5e8, one ulp higher, in k_pose_opt).  Each problem's seed is the first of
# 200 + b + 1000 j (j = 0, 1, ...) that passes pose_outcome_is_rounding_stable; about half the candidates do not.
# test_optimizer_cameras.py checks the list.
POSE_SEEDS = [200, 201, 202, 203, 204, 205, 206, 3207, 208, 1209, 210, 211, 1212, 213, 214, 3215, 216, 217, 4218, 1219, 2220,
              4221, 222, 1223]


def pose_batch():
    """24 pose problems; problem b is observed with CAMERAS[b % 4] (TUM1, EuRoC and perturbed copies of both)."""
    return [synth.synth_pose_problem(POSE_SEEDS[b], n_points=POSE_NP[b], n_lines=POSE_NL[b], K=tuple(CAMERAS[b % 4]))
            for b in range(len(POSE_NP))]


def pose_args(p, K=None):
    """(Tcw0, K, points, lines) of p as the batched kernel reads them: the first CAP_P points and CAP_L lines."""
    n, m = min(len(p["pt_obs"]), CAP_P), min(len(p["line_func"]), CAP_L)
    return (p["Tcw0"], p["K"] if K is None else np.asarray(K, np.float32), p["pt_obs"][:n], p["pt_inv_sigma2"][:n], p["pt_Xw"][:n],
            p["line_func"][:m], p["line_Xw"][:m])


def pose_outcome_is_rounding_stable(p, modes=(0, 1, 2), iterations=True):
    """True if the oracle's inlier count, outlier masks and (with iterations) iteration count for p do not change under its
    rounding variants (k_pose_opt's summation order, the 5e8 Jacobian scale, both): then no LM decision of p that these
    outputs show hangs on the last bits of a sum, and the kernel has to reproduce them exactly."""
    for mode in modes:
        ref = oracle.pose_optimization(mode, *pose_args(p))
        for v in oracle.POSE_VARIANTS:
            r = oracle.pose_optimization(mode, *pose_args(p), variant=v)
            if r[0] != ref[0] or (iterations and r[4] != ref[4]) or not np.array_equal(r[2], ref[2]) or not np.array_equal(r[3], ref[3]):
                return False
    return True


def frontend_problems():
    return [synth.synth_pose_problem(80 + k, K=tuple(CAMERAS[k])) for k in range(4)]


def keyframe_cameras(n_kf, seed, focal=0.03, centre=8.0):
    """TUM1 with each keyframe's focal lengths scaled by up to +-focal and its principal point moved by up to +-centre px."""
    r = np.random.default_rng(seed)
    Ks = np.tile(TUM1, (n_kf, 1))
    Ks[:, :2] *= 1 + r.uniform(-focal, focal, (n_kf, 2))
    Ks[:, 2:] += r.uniform(-centre, centre, (n_kf, 2))
    return Ks.astype(np.float32)


K_END = TUM1 * (1.04, 1.04, 1, 1) + (0, 0, 10, -10)      # the current keyframe's camera, unlike any observing keyframe's


def lba_camera_window():
    """A line-heavy local window (so that the end points' camera moves the poses) with a camera per keyframe and its own K_end."""
    return synth.synth_ba_problem(7, n_free=8, n_fixed=10, n_pt=200, n_ln=300, Ks=keyframe_cameras(18, 107), K_end=K_END)


def without_points(p):
    q = dict(p)
    q.update(pe_kf=p["pe_kf"][:0], pe_pt=p["pe_pt"][:0], pe_obs=p["pe_obs"][:0], pe_inv_sigma2=p["pe_inv_sigma2"][:0])
    return q


def lba_lines_only_window():
    """Lines only (the points stay in the window, unobserved), a camera per keyframe and its own K_end."""
    return without_points(synth.synth_ba_problem(6, n_free=8, n_fixed=10, n_pt=50, n_ln=200, Ks=keyframe_cameras(18, 106), K_end=K_END))


def gba_camera_map():
    return synth.synth_ba_problem(5, n_free=9, n_fixed=0, n_pt=600, n_ln=80, Ks=keyframe_cameras(9, 7))


# ---------------------------------------------------------------------------------------------- pose LM, batched
def _pose_dev(mode, problems):
    """One pl_pose_optimization_dev launch over the problems ([B][cap] torch CUDA buffers, counts unclamped)."""
    import torch
    B = len(problems)
    T0 = np.stack([p["Tcw0"].reshape(16) for p in problems]).astype(np.float32)
    K = np.stack([p["K"] for p in problems]).astype(np.float32)
    npt = np.array([len(p["pt_obs"]) for p in problems], np.int32); nln = np.array([len(p["line_func"]) for p in problems], np.int32)
    obs = np.zeros((B, CAP_P, 2), np.float32); w = np.zeros((B, CAP_P), np.float32); X = np.zeros((B, CAP_P, 3), np.float32)
    lf = np.zeros((B, CAP_L, 3)); lX = np.zeros((B, CAP_L, 6))
    for b, p in enumerate(problems):
        _, _, po, pw, px, plf, plx = pose_args(p)
        obs[b, :len(po)] = po; w[b, :len(po)] = pw; X[b, :len(po)] = px; lf[b, :len(plf)] = plf; lX[b, :len(plf)] = plx
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in dict(T0=T0, K=K, npt=npt, nln=nln, obs=obs, w=w, X=X, lf=lf, lX=lX).items()}
    L = pl.lib()
    L.pl_pose_optimization_scratch_doubles.restype = C.c_size_t
    L.pl_pose_optimization_scratch_doubles.argtypes = [C.c_int] * 3
    scratch = torch.zeros(int(L.pl_pose_optimization_scratch_doubles(B, CAP_P, CAP_L)), dtype=torch.float64, device="cuda")
    Tout = torch.zeros((B, 16), dtype=torch.float32, device="cuda")
    po = torch.full((B, CAP_P), SENTINEL, dtype=torch.uint8, device="cuda"); lo = torch.full((B, CAP_L), SENTINEL, dtype=torch.uint8, device="cuda")
    inl = torch.zeros(B, dtype=torch.int32, device="cuda"); its = torch.zeros(B, dtype=torch.int32, device="cuda")
    f = L.pl_pose_optimization_dev
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_int] + [C.c_void_p] * 9
    ptr = lambda t: C.c_void_p(t.data_ptr())
    torch.cuda.synchronize()
    pl.check(f(mode, B, ptr(d["T0"]), ptr(d["K"]), ptr(d["npt"]), CAP_P, ptr(d["obs"]), ptr(d["w"]), ptr(d["X"]), ptr(d["nln"]), CAP_L,
               ptr(d["lf"]), ptr(d["lX"]), ptr(Tout), ptr(po), ptr(lo), ptr(inl), ptr(its), ptr(scratch), None))
    torch.cuda.synchronize()
    return Tout.cpu().numpy().reshape(B, 4, 4), po.cpu().numpy(), lo.cpu().numpy(), inl.cpu().numpy(), its.cpu().numpy()


def _pose_single(mode, a):
    """pl_pose_optimization (the host entry, one problem) with both masks pre-filled with SENTINEL."""
    Tcw, K, obs, w, X, lf, lX = (np.ascontiguousarray(v) for v in a)
    Tout = np.zeros((4, 4), np.float32)
    po = np.full(max(len(obs), 1), SENTINEL, np.uint8); lo = np.full(max(len(lf), 1), SENTINEL, np.uint8)
    its = C.c_int(-1)
    f = pl.lib().pl_pose_optimization
    f.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 6
    ptr = lambda v: v.ctypes.data_as(C.c_void_p)
    n = pl.check(f(mode, ptr(Tcw), ptr(K), len(obs), ptr(obs), ptr(w), ptr(X), len(lf), ptr(lf), ptr(lX), ptr(Tout), ptr(po), ptr(lo),
                   C.byref(its)))
    return n, Tout, po[:len(obs)], lo[:len(lf)], its.value


SENTINEL = 0xA5       # a mask byte the kernel did not write


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_batched_pose_optimization_with_a_camera_per_problem(mode):
    """Each problem b against the oracle with ITS camera, and bit for bit against the single-problem entry (the kernel has no
    atomics: a problem's arithmetic does not depend on the batch around it).  Problem 13 is over both capacities.  The masks
    the mode defines (points unless mode 2, lines unless mode 1) are compared; the other one, and every byte past a problem's
    count, must be left as the caller passed it, in the batch and in the host entry."""
    probs = pose_batch()
    assert len(probs[13]["pt_obs"]) > CAP_P and len(probs[13]["line_func"]) > CAP_L
    T, po, lo, inl, its = _pose_dev(mode, probs)
    ran = 0
    for b, p in enumerate(probs):
        a = pose_args(p)
        n, m = len(a[2]), len(a[5])
        on, oT, opo, olo, oits = oracle.pose_optimization(mode, *a)
        _close(T[b], oT)
        assert inl[b] == on and its[b] == oits, (b, inl[b], on, its[b], oits)
        sn, sT, spo, slo, sits = _pose_single(mode, a)
        assert sT.tobytes() == T[b].tobytes() and sn == inl[b] and sits == its[b], b
        if mode != 2:
            assert np.array_equal(po[b, :n], opo.astype(np.uint8)) and np.array_equal(spo, po[b, :n]), b
        else:
            assert (po[b, :n] == SENTINEL).all() and (spo == SENTINEL).all(), b
        if mode != 1:
            assert np.array_equal(lo[b, :m], olo.astype(np.uint8)) and np.array_equal(slo, lo[b, :m]), b
        else:
            assert (lo[b, :m] == SENTINEL).all() and (slo == SENTINEL).all(), b
        assert (po[b, n:] == SENTINEL).all() and (lo[b, m:] == SENTINEL).all(), b
        ran += oits > 0
    assert ran >= (18 if mode < 2 else 13)


# ---------------------------------------------------------------------------------------------- local BA
def test_local_ba_with_per_keyframe_cameras_and_current_keyframe_camera():
    p = lba_camera_window()
    assert len(np.unique(p["kf_K"], axis=0)) == len(p["kf_K"]) and not (p["kf_K"] == p["K_end"]).all(axis=1).any()
    check_local(p)


def test_local_ba_lines_only_window():
    p = lba_lines_only_window()
    g, o = check_local(p)
    assert np.array_equal(g["pt_Xw"], p["pt_Xw"]) and o["its"] >= 10


def lba_32_free_window():
    return synth.synth_ba_problem(8, n_free=33, n_fixed=12, n_pt=1500, n_ln=200)


def lba_mirrored_point_window():
    """Window 4 plus a point behind its first free keyframe k at -X_c of a point in front of it, observed by k alone at the pixel
    both project to.  Returns (window, k)."""
    p = synth.synth_ba_problem(4, n_free=8, n_fixed=10, n_pt=600, n_ln=80)
    k = int(np.nonzero(p["kf_fixed"] == 0)[0][0])
    T = p["kf_Tcw"][k].reshape(4, 4).astype(np.float64)
    Xw = (T[:3, :3].T @ (-np.array([0.4, -0.3, 5.0]) - T[:3, 3])).astype(np.float32)
    Xc = T[:3, :3] @ Xw.astype(np.float64) + T[:3, 3]
    K = p["kf_K"][k].astype(np.float64)
    uv = np.array([Xc[0] / Xc[2] * K[0] + K[2], Xc[1] / Xc[2] * K[1] + K[3]], np.float32)
    q = dict(p)
    q.update(pt_Xw=np.concatenate([p["pt_Xw"], Xw[None]]), pe_kf=np.r_[p["pe_kf"], np.int32(k)].astype(np.int32),
             pe_pt=np.r_[p["pe_pt"], np.int32(len(p["pt_Xw"]))].astype(np.int32), pe_obs=np.concatenate([p["pe_obs"], uv[None]]),
             pe_inv_sigma2=np.r_[p["pe_inv_sigma2"], np.float32(1)].astype(np.float32))
    return q, k


def lba_outlier_keyframe_window():
    """Window 6 in which every observation of its second free keyframe k is off by 60-120 px.  k keeps only its observations of
    points that three other keyframes see (a point seen by fewer could be moved onto the wrong observation) and none of its line
    observations (same reason).  Returns (window, k)."""
    p = synth.synth_ba_problem(6, n_free=8, n_fixed=10, n_pt=600, n_ln=80)
    k = int(np.nonzero(p["kf_fixed"] == 0)[0][1])
    others = np.bincount(p["pe_pt"][p["pe_kf"] != k], minlength=len(p["pt_Xw"]))
    keep = (p["pe_kf"] != k) | (others[p["pe_pt"]] >= 3)
    lkeep = p["le_kf"] != k
    q = dict(p)
    q.update({f: p[f][keep] for f in ("pe_kf", "pe_pt", "pe_obs", "pe_inv_sigma2")})
    q.update({f: p[f][lkeep] for f in ("le_kf", "le_ln", "le_func")})
    sel = q["pe_kf"] == k
    r = np.random.default_rng(3)
    a, d = r.uniform(0, 2 * np.pi, sel.sum()), r.uniform(60, 120, sel.sum())
    q["pe_obs"] = q["pe_obs"].copy()
    q["pe_obs"][sel] += (np.stack([np.cos(a), np.sin(a)], 1) * d[:, None]).astype(np.float32)
    return q, k


def test_local_ba_with_32_free_keyframes():
    """32 free keyframes (keyframe 0 is always fixed): a 192 x 192 reduced system, past every earlier window."""
    p = lba_32_free_window()
    assert (p["kf_fixed"] == 0).sum() == 32
    check_local(p)


def test_local_ba_point_erased_by_the_depth_test_alone():
    """The mirrored point's reprojection chi2 stays tiny: only the depth test (!(z > 0), Optimizer.cc:1964-1967) marks and
    erases it."""
    q, k = lba_mirrored_point_window()
    g, o = check_local(q)
    K = q["kf_K"][k].astype(np.float64)
    To = o["kf_Tcw"][k].reshape(4, 4).astype(np.float64)
    c = To[:3, :3] @ o["pt_Xw"][-1].astype(np.float64) + To[:3, 3]
    r = q["pe_obs"][-1] - np.array([c[0] / c[2] * K[0] + K[2], c[1] / c[2] * K[1] + K[3]])
    assert c[2] < 0 and (r * r).sum() < 5.991
    assert o["pe_erase"][-1] and g["pe_erase"][-1]


def test_local_ba_keyframe_with_only_gross_outliers_drops_out():
    """After the robust pass all of k's edges are gated, so the second optimize runs without that keyframe."""
    q, k = lba_outlier_keyframe_window()
    g, o = check_local(q)
    sel = q["pe_kf"] == k
    assert sel.sum() >= 20 and not (q["le_kf"] == k).any()
    assert o["pe_erase"][sel].all()


def test_local_ba_stop_flag_set_before_the_call():
    import torch
    p = synth.synth_ba_problem(4, n_free=8, n_fixed=10, n_pt=600, n_ln=80)
    stop = torch.ones(1, dtype=torch.int32, device="cuda")
    g = pl.LocalBundleAdjustmentWithLine(p, stop.data_ptr())
    o = oracle.local_ba(p, stop_flag=np.array([1], np.int32))
    assert g["its"] == 0 == o["its"]
    assert g["kf_Tcw"].tobytes() == p["kf_Tcw"].tobytes() == o["kf_Tcw"].tobytes()
    assert not g["pe_erase"].any() and not g["le_erase"].any() and not o["pe_erase"].any() and not o["le_erase"].any()
    want = p["le_kf"][np.arange(len(p["le_kf"])) // 2]
    assert np.array_equal(g["le_erase_kf"], want) and np.array_equal(o["le_erase_kf"], want)
    assert np.array_equal(g["pt_Xw"], p["pt_Xw"]) and np.array_equal(g["ln_Xw"], o["ln_Xw"])


# ---------------------------------------------------------------------------------------------- global BA
@pytest.mark.parametrize("n_poses,seed,npt,nln,robust", [(1, 31, 150, 20, True), (5, 32, 500, 60, False), (16, 33, 1200, 150, True),
                                                         (32, 34, 2000, 250, False)])
def test_global_ba_free_pose_counts(n_poses, seed, npt, nln, robust):
    """n = 6, 30, 96, 192: under one 32-wide Cholesky tile, inside one, exactly three tiles (the trsm launch of column 0 has a
    partial CTA: 2 tiles for 4 warps), exactly six tiles (two trsm CTAs, the second with one tile)."""
    p = synth.synth_ba_problem(seed, n_free=n_poses + 1, n_fixed=0, n_pt=npt, n_ln=nln)
    assert (p["kf_fixed"] == 0).sum() == n_poses
    g, o = check_global(p, 6, robust)
    assert g["its"] >= 2


def test_global_ba_every_keyframe_fixed():
    p = synth.synth_ba_problem(35, n_free=6, n_fixed=4, n_pt=500, n_ln=60)
    p["kf_fixed"] = np.ones_like(p["kf_fixed"])
    g, o = check_global(p, 5, True)
    assert g["its"] >= 2 and np.abs(g["kf_Tcw"] - p["kf_Tcw"]).max() < 1e-6


def test_global_ba_free_keyframe_without_observations():
    p = synth.synth_ba_problem(36, n_free=6, n_fixed=0, n_pt=500, n_ln=60)
    T = p["kf_Tcw"][1].reshape(4, 4).copy(); T[:3, 3] += (0.05, -0.02, 0.01)
    p.update(kf_Tcw=np.concatenate([p["kf_Tcw"], T.reshape(1, 16)]), kf_fixed=np.r_[p["kf_fixed"], np.uint8(0)].astype(np.uint8),
             kf_K=np.concatenate([p["kf_K"], p["kf_K"][:1]]))
    g, o = check_global(p, 6, True)
    assert np.abs(g["kf_Tcw"][-1] - p["kf_Tcw"][-1]).max() < 1e-6


def test_global_ba_lines_only_map():
    p = without_points(synth.synth_ba_problem(37, n_free=8, n_fixed=0, n_pt=50, n_ln=150, Ks=keyframe_cameras(8, 137)))
    g, o = check_global(p, 6, True)
    assert np.array_equal(g["pt_Xw"], p["pt_Xw"])


def test_global_ba_with_per_keyframe_cameras():
    p = gba_camera_map()
    assert len(np.unique(p["kf_K"], axis=0)) == len(p["kf_K"])
    check_global(p, 6, True)


# ---------------------------------------------------------------------------------------------- front end
def test_tracking_stage_with_a_camera_per_frame():
    """The tracking stage places frame b's synthetic map on the previous keypoints' rays and projects it with frame b's camera;
    both projection searches and both pose optimisations of every frame equal the oracle's with that frame's K (pose and inlier
    count: the iteration counts of three of these problems depend on rounding, see pose_outcome_is_rounding_stable)."""
    B = 4
    frames = synth.synth_sequence(B, 640, 480, seed=9)
    problems = frontend_problems()
    fe = pl.Frontend(640, 480, max_batch=B, lm_caps=(320, 88))
    fe.set_wrap(True)
    fe.set_pose_problems(problems)
    fe.set_tracking(True)
    out = fe.run(frames)
    t0, t1 = fe.fetch_tracking(B, 0), fe.fetch_tracking(B, 1)
    sf = np.cumprod(np.r_[np.float32(1), np.full(7, np.float32(1.2))]).astype(np.float32)
    bounds = [0, 0, 640, 480]
    for b in range(B):
        a = (b - 1) % B
        K = np.asarray(problems[b]["K"], np.float32)
        n, npv = out["n"][b], out["n"][a]
        ck, cd, pk, pd = out["kps"][b, :n], out["desc"][b, :n], out["kps"][a, :npv], out["desc"][a, :npv]
        T = np.asarray(problems[b]["Tcw0"], np.float32).reshape(4, 4)
        pos = t0["map_pos"][b, :npv]
        Xc = pos.astype(np.float64) @ T[:3, :3].T.astype(np.float64) + T[:3, 3]
        uv = np.stack([Xc[:, 0] / Xc[:, 2] * K[0] + K[2], Xc[:, 1] / Xc[:, 2] * K[1] + K[3]], 1)
        assert npv > 100 and np.abs(uv - np.stack([pk["x"], pk["y"]], 1)).max() < 2e-2 and Xc[:, 2].min() > 1.0, b
        valid = np.ones(npv, np.uint8)
        nm, m = oracle.search_by_projection_last(ck, cd, bounds, T, K, sf, valid, pos, pd, pk["octave"], pk["angle"], 15.0, True)
        if nm < 20:
            nm, m = oracle.search_by_projection_last(ck, cd, bounds, T, K, sf, valid, pos, pd, pk["octave"], pk["angle"], 30.0, True)
        assert t0["n_pt"][b] == nm and np.array_equal(t0["pt_match"][b, :n], m), b
        view = valid.copy(); view[m[m >= 0]] = 0
        nm2, m2 = oracle.search_by_projection_points(ck, cd, bounds, sf, view, np.stack([pk["x"], pk["y"]], 1), pk["octave"],
                                                     np.ones(npv, np.float32), pd, 1.0, 0.8, (m >= 0).astype(np.uint8))
        assert t1["n_pt"][b] == nm2 and np.array_equal(t1["pt_match"][b, :n], m2), b
        p = problems[b]
        on, oT, opo, olo, oits = oracle.pose_optimization(0, *pose_args(p))
        for call in range(2):
            _close(out["poses"][call, b].reshape(4, 4), oT)
            assert out["inliers"][call, b] == on, (call, b)
    assert t0["n_pt"].min() > 50


def test_frontend_refuses_pose_problems_over_its_capacities():
    """pl_frontend_set_pose_problems(_async) return PL_ERR_ARG for a problem with more correspondences than lm_caps, instead of
    dropping the surplus; problems at the capacities are accepted."""
    B, cp, cl = 2, 40, 12
    fe = pl.Frontend(640, 480, max_batch=B, lm_caps=(cp, cl))
    L = pl.lib()
    L.pl_frontend_set_pose_problems_async.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 10
    L.pl_frontend_set_pose_problems_async.restype = C.c_longlong
    arrs = [np.zeros((B, 16), np.float32), np.tile(np.float32(synth.TUM1_K), (B, 1)), None, np.zeros((B, cp, 2), np.float32),
            np.zeros((B, cp), np.float32), np.zeros((B, cp, 3), np.float32), None, np.zeros((B, cl, 3)), np.zeros((B, cl, 6))]
    for npt, nln, ok in [((cp, cp), (cl, 0), True), ((cp, cp + 1), (cl, 0), False), ((cp, 3), (cl + 1, cl), False), ((-1, 3), (0, 0), False)]:
        arrs[2], arrs[6] = np.array(npt, np.int32), np.array(nln, np.int32)
        ptrs = [a.ctypes.data_as(C.c_void_p) for a in arrs]
        rc = L.pl_frontend_set_pose_problems(fe._h, B, *ptrs)
        rca = L.pl_frontend_set_pose_problems_async(fe._h, B, *ptrs, None)
        assert (rc == 0 and rca > 0) if ok else (rc == -1 and rca == -1), (npt, nln, rc, rca)
    import torch
    torch.cuda.synchronize()
