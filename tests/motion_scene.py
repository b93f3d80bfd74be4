"""Test helpers for Tracking::TrackWithMotionModel on the planar scene of tests/track_scene.py: cv::Mat's fp32 4x4 product, the
CPU composites of the motion model (Tracking.cc:1316-1431), of the local-map step after it (with the entries it discarded) and of
the velocity update (:492-501), constant-velocity streams, a map with a few entries moved so that the pose optimisation rejects
them, and the named branch cases the tests run.
"""
import numpy as np

import oracle
from track_scene import (BOUNDS, INV_SIGMA2, K0, K1, LOG_SF, SF, camera_center, features, perturb, pose, scene_map,
                         track_local_map_oracle)


def mat4(A, B):
    """cv::Mat's fp32 4x4 product: ((a0 b0 + a1 b1) + a2 b2) + a3 b3, every operation rounded (the oracle's Mat::operator*)."""
    A = np.asarray(A, np.float32).reshape(4, 4); B = np.asarray(B, np.float32).reshape(4, 4)
    s = A[:, 0:1] * B[0:1, :]
    for k in range(1, 4):
        s = s + A[:, k:k + 1] * B[k:k + 1, :]
    return s.astype(np.float32)


def velocity_oracle(Tcw, Tcw_last):
    """mVelocity = mCurrentFrame.mTcw * LastTwc, LastTwc = [Rcw^T | Ow] of the last frame (Tracking.cc:492-501)."""
    L = np.asarray(Tcw_last, np.float32).reshape(4, 4)
    W = np.eye(4, dtype=np.float32)
    W[:3, :3] = L[:3, :3].T; W[:3, 3] = camera_center(L)
    return mat4(Tcw, W)


def track_motion_model_oracle(m, keys, desc, kl, ldesc, lf, K, last, variant="reference"):
    """One frame of Tracking::TrackWithMotionModel (monocular, localisation mode, Tracking.cc:1316-1431) on the CPU oracles.
    last: dict(keys, kl, point_map, point_outlier, line_map, line_outlier, Tcw, velocity) of the last frame."""
    n, nl = len(keys), len(kl)
    K = np.asarray(K, np.float32)
    G = mat4(last["velocity"], last["Tcw"])
    pm0 = np.asarray(last["point_map"], np.int32); po0 = np.asarray(last["point_outlier"]).astype(bool)
    lm0 = np.asarray(last["line_map"], np.int32); lo0 = np.asarray(last["line_outlier"]).astype(bool)
    Np, Nl = len(m["pt_pos"]), len(m["ln_pos"])
    valid = (pm0 >= 0) & ~po0 & (pm0 < Np)
    prow = np.where(valid, pm0, 0)
    lk = last["keys"]

    def search(th):
        return oracle.search_by_projection_last(keys, desc, BOUNDS, G, K, SF, valid.astype(np.uint8), m["pt_pos"][prow].reshape(-1, 3),
                                                m["pt_desc"][prow].reshape(-1, 32), lk["octave"], lk["angle"], th, True)
    nm1, pm1 = search(15.0)
    lvalid = (lm0 >= 0) & ~lo0 & (lm0 < Nl)
    lrow = np.where(lvalid, lm0, 0)
    liv, lpr, llv, lvc = oracle.is_in_frustum_lines(G, camera_center(G), K, BOUNDS, LOG_SF, 0.5, m["ln_pos"][lrow].reshape(-1, 6),
                                                    m["ln_normal"][lrow].reshape(-1, 3), m["ln_min_dist"][lrow], m["ln_max_dist"][lrow])
    liv[~lvalid] = 0; lpr[~lvalid] = 0; llv[~lvalid] = 0; lvc[~lvalid] = 0
    lmatches, lmatch = oracle.line_search_by_projection_last(kl, lf, ldesc, BOUNDS, liv, lpr, m["ln_desc"][lrow].reshape(-1, 32),
                                                             np.asarray(last["kl"]["lineLength"], np.float32), 15.0)
    retried = nm1 < 20
    nm2, pm2 = search(30.0) if retried else (nm1, pm1)
    nmatches = nm2
    pmatch = np.asarray(pm2[:n], np.int32); lmatch = np.asarray(lmatch[:nl], np.int32)
    point_map = np.where(pmatch >= 0, pm0[np.maximum(pmatch, 0)] if len(pm0) else -1, -1).astype(np.int32)
    line_map = np.where(lmatch >= 0, lm0[np.maximum(lmatch, 0)] if len(lm0) else -1, -1).astype(np.int32)
    r = dict(guess=G, pt_match=np.asarray(pm1[:n], np.int32), pt_match_retry=np.asarray(pm2[:n], np.int32), retried=int(retried),
             ln_match=lmatch, ln_in_view=liv, ln_proj=lpr, ln_level=llv, ln_view_cos=lvc, point_seen=np.full(n, -1, np.int32),
             line_seen=np.full(nl, -1, np.int32))
    if nmatches < 20 and lmatches < 5:        # return false: the guess and the search's matches stay, mbVO is not touched
        empty = dict(pt_obs=np.zeros((0, 2), np.float32), pt_inv_sigma2=np.zeros(0, np.float32), pt_Xw=np.zeros((0, 3), np.float32),
                     line_func=np.zeros((0, 3)), line_Xw=np.zeros((0, 6)))
        return dict(r, Tcw=G, point_map=point_map, line_map=line_map, nmatches=np.array([nmatches, lmatches], np.int32), ok=0, vo=None,
                    problem=empty, prob_n_points=0, prob_n_lines=0, solved=False)
    pi = np.nonzero(point_map >= 0)[0]; li = np.nonzero(line_map >= 0)[0]
    prob = dict(pt_obs=np.stack([keys["x"][pi], keys["y"][pi]], 1).astype(np.float32), pt_inv_sigma2=INV_SIGMA2[keys["octave"][pi]],
                pt_Xw=m["pt_pos"][point_map[pi]].reshape(-1, 3).astype(np.float32),
                line_func=np.asarray(lf, np.float64).reshape(-1, 3)[li], line_Xw=m["ln_pos"][line_map[li]].reshape(-1, 6).astype(np.float64))
    _, T, po, lo, _ = oracle.pose_optimization(0, G, K, prob["pt_obs"], prob["pt_inv_sigma2"], prob["pt_Xw"], prob["line_func"],
                                               prob["line_Xw"], variant=variant)
    pout = pi[po] if len(pi) else pi
    lout = li[lo] if len(li) else li
    r["point_seen"][pout] = point_map[pout]; r["line_seen"][lout] = line_map[lout]
    point_map = point_map.copy(); line_map = line_map.copy()
    point_map[pout] = -1; line_map[lout] = -1
    nm = nmatches - len(pout); lmn = lmatches - len(lout)
    nmatches_map = int((point_map >= 0).sum())     # every entry of a fixed map has Observations() > 0
    return dict(r, Tcw=T, point_map=point_map, line_map=line_map, nmatches=np.array([nm, lmn], np.int32), ok=int(nm > 20),
                vo=int(nmatches_map < 10), problem=prob, prob_n_points=len(pi), prob_n_lines=len(li), solved=True)


def track_local_map_seen_oracle(m, keys, desc, kl, ldesc, lf, Tcw0, K, local_pts, local_lns, frames_since_reloc, max_frames,
                                point_map_in=None, line_map_in=None, point_seen=None, line_seen=None, variant="reference"):
    """track_local_map_oracle after TrackWithMotionModel: the entries it discarded (point_seen / line_seen, -1 none) keep
    mbTrackInView = false like held matches (mnLastFrameSeen == mnId, Tracking.cc:1778, :1833) but are not pre-assigned."""
    n, nl = len(keys), len(kl)
    pm_in = np.full(n, -1, np.int32) if point_map_in is None else np.asarray(point_map_in, np.int32)[:n]
    lm_in = np.full(nl, -1, np.int32) if line_map_in is None else np.asarray(line_map_in, np.int32)[:nl]
    ps = np.full(n, -1, np.int32) if point_seen is None else np.asarray(point_seen, np.int32)[:n]
    ls = np.full(nl, -1, np.int32) if line_seen is None else np.asarray(line_seen, np.int32)[:nl]
    # track_local_map_oracle excludes every index in point_map_in from the frustum test and pre-assigns the features that hold one:
    # run it with the union as "held" for the frustum, then restore the pre-assignment of the real held matches only
    lp = np.asarray(local_pts, np.int64); ll = np.asarray(local_lns, np.int64)
    excl_p = np.isin(lp, np.r_[pm_in[pm_in >= 0], ps[ps >= 0]]); excl_l = np.isin(ll, np.r_[lm_in[lm_in >= 0], ls[ls >= 0]])
    r = track_local_map_oracle(m, keys, desc, kl, ldesc, lf, Tcw0, K, lp[~excl_p], ll[~excl_l], frames_since_reloc, max_frames,
                               pm_in, lm_in, variant)
    # scatter the frustum outputs back to the full lists and renumber the match positions
    pos_p = np.nonzero(~excl_p)[0]; pos_l = np.nonzero(~excl_l)[0]
    for k, cnt, pos, ncol in (("pt_in_view", len(lp), pos_p, 0), ("pt_proj", len(lp), pos_p, 2), ("pt_level", len(lp), pos_p, 0),
                              ("pt_view_cos", len(lp), pos_p, 0), ("ln_in_view", len(ll), pos_l, 0), ("ln_proj", len(ll), pos_l, 4),
                              ("ln_level", len(ll), pos_l, 0), ("ln_view_cos", len(ll), pos_l, 0)):
        full = np.zeros((cnt, ncol) if ncol else cnt, r[k].dtype)
        full[pos] = r[k]
        r[k] = full
    r["pt_match"] = np.where(r["pt_match"] >= 0, pos_p[np.maximum(r["pt_match"], 0)] if len(pos_p) else -1, r["pt_match"]).astype(np.int32)
    r["ln_match"] = np.where(r["ln_match"] >= 0, pos_l[np.maximum(r["ln_match"], 0)] if len(pos_l) else -1, r["ln_match"]).astype(np.int32)
    return r


def shifted_map(n_pts=40, n_lns=12, dx=0.05, seed=7):
    """scene_map() with n_pts map points and n_lns map lines moved dx metres along X on the plane (about 8 px in the image):
    the searches still match them by descriptor, and the pose optimisation flags them as outliers."""
    m = dict(scene_map())
    rng = np.random.default_rng(seed)
    pi = np.sort(rng.choice(len(m["pt_pos"]), n_pts, replace=False)); li = np.sort(rng.choice(len(m["ln_pos"]), n_lns, replace=False))
    m["pt_pos"] = m["pt_pos"].copy(); m["pt_pos"][pi, 0] += np.float32(dx)
    m["ln_pos"] = m["ln_pos"].copy(); m["ln_pos"][li, 0] += dx; m["ln_pos"][li, 3] += dx
    return m, pi, li


# constant-velocity streams: frame k of stream s has pose D_s^k T_s (float64 products, stored in fp32) and camera K_s
STREAMS = [
    (pose((0.01, -0.01, 0.0), (0.06, -0.04, 0.03)), pose((0.002, -0.003, 0.001), (0.015, 0.01, -0.01)), K0),
    (pose((-0.01, 0.005, -0.006), (-0.05, 0.05, -0.04)), pose((-0.003, 0.002, 0.002), (-0.012, 0.014, 0.012)), K1),
    (pose((0.004, 0.012, 0.008), (0.02, 0.08, 0.02)), pose((0.001, -0.004, -0.002), (0.02, -0.012, 0.008)), K0),
]


def stream_pose(s, k):
    T0, D, _ = STREAMS[s]
    T = np.asarray(T0, np.float64)
    for _ in range(k):
        T = np.asarray(D, np.float64) @ T
    return T.astype(np.float32)


def last_frame(m, T, K, Tcw=None, seed=0):
    """A last frame as TrackLocalMapWithLines leaves it: the frame rendered at T, tracked from a guess 6 mm off with the whole map
    as its local map.  Returns dict(keys, kl, point_map, point_outlier, line_map, line_outlier, Tcw) (Tcw: the tracked pose unless
    given)."""
    kps, desc, kl, ldesc, lf = features(T, K)
    r = track_local_map_oracle(m, kps, desc, kl, ldesc, lf, perturb(T, 0.006, seed), K, np.arange(len(m["pt_pos"])),
                               np.arange(len(m["ln_pos"])), 5, 30)
    return dict(keys=kps, kl=kl, point_map=r["point_map"], point_outlier=r["point_outlier"], line_map=r["line_map"],
                line_outlier=r["line_outlier"], Tcw=r["Tcw"] if Tcw is None else np.asarray(Tcw, np.float32))


def motion_cases():
    """The named branch cases of TrackWithMotionModel on shifted_map(): name -> (T_true, K, last with velocity).
      plain:   stream 0, step 1, true velocity; the last frame has point and line outliers (the shifted entries), and the frame
               discards outliers of its own
      retry:   the guess 0.15 m off (about 26 px) and only last-frame keypoints of octave <= 2 valid: th = 15 finds under 20 matches,
               th = 30 finds more
      few:     stream 1, only 8 valid last-frame keypoints: retried, reaches the pose optimisation on its lines with under 10 map
               matches (vo = 1, ok = 0)
      early:   10 valid last-frame keypoints and 3 valid lines: under 20 point and 5 line matches, returns before the optimisation"""
    m, _, _ = shifted_map()
    out = {}
    T1, K = stream_pose(0, 1), STREAMS[0][2]
    last = last_frame(m, T1, K, seed=1)
    out["plain"] = (stream_pose(0, 2), K, dict(last, velocity=STREAMS[0][1]))
    V = np.array(STREAMS[0][1]).copy(); V[0, 3] += np.float32(0.15)
    out["retry"] = (stream_pose(0, 2), K, dict(last, velocity=V,
                                              point_map=np.where(last["keys"]["octave"] <= 2, last["point_map"], -1).astype(np.int32)))
    pv = np.nonzero(last["point_map"] >= 0)[0]; lv = np.nonzero(last["line_map"] >= 0)[0]
    pm = np.full_like(last["point_map"], -1); pm[pv[::40][:10]] = last["point_map"][pv[::40][:10]]
    lm = np.full_like(last["line_map"], -1); lm[lv[:3]] = last["line_map"][lv[:3]]
    out["early"] = (stream_pose(0, 2), K, dict(last, velocity=STREAMS[0][1], point_map=pm, line_map=lm))
    T1, K = stream_pose(1, 1), STREAMS[1][2]
    last = last_frame(m, T1, K, seed=1)
    pv = np.nonzero(last["point_map"] >= 0)[0]
    pm = np.full_like(last["point_map"], -1); pm[pv[::40][:8]] = last["point_map"][pv[::40][:8]]
    out["few"] = (stream_pose(1, 2), K, dict(last, velocity=STREAMS[1][1], point_map=pm))
    return m, out
