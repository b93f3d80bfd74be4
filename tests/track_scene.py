"""Test helpers for Tracking::TrackLocalMapWithLines: a planar scene with known poses, and the CPU composite of the step.

Scene: the textured plane Z = DEPTH (synth_frame) in front of camera 0 (identity pose, TUM1 camera).  Frame k, with pose T_k and its
own K_k, is rendered by casting each pixel's ray onto the plane and sampling frame 0 bilinearly.  The map is frame 0's keypoints and
keylines back-projected onto the plane, with MapPoint.cc:56-64 / MapLine.cpp:50-59's normals and distances and frame 0's descriptors.

track_local_map_oracle() composes the existing CPU oracles in the reference's order (Tracking.cc:1491-1562, 1751-1855).
"""
import functools

import numpy as np

import oracle
from plslam_b200 import synth

W, H = 640, 480
DEPTH = 3.0
K0 = np.array(synth.TUM1_K, np.float32)
NLEV, SCALE = 8, 1.2
SF = np.cumprod(np.r_[np.float32(1), np.full(NLEV - 1, np.float32(SCALE))]).astype(np.float32)   # ORBextractor.cc:419-426
INV_SIGMA2 = (np.float32(1) / (SF * SF)).astype(np.float32)
LOG_SF = float(np.float32(np.log(np.float32(SCALE))))
BOUNDS = np.array([0, 0, W, H], np.float32)


def rot(rx, ry, rz):
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    return (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
            @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))


def pose(r, t):
    T = np.eye(4)
    T[:3, :3] = rot(*r); T[:3, 3] = t
    return T.astype(np.float32)


@functools.lru_cache(maxsize=None)
def frame0():
    return synth.synth_frame(W, H, 1)


def render(T, K):
    """Frame with pose T (Tcw) and camera K: each pixel's ray hits the plane Z = DEPTH, frame 0 is sampled there bilinearly."""
    T = np.asarray(T, np.float64); K = np.asarray(K, np.float64)
    R, t = T[:3, :3], T[:3, 3]
    Ow = -R.T @ t
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    d = np.stack([(u - K[2]) / K[0], (v - K[3]) / K[1], np.ones_like(u)], -1) @ R        # R^T d per pixel
    s = (DEPTH - Ow[2]) / d[..., 2]
    X = Ow[0] + s * d[..., 0]; Y = Ow[1] + s * d[..., 1]
    x0 = X / DEPTH * K0[0] + K0[2]; y0 = Y / DEPTH * K0[1] + K0[3]
    img = frame0().astype(np.float64)
    ix = np.floor(x0).astype(int); iy = np.floor(y0).astype(int); fx = x0 - ix; fy = y0 - iy
    inside = (ix >= 0) & (iy >= 0) & (ix < W - 1) & (iy < H - 1)
    ixc = np.clip(ix, 0, W - 2); iyc = np.clip(iy, 0, H - 2)
    val = (img[iyc, ixc] * (1 - fx) * (1 - fy) + img[iyc, ixc + 1] * fx * (1 - fy) + img[iyc + 1, ixc] * (1 - fx) * fy
           + img[iyc + 1, ixc + 1] * fx * fy)
    return np.where(inside, np.clip(np.rint(val), 0, 255), 128).astype(np.uint8)


@functools.lru_cache(maxsize=None)
def _features(key):
    T, K = key
    img = frame0() if T is None else render(np.array(T, np.float32).reshape(4, 4), np.array(K, np.float32))
    kps, desc = oracle.OrbOracle(1000, SCALE, NLEV, 20, 7).extract(img)
    kl, ldesc, lf = oracle.line_extract(img)
    return kps, desc, kl, ldesc, lf


def features(T=None, K=None):
    """(keys, desc, keylines, line desc, line functions) of frame 0 (T = None) or of the frame rendered with pose T and camera K."""
    key = (None, None) if T is None else (tuple(np.asarray(T, np.float32).ravel().tolist()), tuple(np.asarray(K, np.float32).tolist()))
    return _features(key)


@functools.lru_cache(maxsize=None)
def scene_map():
    """Frame 0's keypoints / keylines on the plane (camera 0 at the origin, so Ow = 0)."""
    kps, desc, kl, ldesc, _ = features()
    z = np.float32(DEPTH)
    pos = np.stack([(kps["x"] - K0[2]) / K0[0] * z, (kps["y"] - K0[3]) / K0[1] * z, np.full(len(kps), z)], 1).astype(np.float32)
    dist = np.linalg.norm(pos.astype(np.float64), axis=1).astype(np.float32)
    normal = (pos / dist[:, None]).astype(np.float32)
    pmax = (dist * SF[kps["octave"]]).astype(np.float32)
    pmin = (pmax / SF[-1]).astype(np.float32)

    def back(x, y):
        return np.stack([(x - K0[2]) / K0[0] * DEPTH, (y - K0[3]) / K0[1] * DEPTH, np.full(len(x), DEPTH)], 1).astype(np.float64)
    lpos = np.concatenate([back(kl["startPointX"].astype(np.float64), kl["startPointY"].astype(np.float64)),
                           back(kl["endPointX"].astype(np.float64), kl["endPointY"].astype(np.float64))], 1)
    mid = 0.5 * (lpos[:, :3] + lpos[:, 3:])
    ldist = np.linalg.norm(mid, axis=1)
    lnormal = mid / ldist[:, None]
    lmax = ldist.astype(np.float32)                 # one line octave: mvScaleFactorsLine = {1}
    return dict(pt_pos=pos, pt_normal=normal, pt_min_dist=pmin, pt_max_dist=pmax, pt_desc=np.ascontiguousarray(desc),
                ln_pos=lpos, ln_normal=lnormal, ln_min_dist=lmax.copy(), ln_max_dist=lmax, ln_desc=np.ascontiguousarray(ldesc))


def camera_center(T):
    """mOw = -mRcw.t() * mtcw (Frame.cc:552-558) in fp32, summed left to right like the device's camera_center."""
    T = np.asarray(T, np.float32).reshape(4, 4)
    Ow = np.zeros(3, np.float32)
    for i in range(3):
        s = np.float32(-T[0, i]) * T[0, 3]
        s = np.float32(s + np.float32(-T[1, i]) * T[1, 3])
        Ow[i] = np.float32(s + np.float32(-T[2, i]) * T[2, 3])
    return Ow


def track_local_map_oracle(m, keys, desc, kl, ldesc, lf, Tcw0, K, local_pts, local_lns, frames_since_reloc, max_frames,
                           point_map_in=None, line_map_in=None, variant="reference"):
    """One frame of Tracking::TrackLocalMapWithLines in localisation mode, on the CPU oracles.  m: scene_map()-style dict."""
    n, nl = len(keys), len(kl)
    Tcw0 = np.asarray(Tcw0, np.float32).reshape(4, 4); K = np.asarray(K, np.float32)
    pm_in = np.full(n, -1, np.int32) if point_map_in is None else np.asarray(point_map_in, np.int32)[:n]
    lm_in = np.full(nl, -1, np.int32) if line_map_in is None else np.asarray(line_map_in, np.int32)[:nl]
    lp = np.asarray(local_pts, np.int64); ll = np.asarray(local_lns, np.int64)
    Ow = camera_center(Tcw0)
    # SearchLocalPoints / SearchLocalLines step 1 and 2: held map points keep mbTrackInView = false, the others go through isInFrustum
    iv, pr, lv, vc = oracle.is_in_frustum_points(Tcw0, Ow, K, BOUNDS, LOG_SF, NLEV, 0.5, m["pt_pos"][lp], m["pt_normal"][lp],
                                                 m["pt_min_dist"][lp], m["pt_max_dist"][lp])
    held = np.isin(lp, pm_in[pm_in >= 0])
    iv[held] = 0; pr[held] = 0; lv[held] = 0; vc[held] = 0
    liv, lpr, llv, lvc = oracle.is_in_frustum_lines(Tcw0, Ow, K, BOUNDS, LOG_SF, 0.5, m["ln_pos"][ll], m["ln_normal"][ll],
                                                    m["ln_min_dist"][ll], m["ln_max_dist"][ll])
    lheld = np.isin(ll, lm_in[lm_in >= 0])
    liv[lheld] = 0; lpr[lheld] = 0; llv[lheld] = 0; lvc[lheld] = 0
    th = 5.0 if frames_since_reloc < 2 else 1.0
    _, pmatch = oracle.search_by_projection_points(keys, desc, BOUNDS, SF, iv, pr, lv, vc, m["pt_desc"][lp].reshape(-1, 32), th, 0.8,
                                                   (pm_in >= 0).astype(np.uint8))
    _, lmatch = oracle.line_search_by_projection_lines(kl, lf, ldesc, BOUNDS, liv, lpr, lvc, m["ln_desc"][ll].reshape(-1, 32), th, 0.7,
                                                       (lm_in >= 0).astype(np.uint8))
    pmatch = np.asarray(pmatch[:n], np.int32); lmatch = np.asarray(lmatch[:nl], np.int32)
    point_map = np.where(pmatch == -2, pm_in, np.where(pmatch >= 0, lp[np.maximum(pmatch, 0)] if len(lp) else -1, -1)).astype(np.int32)
    line_map = np.where(lmatch == -2, lm_in, np.where(lmatch >= 0, ll[np.maximum(lmatch, 0)] if len(ll) else -1, -1)).astype(np.int32)
    pi = np.nonzero(point_map >= 0)[0]; li = np.nonzero(line_map >= 0)[0]
    prob = dict(pt_obs=np.stack([keys["x"][pi], keys["y"][pi]], 1).astype(np.float32), pt_inv_sigma2=INV_SIGMA2[keys["octave"][pi]],
                pt_Xw=m["pt_pos"][point_map[pi]].astype(np.float32), line_func=np.asarray(lf, np.float64).reshape(-1, 3)[li],
                line_Xw=m["ln_pos"][line_map[li]].astype(np.float64))
    nret, T, po, lo, its = oracle.pose_optimization(0, Tcw0, K, prob["pt_obs"], prob["pt_inv_sigma2"], prob["pt_Xw"], prob["line_func"],
                                                   prob["line_Xw"], variant=variant)
    point_outlier = np.zeros(n, np.uint8); point_outlier[pi] = po
    line_outlier = np.zeros(nl, np.uint8); line_outlier[li] = lo
    inl = int((~po).sum()) if len(pi) else 0
    linl = int((~lo).sum()) if len(li) else 0
    ok = int(inl >= (50 if frames_since_reloc < max_frames else 30))
    return dict(Tcw=T, point_map=point_map, point_outlier=point_outlier, line_map=line_map, line_outlier=line_outlier,
                inliers=np.array([inl, linl], np.int32), ok=ok, pt_in_view=iv, pt_proj=pr, pt_level=lv, pt_view_cos=vc,
                ln_in_view=liv, ln_proj=lpr, ln_level=llv, ln_view_cos=lvc, pt_match=pmatch, ln_match=lmatch, problem=prob,
                prob_n_points=len(pi), prob_n_lines=len(li), iterations=its)


def outcome_is_rounding_stable(prob, Tcw0, K):
    """The pose problem ends with the same masks and inlier count under every rounding variant of the LM oracle."""
    outs = [oracle.pose_optimization(0, Tcw0, K, prob["pt_obs"], prob["pt_inv_sigma2"], prob["pt_Xw"], prob["line_func"], prob["line_Xw"],
                                     variant=v) for v in oracle.POSE_VARIANTS]
    return all(o[0] == outs[0][0] and np.array_equal(o[2], outs[0][2]) and np.array_equal(o[3], outs[0][3]) for o in outs)


# frames of the known-answer tests: true pose, camera, and the translation error of the guess
K1 = np.array([480.0, 482.0, 322.0, 236.0], np.float32)     # a second camera in the same batch
TRUE = [
    (pose((0.01, -0.015, 0.005), (0.10, -0.05, 0.08)), K0),
    (pose((-0.012, 0.01, -0.008), (-0.08, 0.06, -0.05)), K1),
    (pose((0.005, 0.02, 0.01), (0.05, 0.10, 0.02)), K0),
    (pose((-0.02, -0.005, 0.012), (-0.12, -0.04, 0.10)), K1),
]


def perturb(T, dt, seed):
    """T with its translation moved by |dt| metres in a seeded direction (1 px at the plane is about DEPTH / fx = 0.006 m)."""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=3); d /= np.linalg.norm(d)
    G = np.array(T, np.float32).copy()
    G[:3, 3] += np.float32(dt) * d.astype(np.float32)
    return G


def plane_reprojection_gap(Ta, Tb, K):
    """Largest distance in pixels between the projections through Ta and Tb (camera K) of a 15 x 11 grid of plane points that
    camera 0 sees from 40 px inside its image border.  On a plane, a translation error along one direction is largely compensated
    by a rotation, so this is the error a user of the pose sees."""
    u, v = np.meshgrid(np.linspace(40, W - 40, 15), np.linspace(40, H - 40, 11))
    X = np.stack([(u.ravel() - K0[2]) / K0[0] * DEPTH, (v.ravel() - K0[3]) / K0[1] * DEPTH, np.full(u.size, DEPTH)], 1)
    K = np.asarray(K, np.float64)

    def proj(T):
        T = np.asarray(T, np.float64).reshape(4, 4)
        c = X @ T[:3, :3].T + T[:3, 3]
        return np.stack([c[:, 0] / c[:, 2] * K[0] + K[2], c[:, 1] / c[:, 2] * K[1] + K[3]], 1)
    return float(np.linalg.norm(proj(Ta) - proj(Tb), axis=1).max())


def pad(a, cap, fill=0):
    out = np.full((cap,) + a.shape[1:], fill, a.dtype)
    out[:len(a)] = a
    return out


def batch_frames(items, cap=None, capL=None):
    """items: list of (T_true, K, Tcw0, point_map_in or None, line_map_in or None) -> the frames dict of plslam_b200.track_local_map."""
    feats = [features(T, K) for T, K, _, _, _ in items]
    cap = cap or max(max(len(f[0]) for f in feats), 1)
    capL = capL or max(max(len(f[2]) for f in feats), 1)
    B = len(items)
    fr = dict(keys_un=np.zeros((B, cap), oracle.KP_DTYPE), desc=np.zeros((B, cap, 32), np.uint8), n=np.zeros(B, np.int32),
              keylines=np.zeros((B, capL), oracle.KEYLINE_DTYPE), line_func=np.zeros((B, capL, 3)), line_desc=np.zeros((B, capL, 32), np.uint8),
              nl=np.zeros(B, np.int32), bounds=BOUNDS, scale_factors=SF, inv_level_sigma2=INV_SIGMA2, log_scale_factor=LOG_SF,
              Tcw0=np.zeros((B, 4, 4), np.float32), K=np.zeros((B, 4), np.float32), point_map_in=np.full((B, cap), -1, np.int32),
              line_map_in=np.full((B, capL), -1, np.int32))
    for b, ((_, K, T0, pm, lm), (kps, desc, kl, ldesc, lf)) in enumerate(zip(items, feats)):
        n, nl = len(kps), len(kl)
        fr["keys_un"][b, :n] = kps; fr["desc"][b, :n] = desc; fr["n"][b] = n
        fr["keylines"][b, :nl] = kl; fr["line_func"][b, :nl] = np.asarray(lf).reshape(-1, 3); fr["line_desc"][b, :nl] = ldesc; fr["nl"][b] = nl
        fr["Tcw0"][b] = T0; fr["K"][b] = K
        if pm is not None:
            fr["point_map_in"][b, :n] = pm
        if lm is not None:
            fr["line_map_in"][b, :nl] = lm
    return fr, feats
