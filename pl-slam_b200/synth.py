"""Deterministic synthetic inputs (SURVEY.md §8d): frames and sequences.

Pure numpy (PCG64 seeds) so the same bytes are produced in the build container and on the GPU box.
"""
import numpy as np

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"),
                     ("response", "<f4"), ("octave", "<i4"), ("class_id", "<i4")])   # cv::KeyPoint, 28 bytes


def _gauss1d(sigma):
    r = int(3 * sigma + 0.5)
    x = np.arange(-r, r + 1, dtype=np.float64)
    k = np.exp(-x * x / (2 * sigma * sigma))
    return k / k.sum()


def _blur(img, sigma):
    k = _gauss1d(sigma)
    r = len(k) // 2
    p = np.pad(img, ((0, 0), (r, r)), mode="reflect")
    out = sum(k[i] * p[:, i:i + img.shape[1]] for i in range(len(k)))
    p = np.pad(out, ((r, r), (0, 0)), mode="reflect")
    return sum(k[i] * p[i:i + img.shape[0], :] for i in range(len(k)))


def synth_frame(w=640, h=480, seed=1, n_rect=60, n_seg=30):
    """Busy grayscale frame: blurred noise + filled rectangles + line segments (config 1)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    base = _blur(rng.random((h, w)), 2.0)
    base = (base - base.min()) / (base.max() - base.min())
    img = (base * 255.0)
    for _ in range(n_rect):
        rw, rh = rng.integers(10, 120, 2)
        x0 = rng.integers(0, max(1, w - rw)); y0 = rng.integers(0, max(1, h - rh))
        img[y0:y0 + rh, x0:x0 + rw] = rng.integers(0, 256)
    yy, xx = np.mgrid[0:h, 0:w]
    for _ in range(n_seg):
        x0, x1 = rng.integers(0, w, 2); y0, y1 = rng.integers(0, h, 2)
        t = rng.integers(1, 4); g = rng.integers(0, 256)
        dx, dy = float(x1 - x0), float(y1 - y0)
        L2 = dx * dx + dy * dy + 1e-9
        u = np.clip(((xx - x0) * dx + (yy - y0) * dy) / L2, 0, 1)
        d2 = (xx - (x0 + u * dx)) ** 2 + (yy - (y0 + u * dy)) ** 2
        img[d2 <= (t * 0.5) ** 2 + 0.25] = g
    # mild sensor noise so the texture statistics resemble a camera image
    img = img + rng.normal(0, 3.0, (h, w))
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def warp_frame(img, seed, max_t=4.0, max_rot_deg=0.5, max_ds=0.005):
    """Similarity-warped copy of img (bilinear, border clamp) — sequence frames (config 2)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    h, w = img.shape
    tx, ty = rng.uniform(-max_t, max_t, 2)
    a = np.deg2rad(rng.uniform(-max_rot_deg, max_rot_deg)); s = 1 + rng.uniform(-max_ds, max_ds)
    c, sn = np.cos(a) * s, np.sin(a) * s
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    cx, cy = w / 2, h / 2
    sx = c * (xx - cx) - sn * (yy - cy) + cx + tx
    sy = sn * (xx - cx) + c * (yy - cy) + cy + ty
    sx = np.clip(sx, 0, w - 1.001); sy = np.clip(sy, 0, h - 1.001)
    x0 = np.floor(sx).astype(np.int64); y0 = np.floor(sy).astype(np.int64)
    fx = sx - x0; fy = sy - y0
    f = img.astype(np.float64)
    out = (f[y0, x0] * (1 - fx) * (1 - fy) + f[y0, x0 + 1] * fx * (1 - fy) +
           f[y0 + 1, x0] * (1 - fx) * fy + f[y0 + 1, x0 + 1] * fx * fy)
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def synth_sequence(n, w=640, h=480, seed=1):
    f0 = synth_frame(w, h, seed)
    return np.stack([f0] + [warp_frame(f0, 1000 * seed + k) for k in range(1, n)])


# ---------------------------------------------------------------------------------------------- PnP with lines
TUM1_K = (517.306408, 516.469215, 318.643040, 255.313989)   # Examples/Monocular/TUM1.yaml:8-11
TUM1_DIST = (0.262383, -0.953104, -0.005358, 0.002628, 1.163314)   # TUM1.yaml:13-17 (k1 k2 p1 p2 k3)
EUROC_K = (458.654, 457.296, 367.215, 248.375)   # Examples/Monocular/EuRoC.yaml:8-11
EUROC_DIST = (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0)   # EuRoC.yaml:13-16


def _rot(rx, ry, rz):
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]); Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def synth_pose_problem(seed=3, n_points=300, n_lines=80, outlier_frac=0.10, K=TUM1_K, w=640, h=480,
                       pert_t=0.02, pert_deg=1.0, noise_px=1.0):
    """One TUM-shaped PoseOptimization problem (SURVEY.md §8d config 3).

    Returns dict with Tcw0 (perturbed initial pose, float32 4x4), Tcw_true, K, pt_obs, pt_inv_sigma2, pt_Xw,
    line_func (normalised 2-D line through the noisy observed end-points), line_Xw (6 doubles).
    """
    rng = np.random.Generator(np.random.PCG64(seed))
    fx, fy, cx, cy = K
    R = _rot(*rng.uniform(-0.2, 0.2, 3)); t = rng.uniform(-0.5, 0.5, 3)
    T = np.eye(4); T[:3, :3] = R; T[:3, 3] = t

    def sample_cam_points(n):
        u = rng.uniform(20, w - 20, n); v = rng.uniform(20, h - 20, n); z = rng.uniform(2.0, 8.0, n)
        return np.stack([(u - cx) / fx * z, (v - cy) / fy * z, z], 1)

    def project(Xc):
        return np.stack([Xc[:, 0] / Xc[:, 2] * fx + cx, Xc[:, 1] / Xc[:, 2] * fy + cy], 1)

    Xc = sample_cam_points(n_points)
    Xw = (Xc - t) @ R          # R^T (Xc - t)
    quota = np.array([217, 181, 151, 126, 105, 87, 73, 60], np.float64)
    octave = rng.choice(8, n_points, p=quota / quota.sum())
    sigma = 1.2 ** octave
    obs = project(Xc) + rng.normal(0, noise_px, (n_points, 2)) * sigma[:, None]
    bad = rng.random(n_points) < outlier_frac
    obs[bad] += rng.uniform(-40, 40, (bad.sum(), 2))
    inv_sigma2 = (1.0 / (np.float32(1.2) ** octave).astype(np.float32) ** 2).astype(np.float32)

    A = sample_cam_points(n_lines)
    Bc = A + rng.uniform(-0.8, 0.8, (n_lines, 3)); Bc[:, 2] = np.clip(Bc[:, 2], 1.5, 9.0)
    lw = np.concatenate([(A - t) @ R, (Bc - t) @ R], 1)
    pa = project(A) + rng.normal(0, noise_px, (n_lines, 2)); pb = project(Bc) + rng.normal(0, noise_px, (n_lines, 2))
    lbad = rng.random(n_lines) < outlier_frac
    pa[lbad] += rng.uniform(-30, 30, (lbad.sum(), 2))
    sp = np.concatenate([pa, np.ones((n_lines, 1))], 1); ep = np.concatenate([pb, np.ones((n_lines, 1))], 1)
    l = np.cross(sp, ep)
    l /= np.sqrt(l[:, 0] ** 2 + l[:, 1] ** 2)[:, None]          # LineExtractor.cpp:82-90

    dR = _rot(*np.deg2rad(rng.uniform(-pert_deg, pert_deg, 3))); dt = rng.uniform(-pert_t, pert_t, 3)
    T0 = np.eye(4); T0[:3, :3] = dR @ R; T0[:3, 3] = dR @ t + dt
    return dict(Tcw0=T0.astype(np.float32), Tcw_true=T, K=np.array(K, np.float32),
                pt_obs=obs.astype(np.float32), pt_inv_sigma2=inv_sigma2, pt_Xw=Xw.astype(np.float32),
                line_func=np.ascontiguousarray(l, np.float64), line_Xw=np.ascontiguousarray(lw, np.float64),
                pt_is_outlier=bad, line_is_outlier=lbad)


# ---------------------------------------------------------------------------------------------- local BA window
def synth_ba_problem(seed=4, n_free=20, n_fixed=40, n_pt=3000, n_ln=400, obs_pt=5, obs_ln=4, K=TUM1_K, w=640, h=480,
                     noise_px=1.0, outlier_frac=0.03, pert_t=0.01, pert_deg=0.3, pert_X=0.02, Ks=None, K_end=None):
    """KITTI/TUM-shaped local-BA window (SURVEY.md §8d config 4): cameras on a smooth path in front of a scene,
    points with ~obs_pt and lines with ~obs_ln observations, noisy observations, a few gross outliers, perturbed
    initial estimates.  Keyframe 0 is fixed (mnId == 0) together with the `n_fixed` covisible-but-not-local ones.

    Ks ([n_kf][4], optional): one camera per keyframe; keyframe k's observations are made with Ks[k] (as float32, the
    precision the optimisers read).  K_end (optional): the current keyframe's camera the local BA projects line end
    points with.  Both default to K; neither draws from the random stream, so the default output does not change."""
    rng = np.random.Generator(np.random.PCG64(seed))
    n_kf = n_free + n_fixed
    if Ks is not None:
        Ks = np.asarray(Ks, np.float32).reshape(n_kf, 4)
    cams = [K] * n_kf if Ks is None else [tuple(float(v) for v in Ks[k]) for k in range(n_kf)]
    Ts = []
    for k in range(n_kf):
        s = k / max(n_kf - 1, 1)
        R = _rot(0.02 * np.sin(3 * s) + rng.normal(0, 0.01), 0.25 * (s - 0.5) + rng.normal(0, 0.01), rng.normal(0, 0.01))
        C = np.array([3.0 * (s - 0.5), 0.1 * np.sin(5 * s), 0.3 * s]) + rng.normal(0, 0.02, 3)
        T = np.eye(4); T[:3, :3] = R; T[:3, 3] = -R @ C
        Ts.append(T)
    Ts = np.array(Ts)
    order = rng.permutation(n_kf)
    Ts = Ts[order]
    fixed = np.zeros(n_kf, np.uint8); fixed[n_free:] = 1; fixed[0] = 1

    def project(k, X):
        fx, fy, cx, cy = cams[k]
        Xc = X @ Ts[k, :3, :3].T + Ts[k, :3, 3]
        return np.stack([Xc[:, 0] / Xc[:, 2] * fx + cx, Xc[:, 1] / Xc[:, 2] * fy + cy], 1), Xc[:, 2]

    Xw = np.stack([rng.uniform(-4, 4, n_pt), rng.uniform(-2, 2, n_pt), rng.uniform(3, 9, n_pt)], 1)
    pe_kf, pe_pt, pe_obs, pe_w = [], [], [], []
    for i in range(n_pt):
        cand = rng.permutation(n_kf)
        got = 0
        for k in cand:
            uv, z = project(k, Xw[i:i + 1])
            if z[0] > 0.5 and 0 < uv[0, 0] < w and 0 < uv[0, 1] < h:
                octv = rng.integers(0, 8)
                o = uv[0] + rng.normal(0, noise_px, 2) * 1.2 ** octv
                if rng.random() < outlier_frac:
                    o = o + rng.uniform(-30, 30, 2)
                pe_kf.append(k); pe_pt.append(i); pe_obs.append(o); pe_w.append(1.0 / (np.float32(1.2) ** octv) ** 2)
                got += 1
                if got >= max(2, rng.poisson(obs_pt)):
                    break
    A = np.stack([rng.uniform(-4, 4, n_ln), rng.uniform(-2, 2, n_ln), rng.uniform(3, 9, n_ln)], 1)
    Bp = A + rng.uniform(-0.8, 0.8, (n_ln, 3))
    Lw = np.concatenate([A, Bp], 1)
    le_kf, le_ln, le_f = [], [], []
    for i in range(n_ln):
        got = 0
        for k in rng.permutation(n_kf):
            ua, za = project(k, A[i:i + 1]); ub, zb = project(k, Bp[i:i + 1])
            if za[0] > 0.5 and zb[0] > 0.5 and 0 < ua[0, 0] < w and 0 < ua[0, 1] < h and 0 < ub[0, 0] < w and 0 < ub[0, 1] < h:
                pa = ua[0] + rng.normal(0, noise_px, 2); pb = ub[0] + rng.normal(0, noise_px, 2)
                if rng.random() < outlier_frac:
                    pa = pa + rng.uniform(-25, 25, 2)
                l = np.cross(np.r_[pa, 1.0], np.r_[pb, 1.0]); l /= np.hypot(l[0], l[1])
                le_kf.append(k); le_ln.append(i); le_f.append(l)
                got += 1
                if got >= max(3, rng.poisson(obs_ln)):
                    break
    T0 = Ts.copy()
    for k in range(n_kf):
        if not fixed[k]:
            dR = _rot(*np.deg2rad(rng.uniform(-pert_deg, pert_deg, 3)))
            T0[k, :3, :3] = dR @ Ts[k, :3, :3]; T0[k, :3, 3] = dR @ Ts[k, :3, 3] + rng.uniform(-pert_t, pert_t, 3)
    return dict(kf_Tcw=T0.astype(np.float32).reshape(n_kf, 16), kf_Tcw_true=Ts, kf_fixed=fixed,
                kf_K=np.tile(np.array(K, np.float32), (n_kf, 1)) if Ks is None else Ks.copy(),
                K_end=np.array(K if K_end is None else K_end, np.float32),
                pt_Xw=(Xw + rng.normal(0, pert_X, Xw.shape)).astype(np.float32), pt_Xw_true=Xw,
                ln_Xw=np.ascontiguousarray(Lw + rng.normal(0, pert_X, Lw.shape)), ln_Xw_true=Lw,
                pe_kf=np.array(pe_kf, np.int32), pe_pt=np.array(pe_pt, np.int32), pe_obs=np.array(pe_obs, np.float32).reshape(-1, 2),
                pe_inv_sigma2=np.array(pe_w, np.float32), le_kf=np.array(le_kf, np.int32), le_ln=np.array(le_ln, np.int32),
                le_func=np.ascontiguousarray(np.array(le_f, np.float64).reshape(-1, 3)))


def synth_map_view(seed=7, n=4000, K=TUM1_K, w=640, h=480, lines=False):
    """A camera pose plus n local-map points (or lines) scattered in front of / around / behind it, for
    Frame::isInFrustum: returns dict(Tcw, Ow, pos, normal, min_dist, max_dist)."""
    rng = np.random.default_rng(seed)
    R = _rot(*(rng.normal(0, 0.2, 3))); t = rng.normal(0, 0.5, 3)
    Tcw = np.eye(4, dtype=np.float32); Tcw[:3, :3] = R.astype(np.float32); Tcw[:3, 3] = t.astype(np.float32)
    Rwc = Tcw[:3, :3].T; Ow = (-Rwc @ Tcw[:3, 3]).astype(np.float32)
    def pts(m):
        z = rng.uniform(-2.0, 12.0, m); x = rng.uniform(-1.2, 1.2, m) * np.abs(z); y = rng.uniform(-1.0, 1.0, m) * np.abs(z)
        Pc = np.stack([x, y, z], 1)
        return (Pc - t) @ R            # Pw = R^T (Pc - t)
    if not lines:
        pos = pts(n).astype(np.float32)
        d = np.linalg.norm(pos - Ow, axis=1)
        nrm = (pos - Ow) / np.maximum(d, 1e-6)[:, None] + rng.normal(0, 0.5, (n, 3))
        nrm = (nrm / np.linalg.norm(nrm, axis=1)[:, None]).astype(np.float32)
    else:
        s = pts(n); e = s + rng.normal(0, 0.4, (n, 3))
        pos = np.concatenate([s, e], 1).astype(np.float64)
        mid = 0.5 * (s + e); d = np.linalg.norm(mid - Ow, axis=1)
        nrm = (mid - Ow) / np.maximum(d, 1e-6)[:, None] + rng.normal(0, 0.5, (n, 3))
        nrm = (nrm / np.linalg.norm(nrm, axis=1)[:, None]).astype(np.float64)
    f = rng.uniform(0.3, 3.0, n)
    max_dist = (d * f * 1.2).astype(np.float32); min_dist = (max_dist / (1.2 ** rng.integers(2, 9, n))).astype(np.float32)
    return dict(Tcw=Tcw, Ow=Ow, pos=pos, normal=nrm, min_dist=min_dist, max_dist=max_dist)


def synth_two_view(seed=5, n_pts=1500, n_clutter=400, K=TUM1_K, w=640, h=480, nlevels=8, scale=1.2):
    """Two keyframes observing the same 3-D points (LocalMapping::CreateNewMapPoints' input to SearchForTriangulation):
    undistorted keypoints with octave / angle, ORB-like 256-bit descriptors (a per-point code with a few flipped bits per
    view), DBoW2-style feature vectors (node id shared by the two views of a point, clutter spread at random), poses, F12."""
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy = K
    Km = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64)
    R1 = _rot(*rng.normal(0, 0.03, 3)); t1 = rng.normal(0, 0.05, 3)
    R2 = _rot(*rng.normal(0, 0.06, 3)); t2 = t1 + np.array([0.35, 0.02, 0.05]) + rng.normal(0, 0.02, 3)
    X = np.stack([rng.uniform(-3, 3, n_pts), rng.uniform(-2, 2, n_pts), rng.uniform(2.5, 9, n_pts)], 1)
    sf = scale ** np.arange(nlevels)

    def view(R, t, flip_seed):
        r = np.random.default_rng(flip_seed)
        Xc = X @ R.T + t
        uv = np.stack([fx * Xc[:, 0] / Xc[:, 2] + cx, fy * Xc[:, 1] / Xc[:, 2] + cy], 1)
        octv = r.integers(0, nlevels, n_pts)
        uv = uv + r.normal(0, 0.6, uv.shape) * sf[octv][:, None]
        ok = (uv[:, 0] > 20) & (uv[:, 0] < w - 20) & (uv[:, 1] > 20) & (uv[:, 1] < h - 20) & (Xc[:, 2] > 0.5)
        return uv, octv, ok
    code = rng.integers(0, 256, (n_pts, 32), dtype=np.uint8)
    base_ang = rng.uniform(0, 360, n_pts)
    node_of = rng.integers(0, 97, n_pts)
    out = {}
    for name, (R, t, fs, drot) in {"1": (R1, t1, 11 + seed, 0.0), "2": (R2, t2, 23 + seed, 12.0)}.items():
        r = np.random.default_rng(fs)
        uv, octv, ok = view(R, t, fs)
        ids = np.nonzero(ok)[0]
        r.shuffle(ids)
        n = len(ids) + n_clutter
        kp = np.zeros(n, KP_DTYPE)
        kp["x"][:len(ids)] = uv[ids, 0]; kp["y"][:len(ids)] = uv[ids, 1]; kp["octave"][:len(ids)] = octv[ids]
        ang = (base_ang[ids] + drot + r.normal(0, 4, len(ids))) % 360
        wrong = r.random(len(ids)) < 0.1                   # some inconsistent rotations for the histogram to remove
        ang[wrong] = r.uniform(0, 360, wrong.sum())
        kp["angle"][:len(ids)] = ang
        kp["x"][len(ids):] = r.uniform(20, w - 20, n_clutter); kp["y"][len(ids):] = r.uniform(20, h - 20, n_clutter)
        kp["octave"][len(ids):] = r.integers(0, nlevels, n_clutter); kp["angle"][len(ids):] = r.uniform(0, 360, n_clutter)
        kp["size"] = 31 * sf[kp["octave"]]; kp["class_id"] = -1
        d = np.empty((n, 32), np.uint8)
        d[:len(ids)] = code[ids]
        flips = r.integers(0, 256, (len(ids), 14)); 
        for j in range(flips.shape[1]):
            sel = r.random(len(ids)) < 0.7
            d[np.nonzero(sel)[0], flips[sel, j] // 8] ^= (1 << (flips[sel, j] % 8)).astype(np.uint8)
        d[len(ids):] = r.integers(0, 256, (n_clutter, 32), dtype=np.uint8)
        nodes = np.concatenate([node_of[ids], r.integers(0, 110, n_clutter)])
        fv = {}
        for i in r.permutation(n):                          # insertion order inside a node is arbitrary
            fv.setdefault(int(nodes[i]), []).append(int(i))
        has_mp = (r.random(n) < 0.3).astype(np.uint8)
        out[name] = dict(keys=kp, desc=d, fv=fv, has_mp=has_mp, R=R.astype(np.float32), t=t.astype(np.float32), pt_id=np.concatenate([ids, -np.ones(n_clutter, np.int64)]))
    # LocalMapping::ComputeF12: F12 = K1^-T [t12]x R12 K2^-1
    R12 = R1 @ R2.T; t12 = -R1 @ R2.T @ t2 + t1
    tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]])
    out["F12"] = (np.linalg.inv(Km).T @ tx @ R12 @ np.linalg.inv(Km)).astype(np.float32)
    out["Cw1"] = (-R1.T @ t1).astype(np.float32)
    out["K"] = np.array(K, np.float32)
    out["scale_factors"] = sf.astype(np.float32); out["level_sigma2"] = (sf * sf).astype(np.float32)
    out["X"] = X
    return out


def synth_fuse_problem(seed=6, n_mp=3000, n_kp=1800, K=TUM1_K, w=640, h=480, nlevels=8, scale=1.2):
    """A keyframe (keypoints, descriptors, pose) and a list of map points to fuse into it (ORBmatcher::Fuse input)."""
    rng = np.random.default_rng(seed)
    v = synth_map_view(seed + 100, n_mp, K, w, h)
    fx, fy, cx, cy = K
    sf = (scale ** np.arange(nlevels)).astype(np.float32)
    T = v["Tcw"].astype(np.float64)
    Pc = v["pos"].astype(np.float64) @ T[:3, :3].T + T[:3, 3]
    with np.errstate(all="ignore"):
        uv = np.stack([fx * Pc[:, 0] / Pc[:, 2] + cx, fy * Pc[:, 1] / Pc[:, 2] + cy], 1)
    vis = np.nonzero((Pc[:, 2] > 0.1) & (uv[:, 0] > 5) & (uv[:, 0] < w - 5) & (uv[:, 1] > 5) & (uv[:, 1] < h - 5))[0]
    mp_desc = rng.integers(0, 256, (n_mp, 32), dtype=np.uint8)
    kp = np.zeros(n_kp, KP_DTYPE); desc = rng.integers(0, 256, (n_kp, 32), dtype=np.uint8)
    m = min(len(vis), n_kp * 2 // 3)
    src = rng.choice(vis, m, replace=False)
    d = np.linalg.norm(v["pos"][src] - v["Ow"], axis=1)
    lvl = np.clip(np.ceil(np.log(v["max_dist"][src] / d) / np.log(scale)), 0, nlevels - 1).astype(int)
    octv = np.clip(lvl - rng.integers(0, 3, m) + 0, 0, nlevels - 1)      # lvl, lvl-1 pass the level filter; lvl-2 does not
    kp["x"][:m] = uv[src, 0] + rng.normal(0, 1.2, m) * sf[octv]; kp["y"][:m] = uv[src, 1] + rng.normal(0, 1.2, m) * sf[octv]
    kp["octave"][:m] = octv
    desc[:m] = mp_desc[src]
    flips = rng.integers(0, 256, (m, 40))
    for j in range(flips.shape[1]):
        sel = rng.random(m) < 0.6
        desc[np.nonzero(sel)[0], flips[sel, j] // 8] ^= (1 << (flips[sel, j] % 8)).astype(np.uint8)
    kp["x"][m:] = rng.uniform(0, w, n_kp - m); kp["y"][m:] = rng.uniform(0, h, n_kp - m); kp["octave"][m:] = rng.integers(0, nlevels, n_kp - m)
    kp["size"] = 31 * sf[kp["octave"]]; kp["class_id"] = -1
    skip = (rng.random(n_mp) < 0.15).astype(np.uint8)
    return dict(keys=kp, desc=desc, bounds=np.array([0, 0, w, h], np.float32), Tcw=v["Tcw"], Ow=v["Ow"], K=np.array(K, np.float32),
                scale_factors=sf, inv_level_sigma2=(1.0 / (sf * sf)).astype(np.float32), log_scale_factor=float(np.float32(np.log(np.float32(scale)))),
                skip=skip, pos=v["pos"], normal=v["normal"], min_dist=v["min_dist"], max_dist=v["max_dist"], mp_desc=mp_desc)
