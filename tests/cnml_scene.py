"""A seeded scene for the line triangulation tests (pl_lsd_triangulate_dev, tests/cnml_oracle.py): a current keyframe and seven
neighbours with their own poses and intrinsics viewing one set of 3-D segments, plus clutter.  Keylines are the projected end
points with a little noise; line functions are formed as Frame does (the cross product of the homogeneous end points over the
norm of its first two entries, in fp64); descriptors are one code per segment with a few bits flipped per view, so the line search
pairs the views of a segment.

Neighbour 5 sits 1 cm from the current keyframe and fails the baseline test, so it is not searched: entries 4 .. of
TotalvMatchedIndices hold the next neighbours' matches but are paired with vpNeighKFs[4] .. (the positional pairing).  Neighbour 7
looks away, so its search finds nothing (an entry with nmatches = 0).  Some keylines hold map lines at the snapshot."""
import numpy as np

from plslam_b200.binding import KEYLINE_DTYPE

f32 = np.float32


def _rot(a):
    cx, sx, cy, sy, cz, sz = np.cos(a[0]), np.sin(a[0]), np.cos(a[1]), np.sin(a[1]), np.cos(a[2]), np.sin(a[2])
    return (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
            @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))


def keylines_of(s, e, octave, rng=None):
    """KEYLINE_DTYPE records and line functions [n][3] (fp64) for end points s, e [n][2]"""
    n = len(s)
    kl = np.zeros(n, KEYLINE_DTYPE)
    kl["startPointX"], kl["startPointY"], kl["endPointX"], kl["endPointY"] = s[:, 0], s[:, 1], e[:, 0], e[:, 1]
    kl["angle"] = np.arctan2(kl["endPointY"].astype(np.float64) - kl["startPointY"], kl["endPointX"].astype(np.float64) - kl["startPointX"])
    kl["octave"] = octave
    kl["ptx"], kl["pty"] = (s[:, 0] + e[:, 0]) / 2, (s[:, 1] + e[:, 1]) / 2
    kl["lineLength"] = np.hypot(e[:, 0] - s[:, 0], e[:, 1] - s[:, 1])
    kl["class_id"] = np.arange(n)
    sp = np.stack([kl["startPointX"], kl["startPointY"], np.ones(n)], 1).astype(np.float64)
    ep = np.stack([kl["endPointX"], kl["endPointY"], np.ones(n)], 1).astype(np.float64)
    f = np.cross(sp, ep)
    f /= np.sqrt(f[:, 0] ** 2 + f[:, 1] ** 2)[:, None]
    return kl, f


def scene(seed=5, n_seg=160, n_clutter=40, w=640, h=480, n_kf=8):
    rng = np.random.default_rng(seed)
    mid = np.stack([rng.uniform(-2.5, 2.5, n_seg), rng.uniform(-1.8, 1.8, n_seg), rng.uniform(3, 8, n_seg)], 1)
    d = rng.normal(size=(n_seg, 3)); d /= np.linalg.norm(d, axis=1)[:, None]
    half = rng.uniform(0.2, 0.8, n_seg)[:, None]
    P0, P1 = mid - half * d, mid + half * d
    code = rng.integers(0, 256, (n_seg, 32), dtype=np.uint8)
    kfs, seg_of, medians = [], [], []
    for k in range(n_kf):
        if k == 0:
            c, ang = np.zeros(3), np.zeros(3)
        elif k == 5:
            c, ang = np.array([0.01, 0.0, 0.0]), rng.normal(0, 0.02, 3)
        elif k == 7:
            c, ang = np.array([0.2, 0.1, 0.0]), np.array([0.0, np.pi, 0.0])
        else:
            c, ang = np.array([0.35 * np.cos(k), 0.15 * np.sin(2 * k), 0.08 * k]), rng.normal(0, 0.04, 3)
        R = _rot(ang)
        T = np.eye(4); T[:3, :3] = R; T[:3, 3] = -R @ c
        K = np.array([517.3, 516.5, 318.6, 255.3]) + (0 if k == 0 else rng.normal(0, 4, 4))
        proj = lambda X: np.stack([K[0] * (X @ R.T + T[:3, 3])[:, 0] / (X @ R.T + T[:3, 3])[:, 2] + K[2],
                                   K[1] * (X @ R.T + T[:3, 3])[:, 1] / (X @ R.T + T[:3, 3])[:, 2] + K[3]], 1)
        z0, z1 = (P0 @ R.T + T[:3, 3])[:, 2], (P1 @ R.T + T[:3, 3])[:, 2]
        s, e = proj(P0) + rng.normal(0, 0.4, (n_seg, 2)), proj(P1) + rng.normal(0, 0.4, (n_seg, 2))
        inside = lambda p: (p[:, 0] > 5) & (p[:, 0] < w - 5) & (p[:, 1] > 5) & (p[:, 1] < h - 5)
        ok = (z0 > 0.1) & (z1 > 0.1) & inside(s) & inside(e) & (rng.random(n_seg) < 0.85)
        ids = rng.permutation(np.nonzero(ok)[0])
        cs, ce = rng.uniform(20, w - 20, (n_clutter, 2)), rng.uniform(20, h - 20, (n_clutter, 2))
        S, E = np.concatenate([s[ids], cs]), np.concatenate([e[ids], ce])
        octave = rng.integers(0, 2, len(S))
        kl, f = keylines_of(S.astype(f32), E.astype(f32), octave)
        desc = np.concatenate([code[ids], rng.integers(0, 256, (n_clutter, 32), dtype=np.uint8)])
        for _ in range(6):
            r = np.nonzero(rng.random(len(ids)) < 0.6)[0]; b = rng.integers(0, 256, len(r))
            desc[r, b // 8] ^= (1 << (b % 8)).astype(np.uint8)
        has_ml = (rng.random(len(S)) < 0.08).astype(np.uint8)
        zs = np.concatenate([(z0[ids] + z1[ids]) / 2, rng.uniform(3, 8, n_clutter)])
        medians.append(f32(np.sort(zs)[(len(zs) - 1) // 2]))
        kfs.append(dict(ldesc=desc, has_ml=has_ml, keylines=kl, line_func=f, Tcw=T.astype(f32).reshape(-1), Ow=c.astype(f32),
                        K=K.astype(f32)))
        seg_of.append(np.concatenate([ids, np.full(n_clutter, -1)]))
    return dict(kfs=kfs, seg_of=seg_of, medians=np.array(medians, f32), level_sigma2_line=np.array([1.0, 1.44], f32))


def searched_neighbours():
    """vpNeighKFs = 1 .. 7 in order; neighbour 5 fails the baseline test"""
    return [1, 2, 3, 4, 6, 7]


def group(sc, problems_of, kf_cur=0, neigh=(1, 2, 3, 4, 5, 6, 7)):
    """The group of kf_cur: entry e = the search problem of the e-th searched neighbour, paired with neigh[e] (positional)"""
    srch = [j for j in neigh if j != 5] if kf_cur == 0 else list(neigh)
    return dict(kf_cur=kf_cur, entries=[(problems_of[j], neigh[e], sc["medians"][neigh[e]]) for e, j in enumerate(srch)])


def truth_matches(sc, kf1, kf2, drop=0.1, seed=1):
    """matches of kf1's keylines in kf2 from the segment ids (the tests' stand-in for the search without a GPU)"""
    rng = np.random.default_rng(seed + 31 * kf1 + kf2)
    a, b = sc["seg_of"][kf1], sc["seg_of"][kf2]
    pos = {int(s): i for i, s in enumerate(b) if s >= 0}
    m = np.array([pos.get(int(s), -1) if s >= 0 else -1 for s in a], np.int32)
    m[rng.random(len(m)) < drop] = -1
    return m


def knife_edge(sc, n_result=12):
    """A two-entry group on keyframes 0, 1, 2 whose view-1 keylines each have an octave of their own, with the level's sigma^2 set
    so that 3.84 sigma^2 lies within one rounding of the triple's squared reprojection error at the start point (alternately just
    above and just below); n_result of the view-2 line functions turned so that |Result1| or |Result2| lands on the last float at or
    below 0.996 or the first above it.  Views 2 and 3 (octaves 0 and 1) have tighter sigma^2 than every level of view 1, so a
    view-2 test with view 1's sigma^2 passes triples that fail (code 12).  Entry 1's median depth is tiny: only entry 0's may be
    read.  Returns (keyframes,
    matches [2][n0], level_sigma2_line); the search problems are (0, 1) and (0, 2)."""
    import cnml_oracle as co
    from plslam_b200 import binding as bd
    kfs = [dict(k, keylines=k["keylines"].copy(), line_func=k["line_func"].copy()) for k in sc["kfs"][:3]]
    n0 = len(kfs[0]["keylines"])
    kfs[0]["keylines"]["octave"] = 2 + np.arange(n0)
    m = np.stack([truth_matches(sc, 0, 1, drop=0), truth_matches(sc, 0, 2, drop=0)])
    kfs[0]["has_ml"] = np.zeros(n0, np.uint8)
    ev = np.nonzero((m[0] >= 0) & (m[1] >= 0))[0]
    # |Result| at 0.996: bisect the direction of view 2's line function
    pc = co.pair_consts(*(np.asarray(kfs[v]["Tcw"], f32).reshape(4, 4) for v in range(3)), *(kfs[v]["K"] for v in range(3)))
    kl0 = kfs[0]["keylines"]

    def res(ikl, th):
        f = np.array([np.cos(th), np.sin(th), 0.0])
        lv = np.array([[-f[1], f[0]]]).astype(f32)
        r = [co._epipolar(pc["F21"][None], kl0[a][ikl:ikl + 1], kl0[b][ikl:ikl + 1], lv)[0] for a, b in
             (("startPointX", "startPointY"), ("endPointX", "endPointY"))]
        return max(abs(float(r[0])), abs(float(r[1])))
    for t, ikl in enumerate(ev[-n_result:]):
        lo, hi = 0.0, 0.5                     # Result near 1 at lo (aligned with the epipolar line), small at hi
        x, y = float(kl0["startPointX"][ikl]), float(kl0["startPointY"][ikl])
        th_ = co._gemm3(pc["F21"][None], np.array([[x, y, 1]], f32))[0]
        phi = np.arctan2(th_[0], th_[1]) + np.pi / 2       # lv2 = (-f1, f0) parallel to Th_ = (-Th1, Th0)
        g = lambda d: res(ikl, phi + d) > 0.996
        if not g(lo) or g(hi):
            continue
        for _ in range(80):
            mid = (lo + hi) / 2
            lo, hi = (mid, hi) if g(mid) else (lo, mid)
        th = phi + (lo if t % 2 else hi)
        kfs[1]["line_func"][m[0][ikl]] = [np.cos(th), np.sin(th), -(np.cos(th) * x + np.sin(th) * y)]
    # reprojection in view 1 at the last rounding of 3.84 sigma^2: view 1's line function enters nothing but that test, so its
    # constant term (a double) moves err onto the threshold, alternately the last value that passes and the first that fails
    k = bd.pack_tri_keyframes(kfs, lines=True)
    q = bd.pack_tri_problems([(0, 1), (0, 2)], k["n"])
    s2 = np.full(2 + n0, 1e30, f32)
    gr = bd.pack_tri_line_groups([dict(kf_cur=0, entries=[(0, 1, sc["medians"][1]), (1, 2, f32(0.05))])], k["n"])
    err = []
    code = co.triangulate_lines(k, q, gr, m.reshape(-1).astype(np.int32), (m >= 0).sum(1).astype(np.int32), np.zeros(2, np.int32),
                                s2, err_out=err)[0]
    evs = np.nonzero((code != co.NO_TRIPLE) & (code != co.HELD))[0]
    if err:
        (es, _, us, vs), (ee, _, _, _) = err[0], err[1]
        # views 2 and 3 (octaves 0 and 1): the triangulation puts the end points on their planes, so their errors are small; a
        # sigma^2 that 40 % of the triples that pass every gate fail there, far below every level of view 1
        e23 = np.max([np.abs(e[0]) for e in err[2:]], 0)[code[evs] == co.COMMITTED]
        s2[:2] = f32(np.quantile(e23 ** 2, 0.6) / 3.84)
        f1 = kfs[0]["line_func"]
        for t, ikl in enumerate(evs):
            d = float(ee[t] - es[t])
            if not (np.isfinite(d) and np.isfinite(es[t])):
                continue
            s2[2 + ikl] = f32(max(abs(d), 3.0) ** 2 * 1.1 / 3.84)
            th = 3.84 * float(s2[2 + ikl])
            sgn = -1.0 if d > 0 else 1.0
            base = f1[ikl, 0] * float(us[t]) + f1[ikl, 1] * float(vs[t])
            c = sgn * np.sqrt(th) - base
            out = lambda x: np.nextafter(x, sgn * np.inf)
            while (base + c) ** 2 > th:
                c = np.nextafter(c, -sgn * np.inf)
            while (base + c) ** 2 <= th:
                c = out(c)
            f1[ikl, 2] = c if t % 2 else np.nextafter(c, -sgn * np.inf)
    return kfs, m, s2


def degenerate_svd(sc):
    """Three keyframes whose triangulation matrix has a fourth column exactly orthogonal to the other three and longer than their
    smallest singular value, so that vt.row(3) is (X, 0): camera 1 at the origin, cameras 2 and 3 at -R^T t and R^T t with one
    rotation and one K, view 3's line function the negative of view 2's.  One keyline each, of a segment all three see."""
    K = np.array([517.3, 516.5, 318.6, 255.3])
    R = _rot(np.array([0.02, -0.03, 0.01]))
    t = np.array([3.0, 0.5, 0.2])
    P0, P1 = np.array([-0.4, 0.2, 5.0]), np.array([0.5, -0.3, 6.0])
    out = []
    for Rv, tv in ((np.eye(3), np.zeros(3)), (R, t), (R, -t)):
        T = np.eye(4); T[:3, :3] = Rv; T[:3, 3] = tv
        pr = lambda X: np.array([K[0] * (Rv @ X + tv)[0] / (Rv @ X + tv)[2] + K[2], K[1] * (Rv @ X + tv)[1] / (Rv @ X + tv)[2] + K[3]])
        kl, f = keylines_of(pr(P0)[None].astype(f32), pr(P1)[None].astype(f32), np.zeros(1, int))
        out.append(dict(ldesc=np.zeros((1, 32), np.uint8), has_ml=np.zeros(1, np.uint8), keylines=kl, line_func=f,
                        Tcw=T.astype(f32).reshape(-1), Ow=(-Rv.T @ tv).astype(f32), K=K.astype(f32)))
    out[2]["line_func"] = -out[1]["line_func"]
    return out
