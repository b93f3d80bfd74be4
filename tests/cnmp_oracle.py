"""CPU oracle of pl_orb_triangulate_dev: the triangulation, the gates and the neighbour-order commit of
LocalMapping::CreateNewMapPoints (src/LocalMapping.cc:417-574, monocular), restated in numpy on the reference's arithmetic and
vectorised over the pairs of a batch.

Every operation is an elementwise numpy operation on float32 or float64 arrays, which rounds once and never contracts, so each
reference expression keeps its C++ promotions and its cv::Mat order:
  Rwc * xn            cv::gemm's small-matrix fp32 order ((a0 b0 + a1 b1) + a2 b2), each operation rounded on its own;
  Mat::dot, cv::norm  products and sums in fp64 from 0, in index order; norm = sqrt of that sum;
  s * M1 - M2         MatExpr's addWeighted: (double) s * M1 - M2 + 0 in fp64, rounded once to fp32 (cv2 shows the fp64 form:
                      tests/test_triangulate_svd.py);
  M / s               M * (float)(1.0 / s) + 0 (convertTo with beta 0), in fp32;
  cv::SVD::compute    svd4 below (one-sided Jacobi, as svd4.cuh states it), pinned to cv2 by tests/golden/orb_cv2_svd4.npz;
  hypot               OpenCV's own formula (cv_hypot), not the C library's.
"""
import numpy as np

f32, f64 = np.float32, np.float64
EPS_SVD = f64(f32(2) * np.finfo(f32).eps)

# code per slot (plslam_b200.h, pl_orb_triangulate_dev)
NO_PAIR, COMMITTED, DROPPED = -1, 0, 1
PARALLAX, W_ZERO, BEHIND1, BEHIND2, REPROJ1, REPROJ2, SCALE = 2, 3, 4, 5, 6, 7, 8
UNWRITTEN = -128      # what the tests pre-fill the code output with


def _dot(x, y):
    """sum_k x[..., k] * y[..., k] in fp64 from 0, k in order (x, y fp32)"""
    s = np.zeros(np.broadcast_shapes(x.shape, y.shape)[:-1], f64)
    for k in range(x.shape[-1]):
        s = s + x[..., k].astype(f64) * y[..., k].astype(f64)
    return s


def _rotate(X, i, j, c, s, m):
    """rows i, j of X[m] <- (c x + s y, -s x + c y) in fp32"""
    x, y = X[m, i].copy(), X[m, j].copy()
    cc, ss = c[:, None], s[:, None]
    X[m, i] = cc * x + ss * y
    X[m, j] = (-ss) * x + cc * y


def cv_hypot(a, b):
    """OpenCV's hypot<double> (lapack.cpp), not the C library's: a > b ? a sqrt(1 + (b/a)^2) : b > 0 ? b sqrt(1 + (a/b)^2) : 0 on
    |a|, |b|, elementwise in fp64"""
    a, b = np.abs(a), np.abs(b)
    with np.errstate(invalid="ignore", divide="ignore"):
        ra, rb = b / a, a / b
        return np.where(a > b, a * np.sqrt(1 + ra * ra), np.where(b > 0, b * np.sqrt(1 + rb * rb), 0.0))


def svd4(A):
    """cv::SVD::compute(A, w, u, vt, MODIFY_A | FULL_UV) for a batch of 4x4 float32 matrices A [N][4][4] -> w [N][4], vt [N][4][4]
    (float32).  All matrices step through the sweeps together; one that had a sweep without a rotation is left alone from then on,
    which is where the scalar algorithm stops."""
    A = np.asarray(A, f32).reshape(-1, 4, 4)
    N = len(A)
    At = np.ascontiguousarray(A.transpose(0, 2, 1))
    V = np.broadcast_to(np.eye(4, dtype=f32), (N, 4, 4)).copy()
    W = _dot(At, At)
    active = np.ones(N, bool)
    for _ in range(30):
        changed = np.zeros(N, bool)
        for i in range(3):
            for j in range(i + 1, 4):
                a, b = W[:, i].copy(), W[:, j].copy()
                p = _dot(At[:, i], At[:, j])
                with np.errstate(invalid="ignore"):
                    m = active & ~(np.abs(p) <= EPS_SVD * np.sqrt(a * b))
                if not m.any():
                    continue
                p, a, b = p[m] * 2, a[m], b[m]
                beta = a - b
                gamma = cv_hypot(p, beta)
                neg = beta < 0
                with np.errstate(invalid="ignore", divide="ignore"):
                    s_neg = np.sqrt(((gamma - beta) * 0.5) / gamma).astype(f32)
                    c_neg = (p / (gamma * s_neg.astype(f64) * 2)).astype(f32)
                    c_pos = np.sqrt((gamma + beta) / (gamma * 2)).astype(f32)
                    s_pos = (p / (gamma * c_pos.astype(f64) * 2)).astype(f32)
                c, s = np.where(neg, c_neg, c_pos), np.where(neg, s_neg, s_pos)
                _rotate(At, i, j, c, s, m)
                W[m, i] = _dot(At[m, i], At[m, i])
                W[m, j] = _dot(At[m, j], At[m, j])
                _rotate(V, i, j, c, s, m)
                changed |= m
        active &= changed
        if not active.any():
            break
    W = np.sqrt(_dot(At, At))
    r = np.arange(N)
    for i in range(3):
        j = np.full(N, i)
        for k in range(i + 1, 4):
            j = np.where(W[r, j] < W[:, k], k, j)
        Wi, Wj = W[:, i].copy(), W[r, j].copy()
        W[:, i], W[r, j] = Wj, Wi
        Vi, Vj = V[:, i].copy(), V[r, j].copy()
        V[:, i], V[r, j] = Vj, Vi
    return W.astype(f32), V


def _gemm3(M, x):
    """M [N][3][3] * x [N][3] in cv::gemm's fp32 order"""
    return (M[..., 0] * x[:, None, 0] + M[..., 1] * x[:, None, 1]) + M[..., 2] * x[:, None, 2]


def _addw(s, a, b):
    """MatExpr s * a - b on CV_32F rows: fp64, one rounding"""
    return ((s.astype(f64)[:, None] * a.astype(f64) - b.astype(f64)) + 0.0).astype(f32)


def linear_triangulation_matrix(xn1, xn2, T1, T2):
    """A (LocalMapping.cc:458-462) for xn [N][3] and Tcw [N][3][4] (float32)"""
    return np.stack([_addw(xn1[:, 0], T1[:, 2], T1[:, 0]), _addw(xn1[:, 1], T1[:, 2], T1[:, 1]),
                     _addw(xn2[:, 0], T2[:, 2], T2[:, 0]), _addw(xn2[:, 1], T2[:, 2], T2[:, 1])], 1)


def gates(kp1, kp2, K1, K2, T1, T2, O1, O2, sigma2_1, sigma2_2, sf1, sf2, scale_factor, e2_out=None):
    """The per-pair body of :433-574 for N pairs.  kp: x, y [N] (float32) as fields of a KP_DTYPE array; K [N][4] fx fy cx cy; T
    [N][3][4] Tcw rows; O [N][3] the camera centres; sigma2_*, sf_* [N] at each keypoint's octave.  Returns (code [N] int8: 0 when
    every gate passes, else the first gate's code; x3D [N][3] float32).  e2_out (a list) receives the squared reprojection error
    in KF1 and in KF2 of every pair (float32 [N] each; meaningful where the depth gates passed)."""
    N = len(kp1)
    code = np.zeros(N, np.int8)
    x1, y1, x2, y2 = (np.asarray(v, f32) for v in (kp1["x"], kp1["y"], kp2["x"], kp2["y"]))
    one = f32(1)
    invfx1, invfy1, invfx2, invfy2 = one / K1[:, 0], one / K1[:, 1], one / K2[:, 0], one / K2[:, 1]
    xn1 = np.stack([(x1 - K1[:, 2]) * invfx1, (y1 - K1[:, 3]) * invfy1, np.ones(N, f32)], 1)
    xn2 = np.stack([(x2 - K2[:, 2]) * invfx2, (y2 - K2[:, 3]) * invfy2, np.ones(N, f32)], 1)
    R1, R2 = T1[:, :, :3], T2[:, :, :3]
    ray1 = _gemm3(R1.transpose(0, 2, 1), xn1)
    ray2 = _gemm3(R2.transpose(0, 2, 1), xn2)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        cos = (_dot(ray1, ray2) / (np.sqrt(_dot(ray1, ray1)) * np.sqrt(_dot(ray2, ray2)))).astype(f32)
        ok = (cos < cos + one) & (cos > 0) & (cos.astype(f64) < 0.9998)
        code[~ok] = PARALLAX
        w, vt = svd4(linear_triangulation_matrix(xn1, xn2, T1, T2))
        x = vt[:, 3]
        code[(code == 0) & (x[:, 3] == 0)] = W_ZERO
        inv = (1.0 / x[:, 3].astype(f64)).astype(f32)
        X = x[:, :3] * inv[:, None] + f32(0)       # convertTo(alpha = 1 / w, beta = 0)
        X[code != 0] = 0
        t1, t2 = T1[:, :, 3], T2[:, :, 3]
        z1 = (_dot(R1[:, 2], X) + t1[:, 2]).astype(f32)
        code[(code == 0) & (z1 <= 0)] = BEHIND1
        z2 = (_dot(R2[:, 2], X) + t2[:, 2]).astype(f32)
        code[(code == 0) & (z2 <= 0)] = BEHIND2
        for K, R, t, z, kx, ky, s2, c in ((K1, R1, t1, z1, x1, y1, sigma2_1, REPROJ1), (K2, R2, t2, z2, x2, y2, sigma2_2, REPROJ2)):
            xc = (_dot(R[:, 0], X) + t[:, 0]).astype(f32)
            yc = (_dot(R[:, 1], X) + t[:, 1]).astype(f32)
            invz = (1.0 / z.astype(f64)).astype(f32)
            u = K[:, 0] * xc * invz + K[:, 2]
            v = K[:, 1] * yc * invz + K[:, 3]
            ex, ey = u - kx, v - ky
            e2 = ex * ex + ey * ey
            if e2_out is not None:
                e2_out.append(e2)
            code[(code == 0) & (e2.astype(f64) > 5.991 * s2.astype(f64))] = c
        dist1 = np.sqrt(_dot(X - O1, X - O1)).astype(f32)
        dist2 = np.sqrt(_dot(X - O2, X - O2)).astype(f32)
        ratio_dist = dist2 / dist1
        ratio_oct = sf1 / sf2
        rf = f32(1.5) * f32(scale_factor)
        bad = (dist1 == 0) | (dist2 == 0) | (ratio_dist * rf < ratio_oct) | (ratio_dist > ratio_oct * rf)
    code[(code == 0) & bad] = SCALE
    return code, X


def commit(code, kf1, status, out_offset, n):
    """The neighbour-order rule on gate results (code per slot: 0 passed, 2..8 rejected, -1 no pair): a slot that passed at problem
    p becomes DROPPED iff an earlier problem q with the same kf1 and status 0 passed at the same idx1.  In place; returns nnew [P]."""
    P = len(kf1)
    nnew = np.zeros(P, np.int32)
    for p in range(P):
        if status[p]:
            continue
        a, m = out_offset[p], n[kf1[p]]
        mine = code[a:a + m]
        passed = mine == COMMITTED
        for q in range(p):
            if status[q] == 0 and kf1[q] == kf1[p]:
                b = out_offset[q]
                earlier = code[b:b + m]
                passed_q = (earlier == COMMITTED) | (earlier == DROPPED)
                mine[passed & passed_q] = DROPPED
                passed &= ~passed_q
        nnew[p] = int(passed.sum())
    return nnew


def triangulate(k, q, matches12, search_status, scale_factor, scale_factors, level_sigma2, drop=True, e2_out=None):
    """pl_orb_triangulate_dev on host arrays: k = pack_tri_keyframes(...), q = pack_tri_problems(...) (binding.py), matches12
    [n_out], search_status [P].  Returns code [n_out] (int8, UNWRITTEN where the call writes nothing), x3D [n_out][3] (NaN where
    not written), nnew [P] (-1 where not written), status [P].  drop=False leaves the neighbour-order rule out (for the tests);
    e2_out (a dict) receives slot [m] and e2 = (KF1, KF2) squared reprojection errors [m] of the gated pairs."""
    P, n_out = q["P"], q["n_out"]
    n_kf, cap = len(k["n"]), k["cap"]
    code = np.full(n_out, UNWRITTEN, np.int8)
    x3D = np.full((n_out, 3), np.nan, f32)
    nnew = np.full(P, -1, np.int32)
    status = np.zeros(P, np.int32)
    sf, s2 = np.asarray(scale_factors, f32), np.asarray(level_sigma2, f32)
    m12 = np.asarray(matches12, np.int32)
    rows = []
    for p in range(P):
        k1, k2 = int(q["kf1"][p]), int(q["kf2"][p])
        if search_status[p]:
            status[p] = search_status[p]; continue
        if not (0 <= k1 < n_kf and 0 <= k2 < n_kf):
            status[p] = 1; continue
        n1, n2 = int(k["n"][k1]), int(k["n"][k2])
        if not (0 <= n1 <= cap and 0 <= n2 <= cap):
            status[p] = 2; continue
        a = int(q["out_offset"][p])
        if a < 0 or a + n1 > n_out:
            status[p] = 1; continue
        m = m12[a:a + n1]
        if ((m < -1) | (m >= n2)).any():
            status[p] = 4; continue
        code[a:a + n1] = NO_PAIR
        i1 = np.nonzero(m >= 0)[0]
        rows.append((p, k1, k2, a + i1, i1, m[i1]))
    if rows:
        slot = np.concatenate([r[3] for r in rows])
        k1 = np.concatenate([np.full(len(r[4]), r[1]) for r in rows])
        k2 = np.concatenate([np.full(len(r[4]), r[2]) for r in rows])
        kp1 = k["keys_un"][k1, np.concatenate([r[4] for r in rows])]
        kp2 = k["keys_un"][k2, np.concatenate([r[5] for r in rows])]
        T = np.asarray(k["Tcw"], f32).reshape(-1, 4, 4)[:, :3, :]
        O, Kc = np.asarray(k["Ow"], f32).reshape(-1, 3), np.asarray(k["K"], f32).reshape(-1, 4)
        o1, o2 = kp1["octave"], kp2["octave"]
        e2 = []
        c, X = gates(kp1, kp2, Kc[k1], Kc[k2], T[k1], T[k2], O[k1], O[k2], s2[o1], s2[o2], sf[o1], sf[o2], scale_factor, e2)
        if e2_out is not None:
            e2_out.update(slot=slot, e2=e2)
        code[slot] = c
        x3D[slot[c == 0]] = X[c == 0]
    if drop:
        written = status == 0
        nnew[written] = commit(code, q["kf1"], status, q["out_offset"], k["n"])[written]
    else:
        for p in range(P):
            if status[p] == 0:
                a = int(q["out_offset"][p]); nnew[p] = int((code[a:a + k["n"][q["kf1"][p]]] == COMMITTED).sum())
    return code, x3D, nnew, status


def triangulation_matrices(rng, n):
    """n triangulation-shaped 4x4 matrices (A of :458-462): TUM-like intrinsics, baselines about 0.3 m, depths 2.5-9 m, a pixel of
    noise"""
    K = np.array([517.3, 516.5, 318.6, 255.3], f32)
    X = np.stack([rng.uniform(-3, 3, n), rng.uniform(-2, 2, n), rng.uniform(2.5, 9, n)], 1)
    T = np.zeros((n, 2, 3, 4))
    xn = np.zeros((n, 2, 3), f32)
    for v in range(2):
        ang = rng.normal(0, 0.05, (n, 3))
        c = np.zeros((n, 3)) if v == 0 else rng.normal(0, 0.3 / np.sqrt(3), (n, 3))
        for i in range(n):
            R = _rot(ang[i])
            T[i, v, :, :3] = R; T[i, v, :, 3] = -R @ c[i]
        Xc = np.einsum("nij,nj->ni", T[:, v, :, :3], X) + T[:, v, :, 3]
        uv = (K[:2] * Xc[:, :2] / Xc[:, 2:] + K[2:] + rng.normal(0, 1, (n, 2))).astype(f32)
        xn[:, v] = np.stack([(uv[:, 0] - K[2]) * (f32(1) / K[0]), (uv[:, 1] - K[3]) * (f32(1) / K[1]), np.ones(n, f32)], 1)
    T = T.astype(f32)
    return linear_triangulation_matrix(xn[:, 0], xn[:, 1], T[:, 0], T[:, 1])


def _rot(a):
    cx, sx, cy, sy, cz, sz = np.cos(a[0]), np.sin(a[0]), np.cos(a[1]), np.sin(a[1]), np.cos(a[2]), np.sin(a[2])
    return (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
            @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))
