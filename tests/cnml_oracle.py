"""CPU oracle of pl_lsd_triangulate_dev: the three-view triangulation, the gates and the commit of
LocalMapping::CreateNewMapLinesConstraint (src/LocalMapping.cc:966-1439, monocular), restated in numpy on the reference's
arithmetic and vectorised over the triples of a batch.

Every operation is an elementwise numpy operation on float32 or float64 arrays, which rounds once and never contracts, so each
reference expression keeps its C++ promotions and its cv::Mat order (DESIGN.md §8f.6; the cv2 pins are in
tests/test_triangulate_lines.py):
  A * B, A * x          cv::gemm's small-matrix fp32 order ((a0 b0 + a1 b1) + a2 b2), each operation rounded on its own;
  klF.t() * M           cv::gemm with GEMM_1_T: products and sums in fp64 from 0, rounded once;
  K.inv() * x           MatExpr makes it cv::solve(K, x, DECOMP_LU): Cramer's rule in fp64 over det3, one product of the second
                        row rounded in fp32 as lapack.cpp writes it;
  (K2.t()).inv() * t21x cv::solve with three columns: LUImpl in fp32 with partial pivoting;
  K1.inv()              cv::invert: the adjugate in fp64 times 1 / det3;
  A - B, Mat::cross     fp32, each operation rounded;
  Mat::dot, cv::norm    fp64 from 0, in index order; norm = sqrt of that sum;
  s * M.row(2) - M.row(k), M / s, M /= s, cv::SVD   as cnmp_oracle states them for points.
"""
import numpy as np

from cnmp_oracle import _addw, _dot, _gemm3, svd4

f32, f64 = np.float32, np.float64
PI = 3.1415926            # LocalMapping.cc:28

NO_TRIPLE, COMMITTED, HELD, TAKEN, EPIPOLAR, ZERO_NORM, COS_SITA, W_ZERO, PARALLAX, NEAR, LONG, BEHIND = -1, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10
REPROJ1, REPROJ2, REPROJ3, OVERLAP1, OVERLAP2, OVERLAP3 = 11, 12, 13, 14, 15, 16
UNWRITTEN = -128
MAX_ENTRIES = 16


def det3(S):
    """det3 of lapack.cpp for S [..., 3, 3] float32, in fp64"""
    m = lambda i, j: S[..., i, j].astype(f64)
    return m(0, 0) * (m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1)) - m(0, 1) * (m(1, 0) * m(2, 2) - m(1, 2) * m(2, 0)) + \
        m(0, 2) * (m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0))


def inv3(S):
    """cv::invert(S, DECOMP_LU) for 3x3 float32 S [..., 3, 3]: zeros where det3 == 0"""
    d = det3(S)
    with np.errstate(divide="ignore"):
        r = np.where(d != 0, 1.0 / d, 0.0)
    m = lambda i, j: S[..., i, j].astype(f64)
    t = [(m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1)), (m(0, 2) * m(2, 1) - m(0, 1) * m(2, 2)), (m(0, 1) * m(1, 2) - m(0, 2) * m(1, 1)),
         (m(1, 2) * m(2, 0) - m(1, 0) * m(2, 2)), (m(0, 0) * m(2, 2) - m(0, 2) * m(2, 0)), (m(0, 2) * m(1, 0) - m(0, 0) * m(1, 2)),
         (m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0)), (m(0, 1) * m(2, 0) - m(0, 0) * m(2, 1)), (m(0, 0) * m(1, 1) - m(0, 1) * m(1, 0))]
    return np.stack([(x * r).astype(f32) for x in t], -1).reshape(S.shape)


def solve3(S, b):
    """cv::solve(S, b, DECOMP_LU) for 3x3 float32 S [N, 3, 3] and b [N, 3]: zeros where det3 == 0"""
    d = det3(S)
    with np.errstate(divide="ignore"):
        r = np.where(d != 0, 1.0 / d, 0.0)
    m = lambda i, j: S[:, i, j].astype(f64)
    B = lambda i: b[:, i].astype(f64)
    t0 = r * (B(0) * (m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1)) - m(0, 1) * (B(1) * m(2, 2) - m(1, 2) * B(2))
              + m(0, 2) * (B(1) * m(2, 1) - m(1, 1) * B(2)))
    q = (b[:, 1] * S[:, 2, 2]).astype(f64)              # bf(1) * Sf(2,2): two floats, rounded in fp32
    t1 = r * (m(0, 0) * (q - m(1, 2) * B(2)) - B(0) * (m(1, 0) * m(2, 2) - m(1, 2) * m(2, 0))
              + m(0, 2) * (m(1, 0) * B(2) - B(1) * m(2, 0)))
    t2 = r * (m(0, 0) * (m(1, 1) * B(2) - B(1) * m(2, 1)) - m(0, 1) * (m(1, 0) * B(2) - B(1) * m(2, 0))
              + B(0) * (m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0)))
    return np.stack([t0, t1, t2], 1).astype(f32)


def lu_solve3(A, B):
    """cv::solve(A, B, DECOMP_LU) for one 3x3 float32 A and a 3-column B: LUImpl in fp32 (zeros when a pivot is below
    10 FLT_EPSILON)"""
    A, B = np.array(A, f32), np.array(B, f32)
    for i in range(3):
        k = i
        for j in range(i + 1, 3):
            if abs(A[j, i]) > abs(A[k, i]):
                k = j
        if abs(A[k, i]) < f32(10) * np.finfo(f32).eps:
            return np.zeros((3, 3), f32)
        if k != i:
            A[[i, k], i:] = A[[k, i], i:]
            B[[i, k]] = B[[k, i]]
        d = f32(-1) / A[i, i]
        for j in range(i + 1, 3):
            al = A[j, i] * d
            A[j, i + 1:] = A[j, i + 1:] + al * A[i, i + 1:]
            B[j] = B[j] + al * B[i]
    for i in range(2, -1, -1):
        for j in range(3):
            s = B[i, j]
            for q in range(i + 1, 3):
                s = s - A[i, q] * B[q, j]
            B[i, j] = s / A[i, i]
    return B


def gemm33(A, B):
    """A * B for 3x3 float32 matrices in cv::gemm's fp32 order"""
    return np.stack([(A[:, 0:1] * B[0:1, c] + A[:, 1:2] * B[1:2, c]) + A[:, 2:3] * B[2:3, c] for c in range(B.shape[1])], 1).reshape(3, -1)


def cross(a, b):
    """Mat::cross on CV_32F 3-vectors [N, 3]"""
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def kmat(k):
    k = np.asarray(k, f32)
    return np.array([[k[0], 0, k[2]], [0, k[1], k[3]], [0, 0, 1]], f32)


def pair_consts(T1, T2, T3, k1, k2, k3):
    """F21, R12, R13, M1, M2, M3 of :1067-1070, :1083-1084, :1123-1125 for Tcw [4][4] and K [4] (float32)"""
    R1, R2, R3 = T1[:3, :3], T2[:3, :3], T3[:3, :3]
    K1, K2, K3 = kmat(k1), kmat(k2), kmat(k3)
    R21 = gemm33(R2, np.ascontiguousarray(R1.T))
    d = _gemm3(R2.T[None], T2[None, :3, 3])[0] - _gemm3(R1.T[None], T1[None, :3, 3])[0]
    t21 = _gemm3(R2[None], d[None])[0]
    tx = np.array([[0, -t21[2], t21[1]], [t21[2], 0, -t21[0]], [-t21[1], t21[0], 0]], f32)
    F21 = gemm33(gemm33(lu_solve3(K2.T, tx), R21), inv3(K1))
    return dict(F21=F21, R12=gemm33(R1, np.ascontiguousarray(R2.T)), R13=gemm33(R1, np.ascontiguousarray(R3.T)),
                M1=gemm33(K1, T1[:3]), M2=gemm33(K2, T2[:3]), M3=gemm33(K3, T3[:3]), K1=K1, K2=K2, K3=K3)


def _norm(v):
    return np.sqrt(_dot(v, v)).astype(f32)


def _scale(v, n):
    with np.errstate(divide="ignore", invalid="ignore"):
        return v * (1.0 / n.astype(f64)).astype(f32)[:, None] + f32(0)


def _epipolar(F, x, y, lv):
    r = np.stack([x, y, np.ones_like(x)], 1)
    th = _gemm3(F, r)
    t = np.stack([-th[:, 1], th[:, 0]], 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        return (_dot(t, lv) / (np.sqrt(_dot(t, t)) * np.sqrt(_dot(lv, lv)))).astype(f32)


def _plane_normal(K, kl):
    s = np.stack([kl["startPointX"], kl["startPointY"], np.ones(len(kl), f32)], 1).astype(f32)
    e = np.stack([kl["endPointX"], kl["endPointY"], np.ones(len(kl), f32)], 1).astype(f32)
    return cross(solve3(K, s), solve3(K, e))


def _klf_row(f, M):
    k = f.astype(f32).astype(f64)
    return ((k[:, 0:1] * M[:, 0].astype(f64) + k[:, 1:2] * M[:, 1].astype(f64)) + k[:, 2:3] * M[:, 2].astype(f64)).astype(f32)


def _endpoint(r01, M1, x, y):
    A = np.concatenate([r01, _addw(x, M1[:, 2], M1[:, 0])[:, None], _addw(y, M1[:, 2], M1[:, 1])[:, None]], 1)
    w, vt = svd4(A)
    v = vt[:, 3]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        X = v[:, :3] * (1.0 / v[:, 3].astype(f64)).astype(f32)[:, None] + f32(0)
    return v[:, 3] == 0, X


def _cam(T, r, X):
    return (_dot(T[:, r, :3], X) + T[:, r, 3].astype(f64)).astype(f32)


def _smin(a, b):
    return np.where(b < a, b, a)


def _smax(a, b):
    return np.where(a < b, b, a)


def overlap_fails(kl, us, vs, ue, ve, pi=PI):
    a = np.abs(kl["angle"]).astype(f64)
    yd = (a < 3.0 * pi / 4.0) & (a > 1.0 * pi / 4.0)
    ps, pe = np.where(yd, vs, us), np.where(yd, ve, ue)
    ks, ke = np.where(yd, kl["startPointY"], kl["startPointX"]), np.where(yd, kl["endPointY"], kl["endPointX"])
    out = (_smin(pe, ps) > _smax(ks, ke)) | (_smin(ks, ke) > _smax(pe, ps))
    hi, lo = _smin(_smax(pe, ps), _smax(ks, ke)), _smax(_smin(pe, ps), _smin(ks, ke))
    with np.errstate(divide="ignore", invalid="ignore"):
        r1 = (hi - lo) / (_smax(pe, ps) - _smin(pe, ps))
        r2 = (hi - lo) / (_smax(ks, ke) - _smin(ks, ke))
    return out | (r1.astype(f64) < 0.85) | (r2.astype(f64) < 0.85)


def gates(pc, T, K, O, kl, f, s2, median, err_out=None, pi=PI):
    """The per-triple body of :1063-1416 for N triples.  pc: per-triple pair constants (F21, R12, R13, M1, M2, M3, K1, K2, K3,
    each [N][..]); T [3][N][4][4], K [3][N][4], O [3][N][3], kl [3] KEYLINE_DTYPE [N], f [3][N][3] float64, s2 [3][N] sigma^2 at
    each keyline's octave, median [N].  Returns (code [N] int8, line3D [N][6] float32).  err_out (a list) receives (err, 3.84
    sigma^2, u, v) of the six reprojections, view by view, start point first."""
    N = len(median)
    code = np.zeros(N, np.int8)
    first = lambda c, m: code.__setitem__((code == 0) & m, c)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        lv2 = np.stack([(-f[1][:, 1]).astype(f32), f[1][:, 0].astype(f32)], 1)
        r1 = _epipolar(pc["F21"], kl[0]["startPointX"], kl[0]["startPointY"], lv2)
        r2 = _epipolar(pc["F21"], kl[0]["endPointX"], kl[0]["endPointY"], lv2)
        first(EPIPOLAR, (np.abs(r1).astype(f64) > 0.996) | (np.abs(r2).astype(f64) > 0.996))
        L1, L2, L3 = (_plane_normal(pc[f"K{v + 1}"], kl[v]) for v in range(3))
        tw = cross(_gemm3(pc["R12"], L2), _gemm3(pc["R13"], L3))
        n = _norm(tw)
        z1 = n == 0
        tw = _scale(tw, n)
        n = _norm(L1)
        L1 = _scale(L1, n)
        first(ZERO_NORM, z1 | (n == 0))
        cos = np.abs(_dot(L1, tw)).astype(f32)
        first(COS_SITA, cos.astype(f64) > 0.0087)
        r01 = np.concatenate([_klf_row(f[2], pc["M3"])[:, None], _klf_row(f[1], pc["M2"])[:, None]], 1)
        ws, s3 = _endpoint(r01, pc["M1"], kl[0]["startPointX"], kl[0]["startPointY"])
        we, e3 = _endpoint(r01, pc["M1"], kl[0]["endPointX"], kl[0]["endPointY"])
        first(W_ZERO, ws | we)
        par = np.zeros(N, bool)
        for X in (s3, e3):
            n1, n2, n3 = X - O[0], X - O[1], X - O[2]
            d1, d2, d3 = _norm(n1), _norm(n2), _norm(n3)
            c1 = (_dot(n1, n2) / (d1 * d2).astype(f64)).astype(f32)
            c2 = (_dot(n1, n3) / (d1 * d3).astype(f64)).astype(f32)
            par |= (c1.astype(f64) >= 0.99998) | (c2.astype(f64) >= 0.99998)
        first(PARALLAX, par)
        near = ((_norm(s3 - O[0]) / median).astype(f64) < 0.3) | ((_norm(s3 - O[1]) / median).astype(f64) < 0.3)
        first(NEAR, near)
        first(LONG, (_norm(e3 - s3) / median).astype(f64) > 1.0)
        zs = [_cam(T[v], 2, s3) for v in range(3)]
        ze = [_cam(T[v], 2, e3) for v in range(3)]
        first(BEHIND, (zs[0] <= 0) | (ze[0] <= 0) | (zs[1] <= 0) | (ze[1] <= 0) | (zs[2] <= 0) | (ze[2] <= 0))
        uv = []
        for v in range(3):
            th = 3.84 * s2[v].astype(f64)
            bad = np.zeros(N, bool)
            pts = []
            for X, z in ((s3, zs[v]), (e3, ze[v])):
                x, y, iz = _cam(T[v], 0, X), _cam(T[v], 1, X), (1.0 / z.astype(f64)).astype(f32)
                u = K[v][:, 0] * x * iz + K[v][:, 2]
                w = K[v][:, 1] * y * iz + K[v][:, 3]
                err = (f[v][:, 0] * u.astype(f64) + f[v][:, 1] * w.astype(f64)) + f[v][:, 2]
                if err_out is not None:
                    err_out.append((err, th, u, w))
                bad |= err * err > th
                pts.append((u, w))
            first(REPROJ1 + v, bad)
            uv.append(pts)
        for v in range(3):
            (us, vs), (ue, ve) = uv[v]
            first(OVERLAP1 + v, overlap_fails(kl[v], us, vs, ue, ve, pi))
    return code, np.concatenate([s3, e3], 1).astype(f32)


def group_status(k, q, gr, g, matches, search_status):
    """status of group g as plslam_b200.h states it (pl_lsd_triangulate_dev)"""
    n_kf, cap, n = len(k["n"]), k["cap"], k["n"]
    kc, e0, E = int(gr["kf_cur"][g]), int(gr["entry_start"][g]), int(gr["n_entries"][g])
    if E < 0 or E > MAX_ENTRIES:
        return 2
    if e0 < 0 or e0 + E > len(gr["entry_kf"]):
        return 1
    ps = [int(gr["entry_problem"][e0 + e]) for e in range(E)]
    rows = [int(gr["entry_kf"][e0 + e]) for e in range(E)]
    if any(p < 0 or p >= q["P"] for p in ps):
        return 1
    for p in ps:
        if search_status[p]:
            return int(search_status[p])
    inside = lambda r: 0 <= r < n_kf
    if not inside(kc) or any(not inside(r) or not inside(q["kf1"][p]) or not inside(q["kf2"][p]) for r, p in zip(rows, ps)):
        return 1
    ok = lambda r: 0 <= n[r] <= cap
    if not ok(kc) or any(not ok(r) or not ok(q["kf1"][p]) or not ok(q["kf2"][p]) for r, p in zip(rows, ps)):
        return 2
    oo = int(gr["out_offset"][g])
    if oo < 0 or oo + E * (E - 1) // 2 * int(n[kc]) > gr["n_out"]:
        return 1
    if any(q["out_offset"][p] < 0 or q["out_offset"][p] + n[q["kf1"][p]] > q["n_out"] for p in ps):
        return 1
    if any(q["kf1"][p] != kc for p in ps):
        return 3
    for p in ps:
        m = matches[q["out_offset"][p]:q["out_offset"][p] + n[kc]]
        if ((m < -1) | (m >= n[q["kf2"][p]])).any():
            return 4
    return 0


def triangulate_lines(k, q, gr, matches, nmatches, search_status, level_sigma2_line, positional=True, commit_state=True,
                      snapshot=True, pi=PI, err_out=None):
    """pl_lsd_triangulate_dev on host arrays: k = pack_tri_keyframes(..., lines=True), q = pack_tri_problems(...), gr =
    pack_tri_line_groups(...) (binding.py).  Returns code [n_out] (int8, UNWRITTEN where the call writes nothing), line3D
    [n_out][6] (NaN where not written), nnew [G] (-1 where not written), status [G].  For the tests' mutants: positional=False
    pairs each entry with its problem's kf2 instead of its positional keyframe; commit_state=False lets a passed slot commit even
    when an earlier commit took one of its slots; snapshot=False ignores has_ml; pi replaces PI in the overlap axis."""
    G, n_out = gr["G"], gr["n_out"]
    code = np.full(n_out, UNWRITTEN, np.int8)
    line3D = np.full((n_out, 6), np.nan, f32)
    nnew = np.full(G, -1, np.int32)
    status = np.zeros(G, np.int32)
    m_all = np.asarray(matches, np.int32)
    s2 = np.asarray(level_sigma2_line, f32)
    cap = k["cap"]
    T = np.asarray(k["Tcw"], f32).reshape(-1, 4, 4)
    Kc, O = np.asarray(k["K"], f32).reshape(-1, 4), np.asarray(k["Ow"], f32).reshape(-1, 3)
    kls, lf, has = k["keylines"], np.asarray(k["line_func"], f64), k["has_ml"].astype(bool)
    if not snapshot:
        has = np.zeros_like(has)
    todo = []       # (g, slots, rows (3), idx (3), pair consts, median)
    walks = []
    for g in range(G):
        status[g] = group_status(k, q, gr, g, m_all, search_status)
        if status[g]:
            continue
        kc, e0, E = int(gr["kf_cur"][g]), int(gr["entry_start"][g]), int(gr["n_entries"][g])
        n = int(k["n"][kc])
        oo = int(gr["out_offset"][g])
        ps = [int(gr["entry_problem"][e0 + e]) for e in range(E)]
        rows = [int(gr["entry_kf"][e0 + e]) if positional else int(q["kf2"][p]) for e, p in enumerate(ps)]
        med = [float(gr["entry_median_depth"][e0 + e]) for e in range(E)]
        pr = 0
        walk = []
        for i in range(E):
            for j in range(i + 1, E):
                base = oo + pr * n
                ikl = np.arange(n)
                i1 = m_all[q["out_offset"][ps[i]] + ikl]
                i2 = m_all[q["out_offset"][ps[j]] + ikl]
                none = (nmatches[ps[i]] == 0) | (nmatches[ps[j]] == 0) | (i1 == -1) | (i2 == -1) | (i1 >= k["n"][rows[i]]) | \
                    (i2 >= k["n"][rows[j]])
                code[base:base + n] = NO_TRIPLE
                held = ~none
                held[~none] = has[kc, ikl[~none]] | has[rows[i], i1[~none]] | has[rows[j], i2[~none]]
                code[base + np.nonzero(held)[0]] = HELD
                ev = np.nonzero(~none & ~held)[0]
                if len(ev):
                    pc = pair_consts(T[kc], T[rows[i]], T[rows[j]], Kc[kc], Kc[rows[i]], Kc[rows[j]])
                    todo.append((base + ev, (kc, rows[i], rows[j]), (ev, i1[ev], i2[ev]), pc, med[i]))
                walk.append((base, i1, i2, rows[i], rows[j]))
                pr += 1
        walks.append((g, kc, rows, n, walk))
    if todo:
        slots = np.concatenate([t[0] for t in todo])
        cnt = [len(t[0]) for t in todo]
        rep = lambda x: np.repeat(np.asarray(x), cnt, axis=0)
        pc = {key: rep([t[3][key] for t in todo]) for key in todo[0][3]}
        rw = [np.concatenate([np.full(len(t[0]), t[1][v]) for t in todo]) for v in range(3)]
        ix = [np.concatenate([t[2][v] for t in todo]) for v in range(3)]
        kl = [kls[rw[v], ix[v]] for v in range(3)]
        c, L = gates(pc, [T[rw[v]] for v in range(3)], [Kc[rw[v]] for v in range(3)], [O[rw[v]] for v in range(3)], kl,
                     [lf[rw[v], ix[v]] for v in range(3)], [s2[kl[v]["octave"]] for v in range(3)], rep([t[4] for t in todo]).astype(f32),
                     err_out, pi)
        code[slots] = c
        line3D[slots[c == 0]] = L[c == 0]
    for g, kc, rows, n, walk in walks:
        taken = {}

        def bits(r):
            if r not in taken:
                taken[r] = has[r].copy()
            return taken[r]
        cnt = 0
        for base, i1, i2, ra, rb in walk:
            for ikl in range(n):
                c = code[base + ikl]
                if not (c == COMMITTED or c >= EPIPOLAR):
                    continue
                t = bits(kc)[ikl] or bits(ra)[i1[ikl]] or bits(rb)[i2[ikl]]
                if t and commit_state:
                    code[base + ikl] = TAKEN
                elif c == COMMITTED:
                    bits(kc)[ikl] = True; bits(ra)[i1[ikl]] = True; bits(rb)[i2[ikl]] = True
                    cnt += 1
        nnew[g] = cnt
    return code, line3D, nnew, status
