"""Generate tests/golden/refcalls/create_new_map_lines.npz: the line half of LocalMapping::CreateNewMapLinesConstraint run as the
reference runs it (monocular), on the seeded scene of tests/cnml_scene.py.  The neighbours that pass the baseline test
(:928-952) are searched in order by the reference's own LSDmatcher::SearchForTriangulation (oracle/_ref/libref_match.so, or its
stored outputs, oracle/refstore.py; th = TH_HIGH = 80, nnratio 0.8, isDouble, :961).  Then the second loop :966-1439 runs triple by
triple, with entry i paired with vpNeighKFs[i] (:976, :1002) and the map-line state updated as each line is created
(:1428-1430).  cv2 does each cv::Mat operation: cv2.gemm (with GEMM_1_T for klF.t() * M), cv2.solve for K.inv() * x and
(K2.t()).inv() * t21x (MatExpr turns an inverse times a Mat into a solve), cv2.invert for K1.inv(), cv2.subtract,
cv2.addWeighted for s * M1.row(2) - M1.row(k), cv2.SVDecomp, cv2.norm; Mat::dot in fp64; Mat::cross in fp32 as OpenCV's
Mat::cross writes it (cv2 has no binding); M / s and M /= s as M * (float)(1.0 / s) + 0.

The fixture holds the scene, which neighbours were searched, the reference searches' matches and counts, and the new lines in
creation order: entry pair (i, j), ikl, idx1, idx2 and the bits of the six floats.  tests/test_triangulate_lines.py replays it on
the oracle (tests/cnml_oracle.py) and tests/test_triangulate_lines_gpu.py through the device calls.

Needs the reference library built (make -C oracle ref) or its stored outputs, and cv2.  Run from the repo root:
    python tools/gen_create_new_map_lines.py
"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle  # noqa: E402
import cnml_scene as cs  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "refcalls", "create_new_map_lines.npz")
f32 = np.float32
PI = 3.1415926
LU = cv2.DECOMP_LU


def dot(a, b):
    return sum(float(x) * float(y) for x, y in zip(np.ravel(a), np.ravel(b)))


def cross(a, b):
    a, b = np.ravel(a).astype(f32), np.ravel(b).astype(f32)
    return np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]], f32).reshape(3, 1)


def col(*v):
    return np.array(v, f32).reshape(-1, 1)


def cam(kf):
    T = kf["Tcw"].reshape(4, 4).astype(f32)
    k = kf["K"]
    K = np.array([[k[0], 0, k[2]], [0, k[1], k[3]], [0, 0, 1]], f32)
    return dict(R=np.ascontiguousarray(T[:3, :3]), Rt=np.ascontiguousarray(T[:3, :3].T), t=np.ascontiguousarray(T[:3, 3:4]),
                T=np.ascontiguousarray(T[:3]), O=kf["Ow"].reshape(3, 1).astype(f32), K=K, k=k)


def overlap_fails(kl, us, vs, ue, ve):
    if abs(float(kl["angle"])) < 3.0 * PI / 4.0 and abs(float(kl["angle"])) > 1.0 * PI / 4.0:
        p1, p2, k1, k2 = ve, vs, kl["startPointY"], kl["endPointY"]
    else:
        p1, p2, k1, k2 = ue, us, kl["startPointX"], kl["endPointX"]
    if min(p1, p2) > max(k1, k2) or min(k1, k2) > max(p1, p2):
        return True
    hi, lo = min(max(p1, p2), max(k1, k2)), max(min(p1, p2), min(k1, k2))
    with np.errstate(divide="ignore", invalid="ignore"):
        r1 = (hi - lo) / (max(p1, p2) - min(p1, p2))
        r2 = (hi - lo) / (max(k1, k2) - min(k1, k2))
    return r1 < 0.85 or r2 < 0.85


def triple(c1, c2, c3, F21, kl, f, median, s2):
    """:1063-1416 for one triple with cv2; returns (code, s3D, e3D)"""
    l1, l2, l3 = kl
    lv2 = col(-f[1][1], f[1][0])
    for x, y in ((l1["startPointX"], l1["startPointY"]), (l1["endPointX"], l1["endPointY"])):
        th = cv2.gemm(F21, col(x, y, 1), 1, None, 0)
        th_ = col(-th[1, 0], th[0, 0])
        r = f32(dot(th_, lv2) / (cv2.norm(th_) * cv2.norm(lv2)))
        if abs(r) > 0.996:
            return 3, None, None
    R12, R13 = cv2.gemm(c1["R"], c2["Rt"], 1, None, 0), cv2.gemm(c1["R"], c3["Rt"], 1, None, 0)
    L = []
    for c, k in ((c1, l1), (c2, l2), (c3, l3)):
        s_ = cv2.solve(c["K"], col(k["startPointX"], k["startPointY"], 1), flags=LU)[1]
        e_ = cv2.solve(c["K"], col(k["endPointX"], k["endPointY"], 1), flags=LU)[1]
        L.append(cross(s_, e_))
    tw = cross(cv2.gemm(R12, L[1], 1, None, 0), cv2.gemm(R13, L[2], 1, None, 0))
    n = f32(cv2.norm(tw))
    if n == 0:
        return 4, None, None
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        tw = tw * f32(1.0 / float(n)) + f32(0)
        n = f32(cv2.norm(L[0]))
        L1 = L[0] * f32(1.0 / float(n)) + f32(0)
    if n == 0:
        return 4, None, None
    if float(f32(abs(dot(L1, tw)))) > 0.0087:
        return 5, None, None
    M1, M2, M3 = (cv2.gemm(c["K"], c["T"], 1, None, 0) for c in (c1, c2, c3))
    kf3, kf2 = np.array(f[2], f32).reshape(3, 1), np.array(f[1], f32).reshape(3, 1)
    r0 = cv2.gemm(kf3, M3, 1, None, 0, flags=cv2.GEMM_1_T)
    r1 = cv2.gemm(kf2, M2, 1, None, 0, flags=cv2.GEMM_1_T)
    P = []
    for x, y in ((l1["startPointX"], l1["startPointY"]), (l1["endPointX"], l1["endPointY"])):
        A = np.concatenate([r0, r1, cv2.addWeighted(M1[2:3], float(x), M1[0:1], -1.0, 0.0),
                            cv2.addWeighted(M1[2:3], float(y), M1[1:2], -1.0, 0.0)])
        w, u, vt = cv2.SVDecomp(A, flags=cv2.SVD_MODIFY_A | cv2.SVD_FULL_UV)
        v = vt[3].reshape(4, 1)
        if v[3, 0] == 0:
            return 6, None, None
        P.append(v[:3] * f32(1.0 / float(v[3, 0])) + f32(0))
    s3, e3 = P
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for X in (s3, e3):
            n1, n2, n3 = (cv2.subtract(X, c["O"]) for c in (c1, c2, c3))
            d1, d2, d3 = (f32(cv2.norm(v)) for v in (n1, n2, n3))
            if float(f32(dot(n1, n2) / float(d1 * d2))) >= 0.99998 or float(f32(dot(n1, n3) / float(d1 * d3))) >= 0.99998:
                return 7, None, None
        if float(f32(cv2.norm(cv2.subtract(s3, c1["O"]))) / median) < 0.3:
            return 8, None, None
        if float(f32(cv2.norm(cv2.subtract(s3, c2["O"]))) / median) < 0.3:
            return 8, None, None
        if float(f32(cv2.norm(cv2.subtract(e3, s3))) / median) > 1:
            return 9, None, None
        z = {}
        for v, c in enumerate((c1, c2, c3)):
            for X, nm in ((s3, "s"), (e3, "e")):
                z[v, nm] = f32(dot(c["R"][2], X) + float(c["t"][2, 0]))
                if z[v, nm] <= 0:
                    return 10, None, None
        uv = {}
        for v, c in enumerate((c1, c2, c3)):
            sig = float(s2[kl[v]["octave"]])
            for X, nm in ((s3, "s"), (e3, "e")):
                x, y = f32(dot(c["R"][0], X) + float(c["t"][0, 0])), f32(dot(c["R"][1], X) + float(c["t"][1, 0]))
                iz = f32(1.0 / float(z[v, nm]))
                u_, v_ = c["k"][0] * x * iz + c["k"][2], c["k"][1] * y * iz + c["k"][3]
                err = f[v][0] * float(u_) + f[v][1] * float(v_) + f[v][2]
                if err * err > 3.84 * sig:
                    return 11 + v, None, None
                uv[v, nm] = (u_, v_)
        for v in range(3):
            (us, vs), (ue, ve) = uv[v, "s"], uv[v, "e"]
            if overlap_fails(kl[v], us, vs, ue, ve):
                return 14 + v, None, None
    return 0, s3.ravel(), e3.ravel()


def reference_loop(s):
    kfs = s["kfs"]
    has = [k["has_ml"].astype(bool).copy() for k in kfs]
    neigh = list(range(1, len(kfs)))                        # vpNeighKFs
    srch = s["searched"]
    entries = []                                            # TotalvMatchedIndices / nTotalMatched
    for j in neigh:
        if srch[j - 1]:
            nm, m = oracle.lsd_search_for_triangulation(kfs[0]["ldesc"], has[0], kfs[j]["ldesc"], has[j], 0.8, True, 80.0, impl="ref")
            entries.append((m, nm))
    cams = [cam(k) for k in kfs]
    new, hist = [], np.zeros(18, np.int64)
    n_cur = len(kfs[0]["keylines"])
    for i in range(len(entries) - 1):
        if entries[i][1] == 0:
            continue
        k2 = neigh[i]
        c1, c2 = cams[0], cams[k2]
        R21 = cv2.gemm(c2["R"], c1["Rt"], 1, None, 0)
        t21 = cv2.gemm(c2["R"], cv2.subtract(cv2.gemm(c2["Rt"], c2["t"], 1, None, 0), cv2.gemm(c1["Rt"], c1["t"], 1, None, 0)), 1, None, 0)
        tx = np.array([[0, -t21[2, 0], t21[1, 0]], [t21[2, 0], 0, -t21[0, 0]], [-t21[1, 0], t21[0, 0], 0]], f32)
        S = cv2.solve(np.ascontiguousarray(c2["K"].T), tx, flags=LU)[1]
        F21 = cv2.gemm(cv2.gemm(S, R21, 1, None, 0), cv2.invert(c1["K"], flags=LU)[1], 1, None, 0)
        for j in range(i + 1, len(entries)):
            if entries[j][1] == 0:
                continue
            k3 = neigh[j]
            c3 = cams[k3]
            for ikl in range(n_cur):
                idx1, idx2 = int(entries[i][0][ikl]), int(entries[j][0][ikl])
                if idx1 == -1 or idx2 == -1 or idx1 >= len(kfs[k2]["keylines"]) or idx2 >= len(kfs[k3]["keylines"]):
                    continue
                if has[0][ikl] or has[k2][idx1] or has[k3][idx2]:
                    hist[1] += 1
                    continue
                kl = (kfs[0]["keylines"][ikl], kfs[k2]["keylines"][idx1], kfs[k3]["keylines"][idx2])
                f = (kfs[0]["line_func"][ikl], kfs[k2]["line_func"][idx1], kfs[k3]["line_func"][idx2])
                c, s3, e3 = triple(c1, c2, c3, F21, kl, f, f32(s["medians"][k2]), s["level_sigma2_line"])
                hist[c] += 1
                if c == 0:
                    new.append((i, j, ikl, idx1, idx2, *np.concatenate([s3, e3]).astype(f32).view(np.uint32)))
                    has[0][ikl] = has[k2][idx1] = has[k3][idx2] = True
    return entries, np.array(new, np.int64), hist


def searched(s):
    """:928-952 monocular: baseline / ComputeSceneMedianDepth(2) >= 0.01"""
    O = [k["Ow"].astype(np.float64) for k in s["kfs"]]
    return np.array([float(f32(np.sqrt(np.sum((O[j] - O[0]) ** 2)))) / s["medians"][j] >= 0.01 for j in range(1, len(O))])


if __name__ == "__main__":
    s = cs.scene()
    s["searched"] = searched(s)
    entries, new, hist = reference_loop(s)
    kfs = s["kfs"]
    out = dict(kf_start=np.concatenate([[0], np.cumsum([len(k["keylines"]) for k in kfs])]).astype(np.int32),
               ldesc=np.concatenate([k["ldesc"] for k in kfs]), has_ml=np.concatenate([k["has_ml"] for k in kfs]),
               keylines=np.concatenate([k["keylines"] for k in kfs]), line_func=np.concatenate([k["line_func"] for k in kfs]),
               Tcw=np.stack([k["Tcw"] for k in kfs]), Ow=np.stack([k["Ow"] for k in kfs]), K=np.stack([k["K"] for k in kfs]),
               medians=s["medians"], level_sigma2_line=s["level_sigma2_line"], searched=s["searched"],
               ref_matches=np.concatenate([e[0] for e in entries]).astype(np.int32),
               ref_nmatches=np.array([e[1] for e in entries], np.int32),
               ref_new=new[:, :5].astype(np.int32), ref_line3D=new[:, 5:].astype(np.uint32).view(np.float32), ref_hist=hist)
    np.savez_compressed(OUT, **out)
    print(f"{OUT}: {len(kfs)} keyframes, searched {s['searched'].astype(int).tolist()}, nmatches {out['ref_nmatches'].tolist()}; "
          f"{len(new)} new lines, per pair {np.unique(new[:, 0] * 100 + new[:, 1], return_counts=True)}; codes 0..17 over the "
          f"reference's triples {hist.tolist()}")
