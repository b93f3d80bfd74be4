"""Generate tests/golden/refcalls/create_new_map_points.npz: the point half of LocalMapping::CreateNewMapPoints run as the reference
runs it, on a seeded scene: the neighbours in order, each searched by the reference's own ORBmatcher::SearchForTriangulation
(oracle/_ref/libref_match.so, ORBmatcher(0.6, false) as LocalMapping.cc:339 makes it) against the map-point state the earlier
neighbours left, then every pair triangulated and gated as LocalMapping.cc:417-574 states it, with cv2 doing each cv::Mat operation
(cv2.gemm for Rwc * xn, cv2.addWeighted for the rows of A, cv2.SVDecomp, cv2.norm; Mat::dot in fp64), and a new map point
registered on both keyframes (AddMapPoint, :582-583).

The scene: a current keyframe and eight neighbours with their own poses and intrinsics, all viewing one set of 3-D points, plus
clutter.  Neighbour 3 sits 9 cm from the current keyframe (the parallax gate), neighbour 6 1 cm (the baseline / median-depth test
of :384-388 skips it, so the reference never searches it).  Some views are "ghosts": the keypoint is moved along the current
keyframe's ray (it stays on the epipolar line) to a point behind the cameras or far away, or across the line (the depth,
reprojection and scale gates).  Octaves are drawn independently of depth (the scale gate).  With F12 = ComputeF12 the search's
band (3.84 sigma^2 in KF2) is narrower than the reprojection gates, and a ghost behind the cameras fails the parallax gate first
(its rays point apart), so the reference's pairs reach codes 2, 4, 5 and 8 here; tests/test_triangulate_batch.py reaches every code
with pairs the search did not choose.  Points seen by several neighbours
are matched at each (the drop rule), and two current-keyframe keypoints share one neighbour keypoint's descriptor (two idx1 with
one idx2).

The fixture holds the scene, which neighbours were searched, and the reference's new points in creation order: neighbour, idx1,
idx2 and the x3D bits.  tests/test_triangulate_batch.py replays it on the oracle (tests/cnmp_oracle.py) with the snapshot
protocol, and tests/test_triangulate_batch_gpu.py through the device calls.

Needs the reference library built (make -C oracle ref) and cv2.  Run from the repo root:  python tools/gen_create_new_map_points.py
"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle  # noqa: E402
from plslam_b200 import synth  # noqa: E402
from plslam_b200.binding import KP_DTYPE  # noqa: E402
import triangulation_protocol as tp  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "refcalls", "create_new_map_points.npz")
f32 = np.float32


def rot(a):
    cx, sx, cy, sy, cz, sz = np.cos(a[0]), np.sin(a[0]), np.cos(a[1]), np.sin(a[1]), np.cos(a[2]), np.sin(a[2])
    return (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
            @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))


def scene(seed=11, n_neigh=8, n_pts=500, n_clutter=100, w=640, h=480, nlevels=8, scale=1.2):
    rng = np.random.default_rng(seed)
    sf = (scale ** np.arange(nlevels)).astype(np.float32)
    n_kf = 1 + n_neigh
    X = np.stack([rng.uniform(-3, 3, n_pts), rng.uniform(-2, 2, n_pts), rng.uniform(2.5, 9, n_pts)], 1)
    code = rng.integers(0, 256, (n_pts, 32), dtype=np.uint8)
    node_of = rng.integers(0, 120, n_pts)
    Tcw = np.zeros((n_kf, 16), np.float32); Ow = np.zeros((n_kf, 3), np.float32); K = np.zeros((n_kf, 4), np.float32)
    kf_start = [0]; keys, desc, has_mp, node, mp_depth = [], [], [], [], []
    C0 = np.zeros(3)
    for k in range(n_kf):
        if k == 0:
            c = C0
        elif k == 3:
            c = np.array([0.09, 0.0, 0.0])
        elif k == 6:
            c = np.array([0.0, 0.01, 0.0])
        else:
            c = np.array([0.3 * np.cos(k), 0.1 * np.sin(2 * k), 0.05 * k]) + rng.normal(0, 0.03, 3)
        R = rot(rng.normal(0, 0.04, 3))
        T = np.eye(4); T[:3, :3] = R; T[:3, 3] = -R @ c
        Tcw[k] = T.reshape(-1); Ow[k] = c
        K[k] = np.array(synth.TUM1_K, np.float32) + (0 if k == 0 else rng.normal(0, 3, 4).astype(np.float32))
        Xv = X.copy()
        if k > 0:                     # ghosts: this view sees a point moved along the current keyframe's ray
            g = rng.random(n_pts)
            Xv[g < 0.04] = C0 - 0.6 * (X[g < 0.04] - C0)                              # behind both cameras
            far = (g >= 0.04) & (g < 0.08)
            Xv[far] = C0 + 2.5 * (X[far] - C0)                                          # the scale gate
            near = (g >= 0.08) & (g < 0.12)
            Xv[near] = C0 + 0.04 * (X[near] - C0)                                       # in front of KF1, behind KF2
        Xc = Xv @ R.T + T[:3, 3]
        uv = np.stack([K[k, 0] * Xc[:, 0] / Xc[:, 2] + K[k, 2], K[k, 1] * Xc[:, 1] / Xc[:, 2] + K[k, 3]], 1)
        octv = rng.integers(0, nlevels, n_pts)
        uv = uv + rng.normal(0, 0.6, uv.shape) * sf[octv][:, None]
        if k > 0:                     # a few views pushed across the epipolar band's middle (the reprojection gates)
            off = rng.random(n_pts) < 0.15
            uv[off] += rng.normal(0, 2.5, (off.sum(), 2)) * sf[octv[off]][:, None]
        ok = (uv[:, 0] > 20) & (uv[:, 0] < w - 20) & (uv[:, 1] > 20) & (uv[:, 1] < h - 20) & (rng.random(n_pts) < 0.85)
        ids = rng.permutation(np.nonzero(ok)[0])
        n = len(ids) + n_clutter
        kp = np.zeros(n, KP_DTYPE)
        kp["x"][:len(ids)], kp["y"][:len(ids)], kp["octave"][:len(ids)] = uv[ids, 0], uv[ids, 1], octv[ids]
        kp["x"][len(ids):], kp["y"][len(ids):] = rng.uniform(20, w - 20, n_clutter), rng.uniform(20, h - 20, n_clutter)
        kp["octave"][len(ids):] = rng.integers(0, nlevels, n_clutter)
        kp["angle"] = rng.uniform(0, 360, n); kp["size"] = 31 * sf[kp["octave"]]; kp["class_id"] = -1
        d = np.concatenate([code[ids], rng.integers(0, 256, (n_clutter, 32), dtype=np.uint8)])
        for _ in range(10):
            r = np.nonzero(rng.random(len(ids)) < 0.7)[0]; b = rng.integers(0, 256, len(r))
            d[r, b // 8] ^= (1 << (b % 8)).astype(np.uint8)
        nd = np.concatenate([node_of[ids], rng.integers(100, 140, n_clutter)]).astype(np.uint32)
        if k == 0:                    # two current-keyframe keypoints with one point's descriptor, next to each other
            src = rng.choice(len(ids), 6, replace=False)
            for t, s in enumerate(src):
                j = len(ids) + t
                kp[j] = kp[s]; kp["x"][j] += 0.7; kp["y"][j] -= 0.4; d[j] = d[s]; nd[j] = nd[s]
        keys.append(kp); desc.append(d)
        hm = (rng.random(n) < 0.2).astype(np.uint8)
        if k == 0:
            hm[len(ids):len(ids) + 6] = 0; hm[src] = 0
        has_mp.append(hm)
        node.append(nd)
        # depths of this keyframe's map points (ComputeSceneMedianDepth): the true points it holds, clutter at random depths
        z = np.concatenate([Xc[ids, 2], rng.uniform(2.5, 9, n_clutter)])
        mp_depth.append(np.where(hm == 1, z, np.nan).astype(np.float32))
        kf_start.append(kf_start[-1] + n)
    Km = lambda k: np.array([[K[k, 0], 0, K[k, 2]], [0, K[k, 1], K[k, 3]], [0, 0, 1]], np.float64)
    T = Tcw.reshape(-1, 4, 4).astype(np.float64)
    F12 = np.zeros((n_neigh, 9), np.float32)
    for j in range(1, n_kf):
        R12 = T[0, :3, :3] @ T[j, :3, :3].T; t12 = -R12 @ T[j, :3, 3] + T[0, :3, 3]
        tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]])
        F12[j - 1] = (np.linalg.inv(Km(0)).T @ tx @ R12 @ np.linalg.inv(Km(j))).reshape(-1)
    return dict(kf_start=np.array(kf_start, np.int32), keys=np.concatenate(keys), desc=np.concatenate(desc),
                has_mp=np.concatenate(has_mp), node=np.concatenate(node), Tcw=Tcw, Ow=Ow, K=K, F12=F12, scale_factors=sf,
                level_sigma2=(sf * sf).astype(np.float32), mp_depth=np.concatenate(mp_depth), scale_factor=np.float32(scale))


def searched(s):
    """:372-389 monocular: baseline / ComputeSceneMedianDepth(2) >= 0.01"""
    out = []
    for j in range(1, len(s["kf_start"]) - 1):
        baseline = f32(np.sqrt(np.sum((s["Ow"][j].astype(np.float64) - s["Ow"][0]) ** 2)))
        a, b = s["kf_start"][j], s["kf_start"][j + 1]
        z = np.sort(s["mp_depth"][a:b][~np.isnan(s["mp_depth"][a:b])])
        med = z[(len(z) - 1) // 2]
        out.append(bool(baseline / med >= 0.01))
    return np.array(out)


def gates_cv2(kp1, kp2, kf1, kf2, sf, s2, scale_factor):
    """:433-574 for one monocular pair with cv2 doing the cv::Mat work.  Returns (code, x3D)."""
    def cam(kf):
        T = kf["Tcw"].reshape(4, 4)
        return T[:3, :3].copy(), T[:3, 3:4].copy(), np.ascontiguousarray(T[:3]), kf["Ow"].reshape(3, 1), kf["K"]
    R1, t1, T1, O1, K1 = cam(kf1)
    R2, t2, T2, O2, K2 = cam(kf2)
    one = f32(1)
    xn1 = np.array([[(f32(kp1["x"]) - K1[2]) * (one / K1[0])], [(f32(kp1["y"]) - K1[3]) * (one / K1[1])], [1]], f32)
    xn2 = np.array([[(f32(kp2["x"]) - K2[2]) * (one / K2[0])], [(f32(kp2["y"]) - K2[3]) * (one / K2[1])], [1]], f32)
    ray1 = cv2.gemm(np.ascontiguousarray(R1.T), xn1, 1, None, 0)
    ray2 = cv2.gemm(np.ascontiguousarray(R2.T), xn2, 1, None, 0)
    dot = lambda a, b: sum(float(x) * float(y) for x, y in zip(a.ravel(), b.ravel()))
    cos = f32(dot(ray1, ray2) / (cv2.norm(ray1) * cv2.norm(ray2)))
    if not (cos < cos + one and cos > 0 and float(cos) < 0.9998):
        return 2, None
    A = np.concatenate([cv2.addWeighted(T1[2:3], float(xn1[0, 0]), T1[0:1], -1.0, 0.0), cv2.addWeighted(T1[2:3], float(xn1[1, 0]), T1[1:2], -1.0, 0.0),
                        cv2.addWeighted(T2[2:3], float(xn2[0, 0]), T2[0:1], -1.0, 0.0), cv2.addWeighted(T2[2:3], float(xn2[1, 0]), T2[1:2], -1.0, 0.0)])
    w, u, vt = cv2.SVDecomp(A, flags=cv2.SVD_MODIFY_A | cv2.SVD_FULL_UV)
    x = vt[3].reshape(4, 1)
    if x[3, 0] == 0:
        return 3, None
    X = x[:3] * f32(1.0 / float(x[3, 0])) + f32(0)
    z1 = f32(dot(R1[2], X) + float(t1[2, 0]))
    if z1 <= 0:
        return 4, None
    z2 = f32(dot(R2[2], X) + float(t2[2, 0]))
    if z2 <= 0:
        return 5, None
    for R, t, K, z, kp, c in ((R1, t1, K1, z1, kp1, 6), (R2, t2, K2, z2, kp2, 7)):
        xc, yc = f32(dot(R[0], X) + float(t[0, 0])), f32(dot(R[1], X) + float(t[1, 0]))
        invz = f32(1.0 / float(z))
        u_, v_ = K[0] * xc * invz + K[2], K[1] * yc * invz + K[3]
        ex, ey = u_ - f32(kp["x"]), v_ - f32(kp["y"])
        if float(ex * ex + ey * ey) > 5.991 * float(s2[kp["octave"]]):
            return c, None
    d1, d2 = f32(cv2.norm(X - O1)), f32(cv2.norm(X - O2))
    if d1 == 0 or d2 == 0:
        return 8, None
    rd, ro, rf = d2 / d1, sf[kp1["octave"]] / sf[kp2["octave"]], f32(1.5) * f32(scale_factor)
    if rd * rf < ro or rd > ro * rf:
        return 8, None
    return 0, X.ravel().astype(f32)


def reference_loop(s):
    kfs = [tp.keyframe(s, k) for k in range(len(s["kf_start"]) - 1)]
    has = [k["has_mp"] for k in kfs]
    srch = s["searched"]
    new, codes = [], []
    for j in range(1, len(kfs)):
        if not srch[j - 1]:
            continue
        m = oracle.search_for_triangulation(*tp.search_args(s, j, has[0], has[j]), False, impl="ref")[1]
        for idx1, idx2 in tp.pairs_of(m):
            c, X = gates_cv2(kfs[0]["keys"][idx1], kfs[j]["keys"][idx2], kfs[0], kfs[j], s["scale_factors"], s["level_sigma2"],
                             s["scale_factor"])
            codes.append(c)
            if c == 0:
                new.append((j, idx1, idx2, *X.view(np.uint32)))
                has[0][idx1] = 1
                has[j][idx2] = 1
    return np.array(new, np.int64), np.bincount(codes, minlength=9)


if __name__ == "__main__":
    s = scene()
    s["searched"] = searched(s)
    new, hist = reference_loop(s)
    s["ref_new"] = new[:, :3].astype(np.int32)
    s["ref_x3D"] = new[:, 3:].astype(np.uint32).view(np.float32)
    np.savez_compressed(OUT, **s)
    print(f"{OUT}: {len(s['keys'])} keypoints in {len(s['kf_start']) - 1} keyframes; searched {s['searched'].astype(int).tolist()}; "
          f"{len(new)} new points, per neighbour {np.bincount(new[:, 0], minlength=len(s['kf_start']) - 1)[1:].tolist()}; "
          f"gate codes 0..8 over the reference's pairs {hist.tolist()}")
