"""Generate tests/golden/refcalls/triangulation_protocol.npz: the neighbour loop of LocalMapping::CreateNewMapPoints run by the
reference's own ORBmatcher::SearchForTriangulation (oracle/_ref/libref_match.so, ORBmatcher(0.6, false) as LocalMapping.cc:339
makes it), on a seeded scene.

The scene: a current keyframe and six neighbours with their own poses and intrinsics, all viewing one set of 3-D points, plus
clutter.  A point's views share a vocabulary node and carry its descriptor with a few flipped bits; some keypoints already hold a
map point.  The triangulation between two searches is a deterministic stand-in (tests/triangulation_protocol.py): a pair with an
even idx1 + idx2 gets a new map point on both keyframes.  A point seen by several neighbours is matched at each of them, so the
later searches skip keypoints that an earlier neighbour triangulated.  The fixture holds the scene and each neighbour's
vMatchedIndices.  tests/test_triangulation_batch.py replays it on the oracle with the snapshot protocol of INTEGRATION.md, and
tests/test_triangulation_batch_gpu.py through the device call.

Needs the reference library built (make -C oracle ref).  Run from the repo root:  python tools/gen_triangulation_protocol.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle  # noqa: E402
from plslam_b200 import synth  # noqa: E402
from plslam_b200.binding import KP_DTYPE  # noqa: E402
import triangulation_protocol as tp  # noqa: E402

OUT = tp.FIXTURE


def rot(a):
    cx, sx, cy, sy, cz, sz = np.cos(a[0]), np.sin(a[0]), np.cos(a[1]), np.sin(a[1]), np.cos(a[2]), np.sin(a[2])
    return (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
            @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))


def scene(seed=4, n_neigh=6, n_pts=400, n_clutter=100, w=640, h=480, nlevels=8, scale=1.2):
    rng = np.random.default_rng(seed)
    sf = (scale ** np.arange(nlevels)).astype(np.float32)
    n_kf = 1 + n_neigh
    X = np.stack([rng.uniform(-3, 3, n_pts), rng.uniform(-2, 2, n_pts), rng.uniform(2.5, 9, n_pts)], 1)
    code = rng.integers(0, 256, (n_pts, 32), dtype=np.uint8)
    node_of = rng.integers(0, 120, n_pts)
    Tcw = np.zeros((n_kf, 16), np.float32); Ow = np.zeros((n_kf, 3), np.float32); K = np.zeros((n_kf, 4), np.float32)
    kf_start = [0]; keys, desc, has_mp, node = [], [], [], []
    for k in range(n_kf):
        c = np.array([0.0, 0.0, 0.0]) if k == 0 else np.array([0.3 * np.cos(k), 0.1 * np.sin(2 * k), 0.05 * k]) + rng.normal(0, 0.03, 3)
        R = rot(rng.normal(0, 0.04, 3))
        T = np.eye(4); T[:3, :3] = R; T[:3, 3] = -R @ c
        Tcw[k] = T.reshape(-1); Ow[k] = c
        K[k] = np.array(synth.TUM1_K, np.float32) + (0 if k == 0 else rng.normal(0, 3, 4).astype(np.float32))
        Xc = X @ R.T + T[:3, 3]
        uv = np.stack([K[k, 0] * Xc[:, 0] / Xc[:, 2] + K[k, 2], K[k, 1] * Xc[:, 1] / Xc[:, 2] + K[k, 3]], 1)
        octv = rng.integers(0, nlevels, n_pts)
        uv = uv + rng.normal(0, 0.6, uv.shape) * sf[octv][:, None]
        ok = (uv[:, 0] > 20) & (uv[:, 0] < w - 20) & (uv[:, 1] > 20) & (uv[:, 1] < h - 20) & (rng.random(n_pts) < 0.85)
        ids = rng.permutation(np.nonzero(ok)[0])
        n = len(ids) + n_clutter
        kp = np.zeros(n, KP_DTYPE)
        kp["x"][:len(ids)], kp["y"][:len(ids)], kp["octave"][:len(ids)] = uv[ids, 0], uv[ids, 1], octv[ids]
        kp["x"][len(ids):], kp["y"][len(ids):] = rng.uniform(20, w - 20, n_clutter), rng.uniform(20, h - 20, n_clutter)
        kp["octave"][len(ids):] = rng.integers(0, nlevels, n_clutter)
        kp["angle"] = rng.uniform(0, 360, n); kp["size"] = 31 * sf[kp["octave"]]; kp["class_id"] = -1
        d = np.concatenate([code[ids], rng.integers(0, 256, (n_clutter, 32), dtype=np.uint8)])
        for _ in range(10):                            # a few flipped bits per view
            r = np.nonzero(rng.random(len(ids)) < 0.7)[0]; b = rng.integers(0, 256, len(r))
            d[r, b // 8] ^= (1 << (b % 8)).astype(np.uint8)
        keys.append(kp); desc.append(d)
        has_mp.append((rng.random(n) < 0.2).astype(np.uint8))
        node.append(np.concatenate([node_of[ids], rng.integers(100, 140, n_clutter)]).astype(np.uint32))
        kf_start.append(kf_start[-1] + n)
    # LocalMapping::ComputeF12(current, neighbour): K1^-T [t12]x R12 K2^-1
    Km = lambda k: np.array([[K[k, 0], 0, K[k, 2]], [0, K[k, 1], K[k, 3]], [0, 0, 1]], np.float64)
    T = Tcw.reshape(-1, 4, 4).astype(np.float64)
    F12 = np.zeros((n_neigh, 9), np.float32)
    for j in range(1, n_kf):
        R12 = T[0, :3, :3] @ T[j, :3, :3].T; t12 = -R12 @ T[j, :3, 3] + T[0, :3, 3]
        tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]])
        F12[j - 1] = (np.linalg.inv(Km(0)).T @ tx @ R12 @ np.linalg.inv(Km(j))).reshape(-1)
    return dict(kf_start=np.array(kf_start, np.int32), keys=np.concatenate(keys), desc=np.concatenate(desc),
                has_mp=np.concatenate(has_mp), node=np.concatenate(node), Tcw=Tcw, Ow=Ow, K=K, F12=F12, scale_factors=sf,
                level_sigma2=(sf * sf).astype(np.float32))


if __name__ == "__main__":
    s = scene()
    ref = lambda j, has: oracle.search_for_triangulation(*tp.search_args(s, j, has[0], has[j]), False, impl="ref")[1]
    lists = tp.create_new_map_points(s, ref)
    s["ref_pairs"] = np.concatenate(lists).astype(np.int32).reshape(-1, 2)
    s["ref_start"] = np.cumsum([0] + [len(x) for x in lists]).astype(np.int32)
    # the snapshot without the drop rule must differ from the reference somewhere, or the fixture tests nothing
    has0 = [tp.keyframe(s, k)["has_mp"] for k in range(len(s["kf_start"]) - 1)]
    snap = [oracle.search_for_triangulation(*tp.search_args(s, j, has0[0], has0[j]), False, impl="ref")[1] for j in range(1, len(has0))]
    assert tp.same_lists(tp.snapshot_protocol(s, snap), lists) and not tp.same_lists(tp.snapshot_protocol(s, snap, drop=False), lists)
    np.savez_compressed(OUT, **s)
    print(f"{OUT}: {len(s['keys'])} keypoints in {len(s['kf_start']) - 1} keyframes; pairs per neighbour {[len(x) for x in lists]}")
