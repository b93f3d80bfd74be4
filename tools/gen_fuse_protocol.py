"""Generate tests/golden/refcalls/fuse_protocol.npz: the first loop of LocalMapping::SearchInNeighbors run by the reference's own
ORBmatcher::Fuse and MapPoint surgery (tools/fuse_protocol_ref.cpp), on a seeded scene.

The scene: a current keyframe whose point list is fused into five targets in order, three more keyframes that only hold
observations, and map points that already observe targets (skipped there), near-duplicate points that observe a target at the
keypoint their twin matches (Replace between two points of the list), and points outside the list that own target keypoints and
observe several targets (the survivor of their Replace becomes skipped at a later target).  Point 0 is built so that the descriptor
it receives from its first Replace picks a different keypoint at a later target than its original descriptor does.
The fixture holds the scene and the reference's final state: every keyframe slot, the bad points, the final descriptors and
Fuse's return values.  tests/test_fuse_batch.py (through tests/fuse_protocol.py) replays it on the oracle with the snapshot
protocol of INTEGRATION.md, and tests/test_fuse_batch_gpu.py through the device call.

Needs the reference tree (REF, default: oracle/Makefile's) and the CPU oracle built (make -C oracle).
Run from the repo root:  python tools/gen_fuse_protocol.py
"""
import ctypes as C
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from plslam_b200 import synth  # noqa: E402
from plslam_b200.binding import KP_DTYPE  # noqa: E402

ORACLE = os.path.join(ROOT, "oracle")
OUT = os.path.join(ROOT, "tests", "golden", "refcalls", "fuse_protocol.npz")


def reference_dir():
    if os.environ.get("REF"):
        return os.environ["REF"]
    return re.search(r"^REF \?= (\S+)", open(os.path.join(ORACLE, "Makefile")).read(), re.M).group(1)


def build_driver(tmp):
    ref = reference_dir()
    dbow, ld = f"{ref}/Thirdparty/DBoW2/DBoW2", f"{ref}/Thirdparty/line_descriptor"
    so = os.path.join(tmp, "libfuse_protocol.so")
    subprocess.check_call(
        ["g++", "-O2", "-std=gnu++14", "-fPIC", "-ffp-contract=off", "-w", "-shared", "-Wl,-Bsymbolic",
         "-Ishim_slam", "-I-", "-Ishim", f"-I{ref}", f"-I{ref}/include", f"-I{dbow}", f"-I{ld}/include", f"-I{ORACLE}", "-o", so,
         f"{ref}/src/ORBmatcher.cc", f"{ref}/src/MapPoint.cc", f"{ref}/src/LSDmatcher.cpp", f"{ref}/src/lineIterator.cpp",
         f"{dbow}/BowVector.cpp", f"{dbow}/FeatureVector.cpp", os.path.join(ROOT, "tools", "fuse_protocol_ref.cpp"), "ref_cv_impl.cpp",
         "-L.", "-loracle", "-lpthread", f"-Wl,-rpath,{ORACLE}"], cwd=ORACLE)
    return C.CDLL(so)


def flip(d, bits):
    d = d.copy()
    for b in bits:
        d[b >> 3] ^= np.uint8(1 << (b & 7))
    return d


def rot(a):
    cx, sx, cy, sy, cz, sz = np.cos(a[0]), np.sin(a[0]), np.cos(a[1]), np.sin(a[1]), np.cos(a[2]), np.sin(a[2])
    return (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
            @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))


def scene(seed=3, n_list=90, n_targets=5, n_extra=3, nlevels=8, scale=1.2):
    rng = np.random.default_rng(seed)
    K = np.array(synth.TUM1_K, np.float32)
    bounds = np.array([0, 0, 640, 480], np.float32)
    sf = (scale ** np.arange(nlevels)).astype(np.float32)
    n_kf = 1 + n_targets + n_extra                   # 0 = current keyframe, 1 .. n_targets = targets, then the extras
    Tcw = np.zeros((n_kf, 16), np.float32); Ow = np.zeros((n_kf, 3), np.float32)
    for k in range(n_kf):
        R = rot(rng.uniform(-0.04, 0.04, 3)); c = rng.uniform(-0.25, 0.25, 3)
        T = np.eye(4); T[:3, :3] = R; T[:3, 3] = -R @ c
        Tcw[k] = T.reshape(-1); Ow[k] = c
    # the list's points, then near-duplicates of some of them, then the points the targets own
    n_dup = 12
    z = rng.uniform(3, 6, n_list)
    pos = np.stack([rng.uniform(-0.3, 0.3, n_list) * z, rng.uniform(-0.25, 0.25, n_list) * z, z], 1)
    dup_of = rng.choice(np.arange(1, n_list), n_dup, replace=False)
    pos = np.concatenate([pos, pos[dup_of] + rng.normal(0, 0.002, (n_dup, 3))])
    base_desc = rng.integers(0, 256, (n_list, 32), dtype=np.uint8)
    desc0 = np.concatenate([base_desc, np.array([flip(base_desc[i], rng.integers(0, 256, 4)) for i in dup_of])])
    centre = Ow[:n_targets + 1].mean(0)
    rows = {k: [] for k in range(n_kf)}              # keyframe -> [(x, y, octave, desc)]
    obs = []                                          # (point, keyframe, slot)

    def slot(k, x, y, octv, d):
        rows[k].append((x, y, octv, d))
        return len(rows[k]) - 1

    def project(k, P):
        T = Tcw[k].reshape(4, 4).astype(np.float64)
        Pc = T[:3, :3] @ P + T[:3, 3]
        return K[0] * Pc[0] / Pc[2] + K[2], K[1] * Pc[1] / Pc[2] + K[3]

    def level(k, m, max_dist):
        d = np.linalg.norm(pos[m] - Ow[k])
        return int(np.clip(np.ceil(np.log(max_dist[m] / d) / np.log(scale)), 0, nlevels - 1))

    n_lm = n_list + n_dup
    dist = np.linalg.norm(pos - centre, axis=1)
    max_dist = (dist * scale ** rng.uniform(0.3, 2.4, n_lm)).astype(np.float32)
    min_dist = (max_dist / scale ** (nlevels - 1)).astype(np.float32)
    normal = ((pos - centre) / dist[::, None]).astype(np.float32)
    # every list point is observed by the current keyframe; its first descriptor is that keyframe's row
    for m in range(n_lm):
        u, v = project(0, pos[m])
        obs.append((m, 0, slot(0, u, v, 0, desc0[m])))
    extra = list(range(1 + n_targets, n_kf))
    foreign = []                                      # (position, descriptor, [(keyframe, slot)]) of points outside the list
    targets = list(range(1, 1 + n_targets))
    for t in targets:
        owner = {}
        for m in range(1, n_lm):
            if m >= n_list and t != 1 + (m % n_targets):
                continue                              # a duplicate appears in one target only, at its twin's keypoint
            if rng.random() > 0.8:
                continue
            u, v = project(t, pos[m])
            lvl = level(t, m, max_dist)
            octv = max(lvl - int(rng.integers(0, 2)), 0)
            s = slot(t, u + rng.normal(0, 0.5) * sf[octv], v + rng.normal(0, 0.5) * sf[octv], octv,
                     flip(desc0[m], rng.integers(0, 256, int(rng.integers(0, 45)))))
            if m >= n_list:                          # the duplicate owns the keypoint its twin will match
                obs.append((m, t, s))
                continue
            r = rng.random()
            if r < 0.15:                              # already observed: skipped at this target
                obs.append((m, t, s))
            elif r < 0.35:                            # owned by a point outside the list, seen by other keyframes too
                owner[m] = s
        for m, s in owner.items():
            more = [(k, slot(k, 0.0, 0.0, 0, flip(desc0[m], rng.integers(0, 256, 10)))) for k in rng.choice(extra, int(rng.integers(0, 3)), replace=False)]
            foreign.append((pos[m], flip(desc0[m], rng.integers(0, 256, 6)), [(t, s)] + more))
        for _ in range(15):                           # clutter
            slot(t, rng.uniform(0, 640), rng.uniform(0, 480), int(rng.integers(0, nlevels)), rng.integers(0, 256, 32, dtype=np.uint8))
    # point 0: its first Replace (at target 1) gives it the descriptor D1; at target 2, D0 picks keypoint A and D1 picks B
    perm = rng.permutation(256)
    D0 = desc0[0]; D1 = flip(D0, perm[:30])
    u, v = project(1, pos[0]); l1 = level(1, 0, max_dist)
    a = slot(1, u + 0.3, v - 0.2, l1, D1)
    e0 = slot(extra[0], 0.0, 0.0, 0, rng.integers(0, 256, 32, dtype=np.uint8))
    obs.append((0, extra[0], e0))
    foreign.append((pos[0], D1, [(1, a), (extra[1], slot(extra[1], 0.0, 0.0, 0, D1))]))
    u, v = project(2, pos[0]); l2 = level(2, 0, max_dist)
    slot(2, u + 0.2, v + 0.1, l2, flip(D0, perm[30:33]))
    slot(2, u - 0.2, v - 0.1, l2, flip(D1, perm[33:36]))
    # the foreign points: observations as listed, then the same geometry as the list point they shadow
    for P, d, where in foreign:
        m = len(pos)
        pos = np.concatenate([pos, P[None]]); desc0 = np.concatenate([desc0, d[None]])
        dd = np.linalg.norm(P - centre)
        normal = np.concatenate([normal, ((P - centre) / dd)[None].astype(np.float32)])
        max_dist = np.concatenate([max_dist, np.float32([dd * scale ** rng.uniform(0.3, 2.4)])])
        min_dist = np.concatenate([min_dist, np.float32([max_dist[-1] / scale ** (nlevels - 1)])])
        for k, s in where:
            obs.append((m, k, s))
    kf_start = np.zeros(n_kf + 1, np.int32)
    kf_start[1:] = np.cumsum([len(rows[k]) for k in range(n_kf)])
    keys = np.zeros(kf_start[-1], KP_DTYPE); desc = np.zeros((kf_start[-1], 32), np.uint8)
    for k in range(n_kf):
        for j, (x, y, o, d) in enumerate(rows[k]):
            i = kf_start[k] + j
            keys[i]["x"], keys[i]["y"], keys[i]["octave"], keys[i]["size"], keys[i]["class_id"] = x, y, o, 31 * sf[o], -1
            desc[i] = d
    obs = np.array(obs, np.int32)
    return dict(kf_start=kf_start, keys=keys, desc=desc, Tcw=Tcw, Ow=Ow, K=np.tile(K, (n_kf, 1)), bounds=np.tile(bounds, (n_kf, 1)),
                scale_factors=sf, inv_level_sigma2=(1.0 / (sf * sf)).astype(np.float32),
                log_scale_factor=np.float32(np.log(np.float32(scale))), pos=pos.astype(np.float32), normal=normal.astype(np.float32),
                min_dist=min_dist.astype(np.float32), max_dist=max_dist.astype(np.float32), mp_desc=desc0,
                obs_mp=obs[:, 0].copy(), obs_kf=obs[:, 1].copy(), obs_idx=obs[:, 2].copy(),
                list=np.arange(n_lm, dtype=np.int32), targets=np.array(targets, np.int32), th=np.float32(3.0))


def run_reference(L, s):
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    n_kf = len(s["Tcw"]); n_mp = len(s["pos"]); n_slots = int(s["kf_start"][-1])
    slots = np.zeros(n_slots, np.int32); bad = np.zeros(n_mp, np.uint8); out_desc = np.zeros((n_mp, 32), np.uint8)
    nfused = np.zeros(len(s["targets"]), np.int32)
    L.ref_fuse_protocol(n_kf, p(s["kf_start"]), p(s["keys"]), p(s["desc"]), p(s["Tcw"]), p(s["Ow"]), p(s["K"]), p(s["bounds"]),
                        p(s["scale_factors"]), p(s["inv_level_sigma2"]), C.c_float(s["log_scale_factor"]), len(s["scale_factors"]),
                        n_mp, p(s["pos"]), p(s["normal"]), p(s["min_dist"]), p(s["max_dist"]), p(s["mp_desc"]), len(s["obs_mp"]),
                        p(s["obs_mp"]), p(s["obs_kf"]), p(s["obs_idx"]), len(s["list"]), p(s["list"]), len(s["targets"]), p(s["targets"]),
                        C.c_float(s["th"]), p(slots), p(bad), p(out_desc), p(nfused))
    return dict(ref_slots=slots, ref_bad=bad, ref_desc=out_desc, ref_nfused=nfused)


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as tmp:
        L = build_driver(tmp)
        s = scene()
        r = run_reference(L, s)
    np.savez_compressed(OUT, **s, **r)
    print(f"{OUT}: {len(s['pos'])} points, {len(s['Tcw'])} keyframes, nFused per target {r['ref_nfused'].tolist()}, "
          f"{int(r['ref_bad'].sum())} bad points")
