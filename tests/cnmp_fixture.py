"""The scene of tests/golden/refcalls/create_new_map_points.npz (tools/gen_create_new_map_points.py) as the batched calls take it:
keyframe dicts for TriangulationProblems / pack_tri_keyframes, one (current keyframe, neighbour, F12) problem per neighbour the
reference searched, in its order, and the reference's new points."""
import os

import numpy as np

import triangulation_protocol as tp

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refcalls", "create_new_map_points.npz")


def load():
    with np.load(FIXTURE) as z:
        return {k: z[k] for k in z.files}


def keyframes(s):
    return [tp.keyframe(s, k) for k in range(len(s["kf_start"]) - 1)]


def problems(s):
    """(0, j, F12) for every neighbour j the reference searched, in its order"""
    return [(0, j, s["F12"][j - 1].reshape(3, 3)) for j in range(1, len(s["kf_start"]) - 1) if s["searched"][j - 1]]


def new_points(code, x3D, problem_list, out_offset, n1):
    """The committed slots applied in problem order, then ascending idx1: (neighbour, idx1) [m][2] and x3D bits [m][3].  idx2 comes
    from matches12 at the caller."""
    rows, X = [], []
    for p, (_, j, _) in enumerate(problem_list):
        a = out_offset[p]
        i = np.nonzero(code[a:a + n1] == 0)[0]
        rows += [(j, int(x)) for x in i]
        X.append(x3D[a + i])
    return np.array(rows, np.int32).reshape(-1, 2), np.concatenate(X).view(np.uint32) if X else np.zeros((0, 3), np.uint32)


def reference(s):
    return s["ref_new"], s["ref_x3D"].view(np.uint32)


def knife_edge(s):
    """The fixture's searches with the current keyframe copied once per searched neighbour (problem p searches copy p against
    neighbour p), every copy's keypoint on its own octave after the fixture's, and that octave's level_sigma2 the largest fp32
    value whose 5.991 * sigma^2 (fp64) lies below the pair's fp32 squared reprojection error in KF1: the reprojection gate of KF1
    then rejects every pair that reaches it by less than one rounding of that error, so an error off by one ulp passes it.
    Returns keyframes, problems, scale_factors, level_sigma2 for TriangulationProblems, and the oracle's codes on them."""
    import cnmp_oracle as co
    from plslam_b200 import binding as bd
    kfs, probs = keyframes(s), problems(s)
    nl, n1 = len(s["scale_factors"]), len(kfs[0]["keys"])
    copies = []
    for p in range(len(probs)):
        c = dict(kfs[0], keys=kfs[0]["keys"].copy())
        c["keys"]["octave"] = nl + p * n1 + np.arange(n1)
        copies.append(c)
    table = copies + kfs[1:]
    P = len(probs)
    kprobs = [(p, P + j - 1, F) for p, (_, j, F) in enumerate(probs)]
    sf = np.concatenate([s["scale_factors"], np.ones(P * n1, np.float32)])
    s2 = np.concatenate([s["level_sigma2"], np.full(P * n1, 1e30, np.float32)])
    k = bd.pack_tri_keyframes(table)
    q = bd.pack_tri_problems(kprobs, k["n"])
    m12 = np.full(q["n_out"], -1, np.int32)
    import oracle
    for p, (_, j, _) in enumerate(probs):
        _, m = oracle.search_for_triangulation(*tp.search_args(s, j, kfs[0]["has_mp"], kfs[j]["has_mp"]), False)
        m12[q["out_offset"][p]:q["out_offset"][p] + n1] = m
    probe = {}
    co.triangulate(k, q, m12, np.zeros(P, np.int32), s["scale_factor"], sf, s2, e2_out=probe)
    E = probe["e2"][0]
    oct1 = np.concatenate([table[p]["keys"]["octave"] for p in range(P)])[probe["slot"]]
    with np.errstate(over="ignore", invalid="ignore"):
        sig = (E.astype(np.float64) / 5.991).astype(np.float32)
        for _ in range(4):                          # the largest fp32 sigma^2 with 5.991 * sigma^2 < E
            up = np.nextafter(sig, np.float32(np.inf))
            sig = np.where(5.991 * up.astype(np.float64) < E, up, sig)
            sig = np.where(5.991 * sig.astype(np.float64) < E, sig, np.nextafter(sig, np.float32(0)))
    ok = np.isfinite(E) & (E > 0)
    s2[oct1[ok]] = sig[ok]
    code, *_ = co.triangulate(k, q, m12, np.zeros(P, np.int32), s["scale_factor"], sf, s2)
    return table, kprobs, sf, s2, code
