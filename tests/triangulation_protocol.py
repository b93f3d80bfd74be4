"""The snapshot protocol of INTEGRATION.md for LocalMapping::CreateNewMapPoints on the scene of
tests/golden/refcalls/triangulation_protocol.npz: every neighbour is searched against the state before the loop, the neighbours are
applied in the reference's order, and a pair is dropped at application when its KF1 keypoint received a map point at an earlier
neighbour.  The triangulation itself is a deterministic stand-in: a pair with an even idx1 + idx2 gets a new map point on both
keyframes (AddMapPoint, LocalMapping.cc:582-583); the others fail its geometric tests."""
import os

import numpy as np

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refcalls", "triangulation_protocol.npz")


def load():
    with np.load(FIXTURE) as z:
        return {k: z[k] for k in z.files}


def keyframe(s, k):
    """Keyframe k of the scene (0 = the current keyframe, 1 .. = its neighbours in the reference's order).  Each keypoint lies in
    one vocabulary node; a node's items are in ascending keypoint order, as DBoW2 inserts them."""
    a, b = s["kf_start"][k], s["kf_start"][k + 1]
    node = s["node"][a:b]
    fv = {int(n): [int(i) for i in np.nonzero(node == n)[0]] for n in np.unique(node)}
    return dict(keys=s["keys"][a:b], desc=s["desc"][a:b], has_mp=s["has_mp"][a:b].copy(), fv=fv, Tcw=s["Tcw"][k], Ow=s["Ow"][k],
                K=s["K"][k])


def search_args(s, j, has_mp1, has_mp2):
    """The arguments of SearchForTriangulation(current keyframe, neighbour j) for ORBmatcher.SearchForTriangulation and the
    oracle, with the map-point flags given."""
    a, b = keyframe(s, 0), keyframe(s, j)
    T = b["Tcw"].reshape(4, 4)
    return (a["keys"], a["desc"], has_mp1, b["keys"], b["desc"], has_mp2, a["fv"], b["fv"], s["F12"][j - 1], a["Ow"],
            np.ascontiguousarray(T[:3, :3]), np.ascontiguousarray(T[:3, 3]), b["K"], s["scale_factors"], s["level_sigma2"])


def pairs_of(matches):
    """vMatchedIndices: (idx1, idx2) in ascending idx1."""
    i = np.nonzero(np.asarray(matches) >= 0)[0]
    return np.stack([i, np.asarray(matches)[i]], 1).astype(np.int32).reshape(-1, 2)


def create_new_map_points(s, matches_at, drop=False):
    """The neighbour loop of CreateNewMapPoints on the scene.  matches_at(j, has_mp) -> matches12 of the current keyframe against
    neighbour j; drop: leave out the pairs whose idx1 holds a map point now.  Returns each neighbour's pairs [m][2]."""
    has = [keyframe(s, k)["has_mp"] for k in range(len(s["kf_start"]) - 1)]
    lists = []
    for j in range(1, len(has)):
        pairs = pairs_of(matches_at(j, has))
        if drop:
            pairs = pairs[has[0][pairs[:, 0]] == 0]
        lists.append(pairs)
        new = pairs[(pairs[:, 0] + pairs[:, 1]) % 2 == 0]
        has[0][new[:, 0]] = 1
        has[j][new[:, 1]] = 1
    return lists


def snapshot_protocol(s, snapshot, drop=True):
    """The protocol on the snapshot searches (matches12 per neighbour, all against the state before the loop)."""
    return create_new_map_points(s, lambda j, has: snapshot[j - 1], drop)


def reference_lists(s):
    st = s["ref_start"]
    return [s["ref_pairs"][st[j]:st[j + 1]] for j in range(len(st) - 1)]


def same_lists(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))
