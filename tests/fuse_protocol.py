"""The snapshot protocol of INTEGRATION.md (LocalMapping::SearchInNeighbors, first loop) on the scene of
tests/golden/refcalls/fuse_protocol.npz: every (target, point) pair is searched against the state before the loop, the results are
applied target by target in the reference's order, the skip test is checked again when a result is applied, and a pair whose
point's descriptor changed since the search is searched again.  The map surgery is ORBmatcher::Fuse's (src/ORBmatcher.cc:1036-1061)
with MapPoint::Replace / AddObservation / ComputeDistinctiveDescriptors (src/MapPoint.cc), restated on plain arrays."""
import os

import numpy as np

import oracle

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refcalls", "fuse_protocol.npz")
TH_LOW = 50


def load():
    with np.load(FIXTURE) as z:
        return {k: z[k] for k in z.files}


def keyframe(s, k):
    a, b = s["kf_start"][k], s["kf_start"][k + 1]
    return dict(keys=s["keys"][a:b], desc=s["desc"][a:b], Tcw=s["Tcw"][k], Ow=s["Ow"][k], K=s["K"][k], bounds=s["bounds"][k])


class MapState:
    """Keyframe slots, observations (keyframe -> slot; keyframes in index order, the address order of the reference's std::map),
    observation counts, bad flags and descriptors of the scene's map points."""

    def __init__(self, s):
        self.kf_desc = [keyframe(s, k)["desc"] for k in range(len(s["Tcw"]))]
        self.slots = [np.full(len(d), -1, np.int32) for d in self.kf_desc]
        n = len(s["pos"])
        self.obs = [dict() for _ in range(n)]
        self.nobs = np.zeros(n, np.int32)
        self.bad = np.zeros(n, bool)
        self.desc = s["mp_desc"].copy()
        for m, k, i in zip(s["obs_mp"], s["obs_kf"], s["obs_idx"]):
            self.add_observation(m, k, i)
            self.slots[k][i] = m

    def skip(self, t, m):
        return bool(self.bad[m]) or t in self.obs[m]

    def add_observation(self, m, k, i):          # monocular: one observation each
        if k in self.obs[m]:
            return
        self.obs[m][k] = int(i)
        self.nobs[m] += 1

    def distinctive(self, m):
        if self.bad[m] or not self.obs[m]:
            return
        rows = np.array([self.kf_desc[k][self.obs[m][k]] for k in sorted(self.obs[m])])
        self.desc[m] = rows[oracle.distinctive_descriptors(rows, np.array([0, len(rows)], np.int32))[0]]

    def replace(self, a, b):                     # a->Replace(b)
        if a == b:
            return
        obs, self.obs[a] = self.obs[a], {}
        self.bad[a] = True
        for k in sorted(obs):
            if k not in self.obs[b]:
                self.slots[k][obs[k]] = b
                self.add_observation(b, k, obs[k])
            else:
                self.slots[k][obs[k]] = -1
        self.distinctive(b)

    def fuse(self, t, m, bi, bd):
        """ORBmatcher::Fuse's action for map point m at target t given its search result; True if it counts in nFused."""
        if bd > TH_LOW:
            return False
        q = self.slots[t][bi]
        if q >= 0:
            if not self.bad[q]:
                if self.nobs[q] > self.nobs[m]:
                    self.replace(m, q)
                else:
                    self.replace(q, m)
        else:
            self.add_observation(m, t, bi)
            self.slots[t][bi] = m
        return True


def oracle_search(s):
    """search(problems, desc) on the CPU oracle: problems = [(target, landmark rows, skip)] -> [(best_idx, best_dist)]."""
    def search(problems, desc):
        out = []
        for t, lm, skip in problems:
            k = keyframe(s, t)
            out.append(oracle.fuse_search(k["keys"], k["desc"], k["bounds"], k["Tcw"], k["Ow"], k["K"], s["scale_factors"],
                                          s["inv_level_sigma2"], float(s["log_scale_factor"]), np.asarray(skip, np.uint8),
                                          s["pos"][lm], s["normal"][lm], s["min_dist"][lm], s["max_dist"][lm], desc[lm], float(s["th"])))
        return out
    return search


def first_loop(s, search, snapshot=True, research=True):
    """The first loop of SearchInNeighbors on the fixture's scene.  snapshot=False: each point is searched when the reference
    reaches it (the reference's own order of reads).  snapshot=True: one search of every pair before the loop, then application
    with the skip re-check and, if research, the re-search of the pairs whose point's descriptor changed.
    Returns (MapState, nFused per target)."""
    M = MapState(s)
    lst, targets = s["list"], [int(t) for t in s["targets"]]
    if snapshot:
        snap = M.desc.copy()
        first = search([(t, lst, [M.skip(t, m) for m in lst]) for t in targets], snap)
    nfused = []
    for ti, t in enumerate(targets):
        nf = 0
        for j, m in enumerate(lst):
            if m < 0 or M.skip(t, m):
                continue
            if snapshot and not (research and (M.desc[m] != snap[m]).any()):
                bi, bd = first[ti][0][j], first[ti][1][j]
            else:
                (bi_, bd_), = search([(t, np.array([m]), [0])], M.desc)
                bi, bd = bi_[0], bd_[0]
            nf += M.fuse(t, m, int(bi), int(bd))
        nfused.append(nf)
    return M, np.array(nfused, np.int32)


def final_slots(M):
    return np.concatenate(M.slots)


def line_results_at_application(bi, bd, stop, live_skip, search_rest):
    """The line half of the protocol at one target.  LSDmatcher::Fuse tests the skip before it stops at a line behind the camera
    (src/LSDmatcher.cpp:886-907), and surgery at an earlier target can turn the skip of the snapshot's stop entry to true; then the
    reference steps over that entry and goes on.  Given the snapshot's (best_idx, best_dist, stop_at) of one problem and the skip
    bytes at application time, return the results and the stop the reference acts on: while the stop entry is skipped now, the
    entries after it are searched again on the current state, search_rest(j0) -> (best_idx, best_dist, stop_at) of entries j0..,
    which also reports the next stop."""
    bi, bd, n = np.array(bi), np.array(bd), len(bi)
    while stop < n and live_skip[stop]:
        j0 = stop + 1
        rbi, rbd, rstop = search_rest(j0)
        bi[j0:], bd[j0:] = rbi, rbd
        stop = j0 + rstop
    return bi, bd, stop
