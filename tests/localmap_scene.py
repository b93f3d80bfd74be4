"""Test helpers for Tracking::UpdateLocalMap (Tracking.cc:1899-2081): keyframe graphs, the reference restated literally, and the
named cases the tests run.

A graph is a dict of per-keyframe lists, keyframes numbered in ascending KeyFrame* address (map<KeyFrame*,int> / set<KeyFrame*>
order): Tcw / Twc [K][4][4], bad [K], parent [K] (-1 none), pt [K] / ln [K] (GetMapPointMatches / GetMapLineMatches in feature
order, map index or -1), cov [K] (mvpOrderedConnectedKeyFrames), children [K] (mspChildrens), n_points, n_lines.  The observations
of a map point (GetObservations) are the keyframes whose slots hold it.

scene_graph() builds one on the planar scene of tests/track_scene.py by the reference's own rules: covisibility weights are the
shared observations, kept at >= 15 or only the strongest if none reaches 15 (KeyFrame.cc:365-389), ordered by (weight, index)
descending (UpdateConnections sorts the pairs and push_fronts them); the parent is the front of that list at a keyframe's first
connection, taken among the keyframes created before it (:408-413).  Creation order and address order differ on purpose.
"""
import numpy as np

import motion_scene as ms
import track_scene as ts

LIMIT = 80      # if(mvpLocalKeyFrames.size()>80) break


def observations(g, which="pt"):
    """map index -> sorted keyframes whose slots hold it."""
    n = g["n_points"] if which == "pt" else g["n_lines"]
    obs = [set() for _ in range(n)]
    for k, slots in enumerate(g[which]):
        for m in slots:
            if m >= 0:
                obs[m].add(k)
    return [sorted(o) for o in obs]


def update_local_map_ref(g, point_map, kf_prev, ref_prev, line_map=None, variant="reference"):
    """Tracking::UpdateLocalMap for one frame, statement by statement.  point_map: the frame's mvpMapPoints (map index or -1);
    kf_prev / ref_prev: mvpLocalKeyFrames and mpReferenceKF before the call.  variant="lines_vote" also counts the observations of
    line_map's lines (what the reference does not do).  Returns dict(kf, ref_kf, points, lines)."""
    obs = observations(g)
    # UpdateLocalKeyFrames (:1973-2081)
    counter = {}
    for m in point_map:
        if m >= 0:
            for k in obs[m]:
                counter[k] = counter.get(k, 0) + 1
    if variant == "lines_vote" and line_map is not None:
        lobs = observations(g, "ln")
        for m in line_map:
            if m >= 0:
                for k in lobs[m]:
                    counter[k] = counter.get(k, 0) + 1
    local, ref = list(kf_prev), ref_prev
    if counter:                                                   # if(keyframeCounter.empty()) return;
        mx, kmax = 0, None
        local, stamped = [], set()
        for k in sorted(counter):                                 # map<KeyFrame*,int> order
            if g["bad"][k]:
                continue
            if counter[k] > mx:
                mx, kmax = counter[k], k
            local.append(k)
            stamped.add(k)
        end = len(local)                                          # itEndKF is fixed before the push_backs
        for i in range(end):
            if len(local) > LIMIT:
                break
            k = local[i]
            for c in g["cov"][k][:10]:                            # GetBestCovisibilityKeyFrames(10)
                if not g["bad"][c]:
                    if c not in stamped:
                        local.append(c); stamped.add(c)
                        break
            for c in sorted(g["children"][k]):
                if not g["bad"][c]:
                    if c not in stamped:
                        local.append(c); stamped.add(c)
                        break
            p = g["parent"][k]
            if p >= 0:
                if p not in stamped:                              # not checked for isBad
                    local.append(p); stamped.add(p)
                    break                                         # leaves the outer loop
        if kmax is not None:
            ref = kmax
    # UpdateLocalPoints / UpdateLocalLines (:1916-1971): mnTrackReferenceForFrame keeps the first occurrence
    out = {}
    for which in ("pt", "ln"):
        seen, lst = set(), []
        for k in local:
            for m in g[which][k]:
                if m >= 0 and m not in seen:
                    lst.append(m); seen.add(m)
        out[which] = lst
    return dict(kf=local, ref_kf=ref, points=out["pt"], lines=out["ln"])


def to_desc(g):
    """The graph as the CSR dict of Map.set_keyframes."""
    def csr(rows):
        off = np.zeros(len(rows) + 1, np.int32)
        off[1:] = np.cumsum([len(r) for r in rows])
        return off, np.asarray([x for r in rows for x in r], np.int32)
    d = dict(Tcw=np.asarray(g["Tcw"], np.float32), Twc=np.asarray(g["Twc"], np.float32), bad=np.asarray(g["bad"], np.uint8),
             parent=np.asarray(g["parent"], np.int32))
    for k, rows in (("pt_slot", g["pt"]), ("ln_slot", g["ln"]), ("cov", g["cov"]), ("child", [sorted(c) for c in g["children"]]),
                    ("obs", observations(g))):
        d[k + "_offset"], d[k] = csr(rows)
    return d


def inverse(T):
    """Twc = [Rcw^T | Ow] in fp32 (KeyFrame::SetPose), Ow summed as Frame::UpdatePoseMatrices does."""
    T = np.asarray(T, np.float32).reshape(4, 4)
    W = np.eye(4, dtype=np.float32)
    W[:3, :3] = T[:3, :3].T; W[:3, 3] = ts.camera_center(T)
    return W


# ---------------------------------------------------------------------------------------------------- the named cases
class _Builder:
    def __init__(self):
        self.g = dict(Tcw=[], Twc=[], bad=[], parent=[], pt=[], ln=[], cov=[], children=[], n_points=0, n_lines=0)
        self.rng = np.random.default_rng(11)

    def kf(self, pt=(), ln=(), bad=False):
        g = self.g
        T = ts.pose(self.rng.uniform(-0.05, 0.05, 3), self.rng.uniform(-0.2, 0.2, 3))
        g["Tcw"].append(T); g["Twc"].append(inverse(T)); g["bad"].append(int(bad)); g["parent"].append(-1)
        g["pt"].append(list(pt)); g["ln"].append(list(ln)); g["cov"].append([]); g["children"].append(set())
        return len(g["bad"]) - 1

    def pts(self, n):
        p = list(range(self.g["n_points"], self.g["n_points"] + n))
        self.g["n_points"] += n
        return p

    def lns(self, n):
        p = list(range(self.g["n_lines"], self.g["n_lines"] + n))
        self.g["n_lines"] += n
        return p

    def parent(self, child, parent):
        self.g["parent"][child] = parent
        self.g["children"][parent].add(child)


def quirk_cases():
    """One graph holding every named case in its own keyframes and map entries.  Returns (graph, cases): name -> dict(point_map,
    line_map, kf_prev, ref_prev) and the keyframes the tests name.
      voter_order:  votes 1, 3, 2 on keyframes a < b < c: the list is index order, not vote order
      first_max:    votes 2, 3, 3 on d < e < f and 5 on the bad g: ref = e
      only_voters:  voter h, its covisible i, i's covisible j: j is not reached
      parent_break: voters k1 < k2, k1's parent q, k2's covisible r: adding q ends the expansion
      bad_skips:    voter v with covisibles (bad cb, cg), children (bad hb < hg) and the bad parent pb
      limit_80:     80 voters; w0's covisible x0 and child x1 are added, then size 82 > 80 stops the loop before w1's x2
      stale:        no matches: the previous list and reference keyframe stay, the points come from that list
      dedup:        y's slots P1 P2 P1 P3, z's P3 P4 P2 -1 (lines L1 L2 L1 / L2 L3): first occurrences P1 P2 P3 P4
      lines_no_vote: t holds the matched point, u only the matched line: u is not a voter
      bad_voters:   only a bad keyframe gets votes: the list is empty and the reference keyframe stays"""
    B = _Builder()
    c = {}
    P = B.pts(6)
    a, b_, cc = B.kf(P[:1]), B.kf(P[1:4]), B.kf(P[4:])
    c["voter_order"] = dict(point_map=P, kfs=dict(a=a, b=b_, c=cc))
    P = B.pts(13)
    d, e, f, g = B.kf(P[:2]), B.kf(P[2:5]), B.kf(P[5:8]), B.kf(P[8:], bad=True)
    c["first_max"] = dict(point_map=P, kfs=dict(d=d, e=e, f=f, g=g))
    P = B.pts(3)
    h, i, j = B.kf(P[:1]), B.kf(P[1:2]), B.kf(P[2:])
    B.g["cov"][h] = [i]; B.g["cov"][i] = [j]
    c["only_voters"] = dict(point_map=P[:1], kfs=dict(h=h, i=i, j=j))
    P = B.pts(4)
    k1, k2, q, r = B.kf(P[:1]), B.kf(P[1:2]), B.kf(P[2:3]), B.kf(P[3:])
    B.parent(k1, q); B.g["cov"][k2] = [r]
    c["parent_break"] = dict(point_map=P[:2], kfs=dict(k1=k1, k2=k2, q=q, r=r))
    P = B.pts(6)
    v, cb, cg, hb, hg, pb = B.kf(P[:1]), B.kf(P[1:2], bad=True), B.kf(P[2:3]), B.kf(P[3:4], bad=True), B.kf(P[4:5]), B.kf(P[5:], bad=True)
    B.g["cov"][v] = [cb, cg]; B.parent(hb, v); B.parent(hg, v); B.parent(v, pb)
    c["bad_skips"] = dict(point_map=P[:1], kfs=dict(v=v, cb=cb, cg=cg, hb=hb, hg=hg, pb=pb))
    P = B.pts(83)
    w = [B.kf(P[n:n + 1]) for n in range(80)]
    x0, x1, x2 = B.kf(P[80:81]), B.kf(P[81:82]), B.kf(P[82:])
    B.g["cov"][w[0]] = [x0]; B.parent(x1, w[0]); B.g["cov"][w[1]] = [x2]
    c["limit_80"] = dict(point_map=P[:80], kfs=dict(w0=w[0], w79=w[79], x0=x0, x1=x1, x2=x2))
    P = B.pts(4); L = B.lns(3)
    y = B.kf([P[0], P[1], P[0], P[2]], [L[0], L[1], L[0]])
    z = B.kf([P[2], P[3], P[1], -1], [L[1], L[2]])
    c["dedup"] = dict(point_map=[P[0], P[3]], kfs=dict(y=y, z=z), P=P, L=L)
    c["stale"] = dict(point_map=[], kf_prev=[y, h, a], ref_prev=h, kfs={})
    P = B.pts(1); L = B.lns(1)
    t, u = B.kf(P), B.kf((), L)
    c["lines_no_vote"] = dict(point_map=P, line_map=L, kfs=dict(t=t, u=u))
    P = B.pts(2)
    gb = B.kf(P, bad=True)
    c["bad_voters"] = dict(point_map=P, kf_prev=[a], ref_prev=b_, kfs=dict(gb=gb))
    for name, cs in c.items():
        cs.setdefault("kf_prev", [])
        cs.setdefault("ref_prev", -1)
        cs.setdefault("line_map", [])
    return B.g, c


def quirk_map(g):
    """A map of g's size for the device (positions and descriptors are not read by UpdateLocalMap)."""
    P, L = max(g["n_points"], 1), max(g["n_lines"], 1)
    return dict(pt_pos=np.zeros((P, 3), np.float32), pt_normal=np.zeros((P, 3), np.float32), pt_min_dist=np.zeros(P, np.float32),
                pt_max_dist=np.ones(P, np.float32), pt_desc=np.zeros((P, 32), np.uint8), ln_pos=np.zeros((L, 6)), ln_normal=np.zeros((L, 3)),
                ln_min_dist=np.zeros(L, np.float32), ln_max_dist=np.ones(L, np.float32), ln_desc=np.zeros((L, 32), np.uint8))


# ---------------------------------------------------------------------------------------------------- the planar scene
def _connections(g, k, among):
    """UpdateConnections of keyframe k against the keyframes in `among`: the ordered covisibles (KeyFrame.cc:304-413)."""
    obs = observations(g)
    cnt = {}
    for m in g["pt"][k]:
        if m >= 0:
            for o in obs[m]:
                if o != k and o in among:
                    cnt[o] = cnt.get(o, 0) + 1
    if not cnt:
        return []
    pairs = [(wt, o) for o, wt in cnt.items() if wt >= 15]
    if not pairs:
        o = max(sorted(cnt), key=lambda x: cnt[x])            # the first strict maximum in map order
        pairs = [(cnt[o], o)]
    return [o for _, o in sorted(pairs, reverse=True)]


def scene_graph(m, seed=5):
    """Ten keyframes over the planar scene (the map's frame, and steps 0, 2, 4 of the three motion_scene streams), each holding the
    map points and lines it sees, numbered by a seeded permutation of their creation order."""
    poses = [(np.eye(4, dtype=np.float32), ts.K0)] + [(ms.stream_pose(s, k), ms.STREAMS[s][2]) for s in range(3) for k in (0, 2, 4)]
    rng = np.random.default_rng(seed)
    idx = rng.permutation(len(poses))                           # creation c gets index idx[c]
    K = len(poses)
    g = dict(Tcw=[None] * K, Twc=[None] * K, bad=[0] * K, parent=[-1] * K, pt=[None] * K, ln=[None] * K, cov=[None] * K,
             children=[set() for _ in range(K)], n_points=len(m["pt_pos"]), n_lines=len(m["ln_pos"]))

    def visible(T, Kc, X):
        T = np.asarray(T, np.float64); X = np.asarray(X, np.float64)
        c = X @ T[:3, :3].T + T[:3, 3]
        u = c[:, 0] / c[:, 2] * Kc[0] + Kc[2]; v = c[:, 1] / c[:, 2] * Kc[1] + Kc[3]
        return (u > 10) & (u < ts.W - 10) & (v > 10) & (v < ts.H - 10) & (c[:, 2] > 0)
    for cidx, (T, Kc) in enumerate(poses):
        k = idx[cidx]
        g["Tcw"][k] = np.asarray(T, np.float32); g["Twc"][k] = inverse(T)
        pv = np.nonzero(visible(T, Kc, m["pt_pos"]))[0]
        lv = np.nonzero(visible(T, Kc, m["ln_pos"][:, :3]) & visible(T, Kc, m["ln_pos"][:, 3:]))[0]
        g["pt"][k] = [int(x) for x in rng.permutation(pv)]   # feature order
        g["ln"][k] = [int(x) for x in rng.permutation(lv)]
    for cidx in range(1, K):
        k = idx[cidx]
        first = _connections(g, k, set(int(x) for x in idx[:cidx]))
        if first:
            g["parent"][k] = first[0]; g["children"][first[0]].add(k)
    for k in range(K):
        g["cov"][k] = _connections(g, k, set(range(K)))
    return g
