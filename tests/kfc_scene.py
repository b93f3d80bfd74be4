"""A seeded scene for LocalMapping::KeyFrameCulling (tests/golden/refcalls/keyframe_culling.npz, tools/gen_keyframe_culling.py).

Random part: keyframe rows of 200-1500 slots along a trajectory; each map point is observed by 1-40 keyframes near its first one,
most by four or more, at octaves drawn towards the fine end, so that some keyframes sit just above or below the 90 % line and the
culls of a list change what the keyframes after them see.  Groups: the covisible keyframes of a current keyframe (the rows sharing
points with it, most shared first), 10-80 long.

Crafted part: one more group whose keyframes each decide one rule of the loop (their points are otherwise seen only by helper
rows that no list holds):
  A   mnId == 0 and redundant                         F  culled; its observations make G's points 4-observer
  G   redundant on the snapshot, not after F's cull   H  culled; four of its points have 3 observers and go bad
  I   redundant only once H's bad points leave nMPs   D  mbNotErase and redundant (code 2); E still sees it
  E   redundant because D erased nothing              B  18 of 20 (a point in two slots, bad points on input)
  B2  9 of 10                                          C  nMPs = 0
  J   observers at octave + 1 count, at + 2 do not    K  holds points it does not observe, Observations() exactly 3
  L   3 other observers of which only 2 are fine enough
"""
import numpy as np

from plslam_b200.binding import KP_DTYPE, pack_cull_groups, pack_cull_keyframes, pack_cull_points


def packed(keyframes, points, groups, cap=None):
    """the scene in the layouts of pl_keyframe_culling_dev, as one dict (the oracle's and the fixture's form)"""
    k = pack_cull_keyframes(keyframes, cap)
    del k["cap"]
    return dict(k, **pack_cull_points(points), **pack_cull_groups(groups))


def split(s):
    """one packed dict -> the (keyframes, points, groups) dicts of KeyFrameCullingProblems"""
    return ({n: s[n] for n in ("keys_un", "n", "mp", "origin", "not_erase")}, {n: s[n] for n in ("bad", "obs_offset", "obs_kf", "obs_idx")},
            {n: s[n] for n in ("offset", "count", "list")})


OCT_P = [0.45, 0.25, 0.12, 0.08, 0.05, 0.03, 0.01, 0.01]


class Builder:
    def __init__(self):
        self.oct, self.mp, self.origin, self.not_erase = [], [], [], []
        self.bad, self.obs = [], []

    def row(self, origin=False, not_erase=False):
        self.oct.append([]); self.mp.append([]); self.origin.append(origin); self.not_erase.append(not_erase)
        return len(self.mp) - 1

    def point(self, bad=False):
        self.bad.append(bad); self.obs.append([])
        return len(self.bad) - 1

    def slot(self, r, p, octave=0, observe=True):
        """a slot of row r holding point p (-1: NULL); observe: the point records it (AddObservation)"""
        self.mp[r].append(p); self.oct[r].append(int(octave))
        if observe and p >= 0:
            self.obs[p].append((r, len(self.mp[r]) - 1))

    def pad(self, r, n):
        while len(self.mp[r]) < n:
            self.slot(r, -1, 0)

    def scene(self, groups):
        keyframes = []
        for o, m, g, ne in zip(self.oct, self.mp, self.origin, self.not_erase):
            keys = np.zeros(len(m), KP_DTYPE)
            keys["octave"] = o
            keys["size"] = 31.0
            keys["class_id"] = -1
            keyframes.append(dict(keys=keys, mp=np.array(m, np.int32), origin=bool(g), not_erase=bool(ne)))
        return keyframes, dict(bad=np.array(self.bad, np.uint8), observations=self.obs), groups


def _random_part(b, rng, n_rows=110, list_lengths=(12, 25, 45, 80, 60)):
    base = len(b.mp)
    rows = [b.row(origin=(k == 0), not_erase=(k % 29 == 13)) for k in range(n_rows)]
    size = rng.integers(200, 700, n_rows)
    size[[5, 37, 71]] = 1500
    free = size.copy()
    dense = 0.78 + 0.2 * (0.5 + 0.5 * np.sin(np.arange(n_rows) / 6.0))     # neighbouring keyframes see alike
    while free.sum() > 0.03 * size.sum():
        owner = int(rng.choice(n_rows, p=free / free.sum()))
        m = 4 + min(int(rng.geometric(0.22)) - 1, 36) if rng.random() < dense[owner] else int(rng.integers(1, 4))
        cand = np.array([k for k in range(max(0, owner - 40), min(n_rows, owner + 41)) if k != owner and free[k] > 0])
        if len(cand):
            w = np.exp(-0.5 * ((cand - owner) / 12.0) ** 2)
            cand = rng.choice(cand, min(m - 1, len(cand)), replace=False, p=w / w.sum())
        p = b.point(bad=rng.random() < 0.01)
        for k in [owner] + [int(c) for c in cand]:
            b.slot(rows[k], p, rng.choice(8, p=OCT_P))
            free[k] -= 1
    for k in range(n_rows):
        held = [p for p in b.mp[rows[k]] if p >= 0]
        if k % 9 == 4 and held:                  # a point held in a second slot, which it does not record
            b.slot(rows[k], held[len(held) // 2], rng.choice(8, p=OCT_P), observe=False)
        b.pad(rows[k], size[k])
    # covisibility: rows sharing points with a current keyframe, most shared first (ties by row)
    share = np.zeros((n_rows, n_rows), np.int64)
    for obs in b.obs:
        ks = sorted({r - base for r, _ in obs if base <= r < base + n_rows})
        for i in ks:
            for j in ks:
                share[i, j] += i != j
    groups = []
    for L, cur in zip(list_lengths, rng.choice(np.arange(20, n_rows - 20), len(list_lengths), replace=False)):
        order = sorted((k for k in range(n_rows) if share[cur, k] > 0), key=lambda k: (-share[cur, k], k))
        groups.append([rows[k] for k in order[:L]])
    if not any(rows[0] in g for g in groups):
        groups[0] = [rows[0]] + groups[0][:-1]
    return groups


def _crafted_part(b):
    h = [b.row() for _ in range(6)]              # helpers: observers that no list holds

    def R(r, octave=0):                          # a point that r and four helpers observe: redundant in r, even after one cull
        p = b.point()
        b.slot(r, p, octave)
        for k in h[:4]:
            b.slot(k, p, 0)
        return p

    def shared(rows_octs, helpers):              # one point observed by the given (row, octave) and helper (index, octave) slots
        p = b.point()
        for r, o in rows_octs:
            b.slot(r, p, o)
        for k, o in helpers:
            b.slot(h[k], p, o)
        return p

    A = b.row(origin=True)
    F, G, H, I, D, E, B, B2, C, J, K, L = [b.row(not_erase=(n == "D")) for n in "FGHIDEBbCJKL"]
    for _ in range(20):
        R(A)
        R(F)
        shared([(F, 0), (G, 0)], [(0, 0), (1, 0)])         # G: 4 observers; after F's cull 3
    for _ in range(40):
        R(H)
    for _ in range(4):
        shared([(H, 0), (I, 0)], [(0, 0)])                 # 3 observers: H's cull leaves 2, the point goes bad
    for _ in range(20):
        R(I)
        shared([(D, 0), (E, 0)], [(0, 0), (1, 0)])         # D keeps its observations (mbNotErase), so E stays redundant
    for _ in range(16):
        R(B)
    twice = R(B)
    b.slot(B, twice, 0, observe=False)                     # the same point in a second slot: 18 redundant slots
    for _ in range(2):
        shared([(B, 0)], [])                               # seen by B alone
    for _ in range(3):
        p = R(B)
        b.bad[p] = True                                    # bad on input
    for _ in range(9):
        R(B2)
    shared([(B2, 0)], [])
    for _ in range(3):
        p = R(C)
        b.bad[p] = True
    for _ in range(20):
        shared([(J, 2)], [(0, 3), (1, 3), (2, 3)])         # octave + 1: counts
    for _ in range(2):
        shared([(J, 2)], [(0, 4), (1, 4), (2, 4)])         # octave + 2: does not
    for _ in range(20):
        p = shared([], [(0, 0), (1, 0), (2, 0)])           # Observations() == 3, K not among them
        b.slot(K, p, 0, observe=False)
        shared([(L, 0)], [(3, 0), (4, 0), (5, 5)])         # two fine-enough others
    for r in (A, F, G, H, I, D, E, B, B2, C, J, K, L):
        b.pad(r, 200)
    for k in h:
        b.pad(k, len(b.mp[k]))
    return [A, F, G, H, I, D, E, B, B2, C, J, K, L]


def bulk(rng, size, heavy=0, heavy_obs=0, window=40):
    """(Builder, rows) of len(size) keyframes along a trajectory filled as the random part fills its rows, after `heavy` points
    observed by `heavy_obs` keyframes each (for the larger scenes of the device test and tools/keyframe_culling_time.py)."""
    b = Builder()
    n_rows = len(size)
    rows = [b.row(origin=(k == 0), not_erase=(k % 29 == 13)) for k in range(n_rows)]
    free = np.asarray(size, np.int64).copy()
    for _ in range(heavy):
        p = b.point()
        for k in rng.choice(n_rows, heavy_obs, replace=False):
            b.slot(rows[k], p, rng.choice(8, p=OCT_P))
            free[k] -= 1
    dense = 0.78 + 0.2 * (0.5 + 0.5 * np.sin(np.arange(n_rows) / 6.0))
    octs = rng.choice(8, int(free.sum()) * 2, p=OCT_P)
    used = 0
    free = np.maximum(free, 0)
    while free.sum() > 0.03 * np.sum(size):
        owner = int(rng.choice(n_rows, p=free / free.sum()))
        m = 4 + min(int(rng.geometric(0.22)) - 1, 36) if rng.random() < dense[owner] else int(rng.integers(1, 4))
        lo, hi = max(0, owner - window), min(n_rows, owner + window + 1)
        cand = np.arange(lo, hi)
        cand = cand[(cand != owner) & (free[lo:hi] > 0)]
        if len(cand):
            w = np.exp(-0.5 * ((cand - owner) / 12.0) ** 2)
            cand = rng.choice(cand, min(m - 1, len(cand)), replace=False, p=w / w.sum())
        p = b.point()
        for k in [owner] + [int(c) for c in cand]:
            b.slot(rows[k], p, octs[used]); used += 1
            free[k] -= 1
    for k in range(n_rows):
        b.pad(rows[k], size[k])
    return b, rows


def scene(seed=11):
    """(keyframes, points, groups): keyframes = dicts (keys [n] KP_DTYPE, mp [n], origin, not_erase), points = dict(bad [n_mp],
    observations = [[(row, idx), ...] per point]), groups = lists of keyframe rows in GetVectorCovisibleKeyFrames() order."""
    rng = np.random.default_rng(seed)
    b = Builder()
    groups = _random_part(b, rng)
    groups.append(_crafted_part(b))
    return b.scene(groups)
