"""CPU oracle of pl_keyframe_culling_dev: LocalMapping::KeyFrameCulling (src/LocalMapping.cc:1835-1899, monocular) restated with
the live state the culls of earlier entries leave (KeyFrame::SetBadFlag, src/KeyFrame.cc:494-508; MapPoint::EraseObservation,
src/MapPoint.cc:111-137), on the packed layouts of include/plslam_b200.h (binding.pack_cull_*).

Each switchable mutant changes one decision of the loop; tests/test_keyframe_culling.py checks that every one of them changes the
reference's result on the scene of tests/kfc_scene.py."""
import numpy as np

MUTANTS = {
    "no_cascade": "every entry judged on the snapshot",
    "no_point_cascade": "an erase never makes a point bad",
    "octave_le": "observers at an octave <= the slot's, not <= + 1",
    "obs_ge3": "Observations() >= 3 instead of > 3",
    "ratio_ge": "nRedundantObservations >= 0.9 * nMPs instead of >",
    "not_erase_erases": "mbNotErase treated as an erase",
    "origin_not_skipped": "mnId == 0 not skipped",
    "self_observer": "the entry itself counted as an observer",
}


def octaves(s):
    return s["keys_un"]["octave"] if "keys_un" in s else s["octave"]


def group_status(s, g):
    """status of group g, the first of plslam_b200.h's pl_keyframe_culling_dev rules that applies"""
    off, cnt = int(s["offset"][g]), int(s["count"][g])
    n_kf, cap, n, mp = len(s["n"]), s["mp"].shape[1], s["n"], s["mp"]
    n_mp, n_obs = len(s["bad"]), len(s["obs_kf"])
    if off < 0 or cnt < 0 or off + cnt > len(s["list"]):
        return 1
    lst = [int(k) for k in s["list"][off:off + cnt]]
    if any(k < 0 or k >= n_kf for k in lst):
        return 1
    if any(n[k] < 0 or n[k] > cap for k in lst):
        return 2
    if len(set(lst)) != len(lst):
        return 3
    pts = np.concatenate([mp[k, :n[k]] for k in lst] + [np.zeros(0, np.int32)])
    if np.any((pts < -1) | (pts >= n_mp)):
        return 4
    pts = np.unique(pts[pts >= 0])
    a, b = s["obs_offset"][pts], s["obs_offset"][pts + 1]
    if np.any((a < 0) | (b < a) | (b > n_obs)):
        return 5
    for p, lo, hi in zip(pts, a, b):
        for k, idx in zip(s["obs_kf"][lo:hi], s["obs_idx"][lo:hi]):
            if k < 0 or k >= n_kf or idx < 0 or idx >= min(n[k], cap) or mp[k, idx] != p:
                return 6
    return 0


def judge(s, k, culled, mutant=None):
    """(nMPs, nRedundantObservations) of keyframe row k, given the rows culled so far (bool [n_kf])"""
    oct_, off = octaves(s).astype(np.int64), s["obs_offset"]
    nm = nr = 0
    for i in range(int(s["n"][k])):
        p = int(s["mp"][k, i])
        if p < 0 or s["bad"][p]:
            continue
        obs_kf, obs_idx = s["obs_kf"][off[p]:off[p + 1]], s["obs_idx"][off[p]:off[p + 1]]
        gone = culled[obs_kf]
        n_culled = int(gone.sum())
        nobs = len(obs_kf) - n_culled                     # Observations(): one per remaining observer
        if n_culled and nobs <= 2 and mutant != "no_point_cascade":
            continue                                      # EraseObservation made it bad (nObs <= 2)
        nm += 1
        if nobs >= 3 if mutant == "obs_ge3" else nobs > 3:
            live = ~gone if mutant == "self_observer" else ~gone & (obs_kf != k)
            gate = oct_[k, i] if mutant == "octave_le" else oct_[k, i] + 1
            if int(np.sum(oct_[obs_kf[live], obs_idx[live]] <= gate)) >= 3:
                nr += 1
    return nm, nr


def cull(s, mutant=None):
    """code, n_mps, n_redundant [n_list] and status [G], as pl_keyframe_culling_dev writes them (untouched entries keep -7)"""
    n_list, G = len(s["list"]), len(s["offset"])
    code = np.full(n_list, -7, np.int8); n_mps = np.full(n_list, -7, np.int32); n_red = np.full(n_list, -7, np.int32)
    status = np.zeros(G, np.int32)
    for g in range(G):
        status[g] = group_status(s, g)
        if status[g]:
            continue
        off, cnt = int(s["offset"][g]), int(s["count"][g])
        culled = np.zeros(len(s["n"]), bool)
        for j in range(off, off + cnt):
            k = int(s["list"][j])
            if s["origin"][k] and mutant != "origin_not_skipped":
                code[j], n_mps[j], n_red[j] = -1, 0, 0
                continue
            nm, nr = judge(s, k, np.zeros_like(culled) if mutant == "no_cascade" else culled, mutant)
            c = 0
            if (nr >= 0.9 * nm) if mutant == "ratio_ge" else (nr > 0.9 * nm):
                c = 2 if s["not_erase"][k] and mutant != "not_erase_erases" else 1
            if c == 1:
                culled[k] = True
            code[j], n_mps[j], n_red[j] = c, nm, nr
    return dict(code=code, n_mps=n_mps, n_redundant=n_red, status=status)
