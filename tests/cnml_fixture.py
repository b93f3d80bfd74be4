"""tests/golden/refcalls/create_new_map_lines.npz (tools/gen_create_new_map_lines.py): the scene of tests/cnml_scene.py, the
reference's own line searches of the neighbours that passed the baseline test, and the lines the reference's
CreateNewMapLinesConstraint loop created from them, in creation order."""
import os

import numpy as np

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refcalls", "create_new_map_lines.npz")


def load():
    with np.load(FIXTURE) as z:
        return {k: z[k] for k in z.files}


def keyframes(s):
    st = s["kf_start"]
    return [dict(ldesc=s["ldesc"][a:b], has_ml=s["has_ml"][a:b], keylines=s["keylines"][a:b], line_func=s["line_func"][a:b],
                 Tcw=s["Tcw"][k], Ow=s["Ow"][k], K=s["K"][k]) for k, (a, b) in enumerate(zip(st[:-1], st[1:]))]


def problems(s):
    """one (current, neighbour) search per neighbour that passed the baseline test, in vpNeighKFs' order"""
    return [(0, j + 1) for j in np.nonzero(s["searched"])[0]]


def group(s, positional=True):
    """entry e = the e-th search, paired with vpNeighKFs[e] = keyframe e + 1 (positional) and its median depth"""
    probs = problems(s)
    rows = [e + 1 if positional else probs[e][1] for e in range(len(probs))]
    return dict(kf_cur=0, entries=[(e, r, s["medians"][r]) for e, r in enumerate(rows)])


def created(code, line3D, n_cur, n_entries, matches_of):
    """the committed slots of one group in slot order -> (rows [m][5]: i, j, ikl, idx1, idx2; line3D [m][6])"""
    rows, L = [], []
    pr = 0
    for i in range(n_entries):
        for j in range(i + 1, n_entries):
            for ikl in np.nonzero(code[pr * n_cur:(pr + 1) * n_cur] == 0)[0]:
                rows.append((i, j, int(ikl), int(matches_of(i)[ikl]), int(matches_of(j)[ikl])))
                L.append(line3D[pr * n_cur + ikl])
            pr += 1
    return np.array(rows, np.int32).reshape(-1, 5), np.array(L, np.float32).reshape(-1, 6)
