"""Generate tests/golden/orb_cv2_svd4.npz: cv2.SVDecomp(A, SVD_MODIFY_A | SVD_FULL_UV) of 4x4 float32 matrices, w and vt, for the
tests of pl-slam_b200/csrc/svd4.cuh and of the oracle's SVD where cv2 is absent (tests/test_triangulate_svd.py).

Four families: triangulation-shaped matrices (LocalMapping.cc:458-462 on two-view problems with TUM-like intrinsics, baselines
about 0.3 m and depths 2.5-9 m, the rows formed as cv2.addWeighted forms them), random matrices whose entries and rows span many
decades, edge cases (zero rows, repeated rows, rank 1 and 2, the zero matrix, diagonal and permutation matrices), and last the
matrices of HYPOT_CASES: uniform random ones on which the Jacobi gives a different vt with the C library's hypot than with
OpenCV's own hypot template (tools/svd4_hypot_search.cpp found them among 3e8; such a matrix is too rare for the random
families to contain one).

Run from the repo root:  python tools/gen_svd4_cv2.py
"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cnmp_oracle as co  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "orb_cv2_svd4.npz")
# 16 fp32 bit patterns each, row-major
HYPOT_CASES = [
    [3198605837, 3200254583, 3204638911, 1063450560, 3209766159, 1060276511, 3210190283, 3199801363, 1056889039, 3212347497, 3196037304, 1064284573, 1034223668, 1050076815, 1057658563, 3208762352],
    [1048895272, 3201376508, 1050393568, 1062681828, 1061437912, 1056256228, 1062840460, 1064389030, 3208240770, 3205423240, 1056801556, 3210722248, 1049265220, 1033617872, 3200906240, 3193642424],
    [3201420728, 3209104022, 1044148896, 3192403432, 1037969968, 3209926634, 1055535648, 3209192406, 3212425006, 1038764592, 1054968128, 1062453134, 1054387284, 1044914608, 3202911684, 1043200328],
    [3208521896, 1048902172, 1010262528, 3205948470, 3193105560, 1057820920, 3200401188, 1007351296, 3205650358, 3207005288, 3202151520, 3208816086, 3205169852, 3207229670, 3205672434, 3201462976],
    [1063575454, 3212025108, 1062734232, 3212080650, 3189734880, 1029004256, 1015155072, 1059145316, 1035129008, 1044447056, 1041789216, 1058871592, 3197873356, 1061316012, 3153509632, 1025644608],
]


def cv2_svd(A):
    w, u, vt = cv2.SVDecomp(A.copy(), flags=cv2.SVD_MODIFY_A | cv2.SVD_FULL_UV)
    return w.ravel(), vt


def matrices(seed=0):
    rng = np.random.default_rng(seed)
    A = [co.triangulation_matrices(rng, 2000)]
    R = rng.normal(size=(1500, 4, 4)) * 10.0 ** rng.uniform(-4, 4, (1500, 1, 1)) * 10.0 ** rng.uniform(-1.5, 1.5, (1500, 4, 1))
    A.append(R.astype(np.float32))
    E = []
    for t in range(500):
        M = (rng.normal(size=(4, 4)) * 10.0 ** rng.uniform(-3, 3)).astype(np.float32)
        kind = t % 8
        if kind == 0: M[rng.integers(4)] = 0
        elif kind == 1: M[rng.choice(4, 2, replace=False)] = 0
        elif kind == 2: M[1] = M[0]
        elif kind == 3: M = np.outer(M[0], M[1]).astype(np.float32)
        elif kind == 4: M[2] = M[0] * np.float32(2); M[3] = M[1] * np.float32(-0.5)
        elif kind == 5: M = np.diag(M[0]).astype(np.float32)
        elif kind == 6: M = np.eye(4, dtype=np.float32)[rng.permutation(4)] * M[0, 0]
        else: M[:, rng.integers(4)] = 0
        E.append(M)
    E[0] = np.zeros((4, 4), np.float32)
    A.append(np.array(E, np.float32))
    A.append(np.array(HYPOT_CASES, np.uint32).view(np.float32).reshape(-1, 4, 4))
    return np.concatenate(A)


if __name__ == "__main__":
    A = matrices()
    w = np.zeros((len(A), 4), np.float32); vt = np.zeros((len(A), 4, 4), np.float32)
    for i, M in enumerate(A):
        w[i], vt[i] = cv2_svd(M)
    np.savez_compressed(OUT, A=A, w=w, vt=vt, n_hypot=np.int32(len(HYPOT_CASES)), cv2_version=np.array(cv2.__version__))
    print(f"{OUT}: {len(A)} matrices, cv2 {cv2.__version__}")
