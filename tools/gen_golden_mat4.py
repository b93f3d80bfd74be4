"""tests/golden/mat4_cv2.npz: cv2.gemm of 512 random fp32 4x4 rigid transforms (A, B, C = A * B), the order the motion model's
guess and velocity products restate (((a0 b0 + a1 b1) + a2 b2) + a3 b3, every operation rounded).  Needs cv2."""
import os

import cv2
import numpy as np


def rigid(rng):
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    w, x, y, z = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    T = np.eye(4); T[:3, :3] = R; T[:3, 3] = rng.normal(size=3)
    return T.astype(np.float32)


def main():
    rng = np.random.default_rng(0)
    A = np.stack([rigid(rng) for _ in range(512)]); B = np.stack([rigid(rng) for _ in range(512)])
    C = np.stack([cv2.gemm(a, b, 1.0, None, 0.0) for a, b in zip(A, B)])
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "mat4_cv2.npz")
    np.savez_compressed(out, A=A, B=B, C=C, cv2_version=cv2.__version__)
    print(out, cv2.__version__)


if __name__ == "__main__":
    main()
