"""Record the pose-only LM's and the global BA's outputs on the GPU -> tests/golden/optimizer_bits.npz (or the path given).

The inputs and the list of arrays are tests/test_optimizer_bits_gpu.optimizer_outputs; that test compares the current library
with this file byte for byte.  Re-record only for a change that is meant to alter the optimisers' results, and say why.

    python tools/gen_optimizer_bits.py [out.npz]
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import plslam_b200  # noqa: F401,E402
from test_optimizer_bits_gpu import optimizer_outputs, GOLDEN  # noqa: E402

out = sys.argv[1] if len(sys.argv) > 1 else GOLDEN
arrays = optimizer_outputs()
os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
np.savez_compressed(out, **arrays)
print(out, {k: (np.asarray(v).dtype.str, np.asarray(v).shape) for k, v in sorted(arrays.items())})
