"""plslam_b200 — H100-native PL-SLAM front-end / LM hot path (host-side Python mirror).

The product is the C-ABI library libplslam_b200.so (include/plslam_b200.h).  This package is a thin
ctypes mirror of the reference's operator classes used by the tests and bench.py; it never imports
the CPU oracle and raises if the CUDA library is missing (no CPU fallback).
"""
from .binding import *  # noqa: F401,F403
from . import synth  # noqa: F401
from . import trajectory  # noqa: F401
