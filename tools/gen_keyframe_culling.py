"""Generate tests/golden/refcalls/keyframe_culling.npz: LocalMapping::KeyFrameCulling on the scene of tests/kfc_scene.py, each group
run by tools/keyframe_culling_ref.cpp (the loop and KeyFrame::SetBadFlag's erasing part restated, every map-point call the
reference's own src/MapPoint.cc) on a fresh copy of the snapshot.

The fixture holds the packed scene (the layouts of pl_keyframe_culling_dev) and the reference's code, nMPs and
nRedundantObservations per list entry.  tests/test_keyframe_culling.py compares the oracle with it, and
tests/test_keyframe_culling_gpu.py the device call.

Needs the reference tree (REF, default: oracle/Makefile's) and the CPU oracle built (make -C oracle).
Run from the repo root:  python tools/gen_keyframe_culling.py
"""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import kfc_scene  # noqa: E402
from gen_fuse_protocol import ORACLE, reference_dir  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "refcalls", "keyframe_culling.npz")


def build_driver(tmp):
    ref = reference_dir()
    dbow, ld = f"{ref}/Thirdparty/DBoW2/DBoW2", f"{ref}/Thirdparty/line_descriptor"
    so = os.path.join(tmp, "libkeyframe_culling.so")
    subprocess.check_call(
        ["g++", "-O2", "-std=gnu++14", "-fPIC", "-ffp-contract=off", "-w", "-shared", "-Wl,-Bsymbolic",
         "-Ishim_slam", "-I-", "-Ishim", f"-I{ref}", f"-I{ref}/include", f"-I{dbow}", f"-I{ld}/include", f"-I{ORACLE}", "-o", so,
         f"{ref}/src/ORBmatcher.cc", f"{ref}/src/MapPoint.cc", f"{ref}/src/LSDmatcher.cpp", f"{ref}/src/lineIterator.cpp",
         f"{dbow}/BowVector.cpp", f"{dbow}/FeatureVector.cpp", os.path.join(ROOT, "tools", "keyframe_culling_ref.cpp"), "ref_cv_impl.cpp",
         "-L.", "-loracle", "-lpthread", f"-Wl,-rpath,{ORACLE}"], cwd=ORACLE)
    return C.CDLL(so)


def run_reference(L, s):
    p = lambda a: np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)
    n_kf, cap = s["mp"].shape
    octave = np.ascontiguousarray(s["keys_un"]["octave"], np.int32)
    n_list = len(s["list"])
    code = np.zeros(n_list, np.int8); n_mps = np.zeros(n_list, np.int32); n_red = np.zeros(n_list, np.int32)
    for off, cnt in zip(s["offset"], s["count"]):
        c, m, r = np.zeros(cnt, np.int8), np.zeros(cnt, np.int32), np.zeros(cnt, np.int32)
        lst = np.ascontiguousarray(s["list"][off:off + cnt])
        L.ref_keyframe_culling(n_kf, cap, p(octave), p(s["n"]), p(s["mp"]), p(s["origin"]), p(s["not_erase"]), len(s["bad"]), p(s["bad"]),
                               p(s["obs_offset"]), p(s["obs_kf"]), p(s["obs_idx"]), int(cnt), p(lst), p(c), p(m), p(r))
        code[off:off + cnt], n_mps[off:off + cnt], n_red[off:off + cnt] = c, m, r
    return dict(ref_code=code, ref_n_mps=n_mps, ref_n_redundant=n_red)


if __name__ == "__main__":
    s = kfc_scene.packed(*kfc_scene.scene())
    with tempfile.TemporaryDirectory() as tmp:
        r = run_reference(build_driver(tmp), s)
    np.savez_compressed(OUT, **s, **r)
    print(f"{OUT}: {len(s['n'])} keyframes, {len(s['bad'])} points, {len(s['offset'])} groups, codes "
          f"{ {int(c): int((r['ref_code'] == c).sum()) for c in (-1, 0, 1, 2)} }")
