"""CPU tests: the line oracle against the reference tree's own line extraction (oracle/_ref/libref_line.so, built by
oracle/Makefile `ref`) at the frame shapes and selection edges test_line_shapes_gpu.py checks the CUDA path at, so that the
GPU test's reference is shown right there on a machine without a GPU.

Every KeyLine of a frame is compared at each shape of line_shapes.SHAPES; LINEextractor's selection (LineExtractor.cpp) at
nfeatures around the line count, min_line_length above every line, equal to a line's length and cutting at the first line, and
with masks that drop lines, on the clamped border too.  Where nfeatures is not below the number of lines the reference appends
a default-constructed KeyLine with indeterminate fields and describes it (LineExtractor.cpp:64; the oracle's is zero), which
is not reproducible: the selection is compared at one line fewer there, where every line is kept and nothing is appended.
The comparisons at line_shapes.REF_SHAPES also run from the reference's stored outputs (tests/golden/refcalls/)."""
import os
import sys
import numpy as np
import pytest
import oracle
from oracle import binding as ob
from plslam_b200 import synth
import line_shapes as LS

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from gen_golden_line_ref import select  # noqa: E402

needs_live = pytest.mark.skipif(not os.path.exists(ob._REF_LINE_LIB), reason="oracle/_ref/libref_line.so not built (needs the reference tree)")


@needs_live
@pytest.mark.parametrize("w,h,seed,cap", LS.SHAPES)
def test_keylines_equal_reference_library(w, h, seed, cap):
    img = synth.synth_frame(w, h, seed)
    rk = oracle.ref_lsd_keylines(img)
    assert len(rk) > 50
    ok = oracle.line_extract(img, nfeatures=100000)[0][:-1]      # every KeyLine, sorted; the appended zero record dropped
    assert ok.tobytes() == select(rk, len(rk)).tobytes()


@pytest.mark.skipif(not oracle.ref_line_available(), reason="neither oracle/_ref/libref_line.so nor its stored outputs exist")
@pytest.mark.parametrize("w,h,seed", LS.REF_SHAPES)
def test_line_extractor_equals_reference_library(w, h, seed):
    img = synth.synth_frame(w, h, seed)
    ok, od, ol = oracle.line_extract(img, nfeatures=200, min_line_length=0.0)
    assert len(ok) == 201
    LS.same_up_to_equal_response_swaps(ok, od, ol, *oracle.ref_line_extract(img, nfeatures=200, min_line_length=0.0))


def _select(img, nf, mll, mask=None):
    ok, od, ol = oracle.line_extract(img, mask=mask, nfeatures=nf, min_line_length=mll)
    LS.same_up_to_equal_response_swaps(ok, od, ol, *oracle.ref_line_extract(img, mask=mask, nfeatures=nf, min_line_length=mll))
    return len(ok)


@needs_live
def test_nfeatures_around_the_line_count():
    img = synth.synth_frame(*LS.SEL_FRAME)
    n = len(oracle.lsd_detect(img))
    assert _select(img, n - 1, 0.0) == n                         # nfeatures + 1 kept: every line, nothing appended
    assert _select(img, n - 2, 0.0) == n - 1
    assert _select(img, 1, 0.0) == 2


@needs_live
def test_min_line_length_edges():
    img = synth.synth_frame(*LS.SEL_FRAME)
    L = oracle.line_extract(img, nfeatures=200)[0]["lineLength"].astype(np.float64)
    assert _select(img, 200, 1e6) == 201
    k = next(i for i in range(100, 190) if L[i - 1] > L[i] > L[i + 1])
    assert _select(img, 200, L[k]) == k + 1
    assert _select(img, k + 1, L[k]) == k + 2
    assert _select(img, 200, (L[0] + L[1]) / 2) == 1


@needs_live
def test_masks_that_drop_lines():
    w, h, seed = LS.SEL_FRAME
    img = synth.synth_frame(w, h, seed)
    some = np.full((h, w), 255, np.uint8)
    some[40:200, 60:260] = 0
    kept = len(oracle.line_extract(img, mask=some, nfeatures=100000)[0]) - 1
    assert _select(img, 200, 0.0, some) == 201
    assert _select(img, kept - 1, 0.0, some) == kept
    # the mask on the last column and row: lines with both end points clamped onto it are dropped, and only those
    w, h = 641, 481
    img = LS.corner(w, h, 3)
    m = LS.border_mask(w, h)
    kept = len(oracle.line_extract(img, mask=m, nfeatures=100000)[0]) - 1
    assert kept < len(oracle.lsd_detect(img))
    assert _select(img, kept - 1, 0.0, m) == kept
