"""pl_local_ba_dev without a GPU: the exported symbols, the argument refusals that come before the device check, the scratch
size query, and the [W][cap] packer of the Python binding."""
import ctypes as C
import numpy as np
import pytest
import plslam_b200 as pl
from plslam_b200 import binding as bd
from plslam_b200 import synth

FAKE = 4096          # a non-NULL, 16-byte aligned address: every call below is refused before anything could read it


def test_symbols_are_exported():
    L = pl.lib()
    for name in ("pl_local_ba", "pl_local_ba_dev", "pl_local_ba_scratch_bytes"):
        assert hasattr(L, name), name


def _args(W=2, caps=(60, 3000, 400, 15000, 1600)):
    return bd.PLBAWindows(W, *caps, *([FAKE] * 18)), bd.PLBAOut(*([FAKE] * 8))


def _call(win, out, scratch=FAKE, use_win=True, use_out=True):
    L = bd._ba_lib()
    return L.pl_local_ba_dev(C.byref(win) if use_win else None, None, C.byref(out) if use_out else None, scratch, None)


@pytest.mark.parametrize("case", ["no windows", "no outputs", "W < 0", "cap_kf 0", "cap_kf 7724", "cap_pt 0", "cap_ln 0",
                                  "cap_pe 0", "cap_le 2^24 + 1", "W * cap over an int", "n_le NULL", "kf_Tcw NULL", "K_end NULL",
                                  "pe_obs NULL", "le_func NULL", "status out NULL", "le_erase_kf out NULL", "scratch NULL",
                                  "scratch misaligned"])
def test_refusals_before_the_device_check(case):
    win, out = _args()
    kw = {}
    if case == "no windows":
        kw["use_win"] = False
    elif case == "no outputs":
        kw["use_out"] = False
    elif case == "W < 0":
        win.W = -1
    elif case.startswith("cap_"):
        name, value = case.split(" ", 1)
        setattr(win, name, {"0": 0, "7724": 7724, "2^24 + 1": (1 << 24) + 1}[value])
    elif case == "W * cap over an int":
        win.W, win.cap_kf, win.cap_pe = 1 << 20, 4, 1 << 12
    elif case.endswith("out NULL"):
        setattr(out, case.split(" ")[0], None)
    elif case.endswith("NULL") and case != "scratch NULL":
        setattr(win, case.split(" ")[0], None)
    if case == "scratch NULL":
        kw["scratch"] = None
    if case == "scratch misaligned":
        kw["scratch"] = FAKE + 8
    assert _call(win, out, **kw) == -1, case


def test_no_windows_enqueue_nothing():
    win, out = _args(W=0)
    assert _call(win, out, scratch=None) == 0


def test_scratch_bytes():
    L = bd._ba_lib()
    one = L.pl_local_ba_scratch_bytes(1, 60, 3000, 400, 15000, 1600)
    assert one >= 8 * 360 * 360 and one % 256 == 0          # the dense reduced system alone is (6 cap_kf)^2 doubles
    assert L.pl_local_ba_scratch_bytes(264, 60, 3000, 400, 15000, 1600) == 264 * one
    assert L.pl_local_ba_scratch_bytes(0, 60, 3000, 400, 15000, 1600) == 0
    assert L.pl_local_ba_scratch_bytes(1, 7723, 1, 1, 1, 1) > 8 * (6 * 7723) ** 2
    for bad in [(-1, 60, 1, 1, 1, 1), (1, 0, 1, 1, 1, 1), (1, 7724, 1, 1, 1, 1), (1, 1, 0, 1, 1, 1), (1, 1, 1, 1, 1, (1 << 24) + 1),
                (1 << 20, 1, 1, 1, 1 << 12, 1)]:
        assert L.pl_local_ba_scratch_bytes(*bad) == 0, bad


def mixed_windows():
    """Windows of different sizes, one without points and one without any edge."""
    a = synth.synth_ba_problem(4, n_free=8, n_fixed=10, n_pt=600, n_ln=80)
    b = synth.synth_ba_problem(6, n_free=3, n_fixed=2, n_pt=50, n_ln=200)
    b.update(pe_kf=b["pe_kf"][:0], pe_pt=b["pe_pt"][:0], pe_obs=b["pe_obs"][:0], pe_inv_sigma2=b["pe_inv_sigma2"][:0])
    c = synth.synth_ba_problem(9, n_free=12, n_fixed=20, n_pt=1500, n_ln=10)
    d = synth.synth_ba_problem(5, n_free=2, n_fixed=1, n_pt=30, n_ln=5)
    d.update({f: d[f][:0] for f in ("pe_kf", "pe_pt", "pe_obs", "pe_inv_sigma2", "le_kf", "le_ln", "le_func")})
    return [a, b, c, d]


def test_packer_round_trips_mixed_size_windows():
    probs = mixed_windows()
    h = bd.pack_ba_windows(probs, fill=0x5A)
    counts = [bd.ba_window_counts(p) for p in probs]
    assert h["W"] == 4 and h["caps"] == {k: max(1, max(n[k] for n in counts)) for k in bd.BA_COUNTS}
    for k in bd.BA_COUNTS:
        assert h["n_" + k].tolist() == [n[k] for n in counts]
    for f, (k, shape, dt) in bd.BA_INPUTS.items():
        assert h[f].shape == (4, h["caps"][k]) + shape and h[f].dtype == dt, f
        for w, n in enumerate(counts):
            assert (h[f][w, n[k]:].view(np.uint8) == 0x5A).all(), (f, w)          # padding rows hold the fill bytes
    assert np.array_equal(h["K_end"], np.stack([np.asarray(p["K_end"], np.float32) for p in probs]))
    # every padding byte changed: what comes back is the same, so no padding row is read back
    for f, (k, _, _) in bd.BA_INPUTS.items():
        for w, n in enumerate(counts):
            h[f][w, n[k]:].view(np.uint8)[...] = 0xC3
    rows = bd.unpack_ba_rows(h, {k: h["n_" + k] for k in bd.BA_COUNTS}, bd.BA_INPUTS)
    for w, p in enumerate(probs):
        for f, (k, shape, dt) in bd.BA_INPUTS.items():
            want = np.asarray(p[f], dt).reshape((-1,) + shape)
            assert rows[w][f].shape == want.shape and rows[w][f].tobytes() == want.tobytes(), (w, f)


def test_packer_takes_larger_capacities_and_refuses_smaller_ones():
    probs = mixed_windows()[:2]
    h = bd.pack_ba_windows(probs, caps=dict(kf=64, le=4000))
    assert h["caps"]["kf"] == 64 and h["caps"]["le"] == 4000 and h["kf_Tcw"].shape == (2, 64, 16)
    with pytest.raises(ValueError):
        bd.pack_ba_windows(probs, caps=dict(pt=10))
