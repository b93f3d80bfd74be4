"""pl_keyframe_culling_dev without a GPU: the exported and declared symbol, the argument refusals that come before the device check,
and the oracle (tests/kfc_oracle.py) against the reference's own culling loop on the scene of tests/kfc_scene.py
(tests/golden/refcalls/keyframe_culling.npz): equal on every entry, while each of its mutants differs somewhere; and the oracle's
status codes on hand-made malformed groups."""
import ctypes as C
import os

import numpy as np
import pytest

import plslam_b200 as pl
from plslam_b200 import binding as bd
import kfc_oracle as ko
import kfc_scene as ks

PL_ERR_ARG = -1
FAKE = 4096          # a non-NULL address: every call below is refused before anything could read it
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "refcalls", "keyframe_culling.npz")


def load():
    with np.load(FIXTURE) as z:
        return {k: z[k] for k in z.files}


def test_symbol_is_exported_and_declared():
    assert hasattr(pl.lib(), "pl_keyframe_culling_dev")
    with open(os.path.join(ROOT, "include", "plslam_b200.h")) as f:
        h = f.read()
    assert "int pl_keyframe_culling_dev(" in h and "typedef struct PLCullGroups" in h


def _call(case):
    k = bd.PLCullKeyframes(4, 300, FAKE, FAKE, FAKE, FAKE, FAKE)
    m = bd.PLCullPoints(10, 30, FAKE, FAKE, FAKE, FAKE)
    g = bd.PLCullGroups(2, FAKE, FAKE, 6, FAKE)
    a = dict(kfs=C.byref(k), points=C.byref(m), groups=C.byref(g), code=FAKE, n_mps=FAKE, n_redundant=FAKE, status=FAKE)
    if case in a:
        a[case] = None
    elif case == "G < 0":
        g.G = -1
    elif case == "n_list < 0":
        g.n_list = -1
    elif case == "n_mp < 0":
        m.n_mp = -1
    elif case == "n_obs < 0":
        m.n_obs = -1
    elif case == "n_kf 0":
        k.n_kf = 0
    elif case == "n_kf over":
        k.n_kf = 65537
    elif case == "cap 0":
        k.cap = 0
    elif case == "cap over":
        k.cap = 6145
    else:
        struct, field = case.split(" ")
        setattr(dict(k=k, m=m, g=g)[struct], field, None)
    return bd._cull_lib().pl_keyframe_culling_dev(a["kfs"], a["points"], a["groups"], a["code"], a["n_mps"], a["n_redundant"],
                                                  a["status"], None)


CASES = ["kfs", "points", "groups", "code", "n_mps", "n_redundant", "status", "G < 0", "n_list < 0", "n_mp < 0", "n_obs < 0",
         "n_kf 0", "n_kf over", "cap 0", "cap over", "k keys_un", "k n", "k mp", "k origin", "k not_erase", "m bad", "m obs_offset",
         "m obs_kf", "m obs_idx", "g offset", "g count", "g list"]


@pytest.mark.parametrize("case", CASES)
def test_refusals_before_the_device_check(case):
    assert _call(case) == PL_ERR_ARG


def test_no_groups_enqueue_nothing():
    g = bd.PLCullGroups(0, None, None, 0, None)
    assert bd._cull_lib().pl_keyframe_culling_dev(None, None, C.byref(g), None, None, None, None, None) == 0


def test_fixture_is_the_scene():
    """the stored scene is what tests/kfc_scene.py builds, so the scene's description holds for the fixture"""
    s, z = ks.packed(*ks.scene()), load()
    for n, a in s.items():
        assert np.array_equal(z[n], a), n


def test_oracle_equals_the_reference():
    s = load()
    r = ko.cull(s)
    assert not r["status"].any()
    assert np.array_equal(r["code"], s["ref_code"])
    assert np.array_equal(r["n_mps"], s["ref_n_mps"])
    assert np.array_equal(r["n_redundant"], s["ref_n_redundant"])
    # the cases the scene is built to reach
    code, nm, nr = s["ref_code"], s["ref_n_mps"], s["ref_n_redundant"]
    assert {-1, 0, 1, 2} <= set(code.tolist())
    assert np.any((nm > 0) & (10 * nr == 9 * nm) & (code == 0))             # exactly 0.9 * nMPs: kept
    assert np.any((nm == 0) & (code == 0))
    assert (s["count"] >= 10).all() and (s["count"] <= 80).all()
    n = s["n"][s["list"]]
    assert n.min() >= 200 and n.max() <= 1500
    obs = np.diff(s["obs_offset"])
    assert obs.min() >= 1 and obs.max() <= 40


@pytest.mark.parametrize("mutant", sorted(ko.MUTANTS))
def test_every_mutant_differs_from_the_reference(mutant):
    s = load()
    r = ko.cull(s, mutant)
    assert (np.any(r["code"] != s["ref_code"]) or np.any(r["n_mps"] != s["ref_n_mps"])
            or np.any(r["n_redundant"] != s["ref_n_redundant"])), ko.MUTANTS[mutant]


def malformed():
    """a small good scene and one copy of it per status code, each broken in one place (status -> packed dict)"""
    b = ks.Builder()
    rows = [b.row() for _ in range(6)]
    for i in range(12):
        p = b.point()
        for r in rows[i % 2:i % 2 + 4]:
            b.slot(r, p, i % 3)
    good = ks.packed(*b.scene([rows[:3], rows[2:5]]))
    out = {}

    def broken(st, **fields):
        s = {n: v.copy() for n, v in good.items()}
        for n, f in fields.items():
            f(s[n])
        out[st] = s

    broken(1, list=lambda a: a.__setitem__(1, 6))
    broken(2, n=lambda a: a.__setitem__(1, good["mp"].shape[1] + 1))
    broken(3, list=lambda a: a.__setitem__(2, a[0]))
    broken(4, mp=lambda a: a.__setitem__((1, 0), len(good["bad"])))
    broken(5, obs_offset=lambda a: a.__setitem__(good["mp"][1, 0] + 1, a[good["mp"][1, 0]] - 1))
    broken(6, obs_idx=lambda a: a.__setitem__(good["obs_offset"][good["mp"][1, 0]], good["mp"].shape[1]))
    return good, out


@pytest.mark.parametrize("st", [1, 2, 3, 4, 5, 6])
def test_oracle_status_codes(st):
    good, bad = malformed()
    assert not ko.cull(good)["status"].any()
    r = ko.cull(bad[st])
    assert r["status"][0] == st
    assert (r["code"][:3] == -7).all()
