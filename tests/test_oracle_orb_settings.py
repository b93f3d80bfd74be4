"""CPU tests: the ORB oracle at extractor settings other than the TUM one (level count, scale factor, FAST thresholds, frame
size) against the reference's own ORBextractor.cc.

(a) committed reference outputs (tests/golden/orb_ref_set_*.npz, tools/gen_golden_orb_ref.py SETTINGS): run everywhere;
(b) where oracle/_ref/libref_orb.so is built, the reference library itself on a second seed: keypoints, descriptors, every
    pyramid level and the constructor tables identical.
"""
import os
import sys
import numpy as np
import pytest
import oracle
from oracle import binding as ob
from plslam_b200 import synth

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from gen_golden_orb_ref import SETTINGS  # noqa: E402

G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("name", sorted(SETTINGS))
def test_oracle_equals_committed_reference_output(name):
    g = np.load(os.path.join(G, f"orb_ref_set_{name}.npz"))
    w, h, seed, nf, nl, ini, mn = [int(v) for v in g["params"]]
    sw, sh, sseed, snf, ssf, snl, sini, smn = SETTINGS[name]     # the fixture is what the table says
    assert (w, h, seed, nf, nl, ini, mn) == (sw, sh, sseed, snf, snl, sini, smn) and g["scale_factor"] == np.float32(ssf)
    img = synth.synth_frame(w, h, seed)
    assert int(img.astype(np.int64).sum()) == int(g["img_sum"])  # the generator is bit-stable
    o = oracle.OrbOracle(nf, float(g["scale_factor"]), nl, ini, mn)
    kps, desc = o.extract(img)
    assert len(kps) == len(g["kps"])
    assert kps.tobytes() == g["kps"].tobytes()
    assert np.array_equal(desc, g["desc"])
    t = o.tables()
    for k in ("scale", "inv_scale", "sigma2", "inv_sigma2"):
        assert t[k].tobytes() == g[k].tobytes(), k
    assert [tuple(d) for d in g["level_dims"]] == [o.level_dims(l) for l in range(nl)]
    assert [int(s) for s in g["level_sums"]] == [int(o.level(l).astype(np.int64).sum()) for l in range(nl)]


@pytest.mark.skipif(not os.path.exists(ob._REF_LIB), reason="oracle/_ref/libref_orb.so not built (needs the reference sources)")
@pytest.mark.parametrize("name", sorted(SETTINGS))
def test_oracle_equals_live_reference(name):
    w, h, seed, nf, sf, nl, ini, mn = SETTINGS[name]
    img = synth.synth_frame(w, h, seed + 100)
    r, o = oracle.RefOrb(nf, sf, nl, ini, mn), oracle.OrbOracle(nf, sf, nl, ini, mn)
    rk, rd = r.extract(img)
    ok, od = o.extract(img)
    for l in range(nl):
        assert r.level_digest(l) == oracle.level_digest_of(o.level(l)), f"pyramid level {l}"
    assert rk.tobytes() == ok.tobytes()
    assert np.array_equal(rd, od)
    rt, ot = r.tables(), o.tables()
    for k in rt:
        assert rt[k].tobytes() == ot[k].tobytes(), k
