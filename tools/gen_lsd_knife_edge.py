"""Generate tests/golden/lsd_cv2_knife_edge.npz: images on which what LSD region growing adds to its float sums decides the segment
list, with cv2's segments for each.

lsd.cpp's region_grow adds  cos(float(angle)), sin(float(angle))  of every pixel it takes to float sums and tests later candidates
against fastAtan2 of those sums.  That line has three plausible arithmetics (oracle/binding.py LSD_ADDENDS): libm's cosf / sinf,
the fp64 functions rounded to fp32, and the fp64 functions added in fp64 to the float sum.  They differ in the last bit of the
addend on about 1.3 % of the gradients, and random images never show it: the difference reaches a segment only when a later
candidate lies within a float ulp of 22.5 degrees from the region angle.  So the images are constructed.

With scale 1.0 cv2's detector grows regions on the image itself: a 2x2 window's gradient is (DA + BC, DA - BC),
DA = I(x+1, y+1) - I(x, y), BC = I(x+1, y) - I(x, y+1).  A 4 x 2 image has exactly three windows, in one row, and its chain of
pixels realises any three gradients gx = gy (mod 2) whose pixel values fit in 0..255:
  - the middle window has the largest gradient g1, so it seeds the only region that matters; the region starts from the fp64
    cos / sin of its angle, the same in every reading;
  - the left window g2 is tested first and is aligned with g1; its addend is one where the readings differ, so the region sum,
    and fastAtan2 of it, differ after it is added;
  - the right window g3 is tested next, against that angle, and its angle lies between the readings' thresholds: aligned in
    one reading and not in the others.
The image's minimum region size is 3, so one reading finds a segment {g2, g1, g3} and the others none.  The search walks the
reachable seeds g1 (defined, gx = gy mod 2) with |g1| <= 160 and every addend-differing g2 aligned with them, and keeps the
triples where cosf is on one side of the threshold and both fp64 readings on the other (it prints how many seeds, pairs and
triples it examined); an image is kept when the oracle's cosf reading gives a segment list different from the two fp64 readings,
which agree, and cv2's segments are stored with it.

Usage: python tools/gen_lsd_knife_edge.py [--want 48]
"""
import argparse
import ctypes as C
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "lsd_cv2_knife_edge.npz")
f32 = np.float32
VARIANTS = ("cosf", "cos_rounded", "cos_double")
D2R = math.pi / 180
PREC = math.pi * 22.5 / 180
RHO2 = 4 * (2.0 / math.sin(PREC)) ** 2


def fast_atan2(y, x):
    """cv::fastAtan2 in degrees, fp32 without contraction (numpy's float32 operations round each step)"""
    y, x = np.asarray(y, f32), np.asarray(x, f32)
    k = f32(180.0 / np.pi)
    p1, p3 = f32(0.9997878412794807) * k, f32(-0.3258083974640975) * k
    p5, p7 = f32(0.1555786518463281) * k, f32(-0.04432655554792128) * k
    eps = f32(2.220446049250313e-16)
    ax, ay = np.abs(x), np.abs(y)
    big = ax >= ay
    with np.errstate(divide="ignore", invalid="ignore"):
        c = np.where(big, ay / (ax + eps), ax / (ay + eps)).astype(f32)
    c2 = c * c
    a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c
    a = np.where(big, a, f32(90) - a)
    a = np.where(x < 0, f32(180) - a, a)
    return np.where(y < 0, f32(360) - a, a).astype(f32)


def aligned(reg, a):
    """LineSegmentDetectorImpl::isAligned of two fp64 angles (radians) at prec = 22.5 degrees"""
    n = np.abs(reg - a)
    n = np.where(n > 1.5 * math.pi, np.abs(n - 2 * math.pi), n)
    return n <= PREC


def gradients(gmax):
    """the defined gradients a 2x2 window can have with |gx|, |gy| <= gmax, their angle (fastAtan2(gx, -gy) degrees, the fp64
    angle) and the three readings of cos / sin of float(angle) (float32; the fp64 reading as float64), and the seed cos / sin"""
    g = np.arange(-gmax, gmax + 1)
    gx, gy = [t.ravel() for t in np.meshgrid(g, g, indexing="ij")]
    ok = ((gx - gy) % 2 == 0) & (gx * gx + gy * gy > RHO2)
    gx, gy = gx[ok], gy[ok]
    deg = fast_atan2(gx.astype(f32), (-gy).astype(f32))
    ang = deg.astype(np.float64) * D2R
    m = C.CDLL("libm.so.6")
    m.cosf.restype = m.sinf.restype = C.c_float
    m.cosf.argtypes = m.sinf.argtypes = [C.c_float]
    af = [float(f32(a)) for a in ang]
    cd = np.array([math.cos(a) for a in af]); sd = np.array([math.sin(a) for a in af])
    return dict(gx=gx, gy=gy, deg=deg, ang=ang, cf=np.array([m.cosf(a) for a in af], f32), sf=np.array([m.sinf(a) for a in af], f32),
                cd=cd, sd=sd, seedc=np.array([math.cos(a) for a in ang], f32), seeds=np.array([math.sin(a) for a in ang], f32))


def region_angles(G, i1, i2):
    """fp64 region angle after the seed i1 and the pixel i2, for each reading"""
    sc, ss = G["seedc"][i1], G["seeds"][i1]
    sums = [(sc + G["cf"][i2], ss + G["sf"][i2]),
            (sc + G["cd"][i2].astype(f32), ss + G["sd"][i2].astype(f32)),
            ((sc.astype(np.float64) + G["cd"][i2]).astype(f32), (ss.astype(np.float64) + G["sd"][i2]).astype(f32))]
    return [fast_atan2(y, x).astype(np.float64) * D2R for x, y in sums]


def image(g2, g1, g3):
    """the 4 x 2 image whose windows have the gradients g2, g1, g3 from left to right, or None if its values do not fit 0..255"""
    r, n = [0], [0]
    for gx, gy in (g2, g1, g3):
        da, bc = (gx + gy) // 2, (gx - gy) // 2
        n.append(r[-1] + da)           # DA = n[k+1] - r[k]
        r.append(n[-2] + bc)           # BC = r[k+1] - n[k]
    img = np.array([r, n])
    img -= img.min()
    return img.astype(np.uint8) if img.max() <= 255 else None


def search(want, gseed=160, gmax=160):
    G = gradients(gmax)
    norm2 = G["gx"] ** 2 + G["gy"] ** 2
    differ = np.flatnonzero((G["cf"] != G["cd"].astype(f32)) | (G["sf"] != G["sd"].astype(f32)))
    order = np.argsort(G["ang"])
    sorted_ang = G["ang"][order]
    found, stats = [], dict(seeds=0, pairs=0, split=0, triples=0)
    for i1 in np.flatnonzero((np.abs(G["gx"]) <= gseed) & (np.abs(G["gy"]) <= gseed)):
        stats["seeds"] += 1
        # pixel 2: an addend-differing gradient aligned with the seed, below it in the seed order (norm well under the seed's)
        i2 = differ[aligned(G["ang"][i1], G["ang"][differ]) & (norm2[differ] * 1.25 < norm2[i1])]
        if not len(i2):
            continue
        stats["pairs"] += len(i2)
        rf, rr, rd = region_angles(G, np.full(len(i2), i1), i2)
        split = (rf != rr) & (rf != rd)
        stats["split"] += int(split.sum())
        for k in np.flatnonzero(split):
            # pixel 3: angles within 1e-6 rad of a threshold 22.5 degrees from the region angle
            for side in (-PREC, PREC):
                t = (rf[k] + side) % (2 * math.pi)
                lo, hi = np.searchsorted(sorted_ang, [t - 1e-6, t + 1e-6])
                for i3 in order[lo:hi]:
                    if norm2[i3] * 1.25 >= norm2[i1]:
                        continue
                    a3 = G["ang"][i3]
                    af, ar, ad = aligned(rf[k], a3), aligned(rr[k], a3), aligned(rd[k], a3)
                    if af == ar or ar != ad:
                        continue
                    img = image(*[(int(G["gx"][j]), int(G["gy"][j])) for j in (i2[k], i1, i3)])
                    if img is None:
                        continue
                    stats["triples"] += 1
                    found.append(img)
                    if len(found) >= want:
                        return found, stats
    return found, stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--want", type=int, default=48)
    args = ap.parse_args()
    import cv2
    from oracle import binding as ob
    cands, stats = search(8 * args.want)
    imgs = []
    for img in cands[::max(1, len(cands) // (2 * args.want))]:     # spread over the seeds the search walked
        outs = [ob.lsd_detect_scale1(img, v) for v in VARIANTS]
        if not np.array_equal(outs[0], outs[1]) and not np.array_equal(outs[0], outs[2]) and np.array_equal(outs[1], outs[2]):
            imgs.append(img)
        if len(imgs) >= args.want:
            break
    print(f"search: {stats}; {len(imgs)} images on which cosf alone gives a different segment list")
    if not imgs:
        sys.exit(1)
    lsd = cv2.createLineSegmentDetector(cv2.LSD_REFINE_STD, 1.0)
    segs = []
    for im in imgs:
        s = lsd.detect(im)[0]
        segs.append(np.zeros((0, 4), f32) if s is None else s.reshape(-1, 4).astype(f32))
    np.savez_compressed(OUT, imgs=np.stack(imgs), nseg=np.array([len(s) for s in segs], np.int32),
                        segs=np.concatenate(segs).astype(f32), cv2_version=np.array(cv2.__version__))
    print("wrote", OUT)


if __name__ == "__main__":
    main()
