"""An INDEPENDENT check of the bundle-adjustment oracle (Optimizer.cc's g2o path cannot be pinned to compiled reference code):
with the robust kernel off, Optimizer::BundleAdjustment is plain Levenberg-Marquardt on
   sum_pe w |obs - proj_K(T_kf X)|^2 + sum_le (l . proj_h(T_kf S))^2 + (l . proj_h(T_kf E))^2     (Optimizer.cc:275-638)
over the free keyframes, the points and the line end points.  scipy.optimize.least_squares (trust-region reflective, rotation-vector
parametrisation, finite-difference Jacobian - none of the oracle's code) must reach the same minimum on a small noisy window."""
import numpy as np
import pytest
import oracle
from plslam_b200 import synth

scipy_opt = pytest.importorskip("scipy.optimize")
from scipy.spatial.transform import Rotation  # noqa: E402
from test_optimizer_edges_gpu import keyframe_cameras  # noqa: E402


def _unpack(x, p, free):
    T = p["kf_Tcw"].reshape(-1, 4, 4).astype(np.float64).copy()
    for j, k in enumerate(free):
        T[k, :3, :3] = Rotation.from_rotvec(x[6 * j:6 * j + 3]).as_matrix() @ T[k, :3, :3]
        T[k, :3, 3] = T[k, :3, 3] + x[6 * j + 3:6 * j + 6]
    o = 6 * len(free)
    X = p["pt_Xw"].astype(np.float64) + x[o:o + 3 * len(p["pt_Xw"])].reshape(-1, 3)
    o += 3 * len(p["pt_Xw"])
    L = p["ln_Xw"].astype(np.float64) + x[o:].reshape(-1, 6)
    return T, X, L


def _residuals(x, p, free, K_end=None):
    """Point and line-end-point residuals, each projected with the observing keyframe's K; with K_end given, the END points
    are projected with K_end instead (the local BA's model, Optimizer.cc:1939-1942)."""
    T, X, L = _unpack(x, p, free)
    K = p["kf_K"].astype(np.float64)

    def proj(kf, P, Kp):
        Pc = np.einsum("nij,nj->ni", T[kf, :3, :3], P) + T[kf, :3, 3]
        return np.stack([Pc[:, 0] / Pc[:, 2] * Kp[:, 0] + Kp[:, 2], Pc[:, 1] / Pc[:, 2] * Kp[:, 1] + Kp[:, 3]], 1)
    kf, pt = p["pe_kf"], p["pe_pt"]
    r = [(np.sqrt(p["pe_inv_sigma2"].astype(np.float64))[:, None] * (p["pe_obs"].astype(np.float64) - proj(kf, X[pt], K[kf]))).ravel()]
    lk, ll, lf = p["le_kf"], p["le_ln"], p["le_func"]
    K_ends = K[lk] if K_end is None else np.broadcast_to(np.asarray(K_end, np.float64), (len(lk), 4))
    for e, Ke in ((L[ll, :3], K[lk]), (L[ll, 3:], K_ends)):
        uv = proj(lk, e, Ke)
        r.append(lf[:, 0] * uv[:, 0] + lf[:, 1] * uv[:, 1] + lf[:, 2])
    return np.concatenate(r)


def _as_x(g, p, free):
    """The oracle's estimate g in the parametrisation of _unpack (increments from p's start)."""
    n_pt = len(p["pt_Xw"])
    To = g["kf_Tcw"].reshape(-1, 4, 4).astype(np.float64); T0 = p["kf_Tcw"].reshape(-1, 4, 4).astype(np.float64)
    x = np.zeros(6 * len(free) + 3 * n_pt + 6 * len(p["ln_Xw"]))
    for j, k in enumerate(free):
        x[6 * j:6 * j + 3] = Rotation.from_matrix(To[k, :3, :3] @ T0[k, :3, :3].T).as_rotvec()
        x[6 * j + 3:6 * j + 6] = To[k, :3, 3] - T0[k, :3, 3]
    o = 6 * len(free)
    x[o:o + 3 * n_pt] = (g["pt_Xw"][:n_pt].astype(np.float64) - p["pt_Xw"].astype(np.float64)).ravel()
    x[o + 3 * n_pt:] = (g["ln_Xw"][:len(p["ln_Xw"])] - p["ln_Xw"]).ravel()
    return x


def _check_global_minimum(p):
    free = [k for k in range(len(p["kf_fixed"])) if not p["kf_fixed"][k]]
    g = oracle.global_ba(p, n_iterations=80, robust=False)
    n = 6 * len(free) + 3 * len(p["pt_Xw"]) + 6 * len(p["ln_Xw"])
    c0 = (_residuals(np.zeros(n), p, free) ** 2).sum()
    sol = scipy_opt.least_squares(_residuals, np.zeros(n), args=(p, free), method="trf", xtol=1e-13, ftol=1e-13, gtol=1e-13, max_nfev=200)
    cs = (sol.fun ** 2).sum()
    co = (_residuals(_as_x(g, p, free), p, free) ** 2).sum()
    assert cs < 0.5 * c0                                   # the start is well away from the minimum
    # g2o's LM stops on the reference's rule - three iterations in a row that improve chi2 by less than 0.1 % (the oracle restates it) -
    # so it ends within a few 1e-4 (relative) of the minimum, never below it; outputs are fp32
    assert cs * (1 - 1e-6) <= co <= cs * (1 + 2e-3), (c0, co, cs)
    Ts, _, _ = _unpack(sol.x, p, free)
    To = g["kf_Tcw"].reshape(-1, 4, 4).astype(np.float64)
    for k in free:
        assert np.abs(Ts[k, :3, :3] - To[k, :3, :3]).max() < 1e-3 and np.linalg.norm(Ts[k, :3, 3] - To[k, :3, 3]) < 1e-2


@pytest.mark.parametrize("seed", [4, 9])
def test_global_ba_reaches_the_least_squares_minimum(seed):
    _check_global_minimum(synth.synth_ba_problem(seed, n_free=4, n_fixed=3, n_pt=120, n_ln=20, outlier_frac=0.0, noise_px=0.5))


def test_global_ba_with_per_keyframe_cameras_reaches_the_least_squares_minimum():
    """Every edge, line end points included, is projected with its observing keyframe's own K (Optimizer.cc:472-475,526-529)."""
    p = synth.synth_ba_problem(9, n_free=4, n_fixed=3, n_pt=120, n_ln=20, outlier_frac=0.0, noise_px=0.5, Ks=keyframe_cameras(7, 19, focal=0.004, centre=1.0))
    assert len(np.unique(p["kf_K"], axis=0)) == 7
    _check_global_minimum(p)


def _check_local_minimum(p):
    free = [k for k in range(len(p["kf_fixed"])) if not p["kf_fixed"][k]]
    g = oracle.local_ba(p)
    assert not g["pe_erase"].any() and not g["le_erase"].any()       # no outlier: the second optimize runs on every edge
    n = 6 * len(free) + 3 * len(p["pt_Xw"]) + 6 * len(p["ln_Xw"])
    n_pr = 2 * len(p["pe_kf"])

    def res(x):
        r = _residuals(x, p, free, K_end=p["K_end"])
        r[n_pr:] *= np.sqrt(0.5)
        return r
    sol = scipy_opt.least_squares(res, np.zeros(n), method="trf", xtol=1e-13, ftol=1e-13, gtol=1e-13, max_nfev=200)
    cs = (sol.fun ** 2).sum()
    co = (res(_as_x(g, p, free)) ** 2).sum()
    c0 = (res(np.zeros(n)) ** 2).sum()
    assert cs < 0.1 * c0
    # 5 + 10 iterations under the reference's stop rule: 99.9 % of the way from the start to the minimum, never below it
    assert cs * (1 - 1e-6) <= co <= cs * (1 + 2e-2), (c0, co, cs)
    assert (co - cs) < 1e-3 * (c0 - cs)


def test_local_ba_ends_at_the_least_squares_minimum_of_its_inliers():
    """Optimizer::LocalBundleAdjustmentWithLine (Optimizer.cc:1645-2100): 5 robust iterations, the chi2 classification, then 10 plain
    iterations on the inliers.  Without outliers the result is (within the stop rule) the minimiser of the same sum with the line terms
    weighted 0.5 (Optimizer.cc:1893); points and line start points are projected with the observing keyframe's K, line END points
    with the CURRENT keyframe's (K_end, the reference's quirk, Optimizer.cc:1939-1942)."""
    _check_local_minimum(synth.synth_ba_problem(6, n_free=4, n_fixed=3, n_pt=120, n_ln=20, outlier_frac=0.0, noise_px=0.5))


def test_local_ba_with_per_keyframe_cameras_ends_at_the_least_squares_minimum():
    """The same with a camera per keyframe and a current-keyframe camera K_end of its own: the sum only has its minimum where the
    oracle ends if each edge uses the camera the reference gives it.  The offsets are small enough that no edge is gated."""
    Ks = keyframe_cameras(7, 16, focal=0.004, centre=1.0)
    p = synth.synth_ba_problem(6, n_free=4, n_fixed=3, n_pt=120, n_ln=20, outlier_frac=0.0, noise_px=0.5, Ks=Ks,
                               K_end=np.array(synth.TUM1_K) * 1.002)
    assert len(np.unique(p["kf_K"], axis=0)) == 7 and not (p["kf_K"] == p["K_end"]).all(axis=1).any()
    _check_local_minimum(p)
