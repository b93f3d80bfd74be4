"""Camera handling of the optimisers' test inputs, without a GPU.

- synth.synth_ba_problem's per-keyframe cameras (Ks, K_end) are opt-in: its default output is pinned byte for byte, and with Ks
  keyframe k's observations are made with Ks[k].
- The GPU comparisons' exact parts (masks, inlier and iteration counts) rest on inputs that keep clear of rounding-level
  decisions: every pose problem's outcome is the same under the oracle's rounding variants, and no edge of a local-BA window
  sits near its chi2 gate.
- Mutant separation: for every camera case of test_optimizer_edges_gpu.py, the oracle run on a copy of the problem with a
  plausible WRONG camera (every K = problem / keyframe 0's, K_end replaced by the observing keyframe's K, start points given
  K_end) ends over 100 x the GPU comparison's translation tolerance away from the oracle's true answer.  So a kernel that used
  such a camera would fail the GPU comparison instead of passing it by accident."""
import hashlib
import numpy as np
import pytest
import oracle
from plslam_b200 import synth
from test_optimizer_edges_gpu import (pose_batch, pose_args, frontend_problems, lba_camera_window, lba_lines_only_window,
                                      gba_camera_map, lba_32_free_window, lba_mirrored_point_window, lba_outlier_keyframe_window,
                                      pose_outcome_is_rounding_stable, POSE_SEEDS)

GPU_REL_TOL = 1e-4        # translations, relative to the largest (test_lm_gpu.py, test_ba_gpu.py)

# SHA-256 of every array of synth_ba_problem(4) and synth_ba_problem(9, n_free=4, n_fixed=3, n_pt=120, n_ln=20, outlier_frac=0.0,
# noise_px=0.5), computed before the per-keyframe camera keywords existed
SYNTH_BA_DIGESTS = {
    4: {"K_end": "7cf2dc968eeb147a7aa2cbf31ee1f8880537c4b446e0758300c261f96fd0f118",
        "kf_K": "ef449fb18c3ef6dc9ca4ae9544f306a4ed1b89010f8945fe2a2caa668801550c",
        "kf_Tcw": "440ffdb1ffd78d28feada47e057e57523d369d6f5945314c602795a0489c8204",
        "kf_Tcw_true": "de91cea8d49e715d110a2506271cf9f852fb749bb5f7bfaa38b669ab6156f495",
        "kf_fixed": "13a1b1161c71f0262d5ce1f1e2da688d5f3b3d9f80390054f153ad6597113a2c",
        "le_func": "45f044976d5991a3abc9616ea14d3ceb3d9e91a70011871c3e663463a861ef13",
        "le_kf": "03b5490559aa0cf6eaf0bcbb79129709dd1ef4ab281a14d25691b5a4087d39b5",
        "le_ln": "bccfec42da97a263d72afdd0058fb5f8b61d4e91101293dddbc95e863e11d79f",
        "ln_Xw": "0dd0c8722afe4c25780210f057cb11bfb062fd2974ae6bc2b1b370baf348a2df",
        "ln_Xw_true": "87e45813885c95e05368c39745f91ad1f7434f331eb91e68a331c8dbc1fac09f",
        "pe_inv_sigma2": "4aeaf27e1f333e6138492d3efdd3579ce94e1ddb1821c3eec8d93da9b8ab28dc",
        "pe_kf": "b243580a387264110dfcd03b536a244d9b7015e4c491d01627080bf8c13e54ac",
        "pe_obs": "7895e717301cdd71772a45d2657ff943648beaaefda8d507f87ebece52cb76a4",
        "pe_pt": "865c2256411fc308269404bd115e2b2b1918ae9154ea70a6b77347ddd4f16ced",
        "pt_Xw": "a6fa4451a8292a03a4e39a68bb7bea66a15377fc83793419cf81da5446648f58",
        "pt_Xw_true": "3eb8bfe0c7c5239030fd80293b51a4b78a7e7b8bcc36d2b17ea73d58ec026d97"},
    9: {"K_end": "7cf2dc968eeb147a7aa2cbf31ee1f8880537c4b446e0758300c261f96fd0f118",
        "kf_K": "c912abeaa5ff1c26d34d566238dc765a454a26313d2a23354c3bc1953c2d273c",
        "kf_Tcw": "bcc57bd81978b2b8cd20ad0bdfcbf4a780337f8ab93d8c6b4ca8a843dc6cc4ec",
        "kf_Tcw_true": "7c4523b1d73e19f4d4d7632e6331516fbb20cf6c5f181285feadcc0e65fc9182",
        "kf_fixed": "5556f5334ec6ddf7f4e37449642147c0de73d8bf7642a4fa04e7c445939c68a3",
        "le_func": "90ac63b8948693cc88c756e696d8e397fc2935394c67ec12b5ea719bdc439751",
        "le_kf": "9e8dc7233865140ccdd277cb79df1921ef8a5644599beebd050ada425228517c",
        "le_ln": "59ce1f0bc3cee7e10f683d7a840da0a24f9f9a681ae05a823ba286347a6d9da7",
        "ln_Xw": "06f7b44fa701bc3c995ea67a7af9da6dacf726b634564ea731ee0c374cf13082",
        "ln_Xw_true": "e89309c77f4d6a847131a485b4906fbe073fb28a304009183465fdaf7a7cdfaa",
        "pe_inv_sigma2": "bb1b9e0613e3d8df4a2a6c954ffc8480d89ca896e2c30c1f34dab03370c3a28d",
        "pe_kf": "dc66ca7efe282f0595a15f10ae33e82fecf7b9b735805b2387959b508e809c2d",
        "pe_obs": "5918877283b6e3328f877774d8b211fd498c86f2262d2f60fe204d553259a58d",
        "pe_pt": "a86967df750c415aa1c37030edd30a563bc53b62205224b95ba71fb2a4b17d86",
        "pt_Xw": "37757d9b8068de39e988f7b123ddad61e88cdb96539beb0b1e47e0d5ca7047d9",
        "pt_Xw_true": "0951fe53ccfb16a08e1f016f1d016ec4347162c4619847ea9e3ce648490c910d"},
}


@pytest.mark.parametrize("seed", [4, 9])
def test_synth_ba_problem_defaults_are_unchanged(seed):
    kw = {} if seed == 4 else dict(n_free=4, n_fixed=3, n_pt=120, n_ln=20, outlier_frac=0.0, noise_px=0.5)
    p = synth.synth_ba_problem(seed, **kw)
    assert sorted(p) == sorted(SYNTH_BA_DIGESTS[seed])
    for k, want in SYNTH_BA_DIGESTS[seed].items():
        assert hashlib.sha256(np.ascontiguousarray(p[k]).tobytes()).hexdigest() == want, k


def test_synth_ba_problem_observes_with_each_keyframes_camera():
    n_kf = 7
    Ks = np.tile(np.float32(synth.TUM1_K), (n_kf, 1)) * np.linspace(0.9, 1.1, n_kf, dtype=np.float32)[:, None]
    K_end = np.array(synth.EUROC_K)
    p = synth.synth_ba_problem(3, n_free=4, n_fixed=3, n_pt=200, n_ln=40, noise_px=0.0, outlier_frac=0.0, Ks=Ks, K_end=K_end)
    assert np.array_equal(p["kf_K"], Ks) and np.array_equal(p["K_end"], np.float32(K_end))
    T, K = p["kf_Tcw_true"], p["kf_K"].astype(np.float64)

    def proj(kf, X):
        c = np.einsum("nij,nj->ni", T[kf, :3, :3], X) + T[kf, :3, 3]
        return np.stack([c[:, 0] / c[:, 2] * K[kf, 0] + K[kf, 2], c[:, 1] / c[:, 2] * K[kf, 1] + K[kf, 3]], 1)
    assert np.abs(p["pe_obs"] - proj(p["pe_kf"], p["pt_Xw_true"][p["pe_pt"]])).max() < 1e-3          # float32 storage only
    for e in (p["ln_Xw_true"][p["le_ln"], :3], p["ln_Xw_true"][p["le_ln"], 3:]):
        uv = proj(p["le_kf"], e)
        assert np.abs(p["le_func"][:, 0] * uv[:, 0] + p["le_func"][:, 1] * uv[:, 1] + p["le_func"][:, 2]).max() < 1e-6
    assert len(np.unique(p["pe_kf"])) == n_kf and len(np.unique(p["le_kf"])) == n_kf


def _t_gap(T, To):
    """max translation difference over poses, in units of the GPU tolerance (GPU_REL_TOL x the largest oracle translation)."""
    t, to = np.asarray(T, np.float64).reshape(-1, 4, 4)[:, :3, 3], np.asarray(To, np.float64).reshape(-1, 4, 4)[:, :3, 3]
    return np.linalg.norm(t - to, axis=1).max() / (GPU_REL_TOL * np.linalg.norm(to, axis=1).max())


@pytest.mark.parametrize("problems", ["batch", "frontend"])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_pose_optimization_with_problem_0s_camera_is_told_apart(problems, mode):
    probs = pose_batch() if problems == "batch" else frontend_problems()
    K0 = probs[0]["K"]
    told = 0
    for b, p in enumerate(probs):
        if np.array_equal(p["K"], K0):
            continue
        on, oT, _, _, oits = oracle.pose_optimization(mode, *pose_args(p))
        if oits == 0:                      # too few correspondences: untouched under any camera
            continue
        _, wT, *_ = oracle.pose_optimization(mode, *pose_args(p, K0))
        assert _t_gap(wT, oT) > 100, b
        told += 1
    assert told >= (3 if problems == "frontend" else 10 if mode == 2 else 13)


@pytest.mark.parametrize("window", ["cameras", "lines_only"])
def test_local_ba_wrong_cameras_are_told_apart(window):
    p = lba_camera_window() if window == "cameras" else lba_lines_only_window()
    o = oracle.local_ba(p)
    k0 = dict(p); k0["kf_K"] = np.tile(p["kf_K"][0], (len(p["kf_K"]), 1))
    for name, w in (("keyframe 0's K", oracle.local_ba(k0)), ("end points with the observing K", oracle.local_ba(p, line_cameras="end_observing_K")),
                    ("start points with K_end", oracle.local_ba(p, line_cameras="start_K_end"))):
        assert _t_gap(w["kf_Tcw"], o["kf_Tcw"]) > 100, name


def test_global_ba_with_keyframe_0s_camera_is_told_apart():
    p = gba_camera_map()
    o = oracle.global_ba(p, 6, True)
    w = dict(p); w["kf_K"] = np.tile(p["kf_K"][0], (len(p["kf_K"]), 1))
    assert _t_gap(oracle.global_ba(w, 6, True)["kf_Tcw"], o["kf_Tcw"]) > 100


def test_pose_problems_do_not_hang_on_rounding():
    """The batched pose test compares inlier and iteration counts and masks exactly; the front-end test compares inlier counts."""
    probs = pose_batch()
    assert [b for b, p in enumerate(probs) if not pose_outcome_is_rounding_stable(p)] == []
    assert all(pose_outcome_is_rounding_stable(p, modes=(0,), iterations=False) for p in frontend_problems())
    # each seed is the first candidate 200 + b + 1000 j that passes, so the list can be re-derived when a size changes
    from test_optimizer_edges_gpu import POSE_NP, POSE_NL, CAMERAS
    for b, sd in enumerate(POSE_SEEDS):
        assert (sd - 200 - b) % 1000 == 0
        for earlier in range(200 + b, sd, 1000):
            q = synth.synth_pose_problem(earlier, n_points=POSE_NP[b], n_lines=POSE_NL[b], K=tuple(CAMERAS[b % 4]))
            assert not pose_outcome_is_rounding_stable(q), (b, earlier)


@pytest.mark.parametrize("window", ["cameras", "lines_only", "32_free", "mirrored_point", "outlier_keyframe"])
def test_local_ba_windows_keep_clear_of_the_chi2_gates(window):
    """k_local_ba sums the reduced system with fp64 atomics, so its chi2 values differ from the oracle's in the last bits: its
    erase masks can only be compared exactly if no edge is within rounding distance of 5.991 / 3.84."""
    p = {"cameras": lba_camera_window, "lines_only": lba_lines_only_window, "32_free": lba_32_free_window,
         "mirrored_point": lambda: lba_mirrored_point_window()[0], "outlier_keyframe": lambda: lba_outlier_keyframe_window()[0]}[window]()
    assert oracle.local_ba(p)["gate_gap"] > 1e-5
