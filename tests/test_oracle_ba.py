"""CPU suite: known-answer scenes for the BA / pose-only restatements (g2o and Ceres are unpinned third-party
code: the pin is the ground truth of the reference's own synthetic fixture, test/test_local_ba.cpp:9-98)."""
import numpy as np

from ygz_slam_b200 import se3, synth


def _g2o(v):  # [upsilon; omega] -> vertex order [omega; upsilon]
    v = np.asarray(v)
    return np.concatenate([v[..., 3:], v[..., :3]], -1)


def test_local_ba_fixture_scene(oracle):
    """8 poses x 16 points of test_local_ba.cpp with its noise recipe (pose 0.1, point 0.1, pixel 1)."""
    rot = [(0, 0, 0), (0.1, 0, 0), (0, 0.1, 0), (0, 0, 0.1), (0, 0, 0), (0, 0, 0), (0, 0, 0), (0, 0, 0)]
    tr = [(0, 0, 0)] * 4 + [(0.1, 0, 0), (0, 0.1, 0), (0, 0, 0.1), (0.1, 0.1, 0.1)]
    poses_true = [se3.se3_exp(np.r_[t, w]) for w, t in zip(rot, tr)]
    pts_true = np.array([[x, y, z] for z in (2, 3, 4, 5) for (x, y) in ((0, 0), (0, 1), (1, 0), (1, 1))], float)
    rng = np.random.default_rng(11)
    logs = np.array([se3.se3_log(T) for T in poses_true])
    noisy = logs.copy()
    noisy[1:] += rng.normal(0, 0.1, (7, 6))
    pts = pts_true + rng.normal(0, 0.1, pts_true.shape)
    kf, pt, px = [], [], []
    for j in range(16):
        for k in range(8):
            pc = poses_true[k][:, :3] @ pts_true[j] + poses_true[k][:, 3]
            kf.append(k)
            pt.append(j)
            px.append([520.9 * pc[0] / pc[2] + 325.1 + rng.normal(0, 1), 521.0 * pc[1] / pc[2] + 249.7 + rng.normal(0, 1)])
    fixed = np.zeros(8, np.uint8)
    fixed[0] = 1
    P, X, outl, st = oracle.local_ba(_g2o(noisy), fixed, pts, kf, pt, px)
    assert st["chi2_final"] < 1e-2 * st["chi2_initial"]
    assert st["chi2_final"] < 2.5 * len(kf)            # ~ pixel noise level (sigma = 1 px, 2 residuals per edge)
    assert np.allclose(P[0], _g2o(noisy)[0])            # keyframe 0 is fixed
    # rotations are observable (scale is not: monocular gauge): they must come back to the truth
    assert np.abs(P[:, :3] - logs[:, 3:]).max() < 0.03
    assert outl.sum() <= 0.1 * len(kf)


def test_local_ba_c4_scene(oracle):
    sc = synth.ba_scene()
    fixed = np.zeros(10, np.uint8)
    fixed[0] = 1
    P, X, outl, st = oracle.local_ba(_g2o(sc["poses_noisy"]), fixed, sc["pts_noisy"], sc["kf_idx"], sc["pt_idx"], sc["px"])
    assert 7000 < len(sc["kf_idx"]) <= 8000
    assert st["chi2_final"] < 2e-3 * st["chi2_initial"]
    est = np.concatenate([P[:, 3:], P[:, :3]], 1)
    assert np.abs(est - sc["poses_true"]).max() < 0.01
    assert np.median(np.abs(X - sc["pts_true"])) < 0.05
    # no robust kernel (the Ceres-flavoured LocalBA has no loss): still converges on outlier-free data
    P2, X2, _, st2 = oracle.local_ba(_g2o(sc["poses_noisy"]), fixed, sc["pts_noisy"], sc["kf_idx"], sc["pt_idx"], sc["px"], huber=0.0)
    assert st2["chi2_final"] < 2e-3 * st2["chi2_initial"]


def test_pose_only_rejects_outliers(oracle):
    sc = synth.ba_scene()
    rng = np.random.default_rng(5)
    sel = sc["kf_idx"] == 3
    pw = sc["pts_true"][sc["pt_idx"][sel]]
    px = sc["px"][sel].copy()
    px[::10] += 30
    T0 = se3.se3_exp(sc["poses_true"][3])
    Tn = se3.se3_exp(sc["poses_true"][3] + rng.normal(0, 0.002, 6))
    T, inl, depth, cnt = oracle.pose_only(pw, px, Tn)
    # the classification of round r uses the pose of round r-1 (BA.cpp:231-251), so the outlier-biased pose of
    # round 0 makes later rounds reject many good points: well below the ~85 % a fresh pose would keep
    assert cnt == inl.sum() and 0.3 * len(pw) < cnt < 0.95 * len(pw)
    assert not inl[::10].any()                          # the +30 px observations are classified as outliers
    _, inl_clean, _, cnt_clean = oracle.pose_only(pw, sc["px"][sel], Tn)
    assert cnt_clean > 0.9 * len(pw)
    err0 = np.linalg.norm(se3.se3_log(se3.mul(Tn, se3.inv(T0))))
    err1 = np.linalg.norm(se3.se3_log(se3.mul(T, se3.inv(T0))))
    assert err1 < err0 and err1 < 2e-3
    assert np.all(depth[inl] > 0)
    # fewer than 10 inliers: the loop breaks and the pose is left at the input (BA.cpp:248-249)
    T2, inl2, _, cnt2 = oracle.pose_only(pw[:8], px[:8] + 100, Tn)
    assert cnt2 == 0 and np.allclose(T2, Tn, atol=1e-12)


def _t_aa(v):  # [upsilon; omega] (se3 log) -> [t; angle-axis] of the same transform (CeresReprojectionError's pose)
    out = []
    for x in np.atleast_2d(v):
        T = se3.se3_exp(x)
        out.append(np.r_[T[:, 3], se3.so3_log(T[:, :3])])
    return np.array(out)


def test_local_ba_ceres_twin_c4_scene(oracle):
    """ba::LocalBA (Ceres flavour, BA.cpp:324-384): normalised residuals, no loss, [t; angle-axis] poses."""
    sc = synth.ba_scene()
    fixed = np.zeros(10, np.uint8)
    fixed[0] = 1
    P0 = _t_aa(sc["poses_noisy"])
    P, X, st = oracle.local_ba_ceres(P0, fixed, sc["pts_noisy"], sc["kf_idx"], sc["pt_idx"], sc["px"])
    assert st["cost_final"] < 2e-3 * st["cost_initial"]
    assert st["termination"] in (1, 2, 3) and 3 <= st["iters"] <= 50
    assert np.allclose(P[0], P0[0])                                      # the first key-frame only has point-only blocks
    assert np.abs(P - _t_aa(sc["poses_true"])).max() < 0.01
    assert np.median(np.abs(X - sc["pts_true"])) < 0.05
    # same minimum as the g2o flavour without its robust kernel (both are exact Gauss-Newton-type solvers of the same
    # least-squares problem up to the residual scaling 1/f): compare the optimised poses as transforms
    Pg, Xg, _, _ = oracle.local_ba(_g2o(sc["poses_noisy"]), fixed, sc["pts_noisy"], sc["kf_idx"], sc["pt_idx"], sc["px"], huber=0.0,
                                   max_iters=50)
    est_g = _t_aa(np.concatenate([Pg[:, 3:], Pg[:, :3]], 1))
    assert np.abs(P - est_g).max() < 2e-3


def test_two_view_ba(oracle):
    """ba::TwoViewBACeres restatement (BA.cpp:11-89): the current pose comes back to the truth (up to the monocular scale,
    which the fixed reference frame does not pin: rotations are compared), the flagged points are re-triangulated from
    (0,0,1) and end up inliers, every point passes the reference's 5.991 px^2 test."""
    sc = synth.two_view_scene()
    T, inl, X, st, cnt = oracle.two_view_ba(sc["T_ref"], sc["T_cur0"], sc["px_ref"], sc["px_cur"], sc["inlier"], sc["X0"])
    assert st["cost_final"] < 0.05 * st["cost_initial"] and st["termination"] in (1, 2, 3)
    assert np.abs(T[:, :3] - sc["T_cur"][:, :3]).max() < 2e-3
    dirn = lambda t: t / np.linalg.norm(t)
    assert np.abs(dirn(T[:, 3]) - dirn(sc["T_cur"][:, 3])).max() < 0.05         # translation direction (scale is gauge)
    assert cnt == inl.sum() and cnt >= len(inl) - 2
    assert inl[sc["inlier"] == 0].sum() >= (sc["inlier"] == 0).sum() - 2        # the restarted points were recovered


def test_local_ba_large_and_sixteen_free_scenes(oracle):
    """The scenes of the GPU suite's staging tests: 10 key-frames x 5,000 landmarks x 20,000 observations, and 17 key-frames
    (16 free) at 150 and 2,000 landmarks.  The oracle must reach the synthetic truth on each, so that the GPU tests compare
    against a validated specification."""
    for n_kf, n_pt, per_pt in ((10, 5000, 4), (17, 150, 8), (17, 2000, 4)):
        sc = synth.ba_scene(n_kf=n_kf, n_pt=n_pt, target_obs=per_pt * n_pt, seed=31 if n_kf == 10 else 40)
        fixed = np.zeros(n_kf, np.uint8)
        fixed[0] = 1
        P, X, outl, st = oracle.local_ba(_g2o(sc["poses_noisy"]), fixed, sc["pts_noisy"], sc["kf_idx"], sc["pt_idx"], sc["px"])
        assert st["chi2_final"] < 2e-3 * st["chi2_initial"], (n_kf, n_pt)
        est = np.concatenate([P[:, 3:], P[:, :3]], 1)
        assert np.abs(est - sc["poses_true"]).max() < 0.01, (n_kf, n_pt)
        assert np.median(np.abs(X - sc["pts_true"])) < 0.05, (n_kf, n_pt)
        assert outl.mean() < 0.05             # ~ the share of 1 px Gaussian residuals above chi2 = 5.991


def test_local_ba_structural_edge_cases(oracle):
    """Landmarks seen only by fixed key-frames, landmarks with one observation, a problem without observations: the oracle
    returns finite results, the constrained part converges to the truth, and an unobserved problem is left as it was."""
    sc = synth.ba_edge_scene()
    fixed = np.zeros(6, np.uint8)
    fixed[:2] = 1
    P, X, outl, st = oracle.local_ba(_g2o(sc["poses_noisy"]), fixed, sc["pts_noisy"], sc["kf_idx"], sc["pt_idx"], sc["px"])
    assert np.isfinite(P).all() and np.isfinite(X).all() and np.isfinite(st["chi2_final"])
    est = np.concatenate([P[:, 3:], P[:, :3]], 1)
    assert np.abs(est - sc["poses_true"]).max() < 0.01
    assert np.median(np.abs(X[:340] - sc["pts_true"][:340])) < 0.05    # every landmark with two or more observations
    e = synth.ba_scene(n_kf=3, n_pt=20, seed=42)
    f3 = np.array([1, 0, 0], np.uint8)
    none = np.zeros(0, np.int32)
    P0, X0, _, st0 = oracle.local_ba(_g2o(e["poses_noisy"]), f3, e["pts_noisy"], none, none, np.zeros((0, 2)))
    assert np.array_equal(P0, _g2o(e["poses_noisy"])) and np.array_equal(X0, e["pts_noisy"]) and st0["chi2_final"] == 0


def test_pose_only_large_frames(oracle):
    """Frames of 40,000 and 45,000 points (the GPU suite's staged and unstaged pose-only paths) with every tenth point
    moved 30 px: the oracle rejects those and comes back to the true pose."""
    for n in (40000, 45000):
        sc = synth.pose_only_scene(n, seed=n)
        px = sc["px"].copy()
        px[::10] += 30
        T, inl, depth, cnt = oracle.pose_only(sc["pw"], px, sc["T0"])
        # (as in test_pose_only_rejects_outliers, the outlier-biased pose of round 0 costs later rounds many good points)
        assert not inl[::10].any() and cnt == inl.sum() and 0.3 * n < cnt < 0.95 * n
        assert np.linalg.norm(se3.se3_log(se3.mul(T, se3.inv(sc["T_true"])))) < 2e-3
        assert np.all(depth[inl] > 0)
