"""CPU suite: known-answer checks of the alignment / Lie-group restatements (no GPU)."""
import numpy as np

from ygz_slam_b200 import se3, synth


def _scene(oracle, k0=1, k1=4):
    g1, d1, T1 = synth.stream_frame(k0)
    g2, _, T2 = synth.stream_frame(k1)
    p1, p2 = oracle.build_pyramid(g1, 3), oracle.build_pyramid(g2, 3)
    f = oracle.detect(p1)
    px = np.stack([f["px"], f["py"]], 1)
    depth = d1[f["py"].astype(int), f["px"].astype(int)]
    Trel = se3.mul(T2, se3.inv(T1))
    Xc = np.stack([(px[:, 0] - synth.CX) * depth / synth.FX, (px[:, 1] - synth.CY) * depth / synth.FY, depth], 1)
    Xc2 = (Trel[:, :3] @ Xc.T).T + Trel[:, 3]
    gt = np.stack([synth.FX * Xc2[:, 0] / Xc2[:, 2] + synth.CX, synth.FY * Xc2[:, 1] / Xc2[:, 2] + synth.CY], 1)
    return dict(p1=p1, p2=p2, f=f, px=px, depth=depth, T1=T1, T2=T2, Trel=Trel, gt=gt)


def test_se3_exp_log_roundtrip(oracle):
    """Sophus ships round-trip tests (thirdparty/Sophus/sophus/test_se3.cpp): exp(log(T)) == T."""
    rng = np.random.default_rng(0)
    for scale in (1e-12, 1e-3, 0.5, 2.0):
        for _ in range(10):
            v = rng.normal(0, scale, 6)
            if np.linalg.norm(v[3:]) > 3.0:     # log() returns the principal rotation (|omega| < pi)
                v[3:] *= 3.0 / np.linalg.norm(v[3:])
            T = oracle.se3_exp(v)
            assert np.allclose(T[:, :3] @ T[:, :3].T, np.eye(3), atol=1e-12)
            assert np.allclose(oracle.se3_log(T), v, atol=1e-9 * max(1, scale))
            assert np.allclose(T, se3.se3_exp(v), atol=1e-10)


def test_se3_exp_log_against_scipy(oracle):
    """Third-party check of the Sophus restatement (se3.cpp:170-220, so3.cpp:127-202): exp([upsilon; omega]) is the matrix
    exponential of the 4 x 4 twist (scipy.linalg.expm), its rotation scipy's Rotation.from_rotvec; log inverts both --
    including tiny angles (Taylor branch) and angles close to pi."""
    from scipy.linalg import expm, logm
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(3)
    for scale in (1e-9, 1e-5, 1e-2, 0.7, 3.0):
        for _ in range(8):
            v = rng.normal(0, 1, 6)
            v[3:] *= scale / np.linalg.norm(v[3:])
            w = v[3:]
            twist = np.zeros((4, 4))
            twist[:3, :3] = [[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]
            twist[:3, 3] = v[:3]
            want = expm(twist)
            T = oracle.se3_exp(v)
            # Sophus evaluates (1 - cos(theta)) / theta^2 literally above SMALL_EPS = 1e-10 (se3.cpp:182-193): for tiny angles the
            # cancellation costs eps / theta^2 in that coefficient, i.e. eps * |upsilon| / theta in the translation -- kept, it is
            # the reference's arithmetic
            tol = 1e-12 * max(1.0, np.abs(want).max()) + 1e-15 * np.linalg.norm(v[:3]) / scale
            assert np.abs(T - want[:3]).max() < tol
            assert np.abs(T[:, :3] - Rotation.from_rotvec(w).as_matrix()).max() < 1e-14
            back = oracle.se3_log(T)
            assert np.abs(back[3:] - Rotation.from_matrix(T[:, :3]).as_rotvec()).max() < 1e-9 * max(1.0, scale) + 1e-15
            if scale >= 1e-2:    # (logm loses digits for tiny rotations; the round trip above covers those)
                L = np.real(logm(np.vstack([T, [0, 0, 0, 1]])))
                assert np.abs(back[:3] - L[:3, 3]).max() < 1e-9 and np.abs(back[3:] - [L[2, 1], L[0, 2], L[1, 0]]).max() < 1e-9


def test_find_direct_projection_converges_to_ground_truth(oracle):
    s = _scene(oracle)
    rng = np.random.default_rng(7)
    init = s["gt"] + rng.uniform(-2, 2, s["gt"].shape)
    I = np.eye(4)[:3]
    cur, lvl, ok = oracle.find_direct_projection(s["p1"], s["p2"], 640, 480, 3, I, s["Trel"], s["px"], s["depth"],
                                                 s["f"]["level"], init)
    assert ok.mean() > 0.9
    assert np.array_equal(lvl, s["f"]["level"])           # |det A| ~ 4^level -> search on the feature's level
    err = np.linalg.norm(cur - s["gt"], axis=1)[ok]
    assert np.median(err) < 0.25 and np.percentile(err, 95) < 0.6


def test_sparse_align_recovers_relative_pose(oracle):
    s = _scene(oracle)
    n = len(s["depth"])
    T, n_meas, iters = oracle.sparse_align(s["p1"], s["p2"], 640, 480, 3, s["px"], s["depth"], np.ones(n, np.uint8), s["T1"], s["T1"])
    err = np.linalg.norm(se3.se3_log(se3.mul(T, se3.inv(s["T2"]))))
    init = np.linalg.norm(se3.se3_log(se3.mul(s["T1"], se3.inv(s["T2"]))))
    assert init > 1e-2 and err < 1e-3
    assert 0 < n_meas <= n
    ok, T2 = oracle.matcher_sparse_alignment(s["p1"], s["p2"], 640, 480, 3, s["px"], s["depth"], np.ones(n, np.uint8), s["T1"], s["T1"])
    assert ok and np.allclose(T2, T)
    # a feature without map point is skipped; no features -> pose untouched, 0 measurements
    T0, nm0, _ = oracle.sparse_align(s["p1"], s["p2"], 640, 480, 3, s["px"], s["depth"], np.zeros(n, np.uint8), s["T1"], s["T1"])
    assert nm0 == 0


def test_sparse_align_dense_pixel_features(oracle):
    """The GPU suite's large sparse-alignment problem: 6,000 random pixels of the rendered frame with their rendered depth
    (not detections), every seventh without a map point.  The oracle recovers the relative pose from them."""
    g1, d1, T1 = synth.stream_frame(1)
    g2, _, T2 = synth.stream_frame(4)
    p1, p2 = oracle.build_pyramid(g1, 3), oracle.build_pyramid(g2, 3)
    px, depth = synth.pixel_features(d1, 6000, seed=61)
    has = np.ones(6000, np.uint8)
    has[::7] = 0
    T, n_meas, iters = oracle.sparse_align(p1, p2, 640, 480, 3, px, depth, has, T1, T1)
    assert np.linalg.norm(se3.se3_log(se3.mul(T, se3.inv(T2)))) < 2e-3
    assert 0.8 * has.sum() < n_meas <= has.sum() and (iters[:3] > 0).all()
