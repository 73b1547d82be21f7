"""SURVEY.md 8f row 1 -- the matching / geometry behind LocalMapping::CreateNewMapPoints: Matcher::SearchForTriangulation with
CheckDistEpipolarLine (Matcher.cpp:86-193, 338-354) and cvutils::DepthFromTriangulation (CVUtils.h:18-38).  The DBoW3
feature vectors are an INPUT here (one vocabulary node per feature; the vocabulary itself is row f2 and out of scope), so the
tests group features with a toy quantiser."""
import numpy as np
import pytest

from ygz_slam_b200 import se3, synth

FX, FY, CX, CY = (float(np.float32(v)) for v in (520.9, 521.0, 325.1, 249.7))


def _scene(oracle, k1=1, k2=6):
    """Two frames of the synthetic stream with detected features, toy BoW nodes and the essential matrix E12 of the true motion."""
    g1, _, T1 = synth.stream_frame(k1)
    g2, _, T2 = synth.stream_frame(k2)
    f1 = oracle.detect(oracle.build_pyramid(g1, 3))
    f2 = oracle.detect(oracle.build_pyramid(g2, 3))
    node = lambda f: (f["desc"][:, 0].astype(np.int32) >> 5) * 8 + (f["desc"][:, 7] >> 5)   # 64 toy nodes from descriptor bits
    n1, n2 = node(f1), node(f2)
    n1[::17] = -1                                          # some features are in no node
    T21 = se3.mul(T2, se3.inv(T1))                         # x2 = R x1 + t
    R, t = T21[:, :3], T21[:, 3]
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    E = tx @ R                                             # x2^T E x1 = 0; the reference's E12 is applied as pt1^T E12 -> line for pt2
    px = lambda f: np.stack([f["px"], f["py"]], 1)
    return f1, f2, px(f1), px(f2), n1, n2, E.T.copy(), T21


def _brute(f1, f2, p1, p2, n1, n2, E12, th_low, dsqr):
    """Plain Python statement of Matcher.cpp:110-156 (candidates in ascending index, `dist > bestDist` skips)."""
    out = np.full(len(n1), -1, np.int32)
    pc = lambda p: ((p[0] - CX) * 1.0 / FX, (p[1] - CY) * 1.0 / FY)
    for i in range(len(n1)):
        if n1[i] < 0:
            continue
        best, bi = 256, -1
        x1, y1 = pc(p1[i])
        a = np.float32(x1 * E12[0, 0] + y1 * E12[1, 0] + E12[2, 0])
        b = np.float32(x1 * E12[0, 1] + y1 * E12[1, 1] + E12[2, 1])
        c = np.float32(x1 * E12[0, 2] + y1 * E12[1, 2] + E12[2, 2])
        den = np.float32(np.float32(a * a) + np.float32(b * b))
        for j in np.nonzero(n2 == n1[i])[0]:
            d = int(np.unpackbits(f1["desc"][i] ^ f2["desc"][j]).sum())
            if d > th_low or d > best:
                continue
            x2, y2 = pc(p2[j])
            num = np.float32(float(a) * x2 + float(b) * y2 + float(c))
            if den < 1e-6:
                continue
            if abs(np.float32(np.float32(num * num) / den)) < np.float32(dsqr):
                best, bi = d, j
        out[i] = bi
    return out


def test_search_for_triangulation_oracle_semantics(oracle):
    f1, f2, p1, p2, n1, n2, E12, _ = _scene(oracle)
    for dsqr in (1e-4, 1e-3):
        got = oracle.search_for_triangulation(f1["desc"], p1, n1, f2["desc"], p2, n2, E12, 65, dsqr)
        want = _brute(f1, f2, p1, p2, n1, n2, E12, 65, dsqr)
        assert np.array_equal(got, want)
        assert (got[n1 < 0] == -1).all()
    assert (got >= 0).sum() > 20                            # the true epipolar geometry lets real matches through
    m = got >= 0
    assert (n2[got[m]] == n1[m]).all()


def test_depth_from_triangulation_recovers_depth(oracle):
    rng = np.random.default_rng(8)
    T = se3.se3_exp(np.array([0.3, -0.05, 0.02, 0.01, 0.03, -0.02]))   # T_search_ref
    X = np.stack([rng.uniform(-1, 1, 50), rng.uniform(-1, 1, 50), rng.uniform(2, 6, 50)], 1)
    f_ref = X / X[:, 2:]
    Xc = (T[:, :3] @ X.T).T + T[:, 3]
    f_cur = Xc / Xc[:, 2:]
    d1, d2, ok = oracle.depth_from_triangulation(T, f_ref, f_cur)
    assert ok.all() and np.abs(d1 - X[:, 2]).max() < 1e-9 and np.abs(d2 - Xc[:, 2]).max() < 1e-9
    # parallel rays (no translation): the 2x2 normal matrix is singular -> rejected
    T0 = np.eye(4)[:3]
    _, _, ok0 = oracle.depth_from_triangulation(T0, f_ref[:5], f_ref[:5])
    assert not ok0.any()


@pytest.mark.gpu
def test_gpu_search_for_triangulation_index_exact(ctx3, oracle):
    a = _scene(oracle, 1, 6)
    b = _scene(oracle, 2, 5)
    off1 = np.cumsum([0, len(a[4]), len(b[4])]).astype(np.int32)
    off2 = np.cumsum([0, len(a[5]), len(b[5])]).astype(np.int32)
    got = ctx3.search_for_triangulation(off1, off2, np.concatenate([a[0]["desc"], b[0]["desc"]]), np.concatenate([a[2], b[2]]),
                                        np.concatenate([a[4], b[4]]), np.concatenate([a[1]["desc"], b[1]["desc"]]),
                                        np.concatenate([a[3], b[3]]), np.concatenate([a[5], b[5]]), np.stack([a[6], b[6]]), 65, 1e-3)
    for p, s in enumerate((a, b)):
        want = oracle.search_for_triangulation(s[0]["desc"], s[2], s[4], s[1]["desc"], s[3], s[5], s[6], 65, 1e-3)
        assert np.array_equal(got[off1[p]:off1[p + 1]], want)
        assert (want >= 0).sum() > 20


@pytest.mark.gpu
def test_gpu_depth_from_triangulation(ctx3, oracle):
    rng = np.random.default_rng(9)
    Ts = np.stack([se3.se3_exp(np.array([0.3, -0.05, 0.02, 0.01, 0.03, -0.02])), np.eye(4)[:3]])
    X = np.stack([rng.uniform(-1, 1, 300), rng.uniform(-1, 1, 300), rng.uniform(2, 6, 300)], 1)
    pose_of = (np.arange(300) % 7 == 0).astype(np.int32)    # every 7th item uses the degenerate identity pose
    f_ref = X / X[:, 2:]
    f_cur = np.empty_like(f_ref)
    for i in range(300):
        Xc = Ts[pose_of[i]][:, :3] @ X[i] + Ts[pose_of[i]][:, 3]
        f_cur[i] = Xc / Xc[2]
    d1, d2, ok = ctx3.depth_from_triangulation(Ts, pose_of, f_ref, f_cur)
    for k in (0, 1):
        sel = pose_of == k
        w1, w2, wok = oracle.depth_from_triangulation(Ts[k], f_ref[sel], f_cur[sel])
        assert np.array_equal(ok[sel], wok)
        assert np.array_equal(d1[sel], w1) and np.array_equal(d2[sel], w2)
    assert ok[pose_of == 0].all() and not ok[pose_of == 1].any()
