"""Triangulation kernels at their decision boundaries: ygzb_search_for_triangulation (Matcher::SearchForTriangulation with
CheckDistEpipolarLine) and ygzb_depth_from_triangulation (cvutils::DepthFromTriangulation) against the oracle, index for
index and bit for bit.

Both kernels decide on values computed in double and, for the epipolar test, rounded to float.  A fused multiply-add in
place of the oracle's separate multiply and add changes those values in their last bits.  At natural scales that rarely
moves a decision, so the cases here are built where it does: essential matrices of ~1e9 whose third row cancels the first
two down to O(1) line coefficients, points within ~1e-12 of the epipolar line, near-parallel rays, and thresholds set to
the oracle's own value and its floating-point neighbours.  The CPU tests state the oracle's arithmetic in Python, check
the oracle against it, and show with exact rationals that each contraction the compiler could make flips decisions on
these cases; the GPU tests then require the kernels to agree with the oracle on all of them."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

from oracle.pyoracle import Camera, default_camera
from ygz_slam_b200 import se3

F32 = np.float32
YGZB_ERR_INVALID = -1
CAM = (520.9, 521.0, 325.1, 249.7)              # the library's and the oracle's default intrinsics
CAM2 = (400.0, 410.5, 300.25, 200.75)           # the second context's
PASS_E = np.array([0, 0, 0, 0, 0, 0, 1.0, 0, 0])  # a = 1, b = c = 0: dsqr = x2^2 with x2 = (u2 - cx) / fx
TH_LOW, TH = 50, 0.25                           # batch parameters: with PASS_E, |u2 - cx| < fx / 2 passes


# ---- the oracle's arithmetic, stated in Python (doubles are IEEE binary64, np.float32 rounds to nearest even) -----------
def _fma(x, y, z):
    """x * y + z rounded once (Fraction -> float is correctly rounded)."""
    return float(Fraction(x) * Fraction(y) + Fraction(z))


def _sum3(p, q, r, s, t, fuse=""):
    """p*q + r*s + t in double: unfused as the oracle evaluates it, or with the first addition fused with the product of p
    (fuse="p") or of r (fuse="r") -- the two contractions a compiler may choose -- and t added separately."""
    if fuse == "p":
        s01 = _fma(p, q, r * s)
    elif fuse == "r":
        s01 = _fma(r, s, p * q)
    else:
        s01 = p * q + r * s
    return s01 + t


def _cam(cam):
    return tuple(float(F32(v)) for v in cam)     # the reference's camera keeps float intrinsics


def _pc(u, v, cam):
    """PinholeCamera::Pixel2Camera at depth 1: double maths on float intrinsics."""
    fx, fy, cx, cy = _cam(cam)
    return (u - cx) * 1.0 / fx, (v - cy) * 1.0 / fy


def _line(x1, y1, E, fuse=""):
    return tuple(F32(_sum3(x1, E[k], y1, E[3 + k], E[6 + k], fuse)) for k in range(3))


def _dsqr(x1, y1, x2, y2, E, fuse_abc="", fuse_num=""):
    """CheckDistEpipolarLine's f32 distance, or None when `den < 1e-6` (a float compared with a double) rejects."""
    a, b, c = _line(x1, y1, E, fuse_abc)
    num = F32(_sum3(float(a), x2, float(b), y2, float(c), fuse_num))
    den = F32(a * a) + F32(b * b)
    if float(den) < 1e-6:
        return None
    return F32(num * num) / den


def _accepts(ds, th):
    return ds is not None and float(abs(ds)) < float(F32(th))


def _search_statement(pr, th_low, th, cam):
    """Matcher.cpp:110-156: candidates in ascending index, `dist > th_low || dist > bestDist` skips."""
    n1, n2 = len(pr["node1"]), len(pr["node2"])
    out = np.full(n1, -1, np.int32)
    if n2 == 0:
        return out
    dist = np.unpackbits(pr["desc1"][:, None, :] ^ pr["desc2"][None, :, :], axis=2).sum(2)
    for i in range(n1):
        if pr["node1"][i] < 0:
            continue
        x1, y1 = _pc(*pr["px1"][i], cam)
        best = 256
        for j in range(n2):
            d = int(dist[i, j])
            if pr["node2"][j] != pr["node1"][i] or d > th_low or d > best:
                continue
            if _accepts(_dsqr(x1, y1, *_pc(*pr["px2"][j], cam), pr["E"]), th):
                best, out[i] = d, j
    return out


# ---- constructed key-frame pairs ------------------------------------------------------------------------------------------
def _flip(d, k, rng):
    """Descriptor d with exactly k of its 256 bits flipped."""
    bits = np.unpackbits(d)
    bits[rng.choice(256, k, replace=False)] ^= 1
    return np.packbits(bits)


def _far(d, n, rng):
    """n descriptors about 230 bits from d (never within 100)."""
    return np.packbits((rng.random((n, 256)) < 0.1).astype(np.uint8), axis=1) ^ ~d


def _u(cam, x):
    fx, _, cx, _ = _cam(cam)
    return cx + x * fx


def _pair(desc1, node1, desc2, node2, cam, rng, E=PASS_E, px1=None, px2=None, expect=None):
    n1, n2 = len(node1), len(node2)
    if px1 is None:
        px1 = np.stack([rng.uniform(20, 620, n1), rng.uniform(20, 460, n1)], 1)
    if px2 is None:   # every candidate passes the PASS_E test at TH
        px2 = np.stack([_u(cam, rng.uniform(-0.4, 0.4, n2)), rng.uniform(20, 460, n2)], 1)
    return dict(desc1=np.asarray(desc1, np.uint8).reshape(n1, 32), px1=np.asarray(px1, np.float64).reshape(n1, 2),
                node1=np.asarray(node1, np.int32), desc2=np.asarray(desc2, np.uint8).reshape(n2, 32),
                px2=np.asarray(px2, np.float64).reshape(n2, 2), node2=np.asarray(node2, np.int32), E=np.asarray(E, np.float64),
                expect=None if expect is None else np.asarray(expect, np.int32))


def _tie_pair(cam, n2, i, j, extra, rng):
    """One key-frame-1 feature.  All n2 candidates share its node; all are out of th_low except i (distance 10) and j > i
    (distance 10 + extra), and a closer candidate (distance 3) right after i fails the epipolar test.  A later candidate of
    equal distance replaces the earlier one, a later one of larger distance is skipped."""
    d1 = rng.integers(0, 256, (1, 32), dtype=np.uint8)
    desc2 = _far(d1[0], n2, rng)
    desc2[i] = _flip(d1[0], 10, rng)
    desc2[j] = _flip(d1[0], 10 + extra, rng)
    px2 = np.stack([_u(cam, rng.uniform(-0.4, 0.4, n2)), rng.uniform(20, 460, n2)], 1)
    if i + 1 < j:
        desc2[i + 1] = _flip(d1[0], 3, rng)
        px2[i + 1, 0] = _u(cam, 0.8)
    return _pair(d1, [4], desc2, np.full(n2, 4), cam, rng, px2=px2, expect=[j if extra == 0 else i])


def _th_low_pair(cam, th_low, rng):
    """Feature 0 (node 0): distance th_low at index 0, th_low + 1 at index 1 -- the first is accepted, the later one is
    out of th_low.  Feature 1 (node 1): its only candidate (index 2) is at th_low + 1.  At th_low = 256 every distance is
    accepted: the later equal candidate wins and feature 1 finds index 2."""
    d1 = rng.integers(0, 256, (2, 32), dtype=np.uint8)
    k = min(th_low + 1, 256)
    desc2 = np.stack([_flip(d1[0], th_low, rng), _flip(d1[0], k, rng), _flip(d1[1], k, rng)])
    expect = [0, -1] if th_low < 256 else [1, 2]
    return _pair(d1, [0, 1], desc2, [0, 0, 1], cam, rng, expect=expect)


def _node_pair(cam, rng):
    """Node -1 on either side and nodes present on one side only never match, whatever the descriptors."""
    d1 = rng.integers(0, 256, (4, 32), dtype=np.uint8)
    desc2 = np.stack([d1[0], d1[0], d1[1], d1[3], d1[2]])
    node1 = [-1, 5, 7, 0]      # feature 0 is in no node; node 7 exists in key-frame 1 only
    node2 = [-1, 0, -1, 0, 9]  # candidate 2 (feature 1's twin) is in no node; node 9 exists in key-frame 2 only
    return _pair(d1, node1, desc2, node2, cam, rng, expect=[-1, -1, -1, 3])


def _dense_pair(cam, n1, n2, n_nodes, rng):
    """Random features over n_nodes nodes (some in none); every key-frame-2 feature is a perturbed copy of a random
    key-frame-1 feature (0..70 bits), and about half of them pass the epipolar test."""
    d1 = rng.integers(0, 256, (n1, 32), dtype=np.uint8)
    node1 = rng.integers(0, n_nodes, n1)
    node1[rng.random(n1) < 0.05] = -1
    src = rng.integers(0, n1, n2)
    desc2 = np.stack([_flip(d1[s], int(rng.integers(0, 71)), rng) for s in src]) if n2 else np.zeros((0, 32), np.uint8)
    node2 = np.where(rng.random(n2) < 0.8, node1[src], rng.integers(-1, n_nodes, n2)) if n2 else np.zeros(0, np.int32)
    px2 = np.stack([_u(cam, rng.uniform(-0.7, 0.7, n2)), rng.uniform(20, 460, n2)], 1)
    return _pair(d1, node1, desc2, node2, cam, rng, px2=px2)


def _epipolar_case(cam, near_line, rng):
    """One feature per side, equal descriptors.  E ~ 1e9 whose third row cancels the first two down to O(1) line
    coefficients.  With near_line, c is 0 and the second point lies within ~1e-12 of the oracle's line, so the two
    products of num = a*x2 + b*y2 + c cancel each other and their rounding decides num."""
    while True:
        u1, v1 = rng.uniform(20, 620), rng.uniform(20, 460)
        x1, y1 = _pc(u1, v1, cam)
        E = np.empty(9)
        for k in range(3):
            E[k], E[3 + k] = rng.uniform(0.5e9, 2e9, 2) * rng.choice([-1, 1], 2)
            E[6 + k] = -(x1 * E[k] + y1 * E[3 + k]) + (0.0 if near_line and k == 2 else rng.uniform(-2, 2))
        u2, v2 = rng.uniform(20, 620), rng.uniform(20, 460)
        if near_line:
            a, b, c = (float(t) for t in _line(x1, y1, E))
            fx, fy, cx, cy = _cam(cam)
            off = rng.uniform(-1e-12, 1e-12)
            if abs(b) > abs(a):
                v2 = (-(a * _pc(u2, v2, cam)[0] + c) / b + off) * fy + cy
            else:
                u2 = (-(b * _pc(u2, v2, cam)[1] + c) / a + off) * fx + cx
        ds = _dsqr(x1, y1, *_pc(u2, v2, cam), E)
        if ds is not None and 1e-30 < float(ds) < 1e30:
            d = rng.integers(0, 256, (1, 32), dtype=np.uint8)
            return _pair(d, [3], d, [3], cam, rng, E=E, px1=[u1, v1], px2=[u2, v2]), ds


def _epipolar_cases(cam=CAM, n=120, seed=31):
    rng = np.random.default_rng(seed)
    return [_epipolar_case(cam, k % 2 == 1, rng) for k in range(n)]


def _thresholds(ds):
    """The oracle's own f32 dsqr and its float neighbours: `fabs(dsqr) < th` rejects the first two, accepts the third."""
    return (np.nextafter(ds, F32(-np.inf)), ds, np.nextafter(ds, F32(np.inf)))


def _den_values():
    """Floats a, b with fl(fl(a*a) + fl(b*b)) equal to the float below 1e-6f, 1e-6f itself (below the double 1e-6: still
    rejected) and the next two floats up (accepted)."""
    t0 = F32(1e-6)
    targets = [np.nextafter(t0, F32(0)), t0, np.nextafter(t0, F32(1)), np.nextafter(np.nextafter(t0, F32(1)), F32(1))]
    out = []
    for t in targets:
        a0 = F32(np.sqrt(float(t)))
        a = a0 - np.arange(0, 400, dtype=np.float32) * np.spacing(a0)
        found = None
        for av in a:
            aa = F32(av * av)
            if aa > t:
                continue
            r = t - aa                              # exact (Sterbenz)
            b0 = F32(np.sqrt(float(r)))
            for bv in (b0, np.nextafter(b0, F32(0)), np.nextafter(b0, F32(1))):
                if F32(aa + F32(bv * bv)) == t:
                    found = (av, bv)
                    break
            if found:
                break
        assert found, t
        out.append((float(found[0]), float(found[1]), t))
    return out


def _den_pairs(cam, rng):
    """E has zero rows 1 and 2, so the line coefficients are the floats in row 3, exactly; the second point sits near the
    principal point so that dsqr is far below TH.  Only `den < 1e-6` decides."""
    pairs = []
    for a, b, t in _den_values():
        d = rng.integers(0, 256, (1, 32), dtype=np.uint8)
        E = np.array([0, 0, 0, 0, 0, 0, a, b, 0.0])
        _, _, cx, cy = _cam(cam)
        px2 = [cx + rng.uniform(-0.5, 0.5), cy + rng.uniform(-0.5, 0.5)]
        pairs.append(_pair(d, [2], d, [2], cam, rng, E=E, px2=px2, expect=[0 if float(t) >= 1e-6 else -1]))
    return pairs


def _structured_pairs(cam, seed):
    """Every constructed pair that runs at the batch parameters (TH_LOW, TH), with its expected result where it has one."""
    rng = np.random.default_rng(seed)
    pairs = []
    for n2, i, j in ((200, 127, 128), (300, 255, 256), (129, 0, 128), (5000, 0, 4999), (128, 126, 127), (2, 0, 1)):
        for extra in (0, 1):
            pairs.append(_tie_pair(cam, n2, i, j, extra, rng))
    pairs.append(_th_low_pair(cam, TH_LOW, rng))
    pairs.append(_node_pair(cam, rng))
    pairs += _den_pairs(cam, rng)
    for n1, n2, nodes in ((1, 0, 4), (5, 0, 1), (7, 1, 1), (200, 127, 3), (260, 128, 3), (130, 129, 2), (300, 3072, 8),
                          (3072, 3072, 1), (60, 5000, 2), (129, 1, 1)):
        pairs.append(_dense_pair(cam, n1, n2, nodes, rng))
    pairs += [p for p, _ in _epipolar_cases(cam, 16, seed + 1)]
    return pairs


# ---- running a batch -----------------------------------------------------------------------------------------------------
def _gpu(ctx, pairs, th_low, th):
    off1 = np.cumsum([0] + [len(p["node1"]) for p in pairs]).astype(np.int32)
    off2 = np.cumsum([0] + [len(p["node2"]) for p in pairs]).astype(np.int32)
    cat = lambda k, shape: np.concatenate([p[k] for p in pairs]) if off2[-1] or k.endswith("1") else np.zeros(shape)
    got = ctx.search_for_triangulation(off1, off2, cat("desc1", None), cat("px1", None), cat("node1", None),
                                       cat("desc2", (0, 32)), cat("px2", (0, 2)), cat("node2", 0),
                                       np.stack([p["E"] for p in pairs]), th_low, th)
    return [got[off1[k]:off1[k + 1]] for k in range(len(pairs))]


def _oracle(oracle, pr, th_low, th, cam=CAM):
    return oracle.search_for_triangulation(pr["desc1"], pr["px1"], pr["node1"], pr["desc2"], pr["px2"], pr["node2"], pr["E"],
                                           th_low, th, cam=Camera(*cam))


# ---- CPU: the constructed cases discriminate -----------------------------------------------------------------------------
def test_epipolar_cases_discriminate(oracle):
    """The Python statement is the oracle's arithmetic on every epipolar case; each contraction of the line coefficients
    or of num changes dsqr, and so flips the decision at one of the three thresholds, on many of them."""
    cases = _epipolar_cases()
    flips = {k: 0 for k in ("abc-p", "abc-r", "num-p", "num-r")}
    for pr, ds in cases:
        want = [_accepts(ds, th) for th in _thresholds(ds)]
        assert want == [False, False, True]
        for th, w in zip(_thresholds(ds), want):
            assert _oracle(oracle, pr, 255, float(th))[0] == (0 if w else -1)
            assert _search_statement(pr, 255, float(th), CAM)[0] == (0 if w else -1)
        x1, y1 = _pc(*pr["px1"][0], CAM)
        x2, y2 = _pc(*pr["px2"][0], CAM)
        for key, kw in (("abc-p", dict(fuse_abc="p")), ("abc-r", dict(fuse_abc="r")), ("num-p", dict(fuse_num="p")),
                        ("num-r", dict(fuse_num="r"))):
            v = _dsqr(x1, y1, x2, y2, pr["E"], **kw)
            flips[key] += [_accepts(v, th) for th in _thresholds(ds)] != want
    # 120 cases, half of them within 1e-12 of the line: measured 44, 48, 59 and 57 flips
    assert flips["abc-p"] >= 35 and flips["abc-r"] >= 35, flips
    assert flips["num-p"] >= 45 and flips["num-r"] >= 45, flips


def test_structured_cases_match_the_statement(oracle):
    """Ties, th_low, nodes and the den boundary: the oracle and the Python statement agree, and give the result each case
    was built for."""
    pairs = _structured_pairs(CAM, 5)
    for k, pr in enumerate(pairs):
        want = _oracle(oracle, pr, TH_LOW, TH)
        if pr["expect"] is not None:
            assert np.array_equal(want, pr["expect"]), k
        if len(pr["node1"]) * len(pr["node2"]) <= 40000:
            assert np.array_equal(want, _search_statement(pr, TH_LOW, TH, CAM)), k
    rng = np.random.default_rng(6)
    for th_low in (0, 1, 255, 256):
        pr = _th_low_pair(CAM, th_low, rng)
        assert np.array_equal(_oracle(oracle, pr, th_low, TH), pr["expect"]), th_low
        assert np.array_equal(_search_statement(pr, th_low, TH, CAM), pr["expect"]), th_low


# ---- DepthFromTriangulation ----------------------------------------------------------------------------------------------
def _depth_statement(T, pose_of, f_ref, f_cur, det_th):
    """CVUtils.h:18-38 in numpy (every operation rounded on its own, as in the oracle): depth1, depth2, ok, det."""
    M = np.asarray(T, np.float64).reshape(-1, 12)[pose_of]
    with np.errstate(all="ignore"):
        a0 = [M[:, 4 * r] * f_ref[:, 0] + M[:, 4 * r + 1] * f_ref[:, 1] + M[:, 4 * r + 2] * f_ref[:, 2] for r in range(3)]
        a1 = [-f_cur[:, r] for r in range(3)]
        m00 = a0[0] * a0[0] + a0[1] * a0[1] + a0[2] * a0[2]
        m01 = a0[0] * a1[0] + a0[1] * a1[1] + a0[2] * a1[2]
        m11 = a1[0] * a1[0] + a1[1] * a1[1] + a1[2] * a1[2]
        det = m00 * m11 - m01 * m01
        ok = ~(det < det_th)
        b0 = a0[0] * M[:, 3] + a0[1] * M[:, 7] + a0[2] * M[:, 11]
        b1 = a1[0] * M[:, 3] + a1[1] * M[:, 7] + a1[2] * M[:, 11]
        inv = 1.0 / det
        d1 = np.abs(-(m11 * inv * b0 + -m01 * inv * b1))
        d2 = np.abs(-(-m01 * inv * b0 + m00 * inv * b1))
    return np.where(ok, d1, 0.0), np.where(ok, d2, 0.0), ok, det, (m00, m01, m11)


def _rays(T, X):
    """Unit-depth rays of world points X in the reference camera (identity) and in T (points behind a camera give rays
    through the opposite direction, which the fabs of the depths folds back)."""
    Xc = X @ T[:, :3].T + T[:, 3]
    return X / X[:, 2:], Xc / Xc[:, 2:]


def _near_parallel(n, seed, baseline=0.01, depth=(50, 400)):
    """A realistic two-view geometry with a short baseline and far points: det is a small difference of two products."""
    rng = np.random.default_rng(seed)
    T = se3.se3_exp(np.array([baseline, -0.3 * baseline, 0.2 * baseline, 0.01, -0.02, 0.005]))
    z = rng.uniform(*depth, n)
    X = np.stack([rng.uniform(-0.5, 0.5, n) * z, rng.uniform(-0.4, 0.4, n) * z, z], 1)
    return T, *_rays(T, X)


def _close(d, up):
    return float(np.nextafter(d, np.inf if up else -np.inf))


def test_depth_cases_discriminate(oracle):
    """The numpy statement is the oracle's arithmetic, depths and decision, at det_th = its own det (accepted) and the
    next double up (rejected); fusing the determinant's product, fma(m00, m11, -m01^2), flips one of the two decisions on
    nearly every near-parallel item."""
    T, fr, fc = _near_parallel(200, 41)
    po = np.zeros(len(fr), np.int32)
    _, _, _, det, (m00, m01, m11) = _depth_statement(T, po, fr, fc, 0.0)
    flips = 0
    for i in range(len(fr)):
        for up in (False, True):
            th = float(det[i]) if not up else _close(det[i], True)
            w1, w2, wok = oracle.depth_from_triangulation(T, fr[i:i + 1], fc[i:i + 1], th)
            s1, s2, sok, _, _ = _depth_statement(T, po[:1], fr[i:i + 1], fc[i:i + 1], th)
            assert wok[0] == (not up) and sok[0] == wok[0], (i, up)
            assert np.array_equal(w1, s1) and np.array_equal(w2, s2), i
        fused = _fma(float(m00[i]), float(m11[i]), -(float(m01[i]) * float(m01[i])))
        flips += [not (fused < float(det[i])), not (fused < _close(det[i], True))] != [True, False]
    assert flips >= 190, flips                                 # measured: 200 of 200


def _check_depth(got, want):
    """Depths bit for bit; NaN (exactly parallel rays with det_th <= 0) by position."""
    for g, w in zip(got[:2], want[:2]):
        assert np.array_equal(np.isnan(g), np.isnan(w))
        m = ~np.isnan(w)
        assert np.array_equal(g[m].view(np.int64), w[m].view(np.int64))
    assert np.array_equal(got[2], want[2])


def _depth_mix(seed):
    """Near-parallel rays, points behind either camera, exactly parallel rays (det = 0) and rounding-level dets of either
    sign, over three poses."""
    rng = np.random.default_rng(seed)
    Ts = [se3.se3_exp(np.array([0.3, -0.05, 0.02, 0.01, 0.03, -0.02])), _near_parallel(1, 1)[0],
          np.concatenate([np.eye(3), [[0.2], [0.1], [0.0]]], 1)]
    fr, fc, po = [], [], []
    for p, T in enumerate(Ts):
        n = 120
        z = rng.uniform(2, 8, n)
        z[::5] *= -1                                           # behind the reference camera
        z[1::7] = rng.uniform(1e3, 1e6, len(z[1::7]))          # (nearly) parallel rays
        X = np.stack([rng.uniform(-0.5, 0.5, n) * np.abs(z), rng.uniform(-0.4, 0.4, n) * np.abs(z), z], 1)
        if p == 0:                                             # behind the current camera: X = R^T (Xc - t) with Xc.z < 0
            X[2::6] = (X[2::6] * [1, 1, -1] - T[:, 3]) @ T[:, :3]
        a, b = _rays(T, X)
        if p == 2:
            b[3::9] = a[3::9]                                  # pure translation and equal rays: det = 0 exactly
        fr.append(a)
        fc.append(b)
        po.append(np.full(n, p, np.int32))
    return np.stack([T.reshape(-1) for T in Ts]), np.concatenate(po), np.concatenate(fr), np.concatenate(fc)


@pytest.mark.gpu
def test_gpu_depth_at_the_determinant_threshold(ctx3, oracle):
    """det_th at the oracle's det of each near-parallel item (accepted) and the next double up (rejected): every call runs
    all items, so the other items are checked at that threshold too."""
    T, fr, fc = _near_parallel(64, 43)
    po = np.zeros(len(fr), np.int32)
    det = _depth_statement(T, po, fr, fc, 0.0)[3]
    for i in range(len(fr)):
        for up in (False, True):
            th = _close(det[i], True) if up else float(det[i])
            got = ctx3.depth_from_triangulation(T.reshape(1, 12), None, fr, fc, th)
            want = _depth_statement(T, po, fr, fc, th)[:3]
            _check_depth(got, want)
            assert got[2][i] == (not up), (i, up)
            w1, w2, wok = oracle.depth_from_triangulation(T, fr[i:i + 1], fc[i:i + 1], th)
            assert wok[0] == got[2][i] and w1[0] == got[0][i] and w2[0] == got[1][i]


@pytest.mark.gpu
@pytest.mark.parametrize("det_th", [1e-5, 0.0, -1e-300, -1.0])
def test_gpu_depth_bit_exact(ctx3, oracle, det_th):
    """Several poses, near-parallel and exactly parallel rays, points behind either camera, at the default det_th, at 0
    and at negative thresholds that admit rounding-level negative dets."""
    Ts, po, fr, fc = _depth_mix(47)
    got = ctx3.depth_from_triangulation(Ts, po, fr, fc, det_th)
    want = _depth_statement(Ts, po, fr, fc, det_th)
    _check_depth(got, want[:3])
    for p in range(len(Ts)):                                   # the statement is the oracle's arithmetic
        sel = po == p
        _check_depth(oracle.depth_from_triangulation(Ts[p], fr[sel], fc[sel], det_th), [w[sel] for w in want[:3]])
    if det_th <= 0:
        assert np.isnan(got[0]).any() and (want[3] == 0).any()
    if det_th < 0:
        assert (want[3] < 0).any()                             # rounding-level negative dets are admitted
    assert got[2].any() and not got[2].all() or det_th < 0


@pytest.mark.gpu
def test_gpu_depth_one_pose_empty_and_invalid(ctx3, oracle):
    T, fr, fc = _near_parallel(300, 44, baseline=0.2, depth=(2, 20))
    got = ctx3.depth_from_triangulation(T.reshape(1, 12), None, fr, fc, 1e-5)
    _check_depth(got, oracle.depth_from_triangulation(T, fr, fc, 1e-5))
    assert got[2].all()
    d1, d2, ok = ctx3.depth_from_triangulation(T.reshape(1, 12), None, np.zeros((0, 3)), np.zeros((0, 3)), 1e-5)
    assert len(d1) == len(d2) == len(ok) == 0
    Ts = np.stack([T.reshape(-1)] * 2)
    d1, d2, ok = (np.full(3, 7.0), np.full(3, 7.0), np.full(3, 9, np.uint8))
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    for po in ([0, 1, 2], [0, -1, 1]):
        po = np.asarray(po, np.int32)
        rc = ctx3.lib.ygzb_depth_from_triangulation(ctx3.h, 3, 2, p(Ts), p(po), p(fr[:3].copy()), p(fc[:3].copy()), C.c_double(1e-5),
                                                     p(d1), p(d2), p(ok))
        assert rc == YGZB_ERR_INVALID
    assert (d1 == 7.0).all() and (ok == 9).all()


@pytest.mark.gpu
def test_gpu_depth_a_million_items(ctx3, oracle):
    """~10^6 items over 4 poses (7,813 blocks), bit for bit against the numpy statement, and every 997th item against the
    oracle itself."""
    rng = np.random.default_rng(48)
    n = 1_000_000
    Ts = np.stack([se3.se3_exp(rng.normal(0, [0.2, 0.2, 0.2, 0.05, 0.05, 0.05])).reshape(-1) for _ in range(4)])
    po = rng.integers(0, 4, n).astype(np.int32)
    z = rng.uniform(1, 30, n)
    z[::11] = rng.uniform(1e3, 1e5, len(z[::11]))
    X = np.stack([rng.uniform(-0.5, 0.5, n) * z, rng.uniform(-0.4, 0.4, n) * z, z], 1)
    fr, fc = np.empty_like(X), np.empty_like(X)
    for p in range(4):
        sel = po == p
        fr[sel], fc[sel] = _rays(Ts[p].reshape(3, 4), X[sel])
    got = ctx3.depth_from_triangulation(Ts, po, fr, fc, 1e-5)
    _check_depth(got, _depth_statement(Ts, po, fr, fc, 1e-5)[:3])
    assert 0.5 < got[2].mean() < 1
    for i in range(0, n, 997):
        w1, w2, wok = oracle.depth_from_triangulation(Ts[po[i]], fr[i:i + 1], fc[i:i + 1], 1e-5)
        assert wok[0] == got[2][i] and w1[0] == got[0][i] and w2[0] == got[1][i], i


# ---- SearchForTriangulation ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_epipolar_threshold(ctx3, oracle):
    """epipolar_dsqr at the oracle's own f32 dsqr and its float neighbours, on ~1e9-scale essential matrices, half of them
    with the second point within 1e-12 of the line."""
    bad = []
    for k, (pr, ds) in enumerate(_epipolar_cases()):
        for th in _thresholds(ds):
            want = _oracle(oracle, pr, 255, float(th))
            got = _gpu(ctx3, [pr], 255, float(th))[0]
            if not np.array_equal(got, want):
                bad.append((k, float(th)))
    assert not bad, f"{len(bad)} of {3 * 120} decisions differ from the oracle: {bad[:5]}"


@pytest.mark.gpu
@pytest.mark.parametrize("th_low", [0, 1, 50, 255, 256])
def test_gpu_distance_threshold(ctx3, oracle, th_low):
    rng = np.random.default_rng(60 + th_low)
    pairs = [_th_low_pair(CAM, th_low, rng) for _ in range(3)]
    for pr, got in zip(pairs, _gpu(ctx3, pairs, th_low, TH)):
        assert np.array_equal(got, pr["expect"]) and np.array_equal(got, _oracle(oracle, pr, th_low, TH))


@pytest.mark.gpu
@pytest.mark.parametrize("cam", [CAM, CAM2], ids=["default-intrinsics", "other-intrinsics"])
def test_gpu_structured_batch(oracle, cam):
    """Ties across the 128-feature staging chunk and at both ends, th_low, nodes, the den boundary, n2 of 0 to 5,000, n1
    up to 3,072 (several blocks per pair next to pairs whose blocks are all idle), all in one batch, each pair alone, and
    the batch reversed."""
    from ygz_slam_b200 import Context
    ctx = Context(0, **dict(zip(("fx", "fy", "cx", "cy"), cam)))
    try:
        pairs = _structured_pairs(cam, 7)
        want = [_oracle(oracle, pr, TH_LOW, TH, cam) for pr in pairs]
        for pr, w in zip(pairs, want):
            if pr["expect"] is not None:
                assert np.array_equal(w, pr["expect"])
        got = _gpu(ctx, pairs, TH_LOW, TH)
        for k, (g, w) in enumerate(zip(got, want)):
            assert np.array_equal(g, w), k
        rev = _gpu(ctx, pairs[::-1], TH_LOW, TH)[::-1]
        for k, (g, w) in enumerate(zip(rev, want)):
            assert np.array_equal(g, w), k
        for k, (pr, w) in enumerate(zip(pairs, want)):
            assert np.array_equal(_gpu(ctx, [pr], TH_LOW, TH)[0], w), k
        assert sum((w >= 0).sum() for w in want) > 1000
    finally:
        ctx.close()


@pytest.mark.gpu
def test_gpu_search_invalid_arguments(ctx3):
    rng = np.random.default_rng(70)
    pr = _dense_pair(CAM, 3, 4, 1, rng)
    out = np.full(3, 5, np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    args = lambda off1, off2, n: (ctx3.h, n, p(off1), p(off2), p(pr["desc1"]), p(pr["px1"]), p(pr["node1"]), p(pr["desc2"]),
                                  p(pr["px2"]), p(pr["node2"]), p(np.tile(pr["E"], 2)), 50, C.c_double(TH), p(out))
    ok1, ok2 = np.array([0, 3], np.int32), np.array([0, 4], np.int32)
    assert ctx3.lib.ygzb_search_for_triangulation(*args(ok1, ok2, 0)) == YGZB_ERR_INVALID
    assert ctx3.lib.ygzb_search_for_triangulation(*args(ok1, ok2, -1)) == YGZB_ERR_INVALID
    assert ctx3.lib.ygzb_search_for_triangulation(*args(np.array([0, 3, 2], np.int32), np.array([0, 2, 4], np.int32), 2)) == YGZB_ERR_INVALID
    assert ctx3.lib.ygzb_search_for_triangulation(*args(np.array([0, 1, 3], np.int32), np.array([0, 3, 2], np.int32), 2)) == YGZB_ERR_INVALID
    assert ctx3.lib.ygzb_search_for_triangulation(*args(np.array([1, 3], np.int32), ok2, 1)) == YGZB_ERR_INVALID
    assert (out == 5).all()
    assert ctx3.lib.ygzb_search_for_triangulation(*args(ok1, ok2, 1)) == 0
