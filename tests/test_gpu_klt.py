"""GPU parity for Tracker::TrackKLT (cv::calcOpticalFlowPyrLK).

klt.cu adds the window sums exactly in 64-bit integers; every other step is explicit round-to-nearest f32.  The oracle's
exact-sum mode does the same, so every comparison with it is bit for bit: positions, status and err.  The comparison with
cv2 itself (f32 sums in its own order) stays a tolerance."""
import numpy as np
import pytest

from ygz_slam_b200 import synth

pytestmark = pytest.mark.gpu


def _assert_same(got, want):
    """GPU (positions, bool status, err) == oracle (positions, u8 status, err), bit for bit."""
    gp, gs, ge = got
    wp, ws, we = want
    bad = np.nonzero((gs != ws.astype(bool)) | (gp != wp).any(1) | (ge.view(np.uint32) != we.view(np.uint32)))[0]
    assert len(bad) == 0, [(int(i), gp[i].tolist(), wp[i].tolist(), bool(gs[i]), int(ws[i]), float(ge[i]), float(we[i])) for i in bad[:5]]


def _klt_one(fr, oracle, imgs, a, b, ref, init, **prm):
    """One pair (slots a -> b) on the GPU and on the exact-sum oracle; asserts they agree and returns the GPU result."""
    got = fr.klt([a], [b], [0, len(ref)], ref, init, **prm)
    _assert_same(got, oracle.klt(imgs[a], imgs[b], ref, init, exact=True, **prm))
    return got


def _features(oracle, g):
    f = oracle.detect(oracle.build_pyramid(g, 3))
    return np.stack([f["px"], f["py"]], 1).astype(np.float32)


@pytest.fixture(scope="module")
def frames3(ctx3, synth_frames):
    """Frames 1, 2, 3 of the synthetic stream in slots 0, 1, 2 of the 3-level context."""
    imgs = [f[0] for f in synth_frames]
    fr = ctx3.frames(3)
    fr.upload(np.stack(imgs))
    yield fr, imgs
    fr.close()


@pytest.mark.parametrize("levels", [3, 8])
def test_klt_matches_oracle_and_cv2(levels, ctx3, ctx8, oracle, synth_frames):
    import cv2
    ctx = ctx3 if levels == 3 else ctx8   # 3 levels: pyramid levels 3 and 4 are built on the fly for the tracker
    g1, g2, g3 = (f[0] for f in synth_frames)
    fr = ctx.frames(3)
    fr.upload(np.stack([g1, g2, g3]))
    ref = _features(oracle, g1)
    extra = np.array([[2.5, 3.0], [637.0, 10.0], [320.0, 478.5], [-30.0, 50.0], [700.0, 500.0]], np.float32)
    ref = np.concatenate([ref, extra])
    n = len(ref)
    init = (ref + np.float32(1.5)).astype(np.float32)
    got, gst, gerr = fr.klt([0, 0], [2, 1], [0, n, 2 * n], np.concatenate([ref, ref]), np.concatenate([init, init]))
    for p, cur in enumerate((g3, g2)):
        s = slice(p * n, (p + 1) * n)
        _assert_same((got[s], gst[s], gerr[s]), oracle.klt(g1, cur, ref, init, exact=True))
        # how far the kernel is from OpenCV's own f32 summation order
        cvp, cvs, _ = cv2.calcOpticalFlowPyrLK(g1, cur, ref.copy(), init.copy(), winSize=(21, 21), maxLevel=4,
                                               criteria=(cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.001),
                                               flags=cv2.OPTFLOW_USE_INITIAL_FLOW)
        cvs = cvs.reshape(-1).astype(bool)
        assert (cvs != gst[s]).mean() < 0.005
        both = cvs & gst[s]
        assert np.percentile(np.abs(got[s][both] - cvp.reshape(-1, 2)[both]).max(1), 99) < 0.01
        assert both.sum() > 0.9 * n
    fr.close()


# (w, h, slot pyramid levels, KLT max_level, grid cell).  KLT depth = levels while larger than the 21-px window:
# 640x480 and 752x480 -> 4, 1281x721 -> 4 (5 with max_level 7), 324x246 -> 3, 128x96 -> 2, 64x48 -> 1, 16x16 -> 0.
# Levels the slot pyramid lacks are built in scratch by pyrdown_ptr_kernel: all of them with one slot level, odd sizes at
# 1281x721 and 324x246.
GEOMETRIES = [(640, 480, 1, 4, 10), (640, 480, 3, 4, 10), (640, 480, 5, 4, 10), (640, 480, 8, 4, 10), (752, 480, 4, 4, 10),
              (1281, 721, 1, 4, 20), (1281, 721, 5, 4, 20), (1281, 721, 1, 7, 20), (324, 246, 3, 4, 10), (128, 96, 1, 4, 10),
              (64, 48, 1, 4, 10), (16, 16, 1, 4, 10)]


@pytest.mark.parametrize("w,h,levels,max_level,cell", GEOMETRIES)
def test_klt_geometries_bit_exact(oracle, w, h, levels, max_level, cell):
    """Textured crops with a known shift, points inside and up to 25 px outside the image."""
    from ygz_slam_b200 import Context
    dx, dy = (7, -5) if w >= 300 else (2, -1)
    g1, g2 = synth.shifted_pair(w, h, dx, dy, seed=w + h)
    rng = np.random.default_rng(w * h)
    ref = np.stack([rng.uniform(-25, w + 25, 400), rng.uniform(-25, h + 25, 400)], 1).astype(np.float32)
    ctx = Context(0, image_width=w, image_height=h, n_levels=levels, cell_size=cell)
    try:
        fr = ctx.frames(2)
        fr.upload(np.stack([g1, g2]))
        got, gst, _ = _klt_one(fr, oracle, [g1, g2], 0, 1, ref, ref.copy(), max_level=max_level)
        if w >= 300:   # the known shift is found where the windows lie inside the images
            truth = ref + np.float32([dx, dy])
            clear = gst & ((ref >= 10) & (ref <= np.float32([w - 11, h - 11]))).all(1)
            assert clear.sum() > 100 and np.median(np.abs(got[clear] - truth[clear]).max(1)) < 0.05
        fr.close()
    finally:
        ctx.close()


PARAMS = [dict(max_iter=0), dict(max_iter=1), dict(max_iter=100), dict(max_iter=500), dict(eps=0.0), dict(eps=1e-3),
          dict(eps=20.0), dict(max_level=0), dict(max_level=2), dict(max_level=4), dict(max_level=6), dict(min_eig=0.0),
          dict(min_eig=1e-3)]


@pytest.mark.parametrize("prm", PARAMS, ids=[",".join(f"{k}={v}" for k, v in p.items()) for p in PARAMS])
def test_klt_params_bit_exact(frames3, oracle, prm):
    """Non-default parameters: max_iter 500 is clamped to 100 and eps 20 to 10 on both sides."""
    fr, imgs = frames3
    ref = _features(oracle, imgs[0])
    got = _klt_one(fr, oracle, imgs, 0, 2, ref, ref + np.float32([1.5, -1.0]), **prm)
    assert got[1].mean() > (0.5 if prm.get("min_eig") == 1e-3 else 0.9)


def test_klt_rejects_other_windows(frames3):
    from ygz_slam_b200.capi import YgzbError
    fr, _ = frames3
    ref = np.float32([[100, 100]])
    with pytest.raises(YgzbError, match=r"rc=-1\)"):
        fr.klt([0], [1], [0, 1], ref, ref, win=19)


def test_klt_min_eig_threshold_edge(frames3, oracle):
    """A point whose level-0 minimum eigenvalue is the float f is kept at min_eig = nextafter(double f, +inf), which rounds
    to f, and dropped at the next float above f."""
    fr, imgs = frames3
    ref = _features(oracle, imgs[0])[::40][:20]
    _, _, f = oracle.klt(imgs[0], imgs[1], ref, ref.copy(), max_level=0, exact=True, get_min_eig=True)
    for i in range(len(ref)):
        p = ref[i:i + 1]
        fi = np.float32(f[i])
        assert fi > 0
        keep = _klt_one(fr, oracle, imgs, 0, 1, p, p.copy(), max_level=0, min_eig=np.nextafter(float(fi), np.inf))
        drop = _klt_one(fr, oracle, imgs, 0, 1, p, p.copy(), max_level=0, min_eig=float(np.nextafter(fi, np.float32(np.inf))))
        assert keep[1][0] and not drop[1][0], i


def _border_points(w0, h0, depth):
    """Reference / initial points that put floor(x / 2^L - 10) at -22, -21, -20, w_L - 2, w_L - 1 and w_L (the -win and >= w
    bounds tests) on each axis and at each level L, points at negative coordinates, and coordinates k + 2^-15 and k + 0.5
    at each level, where a bilinear weight (x 2^14) rounds a half."""
    pts = []
    w, h = w0, h0
    for L in range(depth + 1):
        s = float(1 << L)
        xs = [(k + 10.375) * s for k in (-22, -21, -20, w - 2, w - 1, w)]
        ys = [(k + 10.375) * s for k in (-22, -21, -20, h - 2, h - 1, h)]
        pts += [(x, h0 / 2 + 0.3) for x in xs] + [(w0 / 2 - 0.7, y) for y in ys] + list(zip(xs, ys)) + list(zip(xs, ys[::-1]))
        for k in (7, 13):
            for fx in (2.0 ** -15, 0.5):
                for fy in (0.0, 2.0 ** -15, 0.5):
                    pts.append(((k + fx) * s, (k + 3 + fy) * s))
        w, h = (w + 1) // 2, (h + 1) // 2
    pts += [(-0.5, 100.0), (-5.25, -3.75), (-31.0, -31.0), (100.0, -10.5)]
    return np.array(pts, np.float32)


@pytest.mark.parametrize("levels", [3, 8])
def test_klt_border_branches(levels, ctx3, ctx8, oracle, synth_frames):
    ctx = ctx3 if levels == 3 else ctx8
    imgs = [f[0] for f in synth_frames]
    fr = ctx.frames(2)
    fr.upload(np.stack(imgs[:2]))
    edge = _border_points(640, 480, 4)
    inward = np.where(edge < np.float32([320, 240]), np.float32(3), np.float32(-3))
    # the reference point on the edge; the initial point on the edge with the reference 3 px further in
    _klt_one(fr, oracle, imgs, 0, 1, edge, edge.copy())
    _klt_one(fr, oracle, imgs, 0, 1, edge + inward, edge.copy())
    fr.close()


def _content_frames(ctx, kind):
    rng = np.random.default_rng(3)
    if kind == "blocks":      # 0 / 255 blocks 2 wide, 8 tall, alternating along each row with a random phase per block row:
        # |Ix| = 4080 wherever x - 1 and x + 1 lie in one block row, so A11 sums exceed 2^32
        x = np.arange(640)[None, :] // 2
        g1 = (255 * ((x + rng.integers(0, 2, (60, 1)).repeat(8, 0)) % 2)).astype(np.uint8)
        g2 = np.roll(g1, (1, 2), (0, 1))
    elif kind == "flat":
        g1 = g2 = np.full((480, 640), 128, np.uint8)
    else:                     # vertical stripes: the structure tensor is singular
        g1 = np.repeat(rng.integers(0, 256, (1, 640)), 480, 0).astype(np.uint8)
        g2 = np.roll(g1, 3, 1)
    fr = ctx.frames(2)
    fr.upload(np.stack([g1, g2]))
    return fr, [g1, g2]


def _scharr_dx(g):
    p = np.pad(g.astype(np.int64), 1, mode="reflect")
    t = 3 * (p[:-2] + p[2:]) + 10 * p[1:-1]
    return t[:, 2:] - t[:, :-2]


@pytest.mark.parametrize("kind", ["blocks", "flat", "stripes"])
def test_klt_content_extremes(ctx3, oracle, kind):
    fr, imgs = _content_frames(ctx3, kind)
    rng = np.random.default_rng(11)
    ref = np.stack([rng.integers(30, 610, 300), rng.integers(30, 450, 300)], 1).astype(np.float32)   # integer: weights 2^14, 0
    init = ref + np.float32([0.25, -0.5])
    if kind == "blocks":
        dx = _scharr_dx(imgs[0])
        a11 = [int((dx[int(y) - 10:int(y) + 11, int(x) - 10:int(x) + 11] ** 2).sum()) for x, y in ref]
        assert np.abs(dx).max() == 4080 and max(a11) > 2 ** 32
        got = _klt_one(fr, oracle, imgs, 0, 1, ref, init)
        assert got[1].mean() > 0.5   # the stripes alias: not every point finds the true shift
    elif kind == "flat":
        got = _klt_one(fr, oracle, imgs, 0, 1, ref, init)
        assert not got[1].any() and not got[2].any()
    else:
        _, _, f = oracle.klt(imgs[0], imgs[1], ref, init, min_eig=0.0, exact=True, get_min_eig=True)
        assert (f >= 0).any()   # those points pass the eigenvalue test and fail D < FLT_EPSILON
        got = _klt_one(fr, oracle, imgs, 0, 1, ref, init, min_eig=0.0)
        assert not got[1].any()
    fr.close()


def test_klt_ragged_batch(frames3, oracle):
    """Empty first, middle and last pairs, ref == cur, reversed pairs and one slot shared by many pairs in one call: every
    pair equals a one-pair call and the oracle."""
    fr, imgs = frames3
    feats = _features(oracle, imgs[0])
    rng = np.random.default_rng(2)
    pairs = [(0, 1, 0), (0, 1, 150), (1, 0, 120), (2, 2, 100), (1, 2, 0), (0, 2, 90)]
    pairs += [(0, k % 3, 20 + 7 * k) for k in range(8)] + [(k % 3, 0, 15) for k in range(4)] + [(2, 1, 0)]
    refs = [feats[rng.choice(len(feats), n, replace=False)] for _, _, n in pairs]
    inits = [r + rng.uniform(-2, 2, r.shape).astype(np.float32) if a != b else r.copy() for (a, b, _), r in zip(pairs, refs)]
    off = np.concatenate([[0], np.cumsum([n for _, _, n in pairs])]).astype(np.int32)
    got = fr.klt([a for a, _, _ in pairs], [b for _, b, _ in pairs], off, np.concatenate(refs), np.concatenate(inits))
    for p, (a, b, n) in enumerate(pairs):
        s = slice(off[p], off[p + 1])
        one = _klt_one(fr, oracle, imgs, a, b, refs[p], inits[p])
        _assert_same((got[0][s], got[1][s], got[2][s]), (one[0], one[1].astype(np.uint8), one[2]))
        if a == b and n:   # no motion: the flow is zero up to float rounding
            st = got[1][s]
            assert st.mean() > 0.8 and np.abs(got[0][s][st] - refs[p][st]).max() < 1e-4


def test_klt_40000_pairs(frames3, oracle):
    """40,000 one-point pairs on the 3-level context: KLT levels 3 and 4 are built in scratch for 80,000 images (about
    0.5 GB), more than one launch's gridDim.z (65,535) holds."""
    fr, imgs = frames3
    pool = _features(oracle, imgs[0])[:200]
    n = 40000
    k = np.arange(n)
    a, b, pi = k % 3, (k + 1 + (k // 3) % 2) % 3, k % len(pool)
    ref = pool[pi]
    init = ref + np.float32([1.0, -0.5])
    got = fr.klt(a, b, np.arange(n + 1, dtype=np.int32), ref, init)
    want = (np.empty_like(ref), np.empty(n, np.uint8), np.empty(n, np.float32))
    for sa in range(3):
        for sb in range(3):
            m = (a == sa) & (b == sb)
            if m.any():   # each point of the pool once per slot pair
                u, inv = np.unique(pi[m], return_inverse=True)
                wp, ws, we = oracle.klt(imgs[sa], imgs[sb], pool[u], pool[u] + np.float32([1.0, -0.5]), exact=True)
                want[0][m], want[1][m], want[2][m] = wp[inv], ws[inv], we[inv]
    _assert_same(got, want)
    assert got[1].mean() > 0.9
