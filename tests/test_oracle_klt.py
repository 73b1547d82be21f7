"""CPU suite: the KLT restatement against cv2.calcOpticalFlowPyrLK (the reference's own dependency)."""
import numpy as np
import pytest

from ygz_slam_b200 import synth

cv2 = pytest.importorskip("cv2")

def _points(oracle, synth_frames, shift):
    g1 = synth_frames[0][0]
    f = oracle.detect(oracle.build_pyramid(g1, 3))
    ref = np.stack([f["px"], f["py"]], 1).astype(np.float32)
    # also a few points near / outside the border
    extra = np.array([[2.5, 3.0], [637.0, 10.0], [320.0, 478.5], [-30.0, 50.0], [700.0, 500.0]], np.float32)
    ref = np.concatenate([ref, extra])
    return ref, (ref + np.float32(shift)).astype(np.float32)


def _grid_points(w, h, n, seed):
    """n seeded points inside the image.  (Points whose window is mostly outside are ill-conditioned: there the two f32
    summation orders can drift apart by tenths of a pixel.  The GPU suite covers them bit for bit.)"""
    rng = np.random.default_rng(seed)
    return np.stack([rng.uniform(0, w - 1, n), rng.uniform(0, h - 1, n)], 1).astype(np.float32)


def _cv2_klt(g1, g2, ref, init, max_level=4, max_iter=30, eps=0.001, min_eig=1e-4, flags=0):
    p, s, e = cv2.calcOpticalFlowPyrLK(g1, g2, ref.copy(), init.copy(), winSize=(21, 21), maxLevel=max_level,
                                       criteria=(cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, max_iter, eps),
                                       flags=cv2.OPTFLOW_USE_INITIAL_FLOW | flags, minEigThreshold=min_eig)
    return p.reshape(-1, 2), s.reshape(-1).astype(bool), e.reshape(-1)


# -> image pair, reference and initial points, oracle / cv2 parameters, known flow (or None), least fraction tracked
def _case(kind, oracle, synth_frames):
    prm = {}
    truth = None
    if kind.startswith("size-") or kind == "large-shift":
        # noise-free shifted crops, so the flow is known: other image sizes (odd levels, other depths: 324x246 stops at
        # level 3, 64x48 at level 1), or a shift of tens of pixels that only the coarse levels can find
        w, h, dx, dy = (640, 480, 37, -26) if kind == "large-shift" else (*map(int, kind[5:].split("x")), 3, -2)
        g1, g2 = synth.shifted_pair(w, h, dx, dy, seed=w, noise=0)
        ref = _grid_points(w, h, 400, w)
        init, truth = ref.copy(), ref + np.float32([dx, dy])
        return g1, g2, ref, init, prm, truth, (0.6 if w < 100 else 0.8)   # flat patches fail the min-eigenvalue test
    else:                                          # the tracker's frames 1 -> 3, initial flow off by 1.5 px
        g1, g2 = synth_frames[0][0], synth_frames[2][0]
        shift = 1.5
        if kind in ("0.0", "1.5", "-4.0"):
            shift = float(kind)
        else:
            name, v = kind.split("=")
            prm[name] = float(v) if name == "eps" else int(v)
        ref, init = _points(oracle, synth_frames, shift)
    return g1, g2, ref, init, prm, truth, 0.9


CASES = ["0.0", "1.5", "-4.0", "size-752x480", "size-1281x721", "size-324x246", "size-128x96", "size-64x48", "large-shift",
         "max_iter=0", "max_iter=1", "max_iter=100", "max_iter=500", "eps=0", "eps=0.001", "eps=20",
         "max_level=0", "max_level=2", "max_level=4", "max_level=6"]


@pytest.mark.parametrize("case", CASES)
def test_klt_matches_cv2(oracle, synth_frames, case):
    g1, g2, ref, init, prm, truth, min_tracked = _case(case, oracle, synth_frames)
    want, wst, werr = _cv2_klt(g1, g2, ref, init, **prm)
    got, gst, gerr = oracle.klt(g1, g2, ref, init, **prm)
    gst = gst.astype(bool)
    assert (wst != gst).mean() < 0.005
    both = wst & gst
    d = np.abs(got[both] - want[both]).max(1)
    # OpenCV's SIMD build accumulates the f32 normal equations in a different order: tiny differences
    assert np.percentile(d, 99) < 0.01 and np.median(d) < 1e-3
    # err is taken at the final position: it agrees wherever the positions do.  On the tracker's frames that is every point;
    # the noise-free crops have a few near-singular windows (straight edges of flat shapes) that settle apart
    close = d <= 0.01
    assert close.all() or truth is not None
    assert np.abs(gerr[both][close] - werr[both][close]).max() < 0.05
    inside = ((ref >= 0) & (ref < np.float32(g1.shape[::-1]))).all(1)
    assert both.sum() > min_tracked * inside.sum()
    if truth is not None:   # where both windows lie inside the images, the known shift is found
        lo, hi = np.float32(10), np.float32(g1.shape[::-1]) - 11
        clear = both & ((ref >= lo) & (ref <= hi) & (truth >= lo) & (truth <= hi)).all(1)
        e = np.abs(got[clear] - truth[clear]).max(1)
        assert clear.sum() > 20 and np.median(e) < 0.01 and np.percentile(e, 90) < 0.05, (np.median(e), np.percentile(e, 90))


def test_klt_min_eig_threshold_is_float(oracle, synth_frames):
    """OpenCV keeps minEigThreshold as a float: a point whose level-0 minimum eigenvalue is the float f survives the
    thresholds f and nextafter(double f, +inf) (both round to f) and is dropped at the next float above f."""
    g1, g2 = synth_frames[0][0], synth_frames[1][0]
    pts = _grid_points(640, 480, 400, 5)
    _, _, f = _cv2_klt(g1, g2, pts, pts, max_level=0, flags=cv2.OPTFLOW_LK_GET_MIN_EIGENVALS)
    _, _, of = oracle.klt(g1, g2, pts, pts.copy(), max_level=0, get_min_eig=True)
    same = np.nonzero(of == f)[0][:20]     # points where both sides computed the same f32 eigenvalue
    assert len(same) == 20
    for i in same:
        p = pts[i:i + 1]
        fi = np.float32(f[i])
        for thr, keep in ((float(fi), True), (np.nextafter(float(fi), np.inf), True),
                          (float(np.nextafter(fi, np.float32(np.inf))), False)):
            _, cs, _ = _cv2_klt(g1, g2, p, p, max_level=0, min_eig=thr)
            _, os_, _ = oracle.klt(g1, g2, p, p.copy(), max_level=0, min_eig=thr)
            assert cs[0] == keep and bool(os_[0]) == keep, (i, float(fi), thr)


@pytest.mark.parametrize("exact", [False, True])
def test_klt_min_eig_output_matches_cv2(oracle, synth_frames, exact):
    """get_min_eig writes the level-0 minimum eigenvalue like OPTFLOW_LK_GET_MIN_EIGENVALS.  Both sides round the window
    sums to f32 (in different orders, or once at the end in the exact mode): measured relative difference < 3e-5."""
    g1, g2 = synth_frames[0][0], synth_frames[1][0]
    pts = np.concatenate([_grid_points(640, 480, 400, 9), np.float32([[-40, 10], [700, 300]])])
    _, _, f = _cv2_klt(g1, g2, pts, pts, max_level=0, flags=cv2.OPTFLOW_LK_GET_MIN_EIGENVALS)
    _, _, of = oracle.klt(g1, g2, pts, pts.copy(), max_level=0, get_min_eig=True, exact=exact)
    assert f[-2:].tolist() == [0, 0] and of[-2:].tolist() == [0, 0]     # outside at level 0: err = 0
    nz = f > 0
    assert nz.sum() > 350
    assert np.abs(of[nz] / f[nz] - 1).max() < 1e-4
    assert np.array_equal(of == 0, f == 0)


@pytest.mark.parametrize("kind", ["1.5", "-4.0", "large-shift", "size-1281x721", "max_level=0"])
def test_klt_exact_sums_close_to_f32(oracle, synth_frames, kind):
    """The exact-sum mode (the GPU's arithmetic) changes the result only within the tolerance the cv2 pin allows."""
    g1, g2, ref, init, prm = _case(kind, oracle, synth_frames)[:5]
    a, ast, aerr = oracle.klt(g1, g2, ref, init, **prm)
    b, bst, berr = oracle.klt(g1, g2, ref, init, exact=True, **prm)
    assert (ast != bst).mean() < 0.003
    both = (ast & bst).astype(bool)
    d = np.abs(a[both] - b[both]).max(1)
    assert np.percentile(d, 99) < 0.01 and np.median(d) < 1e-3
    close = d <= 0.01
    if kind != "large-shift":   # see test_klt_matches_cv2: the crops have a few near-singular windows
        assert d.max() < 5e-3
    assert np.abs(aerr[both][close] - berr[both][close]).max() < 0.05
