"""CPU suite: lens undistortion pinned to OpenCV.  tools/undistort_ref.py (numpy, written from the model and OpenCV's fixed-point
rules) must equal cv2.initUndistortRectifyMap(.., CV_16SC2) and cv2.remap bit for bit, live where cv2 is installed and from
tests/golden/cv2_undistort.npz everywhere; the library's host-side ygzb_undistort_map must equal it entry for entry.  Nothing
is loosened: a differing entry fails with the case and the count."""
import hashlib
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import undistort_ref as U  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "cv2_undistort.npz"


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _newK(golden, name):
    return tuple(golden[f"{name}/newK"])


def _mismatches(xy, a, want_xy, want_a):
    return int((xy != want_xy).any(-1).sum() + (a != want_a).sum())


def _Kmat(k):
    return np.array([[k[0], 0, k[2]], [0, k[1], k[3]], [0, 0, 1]], np.float64)


# ---- maps -----------------------------------------------------------------------------------------------------------
def test_reference_maps_match_golden_digests(golden):
    bad = []
    for name, (w, h, K, D, _) in U.CASES.items():
        xy, a = U.undistort_map(w, h, K, D, _newK(golden, name))
        want = golden[f"{name}/sha"]
        if _sha(xy) != want[0] or _sha(a) != want[1]:
            bad.append(name)
    assert not bad, f"maps differ from cv2's digests: {bad}"


def test_reference_maps_match_golden_small(golden):
    for name in U.SMALL:
        w, h, K, D, newK = U.small_case(name)
        xy, a = U.undistort_map(w, h, K, D, newK)
        n = _mismatches(xy, a, golden[f"{name}/map_xy"], golden[f"{name}/map_a"])
        assert n == 0, f"{name}: {n} entries differ from cv2"


def test_reference_maps_match_cv2_live():
    cv2 = pytest.importorskip("cv2")
    counts = {}
    for name, (w, h, K, D, newK) in U.CASES.items():
        if isinstance(newK, str):
            m, _ = cv2.getOptimalNewCameraMatrix(_Kmat(K), np.array(D), (w, h), float(newK[-1]), (w, h))
            newK = (m[0, 0], m[1, 1], m[0, 2], m[1, 2])
        nk = K if newK is None else newK
        m1, m2 = cv2.initUndistortRectifyMap(_Kmat(K), np.array(D, np.float64), None, _Kmat(nk), (w, h), cv2.CV_16SC2)
        xy, a = U.undistort_map(w, h, K, D, newK)
        counts[name] = _mismatches(xy, a, m1, m2)
    assert not any(counts.values()), f"entries differing from cv2 per case: {counts}"


def test_library_map_equals_reference(golden):
    """ygzb_undistort_map (host code of the library: no device needed) against the restatement, every case."""
    from ygz_slam_b200 import capi
    counts = {}
    for name, (w, h, K, D, _) in U.CASES.items():
        nk = _newK(golden, name)
        xy, a = capi.undistort_map(w, h, K, D, nk)
        counts[name] = _mismatches(xy, a, *U.undistort_map(w, h, K, D, nk))
    assert not any(counts.values()), f"entries differing per case: {counts}"
    # newK None = K, and the 4-coefficient model of the reference's camera (k3 = 0)
    w, h, K, D, _ = U.CASES["tum_fr2"]
    xy, a = capi.undistort_map(w, h, K, D[:4])
    assert _mismatches(xy, a, *U.undistort_map(w, h, K, D[:4] + (0.0,))) == 0


def test_library_map_rejects_bad_input():
    from ygz_slam_b200 import capi
    with pytest.raises(capi.YgzbError):
        capi.undistort_map(0, 480, (500.0, 500.0, 320.0, 240.0), (0.1, 0, 0, 0))
    with pytest.raises(capi.YgzbError):
        capi.undistort_map(640, 480, (500.0, 500.0, 320.0, 240.0), (0.1, 0, 0, 0), newK=(0.0, 500.0, 320.0, 240.0))


# ---- remap ----------------------------------------------------------------------------------------------------------
def test_weight_table():
    tab = U.weight_table()
    assert tab.shape == (1024, 4) and (tab.sum(1) == 1 << 15).all()
    fx, fy = np.arange(1024) & 31, np.arange(1024) >> 5
    exact = 32 * np.stack([(32 - fx) * (32 - fy), fx * (32 - fy), (32 - fx) * fy, fx * fy], 1)
    # every entry is the exact product except entry 0, whose 2^15 does not fit OpenCV's int16 table
    assert (tab[1:] == exact[1:]).all() and list(tab[0]) == [32767, 0, 0, 1]


def test_reference_remap_matches_golden(golden):
    seeds = golden["seeds"]
    for name, (w, h, K, D, _) in U.CASES.items():
        xy, a = U.undistort_map(w, h, K, D, _newK(golden, name))
        want = golden[f"{name}/sha"]
        assert _sha(U.remap_gray(U.seeded_image(int(seeds[0]), h, w), xy, a)) == want[2], f"{name}: grey remap"
        assert _sha(U.undistort_image(U.seeded_image(int(seeds[1]), h, w, 3), xy, a)) == want[3], f"{name}: BGR remap"
    for name in U.SMALL:
        w, h, K, D, newK = U.small_case(name)
        xy, a = golden[f"{name}/map_xy"], golden[f"{name}/map_a"]
        got = U.remap_gray(U.seeded_image(int(seeds[0]), h, w), xy, a)
        assert (got != golden[f"{name}/remap_grey"]).sum() == 0, name
        got = U.undistort_image(U.seeded_image(int(seeds[1]), h, w, 3), xy, a)
        assert (got != golden[f"{name}/remap_bgr"]).sum() == 0, name


def every_weight_map(w, h, seed=7):
    """A map that visits all 1024 weight entries, with taps straddling every image edge and lying wholly outside."""
    rng = np.random.default_rng(seed)
    xy = np.stack([rng.integers(-3, w + 2, (h, w)), rng.integers(-3, h + 2, (h, w))], -1).astype(np.int16)
    a = rng.integers(0, 1024, (h, w)).astype(np.uint16)
    a.reshape(-1)[:1024] = np.arange(1024)
    # every edge: the row above / below and the column left / right of the image, each with every fraction
    edges = [(-1, None), (w - 1, None), (None, -1), (None, h - 1)]
    for k, (ex, ey) in enumerate(edges):
        sl = slice(1024 + 1024 * k, 2048 + 1024 * k)
        n = len(a.reshape(-1)[sl])
        a.reshape(-1)[sl] = np.arange(n) % 1024
        if ex is not None:
            xy.reshape(-1, 2)[sl, 0] = ex
        if ey is not None:
            xy.reshape(-1, 2)[sl, 1] = ey
    return xy, a


def test_reference_remap_matches_cv2_live():
    cv2 = pytest.importorskip("cv2")
    h, w = 121, 161
    xy, a = every_weight_map(w, h)
    rng = np.random.default_rng(3)
    images = {"random": rng.integers(0, 256, (h, w), dtype=np.uint8), "flat_0": np.zeros((h, w), np.uint8),
              "flat_255": np.full((h, w), 255, np.uint8)}
    counts = {}
    for name, img in images.items():
        want = cv2.remap(img, xy, a, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
        counts[name] = int((U.remap_gray(img, xy, a) != want).sum())
    bgr = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    want = cv2.remap(cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY), xy, a, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    counts["bgr"] = int((U.undistort_image(bgr, xy, a) != want).sum())
    assert not any(counts.values()), f"pixels differing from cv2.remap: {counts}"
    for name, (w2, h2, K, D, newK) in list(U.CASES.items())[:3]:   # real maps on real-sized seeded images
        m1, m2 = cv2.initUndistortRectifyMap(_Kmat(K), np.array(D), None, _Kmat(K), (w2, h2), cv2.CV_16SC2)
        img = U.seeded_image(11, h2, w2)
        want = cv2.remap(img, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
        assert (U.remap_gray(img, m1, m2) != want).sum() == 0, name


def test_every_weight_map_covers_table_and_edges():
    xy, a = every_weight_map(161, 121)
    assert len(np.unique(a)) == 1024
    x, y = xy[..., 0], xy[..., 1]
    assert (x == -1).any() and (x == 160).any() and (y == -1).any() and (y == 120).any() and (x < -1).any() and (y > 120).any()


# ---- the tracking loop on lens-rendered streams ------------------------------------------------------------------------
# Ground-truth bound of the loop on frames rendered through TUM fr2's lens (synth.lens_stream_frame, stream 0, every 2nd frame
# of 20, key-frames every >= 5 frames at 0.03) with undistortion on.  Measured on the CPU oracle: worst se3 error 1.08e-3
# with undistortion, 7.4e-3 without it (the raw frames tracked as if the camera were a pinhole).
LENS_LOOP_BOUND = 2e-3
LENS_KW = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)


def lens_frames(n_streams, n_frames):
    from ygz_slam_b200 import synth
    fr = [[synth.lens_stream_frame(2 * k, stream=s) for k in range(n_frames)] for s in range(n_streams)]
    return [[f[0] for f in x] for x in fr], [[f[1] for f in x] for x in fr], [[f[2] for f in x] for x in fr]


def lens_maps():
    from ygz_slam_b200 import synth
    return U.undistort_map(640, 480, (synth.FX, synth.FY, synth.CX, synth.CY), synth.LENS_TUM_FR2)


def run_loop(backend, frames, depths, gts):
    """The Python tracking loop; returns it, the trajectories (S, n, 3, 4) and the per-frame ground-truth error (nan: lost)."""
    from ygz_slam_b200 import se3, vo
    S, n = len(frames), len(frames[0])
    V = vo.VisualOdometry(backend, S, **LENS_KW)
    traj, errs = np.zeros((S, n, 3, 4)), np.full((S, n), np.nan)
    for k in range(n):
        V.add_frames([frames[s][k] for s in range(S)], [depths[s][k] for s in range(S)], k)
        for s in range(S):
            st = V.streams[s]
            if not st.lost:
                traj[s, k] = st.T_cw
                errs[s, k] = float(np.linalg.norm(se3.se3_log(se3.mul(st.T_cw, se3.inv(se3.mul(gts[s][k], se3.inv(gts[s][0])))))))
    return V, traj, errs


def test_lens_depth_is_the_undistorted_cameras():
    """The depth map of a lens-rendered frame is that of the pinhole camera with the same K (the undistorted camera)."""
    from ygz_slam_b200 import synth
    _, depth, T = synth.lens_stream_frame(6)
    _, want = synth.render_plane(synth.texture(0x59475A00, 2048), T)
    assert np.allclose(depth, want, rtol=0, atol=1e-12)
    # the renderer's inverse lens model reproduces the forward model
    u, v = np.meshgrid(np.arange(0, 640, 37.0), np.arange(0, 480, 29.0))
    x, y = synth.undistort_rays(u, v, synth.LENS_TUM_FR2)
    k1, k2, p1, p2, k3 = synth.LENS_TUM_FR2
    r2 = x * x + y * y
    kr = 1 + ((k3 * r2 + k2) * r2 + k1) * r2
    assert np.abs(synth.FX * (x * kr + 2 * p1 * x * y + p2 * (r2 + 2 * x * x)) + synth.CX - u).max() < 1e-6


def test_oracle_loop_on_lens_streams_with_undistortion(oracle):
    from oracle.vo_backend import OracleBackend
    frames, depths, gts = lens_frames(1, 20)
    xy, a = lens_maps()
    V, _, errs = run_loop(U.UndistortingBackend(OracleBackend(oracle), xy, a), frames, depths, gts)
    assert not V.streams[0].lost and V.streams[0].stats["keyframes"] >= 3
    worst = float(np.nanmax(errs))
    _, _, raw_errs = run_loop(OracleBackend(oracle), frames, depths, gts)
    print(f"worst ground-truth error: {worst:.3e} undistorted, {np.nanmax(raw_errs):.3e} raw")
    assert worst < LENS_LOOP_BOUND
    assert np.nanmax(raw_errs) > 2 * worst
