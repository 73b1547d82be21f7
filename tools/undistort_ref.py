"""cv2-free restatement of OpenCV's lens undistortion, the checker of ygzb_undistort_map and the device remap (TEST
INFRASTRUCTURE, shared by tests/test_undistort.py, tests/test_gpu_undistort.py and tools/make_undistort_fixture.py).

Written from the model and OpenCV's fixed-point rules, in numpy, independently of the library's C and CUDA code:
  cv::initUndistortRectifyMap(K, D, R = I, newK, size, CV_16SC2), D = (k1, k2, p1, p2, k3):
      newK^-1 by the cofactor formula of cv::invert for 3x3 (d = 1 / det, cofactors times d); per row the homogeneous
      ray (_x, _y, _w) = iR (0, i, 1), per column _x advanced by iR[0][0] (OpenCV's scalar loop); x = _x / _w ...;
      kr = 1 + ((k3 r2 + k2) r2 + k1) r2; u = fx (x kr + 2 p1 x y + p2 (r2 + 2 x^2)) + cx (v likewise);
      cvRound(u * 32) split into u >> 5 (CV_16SC2) and the 5-bit fractions (fy << 5 | fx, CV_16UC1).
  cv::remap(src, map_xy, map_a, INTER_LINEAR, BORDER_CONSTANT, 0) on 8-bit images: OpenCV's 1024-entry table of
      2^15-scaled bilinear weights (float products (1 - x)(1 - y) .., saturated to int16, the rounding corrected so
      that every entry sums to 2^15), result (sum w p + 2^14) >> 15, taps outside the image = 0.
  cv::cvtColor(BGR2GRAY): (B 3735 + G 19235 + R 9798 + 2^14) >> 15.
"""
from fractions import Fraction

import numpy as np

# camera cases of the tests and the fixture: name -> (width, height, K = (fx, fy, cx, cy), D = (k1, k2, p1, p2, k3), newK
# or None = K, or "alpha0" / "alpha1" = cv2.getOptimalNewCameraMatrix at that alpha, stored in the fixture)
TUM_FR1 = ((517.3, 516.5, 318.6, 255.3), (0.2624, -0.9531, -0.0054, 0.0026, 1.1633))
TUM_FR2 = ((520.9, 521.0, 325.1, 249.7), (0.2312, -0.7849, -0.0033, -0.0001, 0.9172))
EUROC_CAM0 = ((458.654, 457.296, 367.215, 248.375), (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0))
CASES = {
    "tum_fr1": (640, 480) + TUM_FR1 + (None,),
    "tum_fr2": (640, 480) + TUM_FR2 + (None,),
    "euroc_cam0": (752, 480) + EUROC_CAM0 + (None,),
    "zero": (640, 480, (517.3, 516.5, 318.6, 255.3), (0.0, 0.0, 0.0, 0.0, 0.0), None),
    # barrel (k1 < 0) seen through a wider undistorted camera: the corners sample far outside the raw image
    "barrel": (640, 480, (300.0, 300.0, 320.0, 240.0), (-0.3, 0.08, 0.001, -0.002, 0.0), (240.0, 240.0, 330.0, 235.0)),
    "pincushion": (640, 480, (500.0, 500.0, 319.5, 239.5), (0.35, 0.1, 0.0, 0.0, 0.05), None),
    "tum_fr1_alpha0": (640, 480) + TUM_FR1 + ("alpha0",),
    "tum_fr1_alpha1": (640, 480) + TUM_FR1 + ("alpha1",),
    "odd_321x241": (321, 241, (260.0, 259.0, 160.3, 120.9), (0.2, -0.5, 0.001, 0.002, 0.3), None),
    # binary-exact camera and coefficients: many u * 32 land on or next to rounding ties, where OpenCV's fused multiply-adds
    # decide; odd sizes exercise the scalar tail of its 8-column loop
    "exact_ties_643x483": (643, 483, (400.0, 400.0, 320.0, 240.0), (0.25, -0.125, 0.0, 0.0, 0.0), (200.0, 200.0, 321.0, 241.0)),
    # a polynomial that explodes inside a wide undistorted view: most samples lie beyond +-32767 px and saturate
    "saturating": (640, 480, (500.0, 500.0, 320.0, 240.0), (2.0, 5.0, 0.0, 0.0, 10.0), (100.0, 100.0, 320.0, 240.0)),
}
# small geometries whose full maps and remaps are stored in the fixture (TUM fr1 scaled to the size)
SMALL = {"small_96x72": (96, 72), "small_161x121": (161, 121)}


def small_case(name):
    w, h = SMALL[name]
    (fx, fy, cx, cy), D = TUM_FR1
    s = w / 640.0
    return w, h, (fx * s, fy * s, cx * s, cy * s), D, None


def _fma(a, b, c):
    """a * b + c rounded once (exact rationals; float() of a Fraction rounds to nearest, ties to even)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def undistort_map(width, height, K, D, newK=None):
    """(map_xy (H, W, 2) int16, map_a (H, W) uint16) of cv::initUndistortRectifyMap(.., CV_16SC2) as OpenCV's x86-64 build
    computes it: its AVX2 loop takes 8 columns per step (_x = start of the group + k iR00, the group start advanced by 8 iR00,
    a scalar tail advanced by iR00) and fuses the row start and the distortion polynomial into multiply-adds.  numpy has no
    fused multiply-add, so the map is computed with plain operations first; fusing changes u or v by a few units in the last
    place, which can only move a value that lies within 1e-6 of a rounding tie of u * 32 or v * 32, and those pixels are
    computed again with exactly rounded multiply-adds."""
    fx, fy, u0, v0 = (float(v) for v in K)
    afx, afy, acx, acy = (float(v) for v in (K if newK is None else newK))
    k1, k2, p1, p2, k3 = (float(v) for v in (tuple(D) + (0.0,) * 5)[:5])
    d = 1.0 / (afx * afy)
    ir0, ir2 = afy * d, -(acx * afy) * d
    ir4, ir5, ir8 = afx * d, -(afx * acy) * d, (afx * afy) * d
    full = width // 8 * 8
    starts = np.add.accumulate(np.concatenate([[ir2], np.full(width // 8, 8 * ir0)]))
    _x = np.empty(width)
    _x[:full] = (starts[:width // 8, None] + np.arange(8) * ir0).reshape(-1)
    _x[full:] = np.add.accumulate(np.concatenate([[starts[width // 8]], np.full(max(width - full - 1, 0), ir0)]))[:width - full]
    w = 1.0 / ir8
    xc = _x * w
    _y = np.arange(height, dtype=np.float64)[:, None] * ir4 + ir5
    x = np.broadcast_to(xc[None, :], (height, width))
    y = np.broadcast_to(_y * w, (height, width))
    x2, y2 = x * x, y * y
    r2 = x2 + y2
    _2xy = 2 * x * y
    kr = 1 + ((k3 * r2 + k2) * r2 + k1) * r2
    su = (fx * (x * kr + p1 * _2xy + p2 * (r2 + 2 * x2)) + u0) * 32
    sv = (fy * (y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy) + v0) * 32
    near = (np.abs(su - np.floor(su) - 0.5) < 1e-6) | (np.abs(sv - np.floor(sv) - 0.5) < 1e-6)
    for i, j in np.argwhere(near):
        yy = _fma(float(i), ir4, ir5) * w
        xx = float(xc[j])
        xx2, yy2 = xx * xx, yy * yy
        rr2 = xx2 + yy2
        t2xy = 2 * xx * yy
        k = _fma(_fma(_fma(k3, rr2, k2), rr2, k1), rr2, 1.0)
        xd = _fma(p2, rr2 + 2 * xx2, _fma(p1, t2xy, xx * k))
        yd = _fma(p2, t2xy, _fma(p1, rr2 + 2 * yy2, yy * k))
        su[i, j] = _fma(fx, xd, u0) * 32
        sv[i, j] = _fma(fy, yd, v0) * 32
    iu = np.rint(np.clip(su, -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)    # cvRound: half to even
    iv = np.rint(np.clip(sv, -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)
    # the integer pixel saturates to int16 (saturate_cast<short>): a ray far outside stays outside the image
    map_xy = np.clip(np.stack([iu >> 5, iv >> 5], -1), -32768, 32767).astype(np.int16)
    map_a = ((iv & 31) * 32 + (iu & 31)).astype(np.uint16)
    return map_xy, map_a


def weight_table():
    """(1024, 4) int64: OpenCV's fixed-point bilinear table, entry fy * 32 + fx, taps (x, y), (x + 1, y), (x, y + 1), (x + 1, y + 1)."""
    t1 = np.arange(32, dtype=np.float32) / np.float32(32)
    tab = np.zeros((1024, 4), np.int64)
    for i in range(32):
        for j in range(32):
            vy = (np.float32(1) - t1[i], t1[i])
            vx = (np.float32(1) - t1[j], t1[j])
            w = [int(np.clip(np.rint(np.float32(vy[k1] * vx[k2]) * np.float32(32768)), -32768, 32767)) for k1 in (0, 1) for k2 in (0, 1)]
            diff = sum(w) - 32768
            if diff:   # only entry 0 (1.0 saturates to 32767): the missing unit goes to the smallest tap
                k = int(np.argmin(w[::-1]))
                w[3 - k] -= diff
            tab[i * 32 + j] = w
    return tab


_TAB = None


def remap_gray(img, map_xy, map_a):
    """cv::remap(img, map_xy, map_a, INTER_LINEAR, BORDER_CONSTANT, 0) of a grey uint8 image."""
    global _TAB
    if _TAB is None:
        _TAB = weight_table()
    img = np.asarray(img, np.uint8)
    H, W = img.shape
    sx = map_xy[..., 0].astype(np.int64)
    sy = map_xy[..., 1].astype(np.int64)
    w = _TAB[np.asarray(map_a, np.int64) & 1023]

    def tap(x, y):
        inside = (x >= 0) & (x < W) & (y >= 0) & (y < H)
        return np.where(inside, img[np.clip(y, 0, H - 1), np.clip(x, 0, W - 1)].astype(np.int64), 0)

    s = w[..., 0] * tap(sx, sy) + w[..., 1] * tap(sx + 1, sy) + w[..., 2] * tap(sx, sy + 1) + w[..., 3] * tap(sx + 1, sy + 1)
    return ((s + (1 << 14)) >> 15).astype(np.uint8)


def bgr2gray(bgr):
    b, g, r = (bgr[..., k].astype(np.int64) for k in range(3))
    return ((b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15).astype(np.uint8)


def undistort_image(img, map_xy, map_a):
    """Level 0 of an undistorting upload: remap of the grey image, or of cvtColor(BGR2GRAY) of a (H, W, 3) image."""
    img = np.asarray(img, np.uint8)
    return remap_gray(bgr2gray(img) if img.ndim == 3 else img, map_xy, map_a)


def seeded_image(seed, height, width, channels=1):
    """The fixture's test images: uniform bytes from numpy's PCG64."""
    shape = (height, width) if channels == 1 else (height, width, channels)
    return np.random.Generator(np.random.PCG64(seed)).integers(0, 256, shape, dtype=np.uint8)


class UndistortingBackend:
    """A tracking-loop backend (ygz_slam_b200.vo) whose uploads are undistorted on the host first: wraps the CPU oracle's
    OracleBackend, so that the oracle loop runs on the same undistorted frames as a GpuBackend with maps."""

    def __init__(self, inner, map_xy, map_a):
        self.inner, self.map_xy, self.map_a = inner, map_xy, map_a

    def upload(self, slots, images):
        self.inner.upload(slots, [undistort_image(im, self.map_xy, self.map_a) for im in images])

    def __getattr__(self, name):
        return getattr(self.inner, name)
