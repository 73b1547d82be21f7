#!/usr/bin/env python3
"""Generates tests/golden/cv2_raw_frames.npz: OpenCV's resampling of raw frames whose size is not the pipeline's, so that
tests/test_vo_raw_frames.py can pin tools/undistort_ref.py (and through it ygzb_undistort_map and the device remap of a
stream's raw frames) without cv2.

A stream whose camera delivers raw frames of another size than the pipeline's W x H is resampled with maps of the OUTPUT's
size, built from the raw camera's K and the stream's camera as newK; only the remap reads the raw frame:
    cv2.initUndistortRectifyMap(K_raw, D, None, newK, (W, H), CV_16SC2), then cv2.remap(raw, .., INTER_LINEAR,
    BORDER_CONSTANT, 0), a BGR raw frame converted with cvtColor(BGR2GRAY) first.
  - every case of CASES: SHA-256 of the two maps and of the remaps of a PCG64-seeded grey and BGR raw frame of the raw
    size (undistort_ref.seeded_image);
  - the small cases of SMALL: the maps and the two remaps in full.
Run once here (cv2 4.13.0): python tools/make_raw_frame_fixture.py"""
import hashlib
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import undistort_ref as U  # noqa: E402

GREY_SEED, BGR_SEED = 3024, 3025
OUT = (640, 480)   # the pipeline's size in every full-size case

# name -> (raw width, raw height, K_raw = (fx, fy, cx, cy), D = (k1, k2, p1, p2, k3), newK = the stream's camera at OUT)
CASES = {
    # an HD lens scaled 1.5x down into 640 x 480 (its 16:9 view cropped at the sides)
    "hd_1280x720_scale": (1280, 720, (780.0, 780.0, 639.5, 359.5), (0.05, -0.1, 0.0005, -0.0003, 0.0), (520.9, 521.0, 325.1, 249.7)),
    # EuRoC's cam0 with its radial-tangential coefficients, cropped to 640 x 480 at the same focal length
    "euroc_752x480_crop": (752, 480) + U.EUROC_CAM0 + ((458.0, 457.0, 320.0, 240.0),),
    # TUM fr2's lens at half resolution, upsampled 2x
    "qvga_320x240_up": (320, 240, (260.45, 260.5, 162.55, 124.85), U.TUM_FR2[1], U.TUM_FR2[0]),
    # odd raw size: the remap's row length and bounds are the raw frame's, not a multiple of anything
    "odd_753x481": (753, 481, (460.0, 459.0, 376.3, 240.7), U.EUROC_CAM0[1], (450.0, 450.0, 320.0, 240.0)),
    # a raw view narrower than the output's: the outer rows and columns sample outside the raw frame and read 0
    "narrow_400x300_outside": (400, 300, (500.0, 500.0, 199.5, 149.5), (0.0,) * 5, (400.0, 400.0, 319.5, 239.5)),
}
# name -> (output width, output height) + a case of the same form: maps and remaps stored in full
SMALL = {
    "small_161x121_to_96x72": ((96, 72), (161, 121, (130.0, 130.0, 80.3, 60.1), U.TUM_FR1[1], (78.0, 78.0, 47.5, 35.5))),
    "small_48x36_to_96x72": ((96, 72), (48, 36, (40.0, 40.0, 23.5, 17.5), (0.1, -0.05, 0.0, 0.0, 0.0), (60.0, 60.0, 47.5, 35.5))),
}


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def Kmat(k):
    return np.array([[k[0], 0, k[2]], [0, k[1], k[3]], [0, 0, 1]], np.float64)


def cv2_case(out, rw, rh, K, D, newK):
    import cv2   # (here, so that the tests can read CASES where cv2 is not installed)
    m1, m2 = cv2.initUndistortRectifyMap(Kmat(K), np.array(D, np.float64), None, Kmat(newK), out, cv2.CV_16SC2)
    grey = U.seeded_image(GREY_SEED, rh, rw)
    bgr = U.seeded_image(BGR_SEED, rh, rw, 3)
    r_grey = cv2.remap(grey, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    r_bgr = cv2.remap(cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY), m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    return m1, m2, r_grey, r_bgr


if __name__ == "__main__":
    import cv2
    out = {"cv2_version": np.array(cv2.__version__), "seeds": np.array([GREY_SEED, BGR_SEED])}
    for name, case in CASES.items():
        m1, m2, rg, rb = cv2_case(OUT, *case)
        out[f"{name}/sha"] = np.array([sha(m1), sha(m2), sha(rg), sha(rb)])
        inside = (m1[..., 0] >= 0) & (m1[..., 0] < case[0] - 1) & (m1[..., 1] >= 0) & (m1[..., 1] < case[1] - 1)
        print(name, "map range", m1.min(), m1.max(), "inside", round(float(inside.mean()), 4))
    for name, (size, case) in SMALL.items():
        m1, m2, rg, rb = cv2_case(size, *case)
        out[f"{name}/map_xy"], out[f"{name}/map_a"], out[f"{name}/remap_grey"], out[f"{name}/remap_bgr"] = m1, m2, rg, rb
    np.savez_compressed(ROOT / "tests" / "golden" / "cv2_raw_frames.npz", **out)
    print("wrote", ROOT / "tests" / "golden" / "cv2_raw_frames.npz")
