#!/usr/bin/env python3
"""Generates tests/golden/cv2_undistort.npz: OpenCV's undistortion maps and remaps, so that tests/test_undistort.py can pin
tools/undistort_ref.py (and through it ygzb_undistort_map and the device remap) without cv2.

  - every camera case of undistort_ref.CASES: the newK the case uses (cv2.getOptimalNewCameraMatrix for the alpha cases),
    SHA-256 of cv2.initUndistortRectifyMap(K, D, None, newK, size, CV_16SC2)'s two maps, and SHA-256 of cv2.remap(INTER_LINEAR,
    BORDER_CONSTANT, 0) of a PCG64-seeded grey image and of cvtColor(BGR2GRAY) of a seeded BGR image through them;
  - the small geometries of undistort_ref.SMALL: the maps and the two remaps in full.
Full 640 x 480 maps would be 1.8 MB each; the digests keep the file small.
Run once here (cv2 4.13.0): python tools/make_undistort_fixture.py"""
import hashlib
import sys
from pathlib import Path

import cv2
import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import undistort_ref as U  # noqa: E402

GREY_SEED, BGR_SEED = 2024, 2025


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def Kmat(k):
    return np.array([[k[0], 0, k[2]], [0, k[1], k[3]], [0, 0, 1]], np.float64)


def resolve_newK(w, h, K, D, newK):
    if isinstance(newK, str):   # "alpha0" / "alpha1"
        m, _ = cv2.getOptimalNewCameraMatrix(Kmat(K), np.array(D, np.float64), (w, h), float(newK[-1]), (w, h))
        return (m[0, 0], m[1, 1], m[0, 2], m[1, 2])
    return K if newK is None else newK


def cv2_case(w, h, K, D, newK):
    m1, m2 = cv2.initUndistortRectifyMap(Kmat(K), np.array(D, np.float64), None, Kmat(newK), (w, h), cv2.CV_16SC2)
    grey = U.seeded_image(GREY_SEED, h, w)
    bgr = U.seeded_image(BGR_SEED, h, w, 3)
    r_grey = cv2.remap(grey, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    r_bgr = cv2.remap(cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY), m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    return m1, m2, r_grey, r_bgr


if __name__ == "__main__":
    out = {"cv2_version": np.array(cv2.__version__), "seeds": np.array([GREY_SEED, BGR_SEED])}
    for name, (w, h, K, D, newK) in U.CASES.items():
        nk = resolve_newK(w, h, K, D, newK)
        m1, m2, rg, rb = cv2_case(w, h, K, D, nk)
        out[f"{name}/newK"] = np.array(nk, np.float64)
        out[f"{name}/sha"] = np.array([sha(m1), sha(m2), sha(rg), sha(rb)])
        print(name, nk, "map range", m1.min(), m1.max())
    for name in U.SMALL:
        w, h, K, D, newK = U.small_case(name)
        m1, m2, rg, rb = cv2_case(w, h, K, D, K)
        out[f"{name}/map_xy"], out[f"{name}/map_a"], out[f"{name}/remap_grey"], out[f"{name}/remap_bgr"] = m1, m2, rg, rb
    np.savez_compressed(ROOT / "tests" / "golden" / "cv2_undistort.npz", **out)
    print("wrote", ROOT / "tests" / "golden" / "cv2_undistort.npz")
