"""ctypes binding of the CPU oracle (oracle/liboracle*.so).

TEST INFRASTRUCTURE ONLY -- imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs; never by the product package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
MAX_LEVELS = 10


def build(force: bool = False) -> None:
    """Compile liboracle.so / liboracle_native.so with oracle/Makefile (g++); make tracks staleness."""
    have = (_HERE / "liboracle.so").exists() and (_HERE / "liboracle_native.so").exists()
    try:
        subprocess.run(["make", "-C", str(_HERE), "-j4"] + (["-B"] if force else []), check=True,
                       stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
    except (subprocess.CalledProcessError, FileNotFoundError) as e:
        if not have:
            raise RuntimeError(f"cannot build the oracle: {getattr(e, 'stderr', e)}")


class DetectParams(C.Structure):
    _fields_ = [("image_width", C.c_int), ("image_height", C.c_int), ("cell_size", C.c_int),
                ("threshold", C.c_int), ("n_levels", C.c_int)]


class Features(C.Structure):
    _fields_ = [("n", C.c_int), ("px", C.c_void_p), ("py", C.c_void_p), ("level", C.c_void_p),
                ("score", C.c_void_p), ("angle", C.c_void_p), ("desc", C.c_void_p), ("cell", C.c_void_p)]


class Camera(C.Structure):
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float)]


class BAParams(C.Structure):
    _fields_ = [("max_iters", C.c_int), ("huber_delta", C.c_double), ("chi2_outlier", C.c_double),
                ("tau", C.c_double), ("max_trials", C.c_int)]


class BAStats(C.Structure):
    _fields_ = [("iters", C.c_int), ("lm_trials", C.c_int), ("chi2_initial", C.c_double),
                ("chi2_final", C.c_double), ("lambda_final", C.c_double), ("n_outliers", C.c_int)]


class CeresStats(C.Structure):
    _fields_ = [("iters", C.c_int), ("successful_steps", C.c_int), ("cost_initial", C.c_double),
                ("cost_final", C.c_double), ("radius_final", C.c_double), ("termination", C.c_int)]


class KLTParams(C.Structure):
    _fields_ = [("win", C.c_int), ("max_level", C.c_int), ("max_iter", C.c_int), ("eps", C.c_double),
                ("min_eig", C.c_double), ("exact_sums", C.c_int), ("get_min_eig", C.c_int)]


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def default_camera() -> Camera:
    return Camera(520.9, 521.0, 325.1, 249.7)


class Oracle:
    """Thin numpy front-end.  `native=True` loads the -O3 AVX2/FMA build (the timed CPU baseline)."""

    def __init__(self, native: bool = False):
        build()
        self.lib = C.CDLL(str(_HERE / ("liboracle_native.so" if native else "liboracle.so")))
        L = self.lib
        L.ora_pyramid_layout.restype = C.c_size_t
        L.ora_shi_tomasi.restype = C.c_float
        L.ora_fast_atan2.restype = C.c_float
        L.ora_fast_atan2.argtypes = [C.c_float, C.c_float]
        L.ora_cv_round_f.argtypes = [C.c_float]
        L.ora_cv_round_d.argtypes = [C.c_double]
        if hasattr(L, "ora_sparse_align"):
            L.ora_sparse_align.restype = C.c_size_t

    # ---- pyramid ---------------------------------------------------------------------------
    def layout(self, w, h, n_levels):
        lw = (C.c_int * MAX_LEVELS)()
        lh = (C.c_int * MAX_LEVELS)()
        off = (C.c_size_t * MAX_LEVELS)()
        total = self.lib.ora_pyramid_layout(w, h, n_levels, lw, lh, off)
        return list(lw)[:n_levels], list(lh)[:n_levels], list(off)[:n_levels], total

    def bgr2gray(self, bgr):
        h, w, _ = bgr.shape
        out = np.empty((h, w), np.uint8)
        self.lib.ora_bgr2gray(_p(np.ascontiguousarray(bgr)), w, h, _p(out))
        return out

    def pyrdown(self, img):
        h, w = img.shape
        out = np.empty(((h + 1) // 2, (w + 1) // 2), np.uint8)
        self.lib.ora_pyrdown(_p(np.ascontiguousarray(img)), w, h, _p(out))
        return out

    def build_pyramid(self, gray, n_levels):
        h, w = gray.shape
        _, _, _, total = self.layout(w, h, n_levels)
        pyr = np.empty(total, np.uint8)
        self.lib.ora_build_pyramid(_p(np.ascontiguousarray(gray)), w, h, n_levels, _p(pyr))
        return pyr

    def level_view(self, pyr, w, h, n_levels, L):
        lw, lh, off, _ = self.layout(w, h, n_levels)
        return pyr[off[L]: off[L] + lw[L] * lh[L]].reshape(lh[L], lw[L])

    # ---- FAST ------------------------------------------------------------------------------
    def fast_detect(self, img, barrier=15, arc=10):
        h, w = img.shape
        img = np.ascontiguousarray(img)
        xy = np.empty((w * h, 2), np.int16)
        n = self.lib.ora_fastN_detect(_p(img), w, h, w, barrier, arc, _p(xy), w * h)
        return xy[:n].copy()

    def fast_score(self, img, xy, barrier=15):
        img = np.ascontiguousarray(img)
        xy = np.ascontiguousarray(xy, np.int16)
        s = np.empty(len(xy), np.int32)
        self.lib.ora_fast10_score(_p(img), img.shape[1], _p(xy), len(xy), barrier, _p(s))
        return s

    def fast_nonmax(self, xy, scores):
        xy = np.ascontiguousarray(xy, np.int16)
        scores = np.ascontiguousarray(scores, np.int32)
        keep = np.empty(max(len(xy), 1), np.int32)
        n = self.lib.ora_fast_nonmax_3x3(_p(xy), _p(scores), len(xy), _p(keep))
        return keep[:n].copy()

    # ---- detector --------------------------------------------------------------------------
    def detect(self, pyr, w=640, h=480, n_levels=3, cell=10, threshold=15, occupied=None):
        prm = DetectParams(w, h, cell, threshold, n_levels)
        ncell = -(-w // cell) * -(-h // cell)
        px = np.empty(ncell, np.float64)
        py = np.empty(ncell, np.float64)
        level = np.empty(ncell, np.int32)
        score = np.empty(ncell, np.float32)
        angle = np.empty(ncell, np.float32)
        desc = np.empty((ncell, 32), np.uint8)
        cellidx = np.empty(ncell, np.int32)
        f = Features(0, *[a.ctypes.data for a in (px, py, level, score, angle, desc, cellidx)])
        occ = None if occupied is None else np.ascontiguousarray(occupied, np.uint8)
        n = self.lib.ora_detect(_p(pyr), C.byref(prm), _p(occ), C.byref(f))
        return dict(n=n, px=px[:n].copy(), py=py[:n].copy(), level=level[:n].copy(), score=score[:n].copy(),
                    angle=angle[:n].copy(), desc=desc[:n].copy(), cell=cellidx[:n].copy())

    def shi_tomasi(self, img, u, v):
        img = np.ascontiguousarray(img)
        return float(self.lib.ora_shi_tomasi(_p(img), img.shape[1], img.shape[0], int(u), int(v)))

    def describe(self, pyr, w, h, n_levels, px, py, level):
        n = len(px)
        px = np.ascontiguousarray(px, np.float64)
        py = np.ascontiguousarray(py, np.float64)
        level = np.ascontiguousarray(level, np.int32)
        angle = np.empty(n, np.float32)
        desc = np.empty((n, 32), np.uint8)
        self.lib.ora_describe(_p(pyr), w, h, n_levels, n, _p(px), _p(py), _p(level), _p(angle), _p(desc))
        return angle, desc

    def fast_atan2(self, y, x):
        return float(self.lib.ora_fast_atan2(float(y), float(x)))

    # ---- matching --------------------------------------------------------------------------
    def match_bf(self, A, B, cross_check=True):
        A = np.ascontiguousarray(A, np.uint8)
        B = np.ascontiguousarray(B, np.uint8)
        idx = np.empty(len(A), np.int32)
        dist = np.empty(len(A), np.int32)
        self.lib.ora_match_bf(_p(A), len(A), _p(B), len(B), int(cross_check), _p(idx), _p(dist))
        return idx, dist

    def good_matches(self, idx, dist):
        keep = np.empty(len(idx), np.uint8)
        n = self.lib.ora_good_matches(_p(np.ascontiguousarray(idx, np.int32)),
                                      _p(np.ascontiguousarray(dist, np.int32)), len(idx), _p(keep))
        return keep.astype(bool), n

    def check_descriptors(self, A, B, ia, ib, init_low=30, init_high=100):
        A = np.ascontiguousarray(A, np.uint8)
        B = np.ascontiguousarray(B, np.uint8)
        ia = np.ascontiguousarray(ia, np.int32)
        ib = np.ascontiguousarray(ib, np.int32)
        dist = np.empty(len(ia), np.int32)
        keep = np.empty(len(ia), np.uint8)
        n = self.lib.ora_check_descriptors(_p(A), _p(B), _p(ia), _p(ib), len(ia), init_low, init_high, _p(dist),
                                           _p(keep))
        return dist, keep.astype(bool), n

    # ---- alignment -------------------------------------------------------------------------
    def align2d(self, img, ref_border, ref, u, v, n_iter=10):
        img = np.ascontiguousarray(img)
        uu = C.c_double(u)
        vv = C.c_double(v)
        ok = self.lib.ora_align2d(_p(img), img.shape[1], img.shape[0], _p(np.ascontiguousarray(ref_border, np.uint8)),
                                  _p(np.ascontiguousarray(ref, np.uint8)), n_iter, C.byref(uu), C.byref(vv))
        return bool(ok), uu.value, vv.value

    def align1d(self, img, dirx, diry, ref_border, ref, u, v, n_iter=10):
        img = np.ascontiguousarray(img)
        uu = C.c_double(u)
        vv = C.c_double(v)
        hinv = C.c_double(0)
        ok = self.lib.ora_align1d(_p(img), img.shape[1], img.shape[0], C.c_float(dirx), C.c_float(diry),
                                  _p(np.ascontiguousarray(ref_border, np.uint8)),
                                  _p(np.ascontiguousarray(ref, np.uint8)), n_iter, C.byref(uu), C.byref(vv),
                                  C.byref(hinv))
        return bool(ok), uu.value, vv.value, hinv.value

    def find_direct_projection(self, ref_pyr, cur_pyr, w, h, n_levels, T_ref, T_cur, ref_px, ref_depth, ref_level,
                               cur_px, cam=None):
        cam = cam or default_camera()
        n = len(ref_depth)
        ref_px = np.ascontiguousarray(ref_px, np.float64)
        cur = np.ascontiguousarray(cur_px, np.float64).copy()
        lvl = np.empty(n, np.int32)
        ok = np.empty(n, np.uint8)
        self.lib.ora_find_direct_projection(_p(ref_pyr), _p(cur_pyr), w, h, n_levels, C.byref(cam),
                                            _p(np.ascontiguousarray(T_ref, np.float64)),
                                            _p(np.ascontiguousarray(T_cur, np.float64)), n, _p(ref_px),
                                            _p(np.ascontiguousarray(ref_depth, np.float64)),
                                            _p(np.ascontiguousarray(ref_level, np.int32)), _p(cur), _p(lvl), _p(ok))
        return cur, lvl, ok.astype(bool)

    def sparse_align(self, ref_pyr, cur_pyr, w, h, n_levels, px, depth, has_mp, T_ref, T_cur, max_level=2,
                     min_level=0, n_iter=30, eps=1e-6, cam=None, exact=False):
        """SparseImgAlign::run.  exact=True sums chi2 in double and rounds it to float once, as the CUDA kernel does, so the
        rollback decisions (and the per-level iteration counts) can be compared exactly."""
        cam = cam or default_camera()
        n = len(depth)
        T = np.ascontiguousarray(T_cur, np.float64).copy()
        iters = np.zeros(MAX_LEVELS, np.int32)
        nm = self.lib.ora_sparse_align(_p(ref_pyr), _p(cur_pyr), w, h, n_levels, C.byref(cam), n,
                                       _p(np.ascontiguousarray(px, np.float64)),
                                       _p(np.ascontiguousarray(depth, np.float64)),
                                       _p(np.ascontiguousarray(has_mp, np.uint8)),
                                       _p(np.ascontiguousarray(T_ref, np.float64)), _p(T), max_level, min_level,
                                       n_iter, C.c_double(eps), _p(iters), int(exact))
        return T, int(nm), iters

    def matcher_sparse_alignment(self, ref_pyr, cur_pyr, w, h, n_levels, px, depth, has_mp, T_ref, T_cur, cam=None):
        cam = cam or default_camera()
        T = np.ascontiguousarray(T_cur, np.float64).copy()
        ok = self.lib.ora_matcher_sparse_alignment(_p(ref_pyr), _p(cur_pyr), w, h, n_levels, C.byref(cam),
                                                   len(depth), _p(np.ascontiguousarray(px, np.float64)),
                                                   _p(np.ascontiguousarray(depth, np.float64)),
                                                   _p(np.ascontiguousarray(has_mp, np.uint8)),
                                                   _p(np.ascontiguousarray(T_ref, np.float64)), _p(T))
        return bool(ok), T

    # ---- Sophus ----------------------------------------------------------------------------
    def se3_exp(self, v):
        T = np.empty(12, np.float64)
        self.lib.ora_se3_exp(_p(np.ascontiguousarray(v, np.float64)), _p(T))
        return T.reshape(3, 4)

    def se3_log(self, T):
        v = np.empty(6, np.float64)
        self.lib.ora_se3_log(_p(np.ascontiguousarray(T, np.float64)), _p(v))
        return v

    # ---- BA --------------------------------------------------------------------------------
    def local_ba(self, poses, fixed, pts, kf_idx, pt_idx, px, max_iters=20, huber=5.991, cam=None, tau=1e-5, max_trials=10,
                 chi2_outlier=5.991):
        cam = cam or default_camera()
        poses = np.ascontiguousarray(poses, np.float64).copy()
        pts = np.ascontiguousarray(pts, np.float64).copy()
        prm = BAParams(max_iters, huber, chi2_outlier, tau, max_trials)
        st = BAStats()
        outl = np.zeros(len(kf_idx), np.uint8)
        self.lib.ora_local_ba_g2o(C.byref(cam), len(poses), _p(poses), _p(np.ascontiguousarray(fixed, np.uint8)),
                                  len(pts), _p(pts), len(kf_idx), _p(np.ascontiguousarray(kf_idx, np.int32)),
                                  _p(np.ascontiguousarray(pt_idx, np.int32)),
                                  _p(np.ascontiguousarray(px, np.float64)), C.byref(prm), _p(outl), C.byref(st))
        stats = {k: getattr(st, k) for k, _ in BAStats._fields_}
        return poses, pts, outl.astype(bool), stats

    def local_ba_ceres(self, poses_t_aa, fixed, pts, kf_idx, pt_idx, px, max_iters=50, huber=0.0, cam=None):
        """ba::LocalBA (Ceres twin): poses as [t; angle-axis]."""
        cam = cam or default_camera()
        poses = np.ascontiguousarray(poses_t_aa, np.float64).copy()
        pts = np.ascontiguousarray(pts, np.float64).copy()
        st = CeresStats()
        self.lib.ora_local_ba_ceres(C.byref(cam), len(poses), _p(poses), _p(np.ascontiguousarray(fixed, np.uint8)),
                                    len(pts), _p(pts), len(kf_idx), _p(np.ascontiguousarray(kf_idx, np.int32)),
                                    _p(np.ascontiguousarray(pt_idx, np.int32)), _p(np.ascontiguousarray(px, np.float64)),
                                    max_iters, C.c_double(huber), C.byref(st))
        return poses, pts, {k: getattr(st, k) for k, _ in CeresStats._fields_}

    def search_for_triangulation(self, desc1, px1, node1, desc2, px2, node2, E12, th_low=65, epipolar_dsqr=1e-4, cam=None):
        cam = cam or default_camera()
        n1, n2 = len(node1), len(node2)
        out = np.full(n1, -1, np.int32)
        self.lib.ora_search_for_triangulation(C.byref(cam), n1, _p(np.ascontiguousarray(desc1, np.uint8)),
                                              _p(np.ascontiguousarray(px1, np.float64)), _p(np.ascontiguousarray(node1, np.int32)), n2,
                                              _p(np.ascontiguousarray(desc2, np.uint8)), _p(np.ascontiguousarray(px2, np.float64)),
                                              _p(np.ascontiguousarray(node2, np.int32)), _p(np.ascontiguousarray(E12, np.float64)),
                                              int(th_low), C.c_double(epipolar_dsqr), _p(out))
        return out

    # ---- DBoW3 (bow.cpp) ----------------------------------------------------------------------
    def vocab_load(self, data: bytes):
        """Vocabulary::loadFromBinaryFile from the file's bytes -> opaque handle (free with vocab_free)."""
        self.lib.ora_vocab_load.restype = C.c_void_p
        self.lib.ora_vocab_load.argtypes = [C.c_char_p, C.c_size_t]
        h = self.lib.ora_vocab_load(data, len(data))
        if not h:
            raise ValueError("malformed vocabulary")
        return C.c_void_p(h)

    def vocab_free(self, v):
        self.lib.ora_vocab_free.argtypes = [C.c_void_p]
        self.lib.ora_vocab_free(v)

    def vocab_info(self, v):
        info = np.zeros(6, np.int32)
        self.lib.ora_vocab_info.argtypes = [C.c_void_p, C.c_void_p]
        self.lib.ora_vocab_info(v, _p(info))
        return dict(zip(("k", "L", "scoring", "weighting", "nodes", "words"), info.tolist()))

    def bow_transform(self, v, desc, levelsup=4):
        desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        n = len(desc)
        word, node, weight = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n)
        bw, bv = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1))
        self.lib.ora_bow_transform.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 5
        m = self.lib.ora_bow_transform(v, n, _p(desc), int(levelsup), _p(word), _p(node), _p(weight), _p(bw), _p(bv))
        return word, node, weight, bw[:m].copy(), bv[:m].copy()

    def search_by_bow(self, desc1, node1, angle1, desc2, node2, angle2, th_low=50, knn_ratio=0.9, check_orientation=False):
        n1, n2 = len(node1), len(node2)
        out = np.full(n1, -1, np.int32)
        self.lib.ora_search_by_bow.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_int, C.c_float, C.c_int, C.c_void_p]
        cnt = self.lib.ora_search_by_bow(n1, _p(np.ascontiguousarray(desc1, np.uint8)), _p(np.ascontiguousarray(node1, np.int32)),
                                         _p(np.ascontiguousarray(angle1, np.float32)), n2, _p(np.ascontiguousarray(desc2, np.uint8)),
                                         _p(np.ascontiguousarray(node2, np.int32)), _p(np.ascontiguousarray(angle2, np.float32)),
                                         int(th_low), float(knn_ratio), int(check_orientation), _p(out))
        return out, cnt

    # ---- Initializer RANSAC (initializer.cpp) ----------------------------------------------------
    def initializer_sets(self, n_points, max_iter=200):
        sets = np.zeros((max_iter, 8), np.int32)
        self.lib.ora_initializer_sets(int(n_points), int(max_iter), _p(sets))
        return sets

    def initializer_ransac(self, px1, px2, sets, sigma=2.0, models=False):
        px1 = np.ascontiguousarray(px1, np.float64).reshape(-1, 2)
        px2 = np.ascontiguousarray(px2, np.float64).reshape(-1, 2)
        sets = np.ascontiguousarray(sets, np.int32).reshape(-1, 8)
        n, iters = len(px1), len(sets)
        H, F = np.zeros(9), np.zeros(9)
        sh, sf = C.c_float(0), C.c_float(0)
        bh, bf = C.c_int32(0), C.c_int32(0)
        ih, jf = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        mod = np.zeros((iters, 18)) if models else None
        self.lib.ora_initializer_ransac.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_float] + [C.c_void_p] * 9
        self.lib.ora_initializer_ransac(n, _p(px1), _p(px2), iters, _p(sets), C.c_float(sigma), _p(H), C.byref(sh), C.byref(bh), _p(ih), _p(F),
                                        C.byref(sf), C.byref(bf), _p(jf), _p(mod))
        out = dict(H21=H.reshape(3, 3), score_H=np.float32(sh.value), best_H=bh.value, inliers_H=ih.astype(bool), F21=F.reshape(3, 3),
                   score_F=np.float32(sf.value), best_F=bf.value, inliers_F=jf.astype(bool))
        if models:
            out["models"] = mod
        return out

    def initializer_reconstruct(self, px1, px2, use_h, model, inliers, K=(520.9, 521.0, 325.1, 249.7), sigma2=4.0, min_parallax=1.0,
                                min_triangulated=8, ratio_h=0.9):
        px1 = np.ascontiguousarray(px1, np.float64).reshape(-1, 2)
        px2 = np.ascontiguousarray(px2, np.float64).reshape(-1, 2)
        n = len(px1)
        # the reference's camera keeps float intrinsics (Camera.h:14-22)
        Kd = np.asarray(K, np.float32).astype(np.float64)
        R, t, p3d = np.zeros(9), np.zeros(3), np.zeros((n, 3))
        tri, ng, par, cand = np.zeros(n, np.uint8), np.zeros(8, np.int32), C.c_double(0), np.zeros((8, 12))
        self.lib.ora_initializer_reconstruct.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float,
                                                         C.c_float, C.c_int, C.c_double] + [C.c_void_p] * 7
        ok = self.lib.ora_initializer_reconstruct(n, _p(px1), _p(px2), int(bool(use_h)), _p(np.ascontiguousarray(model, np.float64).reshape(9)),
                                                  _p(np.ascontiguousarray(inliers, np.uint8)), _p(Kd), C.c_float(sigma2), C.c_float(min_parallax),
                                                  int(min_triangulated), C.c_double(ratio_h), _p(R), _p(t), _p(p3d), _p(tri), _p(ng),
                                                  C.byref(par), _p(cand))
        return dict(ok=bool(ok), R21=R.reshape(3, 3), t21=t, p3d=p3d, triangulated=tri.astype(bool), n_good=ng, parallax=par.value,
                    candidates=cand)

    def depth_from_triangulation(self, T, f_ref, f_cur, det_th=1e-5):
        T = np.ascontiguousarray(T, np.float64).reshape(12)
        f_ref = np.ascontiguousarray(f_ref, np.float64).reshape(-1, 3)
        f_cur = np.ascontiguousarray(f_cur, np.float64).reshape(-1, 3)
        n = len(f_ref)
        d1, d2, ok = np.zeros(n), np.zeros(n), np.zeros(n, bool)
        a, b = C.c_double(0), C.c_double(0)
        for i in range(n):
            ok[i] = bool(self.lib.ora_depth_from_triangulation(_p(T), _p(f_ref[i]), _p(f_cur[i]), C.c_double(det_th), C.byref(a), C.byref(b)))
            if ok[i]:
                d1[i], d2[i] = a.value, b.value
        return d1, d2, ok

    def two_view_ba(self, T_ref, T_cur, px_ref, px_cur, inlier, pts, cam=None):
        """ba::TwoViewBACeres: returns (T_cur 3x4, inlier bool, pts, stats, inlier count)."""
        cam = cam or default_camera()
        n = len(px_ref)
        Tr = np.ascontiguousarray(T_ref, np.float64).reshape(12)
        Tc = np.ascontiguousarray(T_cur, np.float64).reshape(12).copy()
        inl = np.ascontiguousarray(inlier, np.uint8).copy()
        X = np.ascontiguousarray(pts, np.float64).reshape(n, 3).copy()
        st = CeresStats()
        cnt = self.lib.ora_two_view_ba(C.byref(cam), n, _p(Tr), _p(Tc), _p(np.ascontiguousarray(px_ref, np.float64)),
                                       _p(np.ascontiguousarray(px_cur, np.float64)), _p(inl), _p(X), C.byref(st))
        return Tc.reshape(3, 4), inl.astype(bool), X, {k: getattr(st, k) for k, _ in CeresStats._fields_}, int(cnt)

    def pose_only(self, pt_world, px, T_cw, cam=None):
        cam = cam or default_camera()
        n = len(pt_world)
        T = np.ascontiguousarray(T_cw, np.float64).copy()
        inl = np.zeros(n, np.uint8)
        depth = np.zeros(n, np.float64)
        cnt = self.lib.ora_pose_only(C.byref(cam), n, _p(np.ascontiguousarray(pt_world, np.float64)),
                                     _p(np.ascontiguousarray(px, np.float64)), _p(T), _p(inl), _p(depth))
        return T, inl.astype(bool), depth, cnt

    # ---- KLT -------------------------------------------------------------------------------
    def klt(self, ref, cur, ref_xy, cur_xy, win=21, max_level=4, max_iter=30, eps=0.001, min_eig=1e-4, exact=False,
            get_min_eig=False):
        """cv::calcOpticalFlowPyrLK with OPTFLOW_USE_INITIAL_FLOW.  exact=True sums the window in int64 like klt.cu (bit-exact
        to the GPU); the default sums in f32 like OpenCV.  get_min_eig=True returns the level-0 minimum eigenvalue as err."""
        h, w = ref.shape
        n = len(ref_xy)
        out = np.ascontiguousarray(cur_xy, np.float32).copy()
        status = np.zeros(n, np.uint8)
        err = np.zeros(n, np.float32)
        prm = KLTParams(win, max_level, max_iter, eps, min_eig, int(exact), int(get_min_eig))
        self.lib.ora_klt(_p(np.ascontiguousarray(ref)), _p(np.ascontiguousarray(cur)), w, h, n,
                         _p(np.ascontiguousarray(ref_xy, np.float32)), _p(out), _p(status), _p(err), C.byref(prm))
        return out, status, err


def vo_run(oracle: "Oracle", frames, depths, kf_min_frames=10, kf_min_rot=0.1, kf_min_trans=0.1, warm=0, threads=1):
    """The C5 tracking loop on the CPU oracle in C++ (oracle/vo_cpu.cpp), one stream per host thread.
    frames[s]: (n_frames, 480, 640) uint8, depths[s]: (480, 640) float64.
    Returns (trajectory (S, n, 3, 4), stats list of dicts, seconds of frames [warm, n), per-stage seconds dict)."""
    S, n = len(frames), len(frames[0])
    imgs = [np.ascontiguousarray(f, np.uint8) for f in frames]
    deps = [np.ascontiguousarray(d, np.float64) for d in depths]
    ip = (C.c_void_p * S)(*[a.ctypes.data for a in imgs])
    dp = (C.c_void_p * S)(*[a.ctypes.data for a in deps])
    traj = np.zeros((S, n, 12), np.float64)
    stats = np.zeros((S, 8), np.int64)
    stage = np.zeros(7, np.float64)
    sec = C.c_double(0.0)
    fn = oracle.lib.ora_vo_run
    fn.restype = C.c_int
    fn.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_int, C.c_int, C.c_void_p,
                   C.c_void_p, C.c_void_p, C.c_void_p]
    rc = fn(S, n, C.cast(ip, C.c_void_p), C.cast(dp, C.c_void_p), kf_min_frames, kf_min_rot, kf_min_trans, warm, threads,
            traj.ctypes.data, stats.ctypes.data, C.byref(sec), stage.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"ora_vo_run rc={rc}")
    keys = ("lost", "keyframes", "ba", "candidates", "projected", "inliers")
    names = ("pyramid", "sparse_align", "project_align", "pose_only", "detect", "local_ba", "host")
    return (traj.reshape(S, n, 3, 4), [dict(zip(keys, map(int, row[:6]))) for row in stats], sec.value,
            dict(zip(names, map(float, stage))))
