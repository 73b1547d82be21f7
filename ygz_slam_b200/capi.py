"""ctypes binding of libygz_b200.so (include/ygz_b200.h).  Plumbing only: numpy arrays in/out."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
MAX_LEVELS = 10
_LIB = None


class YgzbError(RuntimeError):
    pass


def lib_path() -> Path:
    return HERE / "libygz_b200.so"


class Params(C.Structure):
    _fields_ = [("image_width", C.c_int), ("image_height", C.c_int), ("n_levels", C.c_int), ("cell_size", C.c_int),
                ("fast_threshold", C.c_int), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float)]


class Keypoints(C.Structure):
    _fields_ = [("offsets", C.c_void_p), ("x", C.c_void_p), ("y", C.c_void_p), ("level", C.c_void_p),
                ("score", C.c_void_p), ("angle", C.c_void_p), ("desc", C.c_void_p), ("cell", C.c_void_p),
                ("capacity", C.c_int)]


# every symbol include/ygz_b200.h declares (tests check that the library exports all of them)
EXPORTS = [
    "ygzb_default_params", "ygzb_create", "ygzb_get_params", "ygzb_destroy", "ygzb_last_error", "ygzb_synchronize", "ygzb_stream",
    "ygzb_launch_count", "ygzb_timer_start", "ygzb_timer_stop", "ygzb_profile_enable", "ygzb_profile_read", "ygzb_profile_stage_count",
    "ygzb_profile_stage_name", "ygzb_host_alloc", "ygzb_host_free", "ygzb_frames_create", "ygzb_frames_destroy",
    "ygzb_frames_upload", "ygzb_frames_copy", "ygzb_frames_build_pyramid", "ygzb_frames_layout", "ygzb_frames_device_ptr",
    "ygzb_frames_download_level", "ygzb_detect", "ygzb_grid_dims", "ygzb_describe", "ygzb_fast_debug",
    "ygzb_detect_stats", "ygzb_match_bf", "ygzb_match_frames", "ygzb_hamming_pairs", "ygzb_search_for_triangulation", "ygzb_depth_from_triangulation",
    "ygzb_vocab_create", "ygzb_vocab_destroy", "ygzb_vocab_info", "ygzb_bow_transform", "ygzb_search_by_bow", "ygzb_initializer_ransac", "ygzb_initializer_reconstruct", "ygzb_synchronize_blocking", "ygzb_align2d", "ygzb_align1d",
    "ygzb_project_align", "ygzb_sparse_align", "ygzb_default_ba_params", "ygzb_local_ba", "ygzb_local_ba_ceres", "ygzb_two_view_ba", "ygzb_pose_only",
    "ygzb_default_klt_params", "ygzb_klt",
    "ygzb_tracker_create", "ygzb_tracker_destroy", "ygzb_tracker_set_depth", "ygzb_tracker_upload", "ygzb_tracker_track", "ygzb_tracker_make_keyframes",
    "ygzb_tracker_export", "ygzb_tracker_import", "ygzb_tracker_debug_job", "ygzb_tracker_set_reference_mode", "ygzb_tracker_debug_reference",
    "ygzb_tracker_export_reference", "ygzb_tracker_import_reference", "ygzb_undistort_map", "ygzb_frames_set_undistort",
    "ygzb_tracker_set_start_pose",
]


# Engine threads own two CUDA streams each; with the default 8 hardware work queues the streams of different threads share a
# queue and falsely serialise.  Only effective if the CUDA context
# does not exist yet -- a host process embedding the library exports the variable itself (INTEGRATION.md).
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")


def load_library(build_if_missing: bool = True):
    """Load libygz_b200.so; fails loudly if it is missing and cannot be built (no CPU fallback)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    p = lib_path()
    if not p.exists():
        if not build_if_missing:
            raise YgzbError(f"{p} is missing: build it with `python -m ygz_slam_b200.build` (there is no CPU fallback)")
        from . import build as _build
        _build.build()
    lib = C.CDLL(str(p))
    lib.ygzb_last_error.restype = C.c_char_p
    lib.ygzb_last_error.argtypes = [C.c_void_p]
    lib.ygzb_stream.restype = C.c_void_p
    lib.ygzb_stream.argtypes = [C.c_void_p]
    lib.ygzb_launch_count.restype = C.c_longlong
    lib.ygzb_launch_count.argtypes = [C.c_void_p]
    lib.ygzb_frames_device_ptr.restype = C.c_void_p
    lib.ygzb_frames_device_ptr.argtypes = [C.c_void_p]
    lib.ygzb_destroy.argtypes = [C.c_void_p]
    lib.ygzb_destroy.restype = None
    lib.ygzb_frames_destroy.argtypes = [C.c_void_p]
    lib.ygzb_frames_destroy.restype = None
    lib.ygzb_default_params.restype = None
    lib.ygzb_profile_stage_name.restype = C.c_char_p
    _LIB = lib
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class _Pinned:
    """Keeps a page-locked host allocation (ygzb_host_alloc) alive behind a numpy view."""

    def __init__(self, lib, nbytes):
        self.lib = lib
        self.ptr = C.c_void_p()
        if lib.ygzb_host_alloc(C.byref(self.ptr), C.c_size_t(max(nbytes, 1))) != 0:
            raise YgzbError("ygzb_host_alloc failed")

    def __del__(self):
        try:
            self.lib.ygzb_host_free(self.ptr)
        except Exception:
            pass


def pinned_empty(shape, dtype):
    """numpy array backed by page-locked memory: D2H/H2D copies to it run at full PCIe rate and asynchronously."""
    lib = load_library()
    dtype = np.dtype(dtype)
    n = int(np.prod(shape))
    owner = _Pinned(lib, n * dtype.itemsize)
    buf = (C.c_char * (n * dtype.itemsize)).from_address(owner.ptr.value)
    arr = np.frombuffer(buf, dtype=dtype, count=n).reshape(shape)
    _PINNED_OWNERS[id(arr)] = owner
    import weakref
    weakref.finalize(arr, _PINNED_OWNERS.pop, id(arr), None)
    return arr


_PINNED_OWNERS: dict = {}


def undistort_map(width: int, height: int, K, dist, newK=None):
    """cv2.initUndistortRectifyMap(K, dist, None, newK, (width, height), cv2.CV_16SC2) without OpenCV (ygzb_undistort_map, host
    code): K / newK = (fx, fy, cx, cy), newK None = K; dist = (k1, k2, p1, p2[, k3]).  Returns map_xy (H, W, 2) int16 and
    map_a (H, W) uint16 for Frames.set_undistort."""
    lib = load_library()
    lib.ygzb_undistort_map.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    K = np.ascontiguousarray(K, np.float64).reshape(4)
    d = np.zeros(5)
    d[:len(dist)] = dist
    nk = None if newK is None else np.ascontiguousarray(newK, np.float64).reshape(4)
    map_xy = np.empty((height, width, 2), np.int16)
    map_a = np.empty((height, width), np.uint16)
    rc = lib.ygzb_undistort_map(int(width), int(height), _p(K), _p(d), _p(nk), _p(map_xy), _p(map_a))
    if rc != 0:
        raise YgzbError(f"ygzb_undistort_map failed (rc={rc}): bad size or camera")
    return map_xy, map_a


class Context:
    """One device + one stream (ygzb_ctx)."""

    def __init__(self, device: int = 0, **overrides):
        self.lib = load_library()
        prm = Params()
        self.lib.ygzb_default_params(C.byref(prm))
        for k, v in overrides.items():
            if not hasattr(prm, k):
                raise TypeError(f"unknown parameter {k}")
            setattr(prm, k, v)
        self.params = prm
        self.device_index = device
        h = C.c_void_p()
        rc = self.lib.ygzb_create(device, C.byref(prm), C.byref(h))
        self.h = h
        if rc != 0:
            msg = self.lib.ygzb_last_error(h).decode() if h else ""
            if h:
                self.lib.ygzb_destroy(h)
                self.h = None
            raise YgzbError(f"ygzb_create failed (rc={rc}): {msg or 'no usable sm_90 device; there is no CPU fallback'}")
        rows, cols = C.c_int(), C.c_int()
        self.lib.ygzb_grid_dims(self.h, C.byref(rows), C.byref(cols))
        self.grid_rows, self.grid_cols = rows.value, cols.value
        self.n_cells = rows.value * cols.value
        self.n_levels = prm.n_levels

    def check(self, rc: int, what: str = ""):
        if rc != 0:
            raise YgzbError(f"{what} failed (rc={rc}): {self.lib.ygzb_last_error(self.h).decode()}")

    def close(self):
        if getattr(self, "h", None):
            self.lib.ygzb_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def synchronize(self):
        self.check(self.lib.ygzb_synchronize(self.h), "ygzb_synchronize")

    @property
    def stream(self) -> int:
        return self.lib.ygzb_stream(self.h)

    @property
    def launch_count(self) -> int:
        return self.lib.ygzb_launch_count(self.h)

    def profile(self, on: bool):
        self.check(self.lib.ygzb_profile_enable(self.h, int(on)), "ygzb_profile_enable")

    def profile_read(self) -> dict:
        """{stage: (total ms, launches)} since the last read (CUDA events around each kernel)."""
        n = self.lib.ygzb_profile_stage_count()
        ms = (C.c_double * n)()
        cnt = (C.c_int32 * n)()
        self.check(self.lib.ygzb_profile_read(self.h, ms, cnt), "ygzb_profile_read")
        return {self.lib.ygzb_profile_stage_name(i).decode(): (ms[i], cnt[i]) for i in range(n)}

    def frames(self, capacity: int) -> "Frames":
        return Frames(self, capacity)

    # ---- Matcher -------------------------------------------------------------------------------
    def match_bf(self, A, B, cross_check=True):
        A = np.ascontiguousarray(A, np.uint8).reshape(-1, 32)
        B = np.ascontiguousarray(B, np.uint8).reshape(-1, 32)
        idx = np.full(len(A), -1, np.int32)
        dist = np.full(len(A), -1, np.int32)
        self.check(self.lib.ygzb_match_bf(self.h, _p(A), len(A), _p(B), len(B), int(cross_check), _p(idx), _p(dist)),
                   "ygzb_match_bf")
        return idx, dist

    def hamming_pairs(self, A, B, ia, ib):
        A = np.ascontiguousarray(A, np.uint8).reshape(-1, 32)
        B = np.ascontiguousarray(B, np.uint8).reshape(-1, 32)
        ia = np.ascontiguousarray(ia, np.int32)
        ib = np.ascontiguousarray(ib, np.int32)
        dist = np.empty(len(ia), np.int32)
        self.check(self.lib.ygzb_hamming_pairs(self.h, _p(A), len(A), _p(B), len(B), _p(ia), _p(ib), len(ia), _p(dist)),
                   "ygzb_hamming_pairs")
        return dist


class Frames:
    """Device-resident pyramids + feature store for `capacity` frame slots (ygzb_frames)."""

    def __init__(self, ctx: Context, capacity: int):
        self.ctx = ctx
        self.lib = ctx.lib
        self.capacity = capacity
        h = C.c_void_p()
        ctx.check(self.lib.ygzb_frames_create(ctx.h, capacity, C.byref(h)), "ygzb_frames_create")
        self.h = h
        lw = (C.c_int * MAX_LEVELS)()
        lh = (C.c_int * MAX_LEVELS)()
        lp = (C.c_int * MAX_LEVELS)()
        lo = (C.c_size_t * MAX_LEVELS)()
        ss = C.c_size_t()
        self.lib.ygzb_frames_layout(self.h, lw, lh, lp, lo, C.byref(ss))
        n = ctx.n_levels
        self.lw, self.lh, self.lpitch, self.loff = list(lw)[:n], list(lh)[:n], list(lp)[:n], list(lo)[:n]
        self.slot_stride = ss.value

    def close(self):
        if getattr(self, "h", None) and getattr(self.ctx, "h", None):
            self.lib.ygzb_frames_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def device_ptr(self) -> int:
        return self.lib.ygzb_frames_device_ptr(self.h)

    def upload(self, images, first: int = 0):
        """images: (n,h,w) grey or (n,h,w,3) BGR uint8 (or a raw pointer + n via upload_raw)."""
        images = np.ascontiguousarray(images, np.uint8)
        if images.ndim == 2:
            images = images[None]
        channels = 3 if images.ndim == 4 else 1
        n = images.shape[0]
        stride = int(np.prod(images.shape[1:]))  # bytes per image (numpy may report any stride for a length-1 axis)
        self.ctx.check(self.lib.ygzb_frames_upload(self.h, first, n, _p(images), channels, C.c_size_t(stride)),
                       "ygzb_frames_upload")

    def upload_raw(self, ptr: int, n: int, channels: int, frame_stride: int, first: int = 0):
        self.ctx.check(self.lib.ygzb_frames_upload(self.h, first, n, C.c_void_p(ptr), channels, C.c_size_t(frame_stride)),
                       "ygzb_frames_upload")

    def set_undistort(self, map_xy=None, map_a=None):
        """Undistort every later upload into this pool: level 0 = cv2.remap of the (grey-converted) frame through OpenCV's
        fixed-point maps, map_xy (H, W, 2) int16 and map_a (H, W) uint16 (cv2.initUndistortRectifyMap(.., cv2.CV_16SC2) or
        undistort_map).  No arguments clear the maps."""
        if map_xy is None and map_a is None:
            self.ctx.check(self.lib.ygzb_frames_set_undistort(self.h, None, None), "ygzb_frames_set_undistort")
            return
        H, W = self.lh[0], self.lw[0]
        map_xy = np.ascontiguousarray(map_xy, np.int16)
        map_a = np.ascontiguousarray(map_a, np.uint16)
        if map_xy.shape != (H, W, 2) or map_a.shape != (H, W):
            raise ValueError(f"maps must be ({H}, {W}, 2) int16 and ({H}, {W}) uint16, not {map_xy.shape} and {map_a.shape}")
        self.ctx.check(self.lib.ygzb_frames_set_undistort(self.h, _p(map_xy), _p(map_a)), "ygzb_frames_set_undistort")

    def copy_slot(self, src: int, dst: int):
        self.ctx.check(self.lib.ygzb_frames_copy(self.h, int(src), int(dst)), "ygzb_frames_copy")

    def build_pyramid(self, first: int, count: int):
        self.ctx.check(self.lib.ygzb_frames_build_pyramid(self.h, first, count), "ygzb_frames_build_pyramid")

    def download_level(self, slot: int, level: int) -> np.ndarray:
        out = np.empty((self.lh[level], self.lw[level]), np.uint8)
        self.ctx.check(self.lib.ygzb_frames_download_level(self.h, slot, level, _p(out)), "ygzb_frames_download_level")
        return out

    # ---- FeatureDetector -------------------------------------------------------------------------
    def detect(self, slots, occupied=None, fetch: bool = True):
        slots = np.ascontiguousarray(slots, np.int32)
        n = len(slots)
        occ = None if occupied is None else np.ascontiguousarray(occupied, np.uint8).reshape(n, self.ctx.n_cells)
        if not fetch:
            self.ctx.check(self.lib.ygzb_detect(self.h, _p(slots), n, _p(occ), None), "ygzb_detect")
            return None
        cap = n * self.ctx.n_cells
        if getattr(self, "_kp_cap", 0) < cap:
            self._kp = dict(offsets=np.empty(self.capacity + 1, np.int32), x=np.empty(cap, np.float32),
                            y=np.empty(cap, np.float32), level=np.empty(cap, np.uint8), score=np.empty(cap, np.float32),
                            angle=np.empty(cap, np.float32), desc=np.empty((cap, 32), np.uint8), cell=np.empty(cap, np.int32))
            self._kp_cap = cap
        b = self._kp
        kp = Keypoints(*[b[k].ctypes.data for k in ("offsets", "x", "y", "level", "score", "angle", "desc", "cell")], cap)
        self.ctx.check(self.lib.ygzb_detect(self.h, _p(slots), n, _p(occ), C.byref(kp)), "ygzb_detect")
        off = b["offsets"][: n + 1].copy()
        out = []
        for i in range(n):
            s, e = off[i], off[i + 1]
            out.append(dict(n=int(e - s), px=b["x"][s:e].astype(np.float64), py=b["y"][s:e].astype(np.float64),
                            level=b["level"][s:e].astype(np.int32), score=b["score"][s:e].copy(),
                            angle=b["angle"][s:e].copy(), desc=b["desc"][s:e].copy(), cell=b["cell"][s:e].copy()))
        return out

    def detect_packed(self, slots, occupied=None):
        """Like detect() but returns (offsets[n+1], packed arrays dict) without per-frame splitting."""
        slots = np.ascontiguousarray(slots, np.int32)
        n = len(slots)
        occ = None if occupied is None else np.ascontiguousarray(occupied, np.uint8).reshape(n, self.ctx.n_cells)
        cap = n * self.ctx.n_cells
        if getattr(self, "_kpp_cap", 0) < cap:
            self._kpp = dict(offsets=pinned_empty(self.capacity + 1, np.int32), x=pinned_empty(cap, np.float32),
                             y=pinned_empty(cap, np.float32), level=pinned_empty(cap, np.uint8), score=pinned_empty(cap, np.float32),
                             angle=pinned_empty(cap, np.float32), desc=pinned_empty((cap, 32), np.uint8),
                             cell=pinned_empty(cap, np.int32))
            self._kpp_cap = cap
        b = self._kpp
        kp = Keypoints(*[b[k].ctypes.data for k in ("offsets", "x", "y", "level", "score", "angle", "desc", "cell")], cap)
        self.ctx.check(self.lib.ygzb_detect(self.h, _p(slots), n, _p(occ), C.byref(kp)), "ygzb_detect")
        return b["offsets"][: n + 1], b

    def match_packed(self, a_slots, b_slots, cross_check=True):
        a = np.ascontiguousarray(a_slots, np.int32)
        b = np.ascontiguousarray(b_slots, np.int32)
        n = len(a)
        cap = n * self.ctx.n_cells
        if getattr(self, "_mp_cap", 0) < cap:
            self._mp = (pinned_empty(n + 1, np.int32), pinned_empty(cap, np.int32), pinned_empty(cap, np.int32))
            self._mp_cap = cap
        qoff, idx, dist = self._mp
        if len(qoff) < n + 1:
            qoff = pinned_empty(n + 1, np.int32)
            self._mp = (qoff, idx, dist)
        self.ctx.check(self.lib.ygzb_match_frames(self.h, _p(a), _p(b), n, int(cross_check), _p(qoff), _p(idx), _p(dist),
                                                  cap), "ygzb_match_frames")
        return qoff[: n + 1], idx, dist

    def detect_stats(self, n: int) -> np.ndarray:
        st = np.empty((n, self.ctx.n_levels, 2), np.int32)
        self.ctx.check(self.lib.ygzb_detect_stats(self.h, n, _p(st)), "ygzb_detect_stats")
        return st

    def describe(self, slots, offsets, px, py, level):
        slots = np.ascontiguousarray(slots, np.int32)
        offsets = np.ascontiguousarray(offsets, np.int32)
        px = np.ascontiguousarray(px, np.float64)
        py = np.ascontiguousarray(py, np.float64)
        level = np.ascontiguousarray(level, np.uint8)
        total = int(offsets[-1])
        angle = np.empty(total, np.float32)
        desc = np.empty((total, 32), np.uint8)
        self.ctx.check(self.lib.ygzb_describe(self.h, _p(slots), len(slots), _p(offsets), _p(px), _p(py), _p(level),
                                              _p(angle), _p(desc)), "ygzb_describe")
        return angle, desc

    def fast_debug(self, slot: int, level: int):
        cap = self.lw[level] * self.lh[level]
        xy = np.empty((cap, 2), np.int16)
        scores = np.empty(cap, np.int32)
        nm = np.empty(cap, np.int32)
        nc, nn = C.c_int32(), C.c_int32()
        self.ctx.check(self.lib.ygzb_fast_debug(self.h, slot, level, cap, _p(xy), _p(scores), C.byref(nc), _p(nm),
                                                C.byref(nn)), "ygzb_fast_debug")
        return xy[: nc.value].copy(), scores[: nc.value].copy(), nm[: nn.value].copy()

    # ---- Matcher -----------------------------------------------------------------------------------
    def match(self, a_slots, b_slots, cross_check=True, fetch: bool = True):
        a = np.ascontiguousarray(a_slots, np.int32)
        b = np.ascontiguousarray(b_slots, np.int32)
        n = len(a)
        if not fetch:
            self.ctx.check(self.lib.ygzb_match_frames(self.h, _p(a), _p(b), n, int(cross_check), None, None, None, 0),
                           "ygzb_match_frames")
            return None
        cap = n * self.ctx.n_cells
        if getattr(self, "_m_cap", 0) < cap:
            self._m = (np.empty(self.capacity * 4 + 1, np.int32), np.empty(cap, np.int32), np.empty(cap, np.int32))
            self._m_cap = cap
        qoff, idx, dist = self._m
        if len(qoff) < n + 1:
            qoff = np.empty(n + 1, np.int32)
        self.ctx.check(self.lib.ygzb_match_frames(self.h, _p(a), _p(b), n, int(cross_check), _p(qoff), _p(idx), _p(dist),
                                                  cap), "ygzb_match_frames")
        return [(idx[qoff[i]: qoff[i + 1]].copy(), dist[qoff[i]: qoff[i + 1]].copy()) for i in range(n)]


# ---- photometric alignment (methods attached to Frames) ------------------------------------------------
def _align2d(self, slot, level, ref_border, ref, uv, n_iter=10):
    slot = np.ascontiguousarray(slot, np.int32)
    n = len(slot)
    level = np.ascontiguousarray(level, np.uint8)
    rb = np.ascontiguousarray(ref_border, np.uint8).reshape(n, 100)
    rf = None if ref is None else np.ascontiguousarray(ref, np.uint8).reshape(n, 64)
    uv = np.ascontiguousarray(uv, np.float64).reshape(n, 2).copy()
    ok = np.zeros(n, np.uint8)
    self.ctx.check(self.lib.ygzb_align2d(self.h, n, _p(slot), _p(level), _p(rb), _p(rf), n_iter, _p(uv), _p(ok)), "ygzb_align2d")
    return uv, ok.astype(bool)


def _project_align(self, ref_slot, cur_slot, poses, ref_pose, cur_pose, ref_px, ref_depth, ref_level, cur_px):
    ref_slot = np.ascontiguousarray(ref_slot, np.int32)
    n = len(ref_slot)
    cur_slot = np.ascontiguousarray(cur_slot, np.int32)
    poses = np.ascontiguousarray(poses, np.float64).reshape(-1, 12)
    cur = np.ascontiguousarray(cur_px, np.float64).reshape(n, 2).copy()
    lvl = np.zeros(n, np.uint8)
    ok = np.zeros(n, np.uint8)
    self.ctx.check(self.lib.ygzb_project_align(
        self.h, n, _p(ref_slot), _p(cur_slot), len(poses), _p(poses), _p(np.ascontiguousarray(ref_pose, np.int32)),
        _p(np.ascontiguousarray(cur_pose, np.int32)), _p(np.ascontiguousarray(ref_px, np.float64)),
        _p(np.ascontiguousarray(ref_depth, np.float64)), _p(np.ascontiguousarray(ref_level, np.uint8)), _p(cur), _p(lvl), _p(ok)),
        "ygzb_project_align")
    return cur, lvl.astype(np.int32), ok.astype(bool)


def _sparse_align(self, ref_slot, cur_slot, offsets, px, depth, has_mp, T_ref, T_cur, max_level=2, min_level=0, n_iter=30, eps=1e-6):
    ref_slot = np.ascontiguousarray(ref_slot, np.int32)
    P = len(ref_slot)
    T = np.ascontiguousarray(T_cur, np.float64).reshape(P, 12).copy()
    nm = np.zeros(P, np.int32)
    iters = np.zeros((P, MAX_LEVELS), np.int32)
    self.ctx.check(self.lib.ygzb_sparse_align(
        self.h, P, _p(ref_slot), _p(np.ascontiguousarray(cur_slot, np.int32)), _p(np.ascontiguousarray(offsets, np.int32)),
        _p(np.ascontiguousarray(px, np.float64)), _p(np.ascontiguousarray(depth, np.float64)),
        _p(np.ascontiguousarray(has_mp, np.uint8)), _p(np.ascontiguousarray(T_ref, np.float64).reshape(P, 12)), _p(T),
        max_level, min_level, n_iter, C.c_double(eps), _p(nm), _p(iters)), "ygzb_sparse_align")
    return T.reshape(P, 3, 4), nm, iters


def _align1d(self, slot, level, direction, ref_border, ref, uv, n_iter=10):
    slot = np.ascontiguousarray(slot, np.int32)
    n = len(slot)
    rb = np.ascontiguousarray(ref_border, np.uint8).reshape(n, 100)
    rf = None if ref is None else np.ascontiguousarray(ref, np.uint8).reshape(n, 64)
    uv = np.ascontiguousarray(uv, np.float64).reshape(n, 2).copy()
    ok = np.zeros(n, np.uint8)
    hinv = np.zeros(n, np.float64)
    self.ctx.check(self.lib.ygzb_align1d(self.h, n, _p(slot), _p(np.ascontiguousarray(level, np.uint8)),
                                         _p(np.ascontiguousarray(direction, np.float32).reshape(n, 2)), _p(rb), _p(rf), n_iter, _p(uv),
                                         _p(ok), _p(hinv)), "ygzb_align1d")
    return uv, ok.astype(bool), hinv


Frames.align2d = _align2d
Frames.align1d = _align1d
Frames.project_align = _project_align
Frames.sparse_align = _sparse_align


# ---- bundle adjustment (methods attached to Context) ---------------------------------------------------
class BAParams(C.Structure):
    _fields_ = [("max_iters", C.c_int), ("huber_delta", C.c_double), ("chi2_outlier", C.c_double), ("tau", C.c_double),
                ("max_trials", C.c_int)]


class BAStats(C.Structure):
    _fields_ = [("iters", C.c_int), ("lm_trials", C.c_int), ("chi2_initial", C.c_double), ("chi2_final", C.c_double),
                ("lambda_final", C.c_double), ("n_outliers", C.c_int)]


def _local_ba(self, kf_off, pt_off, obs_off, poses, fixed, pts, kf_idx, pt_idx, px, max_iters=20, huber=5.991, tau=1e-5,
              max_trials=10, chi2_outlier=5.991):
    """Batched ba::LocalBAG2O.  poses: (n_kf, 6) in g2o order [omega; upsilon]."""
    kf_off = np.ascontiguousarray(kf_off, np.int32)
    P = len(kf_off) - 1
    poses = np.ascontiguousarray(poses, np.float64).copy()
    pts = np.ascontiguousarray(pts, np.float64).copy()
    prm = BAParams()
    self.lib.ygzb_default_ba_params(C.byref(prm))
    prm.max_iters = max_iters
    prm.huber_delta = huber
    prm.tau = tau
    prm.max_trials = max_trials
    prm.chi2_outlier = chi2_outlier
    outl = np.zeros(len(kf_idx), np.uint8)
    st = (BAStats * P)()
    self.check(self.lib.ygzb_local_ba(self.h, P, _p(kf_off), _p(np.ascontiguousarray(pt_off, np.int32)),
                                      _p(np.ascontiguousarray(obs_off, np.int32)), _p(poses),
                                      _p(np.ascontiguousarray(fixed, np.uint8)), _p(pts),
                                      _p(np.ascontiguousarray(kf_idx, np.int32)), _p(np.ascontiguousarray(pt_idx, np.int32)),
                                      _p(np.ascontiguousarray(px, np.float64)), C.byref(prm), _p(outl), st), "ygzb_local_ba")
    stats = [{k: getattr(s_, k) for k, _ in BAStats._fields_} for s_ in st]
    return poses, pts, outl.astype(bool), stats


class CeresStats(C.Structure):
    _fields_ = [("iters", C.c_int), ("successful_steps", C.c_int), ("cost_initial", C.c_double), ("cost_final", C.c_double),
                ("radius_final", C.c_double), ("termination", C.c_int)]


def _local_ba_ceres(self, kf_off, pt_off, obs_off, poses_t_aa, fixed, pts, kf_idx, pt_idx, px, max_iters=50, huber=0.0):
    """Batched ba::LocalBA (Ceres twin).  poses: (n_kf, 6) as [t; angle-axis]."""
    kf_off = np.ascontiguousarray(kf_off, np.int32)
    P = len(kf_off) - 1
    poses = np.ascontiguousarray(poses_t_aa, np.float64).copy()
    pts = np.ascontiguousarray(pts, np.float64).copy()
    st = (CeresStats * P)()
    self.check(self.lib.ygzb_local_ba_ceres(self.h, P, _p(kf_off), _p(np.ascontiguousarray(pt_off, np.int32)),
                                            _p(np.ascontiguousarray(obs_off, np.int32)), _p(poses),
                                            _p(np.ascontiguousarray(fixed, np.uint8)), _p(pts),
                                            _p(np.ascontiguousarray(kf_idx, np.int32)), _p(np.ascontiguousarray(pt_idx, np.int32)),
                                            _p(np.ascontiguousarray(px, np.float64)), max_iters, C.c_double(huber), st),
               "ygzb_local_ba_ceres")
    return poses, pts, [{k: getattr(s_, k) for k, _ in CeresStats._fields_} for s_ in st]


def _pose_only(self, offsets, pt_world, px, T_cw):
    offsets = np.ascontiguousarray(offsets, np.int32)
    P = len(offsets) - 1
    n = int(offsets[-1])
    T = np.ascontiguousarray(T_cw, np.float64).reshape(P, 12).copy()
    inl = np.zeros(n, np.uint8)
    depth = np.zeros(n, np.float64)
    cnt = np.zeros(P, np.int32)
    self.check(self.lib.ygzb_pose_only(self.h, P, _p(offsets), _p(np.ascontiguousarray(pt_world, np.float64)),
                                       _p(np.ascontiguousarray(px, np.float64)), _p(T), _p(inl), _p(depth), _p(cnt)),
               "ygzb_pose_only")
    return T.reshape(P, 3, 4), inl.astype(bool), depth, cnt


def _two_view_ba(self, offsets, T_ref, T_cur, px_ref, px_cur, inlier, pts):
    """Batched ba::TwoViewBACeres.  Returns (T_cur (P,3,4), inlier bool, pts, stats)."""
    offsets = np.ascontiguousarray(offsets, np.int32)
    P = len(offsets) - 1
    n = int(offsets[-1])
    Tr = np.ascontiguousarray(T_ref, np.float64).reshape(P, 12)
    Tc = np.ascontiguousarray(T_cur, np.float64).reshape(P, 12).copy()
    inl = np.ascontiguousarray(inlier, np.uint8).copy()
    X = np.ascontiguousarray(pts, np.float64).reshape(n, 3).copy()
    st = (CeresStats * P)()
    self.check(self.lib.ygzb_two_view_ba(self.h, P, _p(offsets), _p(Tr), _p(Tc), _p(np.ascontiguousarray(px_ref, np.float64)),
                                         _p(np.ascontiguousarray(px_cur, np.float64)), _p(inl), _p(X), st), "ygzb_two_view_ba")
    return Tc.reshape(P, 3, 4), inl.astype(bool), X, [{k: getattr(s_, k) for k, _ in CeresStats._fields_} for s_ in st]


def _search_for_triangulation(self, off1, off2, desc1, px1, node1, desc2, px2, node2, E12, th_low=65, epipolar_dsqr=1e-4):
    """Batched Matcher::SearchForTriangulation: match12 per key-frame-1 feature (index local to key-frame 2 of its pair, or -1)."""
    off1 = np.ascontiguousarray(off1, np.int32)
    off2 = np.ascontiguousarray(off2, np.int32)
    out = np.full(int(off1[-1]), -1, np.int32)
    self.check(self.lib.ygzb_search_for_triangulation(self.h, len(off1) - 1, _p(off1), _p(off2), _p(np.ascontiguousarray(desc1, np.uint8)),
                                                      _p(np.ascontiguousarray(px1, np.float64)), _p(np.ascontiguousarray(node1, np.int32)),
                                                      _p(np.ascontiguousarray(desc2, np.uint8)), _p(np.ascontiguousarray(px2, np.float64)),
                                                      _p(np.ascontiguousarray(node2, np.int32)), _p(np.ascontiguousarray(E12, np.float64)),
                                                      int(th_low), C.c_double(epipolar_dsqr), _p(out)), "ygzb_search_for_triangulation")
    return out


def _depth_from_triangulation(self, T, pose_of, f_ref, f_cur, det_th=1e-5):
    T = np.ascontiguousarray(T, np.float64).reshape(-1, 12)
    f_ref = np.ascontiguousarray(f_ref, np.float64).reshape(-1, 3)
    n = len(f_ref)
    d1, d2, ok = np.zeros(n), np.zeros(n), np.zeros(n, np.uint8)
    po = None if pose_of is None else np.ascontiguousarray(pose_of, np.int32)
    self.check(self.lib.ygzb_depth_from_triangulation(self.h, n, len(T), _p(T), _p(po), _p(f_ref), _p(np.ascontiguousarray(f_cur, np.float64)),
                                                      C.c_double(det_th), _p(d1), _p(d2), _p(ok)), "ygzb_depth_from_triangulation")
    return d1, d2, ok.astype(bool)


class Vocabulary:
    """DBoW3 vocabulary resident on the device (ygzb_vocab_*): Vocabulary::loadFromBinaryFile + transform."""

    def __init__(self, ctx, data: bytes):
        self.ctx = ctx
        self.h = C.c_void_p()
        ctx.lib.ygzb_vocab_create.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_void_p]
        ctx.check(ctx.lib.ygzb_vocab_create(ctx.h, data, len(data), C.byref(self.h)), "ygzb_vocab_create")

    def close(self):
        if self.h:
            self.ctx.lib.ygzb_vocab_destroy.argtypes = [C.c_void_p]
            self.ctx.lib.ygzb_vocab_destroy.restype = None
            self.ctx.lib.ygzb_vocab_destroy(self.h)
            self.h = C.c_void_p()

    def info(self):
        out = np.zeros(6, np.int32)
        self.ctx.check(self.ctx.lib.ygzb_vocab_info(self.h, _p(out)), "ygzb_vocab_info")
        return dict(zip(("k", "L", "scoring", "weighting", "nodes", "words"), out.tolist()))

    def transform(self, offsets, desc, levelsup=4):
        """-> word, node, weight per descriptor and, per frame, the BowVector as (word ids ascending, values)."""
        offsets = np.ascontiguousarray(offsets, np.int32)
        n, F = int(offsets[-1]), len(offsets) - 1
        word, node, weight = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n)
        cnt, bw, bv = np.zeros(F, np.int32), np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1))
        self.ctx.check(self.ctx.lib.ygzb_bow_transform(self.h, F, _p(offsets), _p(np.ascontiguousarray(desc, np.uint8)), int(levelsup), _p(word),
                                                       _p(node), _p(weight), _p(cnt), _p(bw), _p(bv)), "ygzb_bow_transform")
        bows = [(bw[offsets[f]:offsets[f] + cnt[f]].copy(), bv[offsets[f]:offsets[f] + cnt[f]].copy()) for f in range(F)]
        return word, node, weight, bows


def _search_by_bow(self, off1, off2, desc1, node1, angle1, desc2, node2, angle2, th_low=50, knn_ratio=0.9, check_orientation=False):
    """Batched Matcher::SearchByBoW -> (match12, count per pair)."""
    off1 = np.ascontiguousarray(off1, np.int32)
    off2 = np.ascontiguousarray(off2, np.int32)
    P = len(off1) - 1
    out = np.full(int(off1[-1]), -1, np.int32)
    cnt = np.zeros(P, np.int32)
    a1 = None if angle1 is None else np.ascontiguousarray(angle1, np.float32)
    a2 = None if angle2 is None else np.ascontiguousarray(angle2, np.float32)
    self.lib.ygzb_search_by_bow.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 8 + [C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_void_p]
    self.check(self.lib.ygzb_search_by_bow(self.h, P, _p(off1), _p(off2), _p(np.ascontiguousarray(desc1, np.uint8)),
                                           _p(np.ascontiguousarray(node1, np.int32)), _p(a1), _p(np.ascontiguousarray(desc2, np.uint8)),
                                           _p(np.ascontiguousarray(node2, np.int32)), _p(a2), int(th_low), float(knn_ratio),
                                           int(check_orientation), _p(out), _p(cnt)), "ygzb_search_by_bow")
    return out, cnt


def _initializer_ransac(self, offsets, px1, px2, sets, sigma=2.0, models=False):
    """Batched Initializer::FindHomography + FindFundamental; sets: [n_lists][max_iter][8] indices local to each list."""
    offsets = np.ascontiguousarray(offsets, np.int32)
    P, N = len(offsets) - 1, int(offsets[-1])
    sets = np.ascontiguousarray(sets, np.int32).reshape(P, -1, 8)
    I = sets.shape[1]
    H, F = np.zeros((P, 9)), np.zeros((P, 9))
    sh, sf = np.zeros(P, np.float32), np.zeros(P, np.float32)
    bh, bf = np.zeros(P, np.int32), np.zeros(P, np.int32)
    ih, jf = np.zeros(max(N, 1), np.uint8), np.zeros(max(N, 1), np.uint8)
    mod = np.zeros((P, I, 18)) if models else None
    self.lib.ygzb_initializer_ransac.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_float] + [C.c_void_p] * 9
    self.check(self.lib.ygzb_initializer_ransac(self.h, P, _p(offsets), _p(np.ascontiguousarray(px1, np.float64)), _p(np.ascontiguousarray(px2, np.float64)),
                                                I, _p(sets), C.c_float(sigma), _p(H), _p(sh), _p(bh), _p(ih), _p(F), _p(sf), _p(bf), _p(jf), _p(mod)),
               "ygzb_initializer_ransac")
    out = dict(H21=H.reshape(P, 3, 3), score_H=sh, best_H=bh, inliers_H=ih[:N].astype(bool), F21=F.reshape(P, 3, 3), score_F=sf, best_F=bf,
               inliers_F=jf[:N].astype(bool))
    if models:
        out["models"] = mod
    return out


def _initializer_reconstruct(self, offsets, px1, px2, use_h, model, inliers, sigma2=4.0, min_parallax=1.0, min_triangulated=8, ratio_h=0.9):
    """Batched Initializer::ReconstructH / ReconstructF on the chosen models."""
    offsets = np.ascontiguousarray(offsets, np.int32)
    P, N = len(offsets) - 1, int(offsets[-1])
    ok, R, t = np.zeros(P, np.int32), np.zeros((P, 9)), np.zeros((P, 3))
    p3d, tri, ng, par, cand = np.zeros((N, 3)), np.zeros(N, np.uint8), np.zeros((P, 8), np.int32), np.zeros(P), np.zeros((P, 8, 12))
    self.lib.ygzb_initializer_reconstruct.argtypes = ([C.c_void_p, C.c_int] + [C.c_void_p] * 6 + [C.c_float, C.c_float, C.c_int, C.c_double]
                                                      + [C.c_void_p] * 8)
    self.check(self.lib.ygzb_initializer_reconstruct(self.h, P, _p(offsets), _p(np.ascontiguousarray(px1, np.float64)),
                                                     _p(np.ascontiguousarray(px2, np.float64)), _p(np.ascontiguousarray(use_h, np.int32)),
                                                     _p(np.ascontiguousarray(model, np.float64).reshape(P, 9)),
                                                     _p(np.ascontiguousarray(inliers, np.uint8)), C.c_float(sigma2), C.c_float(min_parallax),
                                                     int(min_triangulated), C.c_double(ratio_h), _p(ok), _p(R), _p(t), _p(p3d), _p(tri), _p(ng),
                                                     _p(par), _p(cand)), "ygzb_initializer_reconstruct")
    return dict(ok=ok.astype(bool), R21=R.reshape(P, 3, 3), t21=t, p3d=p3d, triangulated=tri.astype(bool), n_good=ng, parallax=par,
                candidates=cand)


Context.initializer_reconstruct = _initializer_reconstruct
Context.initializer_ransac = _initializer_ransac
Context.search_by_bow = _search_by_bow
Context.vocabulary = lambda self, data: Vocabulary(self, data)
Context.search_for_triangulation = _search_for_triangulation
Context.depth_from_triangulation = _depth_from_triangulation
Context.local_ba = _local_ba
Context.local_ba_ceres = _local_ba_ceres
Context.pose_only = _pose_only
Context.two_view_ba = _two_view_ba


# ---- KLT (method attached to Frames) -------------------------------------------------------------------
class KLTParams(C.Structure):
    _fields_ = [("win", C.c_int), ("max_level", C.c_int), ("max_iter", C.c_int), ("eps", C.c_double), ("min_eig", C.c_double)]


def _klt(self, ref_slot, cur_slot, offsets, ref_xy, cur_xy, **overrides):
    """Batched calcOpticalFlowPyrLK; keyword overrides (win, max_level, max_iter, eps, min_eig) replace fields of
    ygzb_default_klt_params."""
    ref_slot = np.ascontiguousarray(ref_slot, np.int32)
    offsets = np.ascontiguousarray(offsets, np.int32)
    n = int(offsets[-1])
    out = np.ascontiguousarray(cur_xy, np.float32).reshape(n, 2).copy()
    status = np.zeros(n, np.uint8)
    err = np.zeros(n, np.float32)
    prm = KLTParams()
    self.lib.ygzb_default_klt_params(C.byref(prm))
    for k, v in overrides.items():
        if k not in ("win", "max_level", "max_iter", "eps", "min_eig"):
            raise TypeError(f"unknown KLT parameter {k}")
        setattr(prm, k, v)
    self.ctx.check(self.lib.ygzb_klt(self.h, len(ref_slot), _p(ref_slot), _p(np.ascontiguousarray(cur_slot, np.int32)), _p(offsets),
                                     _p(np.ascontiguousarray(ref_xy, np.float32)), _p(out), _p(status), _p(err), C.byref(prm)),
                   "ygzb_klt")
    return out, status.astype(bool), err


Frames.klt = _klt


# ---- map records of the device-resident tracker (ygzb_tracker_export / _import) ------------------------------------------
TRACK_RING = 4          # YGZB_TRACK_RING
MAP_OBS_PER_CELL = 4    # YGZB_MAP_OBS_PER_CELL
_MAP_ARRAYS = ("entry", "T_cw", "mp0", "n_features", "n_obs", "image", "px", "level", "depth", "pw", "obs_id", "obs_px")


class MapRecord(C.Structure):
    _fields_ = ([("width", C.c_int32), ("height", C.c_int32), ("cells", C.c_int32), ("n_levels", C.c_int32), ("K", C.c_double * 4),
                 ("n_keyframes", C.c_int32), ("pad", C.c_int32)] + [(k, C.c_void_p) for k in _MAP_ARRAYS])


class MapBuffers:
    """A ygzb_map_record with numpy arrays behind it, sized for `capacity` key-frames of a `width` x `height` image with
    `cells` grid cells.  `rec` may be an existing MapRecord (e.g. an element of a ctypes array) to point at the arrays."""

    def __init__(self, capacity, width, height, cells, images=True, rec=None):
        F, O = capacity * cells, capacity * MAP_OBS_PER_CELL * cells
        self.a = dict(entry=np.zeros(capacity, np.int32), T_cw=np.zeros((capacity, 12)), mp0=np.zeros(capacity, np.int64),
                      n_features=np.zeros(capacity, np.int32), n_obs=np.zeros(capacity, np.int32),
                      image=np.zeros((capacity, height, width), np.uint8) if images else None, px=np.zeros((F, 2)),
                      level=np.zeros(F, np.uint8), depth=np.zeros(F), pw=np.zeros((F, 3)), obs_id=np.zeros(O, np.int64),
                      obs_px=np.zeros((O, 2)))
        self.rec = MapRecord() if rec is None else rec
        for k in _MAP_ARRAYS:
            setattr(self.rec, k, None if self.a[k] is None else self.a[k].ctypes.data)

    @property
    def header(self):
        r = self.rec
        return dict(width=r.width, height=r.height, cells=r.cells, n_levels=r.n_levels, K=tuple(r.K), n_keyframes=r.n_keyframes)

    def keyframes(self):
        """Per key-frame dict of its live rows (copies): entry, T_cw (3x4), mp0, px, level, depth, pw, obs_id, obs_px, image."""
        a, out, f0, o0 = self.a, [], 0, 0
        for k in range(self.rec.n_keyframes):
            nf, no = int(a["n_features"][k]), int(a["n_obs"][k])
            out.append(dict(entry=int(a["entry"][k]), T_cw=a["T_cw"][k].reshape(3, 4).copy(), mp0=int(a["mp0"][k]), px=a["px"][f0:f0 + nf].copy(),
                            level=a["level"][f0:f0 + nf].copy(), depth=a["depth"][f0:f0 + nf].copy(), pw=a["pw"][f0:f0 + nf].copy(),
                            obs_id=a["obs_id"][o0:o0 + no].copy(), obs_px=a["obs_px"][o0:o0 + no].copy(),
                            image=None if a["image"] is None else a["image"][k].copy()))
            f0 += nf
            o0 += no
        return out

    def copy(self):
        """An independent record with the same header and array contents."""
        cap = len(self.a["entry"])
        other = MapBuffers(cap, self.rec.width, self.rec.height, self.a["level"].shape[0] // cap, images=self.a["image"] is not None)
        for k in _MAP_ARRAYS:
            if self.a[k] is not None:
                other.a[k][...] = self.a[k]
        for k in ("width", "height", "cells", "n_levels", "n_keyframes", "pad"):
            setattr(other.rec, k, getattr(self.rec, k))
        other.rec.K[:] = list(self.rec.K)
        return other


# ---- reference records of the previous-frame mode (ygzb_tracker_export_reference / _import_reference) ----------------------
REF_FEATURES_PER_CELL = TRACK_RING + 1   # YGZB_TRACK_REF_FEATURES_PER_CELL
_REF_ARRAYS = ("px", "depth", "image")


class ReferenceRecord(C.Structure):
    _fields_ = ([("width", C.c_int32), ("height", C.c_int32), ("cells", C.c_int32), ("n_levels", C.c_int32), ("K", C.c_double * 4),
                 ("capacity", C.c_int32), ("n", C.c_int32), ("T_cw", C.c_double * 12)] + [(k, C.c_void_p) for k in _REF_ARRAYS])


class ReferenceBuffers:
    """A ygzb_reference_record with numpy arrays behind it, sized for a `width` x `height` image with `cells` grid cells
    (capacity REF_FEATURES_PER_CELL * cells).  `rec` may be an existing ReferenceRecord to point at the arrays."""

    def __init__(self, width, height, cells, rec=None):
        cap = REF_FEATURES_PER_CELL * cells
        self.a = dict(px=np.zeros((cap, 2)), depth=np.zeros(cap), image=np.zeros((height, width), np.uint8))
        self.rec = ReferenceRecord() if rec is None else rec
        self.rec.capacity = cap
        for k in _REF_ARRAYS:
            setattr(self.rec, k, self.a[k].ctypes.data)

    @property
    def header(self):
        r = self.rec
        return dict(width=r.width, height=r.height, cells=r.cells, n_levels=r.n_levels, K=tuple(r.K), capacity=r.capacity, n=r.n)

    @property
    def T_cw(self):
        return np.array(self.rec.T_cw).reshape(3, 4)

    def copy(self):
        """An independent record with the same header, pose and array contents."""
        h, w = self.a["image"].shape
        other = ReferenceBuffers(w, h, self.a["depth"].shape[0] // REF_FEATURES_PER_CELL)
        for k in _REF_ARRAYS:
            other.a[k][...] = self.a[k]
        for k in ("width", "height", "cells", "n_levels", "capacity", "n"):
            setattr(other.rec, k, getattr(self.rec, k))
        other.rec.K[:] = list(self.rec.K)
        other.rec.T_cw[:] = list(self.rec.T_cw)
        return other


class TrackJob(C.Structure):
    _fields_ = [("stream", C.c_int32), ("cur_slot", C.c_int32), ("n_local", C.c_int32), ("entry", C.c_int32 * TRACK_RING), ("pad", C.c_int32)]


class TrackResult(C.Structure):
    _fields_ = [("T_cw", C.c_double * 12), ("n_meas", C.c_int32), ("aligned", C.c_int32), ("n_candidates", C.c_int32),
                ("n_projected", C.c_int32), ("n_inliers", C.c_int32), ("pad", C.c_int32 * 3)]


class KeyframeJob(C.Structure):
    _fields_ = [("stream", C.c_int32), ("frame_slot", C.c_int32), ("kf_slot", C.c_int32), ("entry", C.c_int32), ("track_job", C.c_int32),
                ("n_local", C.c_int32), ("local_entry", C.c_int32 * TRACK_RING), ("run_ba", C.c_int32), ("pad", C.c_int32), ("mp0", C.c_int64)]


class KeyframeResult(C.Structure):
    _fields_ = [("n_features", C.c_int32), ("ba_points", C.c_int32), ("ba_observations", C.c_int32), ("ba_iters", C.c_int32),
                ("ba_trials", C.c_int32), ("pad", C.c_int32), ("chi2_initial", C.c_double), ("chi2_final", C.c_double),
                ("T_cw", C.c_double * (12 * TRACK_RING))]


_DEBUG_ARRAYS = ("cand_ok", "cand_px", "c_src", "c_px", "c_pw", "inlier")


class TrackDebug(C.Structure):
    _fields_ = ([("T_aligned", C.c_double * 12), ("rel", C.c_double * (12 * TRACK_RING)), ("n_local", C.c_int32), ("n_meas", C.c_int32),
                 ("aligned", C.c_int32), ("n_candidates", C.c_int32), ("n_projected", C.c_int32), ("n_inliers", C.c_int32)]
                + [(k, C.c_void_p) for k in _DEBUG_ARRAYS])


def _record(s):
    """dict of a ctypes record without its padding; array fields as float64 numpy arrays."""
    return {k: (np.array(getattr(s, k)[:]) if isinstance(getattr(s, k), C.Array) else getattr(s, k)) for k, _ in s._fields_ if k != "pad"}


class Tracker:
    """The device-resident tracker (ygzb_tracker) on a frame pool: its map records (export / import) and thin wrappers of the
    tracking entry points, each followed by a synchronisation."""

    def __init__(self, frames: Frames, n_streams: int, max_jobs: int, K):
        self.frames, self.ctx, self.lib = frames, frames.ctx, frames.lib
        self.lib.ygzb_tracker_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        self.lib.ygzb_tracker_destroy.argtypes = [C.c_void_p]
        self.lib.ygzb_tracker_destroy.restype = None
        self.lib.ygzb_tracker_export.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        self.lib.ygzb_tracker_import.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        self.lib.ygzb_tracker_set_depth.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        self.lib.ygzb_tracker_set_start_pose.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        self.lib.ygzb_tracker_upload.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
        self.lib.ygzb_tracker_track.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        self.lib.ygzb_tracker_make_keyframes.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        self.lib.ygzb_tracker_debug_job.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        self.lib.ygzb_tracker_set_reference_mode.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        self.lib.ygzb_tracker_debug_reference.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        self.lib.ygzb_tracker_export_reference.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        self.lib.ygzb_tracker_import_reference.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        Kd = np.ascontiguousarray(K, np.float64)
        h = C.c_void_p()
        self.ctx.check(self.lib.ygzb_tracker_create(frames.h, n_streams, max_jobs, _p(Kd), C.byref(h)), "ygzb_tracker_create")
        self.h = h
        self.n_streams = n_streams

    def close(self):
        if getattr(self, "h", None) and getattr(self.ctx, "h", None):
            self.lib.ygzb_tracker_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def export(self, stream: int, entries, images: bool = True, out: MapBuffers | None = None) -> MapBuffers:
        """Map record of ring entries `entries` of `stream`, complete (the call synchronises the context)."""
        entries = np.ascontiguousarray(entries, np.int32)
        if out is None:
            f = self.frames
            out = MapBuffers(TRACK_RING, f.lw[0], f.lh[0], self.ctx.n_cells, images=images)
        self.ctx.check(self.lib.ygzb_tracker_export(self.h, int(stream), len(entries), _p(entries), C.byref(out.rec)), "ygzb_tracker_export")
        self.ctx.synchronize()
        return out

    def import_(self, stream: int, entries, kf_slots, rec: MapBuffers):
        entries = np.ascontiguousarray(entries, np.int32)
        kf_slots = np.ascontiguousarray(kf_slots, np.int32)
        self.ctx.check(self.lib.ygzb_tracker_import(self.h, int(stream), _p(entries), _p(kf_slots), C.byref(rec.rec)), "ygzb_tracker_import")
        self.ctx.synchronize()

    def export_reference(self, stream: int, out: ReferenceBuffers | None = None) -> ReferenceBuffers:
        """Reference record of `stream` (previous-frame mode), complete (the call synchronises the context)."""
        if out is None:
            f = self.frames
            out = ReferenceBuffers(f.lw[0], f.lh[0], self.ctx.n_cells)
        self.ctx.check(self.lib.ygzb_tracker_export_reference(self.h, int(stream), C.byref(out.rec)), "ygzb_tracker_export_reference")
        self.ctx.synchronize()
        return out

    def import_reference(self, stream: int, rec: ReferenceBuffers):
        """`rec` becomes the current reference of `stream`; import the stream's map first."""
        self.ctx.check(self.lib.ygzb_tracker_import_reference(self.h, int(stream), C.byref(rec.rec)), "ygzb_tracker_import_reference")
        self.ctx.synchronize()

    def set_depth(self, stream: int, depth):
        """Depth image (H, W) that initialises the map points of `stream`'s next key-frame."""
        depth = np.ascontiguousarray(depth, np.float64)
        self.ctx.check(self.lib.ygzb_tracker_set_depth(self.h, int(stream), _p(depth)), "ygzb_tracker_set_depth")
        self.ctx.synchronize()

    def set_start_pose(self, stream: int, T_cw):
        """T_cw (3, 4) that `stream`'s next first key-frame (a key-frame job with track_job = -1) takes; identity by default."""
        T = np.ascontiguousarray(T_cw, np.float64).reshape(12)
        self.ctx.check(self.lib.ygzb_tracker_set_start_pose(self.h, int(stream), _p(T)), "ygzb_tracker_set_start_pose")

    def upload(self, first: int, images):
        """Grey frames (n, H, W) into slots [first, first + n)."""
        images = np.ascontiguousarray(images, np.uint8)
        if images.ndim == 2:
            images = images[None]
        self.ctx.check(self.lib.ygzb_tracker_upload(self.h, int(first), len(images), _p(images), C.c_size_t(images[0].size)),
                       "ygzb_tracker_upload")
        self.ctx.synchronize()

    def track(self, jobs):
        """jobs: (stream, cur_slot, ring entries of the local key-frames, oldest first).  One result dict per job: T_cw (3, 4),
        n_meas, aligned, n_candidates, n_projected, n_inliers."""
        arr = (TrackJob * len(jobs))()
        for q, (stream, slot, entries) in zip(arr, jobs):
            q.stream, q.cur_slot, q.n_local = int(stream), int(slot), len(entries)
            q.entry[:len(entries)] = [int(e) for e in entries]
        res = (TrackResult * len(jobs))()
        self.ctx.check(self.lib.ygzb_tracker_track(self.h, len(jobs), arr, res), "ygzb_tracker_track")
        self.ctx.synchronize()
        out = [_record(r) for r in res]
        for r in out:
            r["T_cw"] = r["T_cw"].reshape(3, 4)
        return out

    def make_keyframes(self, jobs, ba: BAParams | None = None):
        """jobs: dicts with the fields of ygzb_keyframe_job (local_entry: a list, oldest first; run_ba and mp0 default to 0).
        One result dict per job: n_features, ba_points, ba_observations, ba_iters, ba_trials, chi2_initial, chi2_final and
        T_cw (n_local, 3, 4)."""
        arr = (KeyframeJob * len(jobs))()
        for q, j in zip(arr, jobs):
            q.stream, q.frame_slot, q.kf_slot, q.entry, q.track_job = (int(j[k]) for k in ("stream", "frame_slot", "kf_slot", "entry", "track_job"))
            q.n_local = len(j["local_entry"])
            q.local_entry[:q.n_local] = [int(e) for e in j["local_entry"]]
            q.run_ba, q.mp0 = int(j.get("run_ba", 0)), int(j.get("mp0", 0))
        if ba is None:
            ba = BAParams()
            self.lib.ygzb_default_ba_params(C.byref(ba))
        res = (KeyframeResult * len(jobs))()
        self.ctx.check(self.lib.ygzb_tracker_make_keyframes(self.h, len(jobs), arr, C.byref(ba), res), "ygzb_tracker_make_keyframes")
        self.ctx.synchronize()
        out = [_record(r) for r in res]
        for r, q in zip(out, arr):
            r["T_cw"] = r["T_cw"].reshape(TRACK_RING, 3, 4)[:q.n_local]
        return out

    def debug_job(self, job: int):
        """ygzb_tracker_debug_job: the intermediate state of job `job` of the last track() batch.  The dense arrays (cand_ok,
        cand_px) cover MAP_OBS_PER_CELL * cells entries; the compacted ones (c_src, c_px, c_pw, inlier) are cut to
        n_projected; rel to n_local."""
        cap = MAP_OBS_PER_CELL * self.ctx.n_cells
        a = dict(cand_ok=np.zeros(cap, np.uint8), cand_px=np.zeros((cap, 2)), c_src=np.zeros(cap, np.int32), c_px=np.zeros((cap, 2)),
                 c_pw=np.zeros((cap, 3)), inlier=np.zeros(cap, np.uint8))
        d = TrackDebug()
        for k in _DEBUG_ARRAYS:
            setattr(d, k, a[k].ctypes.data)
        self.ctx.check(self.lib.ygzb_tracker_debug_job(self.h, int(job), C.byref(d)), "ygzb_tracker_debug_job")
        out = _record(d)
        n = d.n_projected
        out.update(T_aligned=out["T_aligned"].reshape(3, 4), rel=out["rel"].reshape(TRACK_RING, 3, 4)[:d.n_local], cand_ok=a["cand_ok"].astype(bool),
                   cand_px=a["cand_px"], c_src=a["c_src"][:n], c_px=a["c_px"][:n], c_pw=a["c_pw"][:n], inlier=a["inlier"][:n].astype(bool))
        return out

    def set_reference_mode(self, mode: str, ref_slots=None):
        """ygzb_tracker_set_reference_mode: "keyframe" or "previous" (ref_slots: one frame slot per stream)."""
        slots = None if ref_slots is None else np.ascontiguousarray(ref_slots, np.int32)
        self.ctx.check(self.lib.ygzb_tracker_set_reference_mode(self.h, {"keyframe": 0, "previous": 1}.get(mode, -1),
                                                                 None if slots is None else _p(slots)), "ygzb_tracker_set_reference_mode")

    def debug_reference(self, stream: int):
        """ygzb_tracker_debug_reference: the stream's current reference -- dict(slot, T_cw (3, 4), px (n, 2), depth (n,))."""
        cap = (TRACK_RING + 1) * self.ctx.n_cells
        px, depth = np.zeros((cap, 2)), np.zeros(cap)
        r = TrackReference()
        r.capacity = cap
        r.px, r.depth = px.ctypes.data, depth.ctypes.data
        self.ctx.check(self.lib.ygzb_tracker_debug_reference(self.h, int(stream), C.byref(r)), "ygzb_tracker_debug_reference")
        return dict(slot=r.slot, T_cw=np.array(r.T_cw).reshape(3, 4), px=px[:r.n].copy(), depth=depth[:r.n].copy())


class TrackReference(C.Structure):
    _fields_ = [("slot", C.c_int32), ("n", C.c_int32), ("capacity", C.c_int32), ("pad", C.c_int32), ("T_cw", C.c_double * 12),
                ("px", C.c_void_p), ("depth", C.c_void_p)]


Frames.tracker = lambda self, n_streams, max_jobs, K: Tracker(self, n_streams, max_jobs, K)
