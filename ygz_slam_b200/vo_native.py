"""ctypes harness for the native tracking loop (host/vo_driver.cpp -> libygz_vo.so): the C++ twin of
vo.VisualOdometry with the GPU backend, used by bench.py for BASELINE config C5 and by the tests to compare both loops."""
from __future__ import annotations

import ctypes as C
from operator import itemgetter
from pathlib import Path

import numpy as np

from . import build
from .capi import INFO_DTYPE, MAP_POINT_DTYPE, unpack_sym6

_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        path = Path(build.VO_LIB)
        if not path.exists():
            build.build()          # builds libygz_b200.so first if needed, then the driver
        _LIB = C.CDLL(str(path))
        _LIB.ygz_vo_run.restype = C.c_int
        _LIB.ygz_vo_run.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                    C.c_double, C.c_double, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.ygz_vo_run_ex.restype = C.c_int
        _LIB.ygz_vo_run_ex.argtypes = _LIB.ygz_vo_run.argtypes + [C.c_int]
        _LIB.ygz_vo_run_handoff.restype = C.c_int
        _LIB.ygz_vo_run_handoff.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                            C.c_double, C.c_double, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.ygz_vo_run_handoff_ex.restype = C.c_int
        _LIB.ygz_vo_run_handoff_ex.argtypes = (_LIB.ygz_vo_run_handoff.argtypes[:15] + [C.c_void_p] + _LIB.ygz_vo_run_handoff.argtypes[15:]
                                               + [C.c_int])
        _LIB.ygz_vo_run_stages.restype = C.c_int
        _LIB.ygz_vo_run_stages.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                           C.c_double, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.ygz_vo_create.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.ygz_vo_push.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
        _LIB.ygz_vo_restart.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _LIB.ygz_vo_set_camera.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _LIB.ygz_vo_get_camera.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _LIB.ygz_vo_set_lens.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _LIB.ygz_vo_get_lens.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.ygz_vo_set_frame_format.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        _LIB.ygz_vo_get_frame_format.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.ygz_vo_step.argtypes = [C.c_void_p]
        _LIB.ygz_vo_flush.argtypes = [C.c_void_p]
        _LIB.ygz_vo_poll.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        _LIB.ygz_vo_set_observations.argtypes = [C.c_void_p, C.c_int]
        _LIB.ygz_vo_poll_observations.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        _LIB.ygz_vo_set_information.argtypes = [C.c_void_p, C.c_int]
        _LIB.ygz_vo_poll_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        _LIB.ygz_vo_set_map_updates.argtypes = [C.c_void_p, C.c_int]
        _LIB.ygz_vo_poll_map_updates.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        _LIB.ygz_vo_stream_stats.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _LIB.ygz_vo_export_map.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _LIB.ygz_vo_stream_record_bound.argtypes = [C.c_void_p, C.c_void_p]
        _LIB.ygz_vo_save_stream.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]
        _LIB.ygz_vo_load_stream.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]
        _LIB.ygz_vo_destroy.argtypes = [C.c_void_p]
        _LIB.ygz_vo_destroy.restype = None
    return _LIB


def stack_pinned(frames):
    """[stream][frame][H][W] uint8 in page-locked memory (where a camera / decoder would deliver frames): equally spaced,
    so the driver uploads a lock-step frame with one strided copy at the full PCIe rate."""
    from .capi import pinned_empty
    S, n = len(frames), len(frames[0])
    stacked = pinned_empty((S, n) + tuple(np.shape(frames[0])[1:]), np.uint8)
    for s_, f in enumerate(frames):
        stacked[s_] = f
    return stacked


_REF_MODES = {"keyframe": 0, "previous": 1}   # YGZB_TRACK_REF_KEYFRAME / _PREVIOUS
# names of the first 12 of a stream's 16 counters (ygz_vo_run's stats, ygz_vo_stream_stats); counter 12 counts restarts
_STAT_KEYS = ("lost", "keyframes", "ba", "candidates", "projected", "inliers", "ba_obs", "ba_pts", "ba_kfs", "ba_trials", "ba_iters", "ba_flops")


def run(ctx, frames, depths, kf_min_frames=10, kf_min_rot=0.1, kf_min_trans=0.1, warm=0, threads=1, device_frames=None,
        return_device_ms=False, details=False, window=1, engine="resident", handoff=None, return_maps=False, ref_mode="keyframe"):
    """frames: list of (n_frames, 480, 640) uint8 arrays or one stacked (S, n, 480, 640) array (ideally from stack_pinned);
    depths[s]: (480, 640) float64.  device_frames = (device pointer, S, n): the same stacked layout already resident in
    HBM (the "value" leg of bench.py) -- the driver then copies device-to-device.  The context must use the 3-level pyramid.
    threads > 1 splits the streams over that many host threads, each with its own context (CUDA stream) on the device.
    engine = "resident": the device-resident engine (ygzb_tracker_*; `window` = frames of one stream in flight per round);
    engine = "stages": the per-stage C-ABI path (one blocking call per stage and lock-step frame).
    handoff = frame h (resident engine only): at h every stream's local map (and, with ref_mode="previous", its reference)
    is exported, the tracker torn down and the streams carried over to a fresh tracker on a new context in reverse order
    (ygz_vo_run_handoff_ex); the results equal a run with warm = h.  return_maps (with handoff): also return the maps
    exported at h, one capi.MapBuffers per stream, and with ref_mode="previous" the references, one capi.ReferenceBuffers
    per stream (n = 0 for a stream that had no key-frame yet).
    ref_mode (resident engine): "keyframe" aligns every frame against the newest key-frame; "previous" against the previous
    frame, the reference's rule (ygz_vo_run_ex, YGZB_TRACK_REF_PREVIOUS).
    Returns (trajectory (S, n_frames, 3, 4), stats list of dicts, seconds of frames [warm, n_frames)[, device ms][, maps]
    [, references])."""
    if ref_mode not in _REF_MODES:
        raise ValueError(f"ref_mode must be 'keyframe' or 'previous', not {ref_mode!r}")
    if ref_mode != "keyframe" and engine != "resident":
        raise ValueError("the previous-frame reference is only offered by the resident engine")
    if device_frames is not None:
        base, S, n = device_frames
        ptrs = [base + s * n * 480 * 640 for s in range(S)]
    else:
        stacked = frames if isinstance(frames, np.ndarray) and frames.ndim == 4 else stack_pinned(frames)
        S, n = stacked.shape[:2]
        ptrs = [stacked[s].ctypes.data for s in range(S)]
    deps = [np.ascontiguousarray(d, np.float64) for d in depths]
    ip = (C.c_void_p * S)(*ptrs)
    dp = (C.c_void_p * S)(*[a.ctypes.data for a in deps])
    traj = np.zeros((S, n, 12), np.float64)
    stats = np.zeros((S, 16), np.int64)
    totals = np.zeros(8, np.int64)
    sec = C.c_double(0.0)
    dev_ms = C.c_double(0.0)
    if engine == "stages":
        rc = _lib().ygz_vo_run_stages(ctx.h, ctx.device_index, C.byref(ctx.params), threads, S, n, C.cast(ip, C.c_void_p),
                                      C.cast(dp, C.c_void_p), kf_min_frames, kf_min_rot, kf_min_trans, warm, traj.ctypes.data,
                                      stats.ctypes.data, C.byref(sec), C.byref(dev_ms), totals.ctypes.data)
    elif handoff is not None:
        from .capi import TRACK_RING, MapBuffers, MapRecord, ReferenceBuffers, ReferenceRecord
        recs = (MapRecord * S)() if return_maps else None
        maps = [MapBuffers(TRACK_RING, 640, 480, ctx.n_cells, rec=recs[s_]) for s_ in range(S)] if return_maps else None
        with_refs = return_maps and ref_mode == "previous"
        ref_recs = (ReferenceRecord * S)() if with_refs else None
        refs = [ReferenceBuffers(640, 480, ctx.n_cells, rec=ref_recs[s_]) for s_ in range(S)] if with_refs else None
        rc = _lib().ygz_vo_run_handoff_ex(ctx.h, ctx.device_index, C.byref(ctx.params), threads, S, n, C.cast(ip, C.c_void_p),
                                          C.cast(dp, C.c_void_p), kf_min_frames, kf_min_rot, kf_min_trans, warm, int(window), int(handoff),
                                          C.cast(recs, C.c_void_p) if return_maps else None,
                                          C.cast(ref_recs, C.c_void_p) if with_refs else None, traj.ctypes.data, stats.ctypes.data,
                                          C.byref(sec), C.byref(dev_ms), totals.ctypes.data, _REF_MODES[ref_mode])
    else:
        rc = _lib().ygz_vo_run_ex(ctx.h, ctx.device_index, C.byref(ctx.params), threads, S, n, C.cast(ip, C.c_void_p), C.cast(dp, C.c_void_p),
                                  kf_min_frames, kf_min_rot, kf_min_trans, warm, int(window), traj.ctypes.data, stats.ctypes.data,
                                  C.byref(sec), C.byref(dev_ms), totals.ctypes.data, _REF_MODES[ref_mode])
    ctx.check(rc, "ygz_vo_run")
    if handoff is not None and return_maps:
        return _result(traj, stats, totals, sec, dev_ms, S, n, details, return_device_ms) + (maps,) + ((refs,) if refs else ())
    return _result(traj, stats, totals, sec, dev_ms, S, n, details, return_device_ms)


def _result(traj, stats, totals, sec, dev_ms, S, n, details, return_device_ms):
    out = (traj.reshape(S, n, 3, 4), [dict(zip(_STAT_KEYS, map(int, row[:12]))) for row in stats], sec.value)
    if details:   # timed region only: device ms (CUDA events), kernel launches, bytes through the C ABI
        return out + (dict(device_ms=dev_ms.value, gpu_launches=int(totals[0]), h2d_image_bytes=int(totals[1]),
                           h2d_other_bytes=int(totals[2]), d2h_bytes=int(totals[3])),)
    return out + (dev_ms.value,) if return_device_ms else out


class VoConfig(C.Structure):
    _fields_ = [("n_streams", C.c_int), ("window", C.c_int), ("ref_mode", C.c_int), ("kf_min_frames", C.c_int), ("kf_min_rot", C.c_double),
                ("kf_min_trans", C.c_double), ("min_inliers", C.c_int), ("K", C.c_double * 4)]


STATUS = ("tracked", "keyframe", "lost")   # YGZ_VO_TRACKED / _KEYFRAME / _LOST
RESULT_DTYPE = np.dtype([("stream", np.int32), ("frame", np.int32), ("tag", np.int64), ("status", np.int32), ("n_inliers", np.int32),
                         ("T_cw", np.float64, (12,))])   # ygz_vo_result
OBS_DTYPE = np.dtype([("id", np.int64), ("px", np.float64, (2,)), ("pw", np.float64, (3,))])   # ygzb_observation
MAP_UPDATE_DTYPE = np.dtype([("stream", np.int32), ("frame", np.int32), ("sequence", np.int64), ("n_local", np.int32),
                             ("retired_frame", np.int32), ("local_frame", np.int32, (4,)), ("n_moved", np.int32), ("n_new", np.int32),
                             ("T_cw", np.float64, (4, 12))])   # ygz_vo_map_update
_ERR_CAPACITY = -4   # YGZB_ERR_CAPACITY


# the int64 counters of a stream record's host state, in order (include/ygz_vo.h)
_COUNTERS = ("n_keyframes", "n_ba", "n_candidates", "n_projected", "n_inliers", "ba_obs", "ba_pts", "ba_kfs", "ba_trials", "ba_iters",
             "n_restarts")


_LENS_VERSION = 2   # YGZ_VO_STREAM_RECORD_VERSION_LENS: a 72-byte lens block (K[4], dist[5]) follows the header
# YGZ_VO_STREAM_RECORD_VERSION_FORMAT: a 16-byte format block (width, height, channels, has_lens) follows the header, then
# the lens block if has_lens
_FORMAT_VERSION = 3


def _record_head(rec):
    """Bytes before a stream record's host state: the 68-byte header and the format and lens blocks its version has."""
    version = int(rec[4:8].view("<u4")[0])
    if version == _FORMAT_VERSION:
        return 68 + 16 + (72 if int(rec[80:84].view("<i4")[0]) else 0)
    return 68 + (72 if version == _LENS_VERSION else 0)


def stream_record_next_frame(rec):
    """next_frame of a stream record (uint8 array) from its fixed offset: the 68-byte header, the format and lens blocks of
    its version, n_kf, n_kf key-frames of 116 bytes, the two poses, the four flags and frames_since_kf come before it."""
    head = _record_head(rec)
    n_kf = int(rec[head:head + 4].view("<i4")[0])
    off = head + 4 + 116 * n_kf + 2 * 96 + 4 + 4
    return int(rec[off:off + 4].view("<i4")[0])


def parse_stream_record(data):
    """The fields of a stream record (ygz_vo_save_stream, layout in include/ygz_vo.h) by name: (byte offset, value), with
    per-key-frame fields named like "kf[1].entry" (host state) and "map[1].n_features" (map).  Values are numpy scalars
    and arrays read from `data`; raises ValueError if the record is shorter than its counts say."""
    buf = memoryview(bytes(data))
    out, pos = {}, 0

    def take(name, dtype, count=1):
        nonlocal pos
        dt = np.dtype(dtype).newbyteorder("<")
        size = dt.itemsize * int(count)
        if count < 0 or pos + size > len(buf):
            raise ValueError(f"stream record ends inside {name}")
        v = np.frombuffer(buf, dt, int(count), pos)
        out[name] = (pos, v[0] if count == 1 else v)
        pos += size
        return out[name][1]

    take("magic", "u1", 4)
    version = take("version", "u4")
    take("size", "u8")
    W, H = take("width", "i4"), take("height", "i4")
    take("cells", "i4"); take("n_levels", "i4"); take("K", "f8", 4)
    mode = take("ref_mode", "i4")
    has_lens = version == _LENS_VERSION
    if version == _FORMAT_VERSION:
        take("format.width", "i4"); take("format.height", "i4"); take("format.channels", "i4")
        has_lens = bool(take("format.has_lens", "i4"))
    if has_lens:
        take("lens.K", "f8", 4); take("lens.dist", "f8", 5)
    n_kf = take("n_kf", "i4")
    for k in range(n_kf):
        take(f"kf[{k}].entry", "i4"); take(f"kf[{k}].n", "i4"); take(f"kf[{k}].frame_id", "i4"); take(f"kf[{k}].mp0", "i8")
        take(f"kf[{k}].T_cw", "f8", 12)
    take("T_cw", "f8", 12); take("start", "f8", 12)
    take("restart_pending", "u1"); take("has_pose", "u1"); take("lost", "u1")
    has_depth = take("has_depth", "u1")
    take("frames_since_kf", "i4"); take("next_frame", "i4"); take("next_mp", "i8")
    for c in _COUNTERS:
        take(c, "i8")
    take("ba_flops", "f8")
    nk = take("n_keyframes", "i4")
    F = O = 0
    for k in range(nk):
        take(f"map[{k}].entry", "i4")
        F += int(take(f"map[{k}].n_features", "i4"))
        O += int(take(f"map[{k}].n_obs", "i4"))
        take(f"map[{k}].mp0", "i8"); take(f"map[{k}].T_cw", "f8", 12); take(f"map[{k}].image", "u1", W * H)
    take("px", "f8", 2 * F); take("level", "u1", F); take("depth", "f8", F); take("pw", "f8", 3 * F)
    take("obs_id", "i8", O); take("obs_px", "f8", 2 * O)
    if mode == _REF_MODES["previous"] and n_kf > 0:
        n = take("ref.n", "i4")
        take("ref.T_cw", "f8", 12); take("ref.px", "f8", 2 * n); take("ref.depth", "f8", n); take("ref.image", "u1", W * H)
    if has_depth:
        take("depth_map", "f8", W * H)
    out["end"] = (pos, None)
    return out


class Engine:
    """The device-resident engine fed frame by frame (include/ygz_vo.h): push frames per stream as they arrive, step or
    flush, poll the final results.  The image size is the context's; K (fx, fy, cx, cy in double) defaults to the
    context's camera at the shortest decimal that rounds to it (520.9 for the float 520.9f), which is the TUM camera the
    batch functions (run) use.  The pushed arrays are kept alive here until their results have been polled.
    observations=True: every result carries the map points its pose rests on (ygz_vo_set_observations), and poll
    returns them too.  information=True: every result carries how well its pose is determined (ygz_vo_set_information):
    poll also returns an [n, 2, 6, 6] array, the sparse alignment's Fisher information and pose-only's information
    matrix of each result as full symmetric matrices.  map_updates=True: every key-frame insertion queues what it changed
    in the local map (ygz_vo_set_map_updates), which poll_map_updates returns.  cameras: None, or one (fx, fy, cx, cy)
    per stream (None: K), set before any push (ygz_vo_set_camera).  lenses: None, or one (K, dist) or None per stream:
    the stream's raw frames are those of camera K = (fx, fy, cx, cy) with distortion dist = (k1, k2, p1, p2, k3), and the
    engine undistorts them on the device to the stream's camera (ygz_vo_set_lens).  frame_formats: None, or one (width,
    height, channels) or None per stream: the frames the stream pushes, grey (channels 1) or BGR (3), of the context's size
    or, with a lens whose K is that raw camera's, of any size (ygz_vo_set_frame_format)."""

    def __init__(self, ctx, n_streams, window=8, ref_mode="keyframe", kf_min_frames=10, kf_min_rot=0.1, kf_min_trans=0.1,
                 min_inliers=30, K=None, observations=False, information=False, map_updates=False, cameras=None, lenses=None,
                 frame_formats=None):
        if ref_mode not in _REF_MODES:
            raise ValueError(f"ref_mode must be 'keyframe' or 'previous', not {ref_mode!r}")
        p = ctx.params
        if K is None:
            K = [float(str(np.float32(v))) for v in (p.fx, p.fy, p.cx, p.cy)]
        self.ctx, self.n_streams, self.shape = ctx, int(n_streams), (p.image_height, p.image_width)
        self.cfg = VoConfig(int(n_streams), int(window), _REF_MODES[ref_mode], int(kf_min_frames), float(kf_min_rot), float(kf_min_trans),
                            int(min_inliers), (C.c_double * 4)(*map(float, K)))
        self.lib = _lib()
        self.h = C.c_void_p()
        ctx.check(self.lib.ygz_vo_create(ctx.h, C.byref(self.cfg), C.byref(self.h)), "ygz_vo_create")
        self._pushed = [0] * self.n_streams
        self._alive = {}   # (stream, frame) -> the arrays its result still needs
        self._rows = {}   # row dtype -> the row buffer of one poll call, grown on demand
        self.observations = False
        if observations:
            self.set_observations(True)
        self.information = False
        if information:
            self.set_information(True)
        self.map_updates = False
        if map_updates:
            self.set_map_updates(True)
        for name, noun, per_stream, apply in (("cameras", "cameras", cameras, self.set_camera),
                                              ("lenses", "lenses", lenses, lambda s, lens: self.set_lens(s, *lens)),
                                              ("frame_formats", "formats", frame_formats, lambda s, fmt: self.set_frame_format(s, *fmt))):
            if per_stream is None:
                continue
            if len(per_stream) != self.n_streams:
                raise ValueError(f"{name}: {len(per_stream)} {noun} for {self.n_streams} streams")
            for s, v in enumerate(per_stream):
                if v is not None:
                    apply(s, v)

    def set_camera(self, stream, K):
        """K = (fx, fy, cx, cy) of `stream`'s next sequence (ygz_vo_set_camera): only before its first push or while a
        restart is pending; frames pushed before the restart keep the old camera."""
        K = np.ascontiguousarray(K, np.float64).reshape(4)
        self.ctx.check(self.lib.ygz_vo_set_camera(self.h, int(stream), K.ctypes.data), "ygz_vo_set_camera")

    def camera(self, stream):
        """The camera (fx, fy, cx, cy) set_camera last gave `stream` (the engine's K until then)."""
        K = np.zeros(4, np.float64)
        self.ctx.check(self.lib.ygz_vo_get_camera(self.h, int(stream), K.ctypes.data), "ygz_vo_get_camera")
        return K

    def set_lens(self, stream, K=None, dist=None):
        """The lens of `stream`'s next sequence (ygz_vo_set_lens): raw camera K = (fx, fy, cx, cy) and dist = (k1, k2, p1,
        p2[, k3]); no arguments: none.  At the times set_camera is accepted; frames pushed before the restart keep the old
        lens."""
        if K is None and dist is None:
            self.ctx.check(self.lib.ygz_vo_set_lens(self.h, int(stream), None, None), "ygz_vo_set_lens")
            return
        K = np.ascontiguousarray(K, np.float64).reshape(4)
        d = np.zeros(5)
        d[:len(dist)] = dist
        self.ctx.check(self.lib.ygz_vo_set_lens(self.h, int(stream), K.ctypes.data, d.ctypes.data), "ygz_vo_set_lens")

    def lens(self, stream):
        """The lens set_lens last gave `stream`: (K, dist) arrays, or None for none."""
        has, K, d = C.c_int(0), np.zeros(4, np.float64), np.zeros(5, np.float64)
        self.ctx.check(self.lib.ygz_vo_get_lens(self.h, int(stream), C.byref(has), K.ctypes.data, d.ctypes.data), "ygz_vo_get_lens")
        return (K, d) if has.value else None

    def set_frame_format(self, stream, width, height, channels=1):
        """The frames of `stream`'s next sequence (ygz_vo_set_frame_format): width x height, grey (channels 1) or BGR (3).
        A size other than the context's needs a lens (set_lens) by the sequence's first push.  At the times set_camera is
        accepted; frames pushed before the restart keep the old format."""
        self.ctx.check(self.lib.ygz_vo_set_frame_format(self.h, int(stream), int(width), int(height), int(channels)),
                       "ygz_vo_set_frame_format")

    def frame_format(self, stream):
        """The format (width, height, channels) set_frame_format last gave `stream` (the context's size, grey, until then)."""
        w, h, c = C.c_int(0), C.c_int(0), C.c_int(0)
        self.ctx.check(self.lib.ygz_vo_get_frame_format(self.h, int(stream), C.byref(w), C.byref(h), C.byref(c)),
                       "ygz_vo_get_frame_format")
        return w.value, h.value, c.value

    def set_observations(self, on):
        """Switch the observation rows of the results on or off (ygz_vo_set_observations): only while the engine is
        idle -- nothing queued or pending, every result polled."""
        self.ctx.check(self.lib.ygz_vo_set_observations(self.h, int(bool(on))), "ygz_vo_set_observations")
        self.observations = bool(on)

    def set_information(self, on):
        """Switch the information records of the results on or off (ygz_vo_set_information): only while the engine is
        idle, as set_observations."""
        self.ctx.check(self.lib.ygz_vo_set_information(self.h, int(bool(on))), "ygz_vo_set_information")
        self.information = bool(on)

    def set_map_updates(self, on):
        """Switch the map updates of key-frame insertions on or off (ygz_vo_set_map_updates): only while the engine is
        idle, as set_observations, with no update waiting either."""
        self.ctx.check(self.lib.ygz_vo_set_map_updates(self.h, int(bool(on))), "ygz_vo_set_map_updates")
        self.map_updates = bool(on)

    def _drain(self, call, name, capacity, dtypes, row_dtype=None, row_count=None):
        """Polls until nothing is left: call(records, n, rows, row_capacity, n_rows) gets one array of `capacity` records per
        dtype in `dtypes` and the row buffer (None and 0 without a row dtype), and returns the C status; YGZB_ERR_CAPACITY
        (the next record's rows do not fit) grows the row buffer and asks again.  Returns the records, one array per dtype,
        and with a row dtype the rows, one array per record of row_count(records[0]) rows."""
        recs, rows = [[] for _ in dtypes], []
        while True:
            bufs = [np.zeros(capacity, dt) for dt in dtypes]
            n, n_rows = C.c_int(0), C.c_size_t(0)
            if row_dtype is None:
                rc = call(bufs, C.byref(n), None, 0, C.byref(n_rows))
            else:
                buf = self._rows.get(row_dtype)
                if buf is None:
                    buf = self._rows[row_dtype] = np.zeros(4 * 4096, row_dtype)
                rc = call(bufs, C.byref(n), buf.ctypes.data, len(buf), C.byref(n_rows))
                if rc == _ERR_CAPACITY:
                    self._rows[row_dtype] = np.zeros(max(2 * len(buf), n_rows.value), row_dtype)
                    continue
            self.ctx.check(rc, name)
            if n.value == 0:
                break
            for r, b in zip(recs, bufs):
                r.append(b[:n.value])
            if row_dtype is None and n.value < capacity:   # (without rows, a short answer has drained the queue)
                break
            if row_dtype is not None:
                ends = np.cumsum(row_count(bufs[0][:n.value]))
                assert ends[-1] == n_rows.value
                rows.extend(np.split(buf[:n_rows.value].copy(), ends[:-1]))
        return [np.concatenate(r) if r else np.zeros(0, dt) for r, dt in zip(recs, dtypes)], rows

    def poll_map_updates(self, capacity=256):
        """Map updates since the last call, oldest first: (updates, rows) -- a MAP_UPDATE_DTYPE array and, per update, a
        MAP_POINT_DTYPE array of its n_moved rows (the local BA's points) followed by its n_new rows (the new key-frame's
        points).  Independent of poll: results and updates have queues of their own."""
        lib, h = self.lib, self.h
        (upd,), rows = self._drain(lambda out, n, *r: lib.ygz_vo_poll_map_updates(h, out[0].ctypes.data, capacity, n, *r),
                                   "ygz_vo_poll_map_updates", capacity, (MAP_UPDATE_DTYPE,), MAP_POINT_DTYPE,
                                   lambda u: u["n_moved"].astype(np.int64) + u["n_new"])
        return upd, rows

    def push(self, stream, image, depth=None, tag=None):
        """Queue `image` of `stream` in the stream's frame format (frame_format: (h, w) grey or (h, w, 3) BGR uint8; by
        default (H, W) grey) with its depth map (H, W) float64 at the context's size, or None to keep the stream's current
        map.  Returns the frame's index in its stream; tag (default: that index) comes back with its result."""
        if not 0 <= stream < self.n_streams:
            raise ValueError(f"stream {stream} out of range [0, {self.n_streams})")
        img = np.ascontiguousarray(image, np.uint8)
        dep = None if depth is None else np.ascontiguousarray(depth, np.float64)
        w, h, c = self.frame_format(stream)
        shape = (h, w) if c == 1 else (h, w, c)
        if img.shape != shape or (dep is not None and dep.shape != self.shape):
            raise ValueError(f"image must be {shape} and depth {self.shape}, not {img.shape} and {None if dep is None else dep.shape}")
        frame = self._pushed[stream]
        tag = frame if tag is None else int(tag)
        self.ctx.check(self.lib.ygz_vo_push(self.h, int(stream), img.ctypes.data, None if dep is None else dep.ctypes.data, tag),
                       "ygz_vo_push")
        self._alive[(stream, frame)] = (img, dep)
        self._pushed[stream] += 1
        return frame

    def restart(self, stream, T_cw=None):
        """Start a new sequence of `stream` with the next push, whose frame becomes the first key-frame at T_cw (3, 4)
        (None: identity) and must bring a depth map; frames pushed before keep their results (ygz_vo_restart).  Before
        the stream's first push it only sets the pose of its first key-frame."""
        if not 0 <= stream < self.n_streams:
            raise ValueError(f"stream {stream} out of range [0, {self.n_streams})")
        T = None if T_cw is None else np.ascontiguousarray(T_cw, np.float64).reshape(12)
        self.ctx.check(self.lib.ygz_vo_restart(self.h, int(stream), None if T is None else T.ctypes.data), "ygz_vo_restart")

    def step(self):
        self.ctx.check(self.lib.ygz_vo_step(self.h), "ygz_vo_step")

    def flush(self):
        self.ctx.check(self.lib.ygz_vo_flush(self.h), "ygz_vo_flush")

    def poll(self, capacity=4096):
        """Final results since the last poll, oldest first: a RESULT_DTYPE array (status indexes STATUS).  With
        observations on, (results, rows): rows[k] is an OBS_DTYPE array of result k's n_inliers observations.  With
        information on, (results, info) or (results, rows, info): info[k] = [alignment Fisher, pose information] of
        result k, [n, 2, 6, 6] (zeros for a sequence's first key-frame and for LOST results)."""
        lib, h, obs = self.lib, self.h, self.observations
        row_dtype, n_inliers = (OBS_DTYPE if obs else None), itemgetter("n_inliers")
        if self.information:
            (res, info), rows = self._drain(
                lambda out, n, *r: lib.ygz_vo_poll_ex(h, out[0].ctypes.data, capacity, n, out[1].ctypes.data, *r), "ygz_vo_poll_ex",
                capacity, (RESULT_DTYPE, INFO_DTYPE), row_dtype, n_inliers)
            full = np.stack([unpack_sym6(info["align_fisher"]), unpack_sym6(info["pose_info"])], axis=1)
            return (self._release(res), rows, full) if obs else (self._release(res), full)
        if obs:
            (res,), rows = self._drain(lambda out, n, *r: lib.ygz_vo_poll_observations(h, out[0].ctypes.data, capacity, n, *r),
                                       "ygz_vo_poll_observations", capacity, (RESULT_DTYPE,), row_dtype, n_inliers)
            return self._release(res), rows
        (res,), _ = self._drain(lambda out, n, *r: lib.ygz_vo_poll(h, out[0].ctypes.data, capacity, n), "ygz_vo_poll", capacity,
                                (RESULT_DTYPE,))
        return self._release(res)

    def _release(self, res):
        for s_, f in zip(res["stream"].tolist(), res["frame"].tolist()):
            self._alive.pop((s_, f), None)
        return res

    def _stat_row(self, stream):
        row = np.zeros(16, np.int64)
        self.ctx.check(self.lib.ygz_vo_stream_stats(self.h, int(stream), row.ctypes.data), "ygz_vo_stream_stats")
        return row

    def stats(self, stream):
        """The counters of ygz_vo_run for one stream, as run's dicts."""
        return dict(zip(_STAT_KEYS, map(int, self._stat_row(stream)[:12])))

    def restarts(self, stream):
        """How many restarts (ygz_vo_restart) have started a new sequence of `stream`: counter 12 of ygz_vo_stream_stats."""
        return int(self._stat_row(stream)[12])

    def export_map(self, stream):
        """The stream's local map (every key-frame still in its ring, oldest first) as a capi.MapBuffers; call after flush."""
        from .capi import TRACK_RING, MapBuffers
        m = MapBuffers(TRACK_RING, self.shape[1], self.shape[0], self.ctx.n_cells)
        self.ctx.check(self.lib.ygz_vo_export_map(self.h, int(stream), C.byref(m.rec)), "ygz_vo_export_map")
        self.ctx.synchronize()
        return m

    def stream_record_bound(self):
        """The most bytes a stream record of this engine can take (ygz_vo_stream_record_bound)."""
        n = C.c_size_t(0)
        self.ctx.check(self.lib.ygz_vo_stream_record_bound(self.h, C.byref(n)), "ygz_vo_stream_record_bound")
        return n.value

    def save_stream(self, stream):
        """The whole state of `stream` as a stream record (bytes, the layout of include/ygz_vo.h); flush first.  The stream
        is unchanged and may go on tracking."""
        bound = self.stream_record_bound()   # (grows by the lens block once a stream has a lens)
        if getattr(self, "_record_buf", None) is None or self._record_buf.size < bound:
            self._record_buf = np.empty(bound, np.uint8)
        buf, n = self._record_buf, C.c_size_t(0)
        self.ctx.check(self.lib.ygz_vo_save_stream(self.h, int(stream), buf.ctypes.data, buf.size, C.byref(n)), "ygz_vo_save_stream")
        return buf[:n.value].tobytes()

    def load_stream(self, stream, data):
        """`stream` continues the stream saved in `data` (save_stream of any engine with the same geometry, camera and
        reference mode): its next push gets the saved stream's next frame index."""
        rec = np.frombuffer(data, np.uint8)
        self.ctx.check(self.lib.ygz_vo_load_stream(self.h, int(stream), rec.ctypes.data, rec.size), "ygz_vo_load_stream")
        self._pushed[stream] = stream_record_next_frame(rec)

    def close(self):
        if self.h:
            self.lib.ygz_vo_destroy(self.h)
            self.h = C.c_void_p()
        self._alive.clear()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
