"""ctypes harness for the native tracking loop (host/vo_driver.cpp -> libygz_vo.so): the C++ twin of
vo.VisualOdometry with the GPU backend, used by bench.py for BASELINE config C5 and by the tests to compare both loops."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from . import build

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
    keys = ("lost", "keyframes", "ba", "candidates", "projected", "inliers", "ba_obs", "ba_pts", "ba_kfs", "ba_trials", "ba_iters", "ba_flops")
    out = (traj.reshape(S, n, 3, 4), [dict(zip(keys, map(int, row[:12]))) for row in stats], sec.value)
    if details:   # timed region only: device ms (CUDA events), kernel launches, bytes through the C ABI
        return out + (dict(device_ms=dev_ms.value, gpu_launches=int(totals[0]), h2d_image_bytes=int(totals[1]),
                           h2d_other_bytes=int(totals[2]), d2h_bytes=int(totals[3])),)
    return out + (dev_ms.value,) if return_device_ms else out
