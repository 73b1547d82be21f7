"""Throughput of the streaming API (include/ygz_vo.h) against the batch entry point on the same frames, in one process.

8 synthetic streams (shift_stream) at bench.py's key-frame policy.  Legs, alternated `--repeats` times:
- batch:          ygz_vo_run at window 8 on the stacked page-locked sequences (`seconds` of the run, warm = 0);
- stream:         ygz_vo_push of one frame per stream, each with its depth map, then ygz_vo_step and ygz_vo_poll, frame after
                  frame, then ygz_vo_flush: host clock from the first push to the end of the flush.  Every key-frame uploads
                  its frame's depth map (W*H doubles, page-locked) before its insertion;
- stream_nodepth: the same with a depth map on each stream's first frame only (NULL afterwards): the difference to `stream`
                  is the cost of the per-key-frame depth uploads;
- burst:          8 frames per stream pushed before each step (windows of up to 8 frames, as in the batch run), each from
                  its own page-locked buffer and uploaded by its own copy; against `batch`, which uploads a window with one
                  strided copy, this bounds what a staging ring for one strided copy per window could gain; burst_nodepth
                  is the same without the per-key-frame depth uploads.
Upload micro-benchmark (one frame pool, device-synchronised, median us per 8 frames): 8 single-frame ygzb_frames_upload
calls from separate page-locked frames (what the engine does with pushed frames), one strided call over 8 stacked frames,
and a staging ring's way: a host copy of the 8 separate frames into one page-locked buffer, then one strided call.
Every streaming leg must give the batch trajectory bit for bit.  Rates are tracked frames/s over all streams.  Prints one
JSON line of medians with the GPU's name and power limit, read in the same run."""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import numpy as np  # noqa: E402

from ygz_slam_b200 import Context, synth, vo_native  # noqa: E402
from ygz_slam_b200.capi import pinned_empty  # noqa: E402

POLICY = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)   # bench.py's KF_POLICY: a key-frame every >= 5 frames


def gpu_name_and_power():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def stream_run(ctx, images, depths, window, burst, depth_every_frame):
    """images[s][k]: frame pointers; one ygz_vo per run, created outside the timed region.  Returns (seconds, trajectory)."""
    lib = vo_native._lib()
    S, n = len(images), len(images[0])
    eng = vo_native.Engine(ctx, S, window=window, **POLICY)
    out = np.zeros(S * n, vo_native.RESULT_DTYPE)
    got = C.c_int(0)
    n_out = 0
    ctx.synchronize()
    t0 = time.perf_counter()
    for k0 in range(0, n, burst):
        for s in range(S):
            for k in range(k0, min(n, k0 + burst)):
                ctx.check(lib.ygz_vo_push(eng.h, s, images[s][k], depths[s] if depth_every_frame or k == 0 else None, k), "ygz_vo_push")
        ctx.check(lib.ygz_vo_step(eng.h), "ygz_vo_step")
        ctx.check(lib.ygz_vo_poll(eng.h, out[n_out:].ctypes.data, len(out) - n_out, C.byref(got)), "ygz_vo_poll")
        n_out += got.value
    ctx.check(lib.ygz_vo_flush(eng.h), "ygz_vo_flush")
    sec = time.perf_counter() - t0
    ctx.check(lib.ygz_vo_poll(eng.h, out[n_out:].ctypes.data, len(out) - n_out, C.byref(got)), "ygz_vo_poll")
    n_out += got.value
    eng.close()
    assert n_out == S * n
    traj = np.zeros((S, n, 12))
    traj[out["stream"], out["frame"]] = out["T_cw"]
    return sec, traj.reshape(S, n, 3, 4)


def upload_micro(ctx, stacked8, separate8, reps=200):
    lib = ctx.lib
    fr = ctx.frames(8)
    fb = stacked8[0].size
    staging = pinned_empty(stacked8.shape, np.uint8)

    def per_frame():
        for t, f in enumerate(separate8):
            ctx.check(lib.ygzb_frames_upload(fr.h, t, 1, C.c_void_p(f.ctypes.data), 1, C.c_size_t(fb)), "ygzb_frames_upload")

    def strided():
        ctx.check(lib.ygzb_frames_upload(fr.h, 0, 8, C.c_void_p(stacked8.ctypes.data), 1, C.c_size_t(fb)), "ygzb_frames_upload")

    def staged():
        for t, f in enumerate(separate8):
            staging[t] = f
        ctx.check(lib.ygzb_frames_upload(fr.h, 0, 8, C.c_void_p(staging.ctypes.data), 1, C.c_size_t(fb)), "ygzb_frames_upload")

    out = {}
    for name, fn in (("per_frame", per_frame), ("strided", strided), ("staging_ring", staged)):
        times = []
        for r in range(reps + 10):
            ctx.synchronize()
            t0 = time.perf_counter()
            fn()
            ctx.synchronize()
            if r >= 10:
                times.append((time.perf_counter() - t0) * 1e6)
        out[name] = float(np.median(times))
    fr.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--frames", type=int, default=240)
    ap.add_argument("--window", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=9)
    a = ap.parse_args()
    ctx = Context(0)
    S, n = a.streams, a.frames
    data = [synth.shift_stream(s, n) for s in range(S)]
    stacked = vo_native.stack_pinned([d[0] for d in data])
    depths = [d[1] for d in data]
    pinned_depths = []
    for d in depths:
        p = pinned_empty(d.shape, np.float64)
        p[...] = d
        pinned_depths.append(p)
    separate = [[pinned_empty(stacked.shape[2:], np.uint8) for _ in range(n)] for _ in range(S)]
    for s in range(S):
        for k in range(n):
            separate[s][k][...] = stacked[s, k]
    ptr_separate = [[separate[s][k].ctypes.data for k in range(n)] for s in range(S)]
    ptr_depth = [d.ctypes.data for d in pinned_depths]

    def batch():
        traj, _, sec = vo_native.run(ctx, stacked, depths, window=a.window, **POLICY)
        return sec, traj

    legs = {"batch": batch,
            "stream": lambda: stream_run(ctx, ptr_separate, ptr_depth, a.window, 1, True),
            "stream_nodepth": lambda: stream_run(ctx, ptr_separate, ptr_depth, a.window, 1, False),
            "burst": lambda: stream_run(ctx, ptr_separate, ptr_depth, a.window, 8, True),
            "burst_nodepth": lambda: stream_run(ctx, ptr_separate, ptr_depth, a.window, 8, False)}
    ref = batch()[1]   # warm-up, and the trajectory every leg must reproduce
    for fn in legs.values():
        fn()
    fps = {k: [] for k in legs}
    for _ in range(a.repeats):
        for name, fn in legs.items():
            sec, traj = fn()
            assert np.array_equal(traj, ref), name
            fps[name].append(S * n / sec)
    med = {k: float(np.median(v)) for k, v in fps.items()}
    uploads = upload_micro(ctx, stacked[0, :8], separate[0][:8])
    _, stats, _ = vo_native.run(ctx, stacked, depths, window=a.window, **POLICY)
    keyframes = sum(st["keyframes"] for st in stats)
    per_kf_us = (S * n / med["stream"] - S * n / med["stream_nodepth"]) / keyframes * 1e6
    print(json.dumps(dict(metric="tracked frames/s", gpu=gpu_name_and_power(), streams=S, frames=n, window=a.window, keyframes=keyframes,
                          median_fps=med, depth_upload_us_per_keyframe=per_kf_us, upload_us_per_8_frames=uploads,
                          runs={k: [round(x, 1) for x in v] for k, v in fps.items()})))
    ctx.close()


if __name__ == "__main__":
    main()
