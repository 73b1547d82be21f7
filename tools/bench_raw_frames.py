"""Cost of pushing raw frames of another size and colour to the streaming engine (ygz_vo_set_frame_format) at bench.py's
C5 shape: 8 streams on one engine, window 8, bench.py's key-frame policy, 8 frames per stream pushed before each
ygz_vo_step.  Two runs, alternated `--repeats` times:
- raw: 1280 x 720 BGR frames of an HD camera (K_raw = RAW_K, no distortion) pushed as they are; every stream has that
       format and lens, so the engine uploads 2.76 MB per frame and resamples it into the 640 x 480 pipeline on the device;
- pre: the same frames resampled to 640 x 480 grey before the run and pushed in the default format (0.31 MB per frame) --
       what a caller does without formats, minus the host's own resampling.  Both legs must give the same trajectories.
The raw frames are made from synth.shift_stream's frames: each raw pixel takes the bilinear sample of the 640 x 480 frame
at its ray, grey copied into three different channels.  The pre-resampled frames come from a tracker stream with the same
format and maps (tests/test_vo_raw_frames.py pins that upload to numpy and cv2).
Host clock from the first push to the end of the flush gives tracked frames/s; a separate torch.profiler run of the raw
leg gives the device time of remap_gray_kernel per tracked frame (speculative frames are uploaded again, so a frame may be
resampled more than once).  Prints one JSON line of medians with the GPU's name and power limit, read in the same run."""
import argparse
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

import numpy as np  # noqa: E402

from bench_lens import POLICY, gpu_name_and_power, remap_us  # noqa: E402
from ygz_slam_b200 import Context, capi, synth, vo_native  # noqa: E402

K = (synth.FX, synth.FY, synth.CX, synth.CY)
RW, RH = 1280, 720
RAW_K = (780.0, 780.0, 639.5, 359.5)
DIST = (0.0,) * 5


def raw_frames(frames):
    """HD BGR frames whose view through RAW_K, resampled with newK = K, is `frames` (where the view covers it)."""
    u, v = np.meshgrid(np.arange(RW, dtype=np.float64), np.arange(RH, dtype=np.float64))
    px = (u - RAW_K[2]) / RAW_K[0] * K[0] + K[2]
    py = (v - RAW_K[3]) / RAW_K[1] * K[1] + K[3]
    inside = (px >= 0) & (px <= synth.W - 1) & (py >= 0) & (py <= synth.H - 1)
    x0 = np.clip(np.floor(px), 0, synth.W - 2).astype(np.int64)
    y0 = np.clip(np.floor(py), 0, synth.H - 2).astype(np.int64)
    ax, ay = (px - x0).astype(np.float32), (py - y0).astype(np.float32)
    i00 = y0 * synth.W + x0
    out = np.empty((len(frames), RH, RW, 3), np.uint8)
    for k, f in enumerate(frames):
        g = f.reshape(-1).astype(np.float32)
        val = (1 - ay) * ((1 - ax) * g[i00] + ax * g[i00 + 1]) + ay * ((1 - ax) * g[i00 + synth.W] + ax * g[i00 + synth.W + 1])
        grey = np.where(inside, np.clip(np.rint(val), 0, 255), 0).astype(np.int32)
        out[k] = np.stack([grey, np.clip(grey * 3 // 4 + 40, 0, 255), 255 - grey // 2], -1)
    return out


def resample(ctx, frames, maps, chunk=64):
    """Level 0 of the frames as a tracker stream of their format and maps uploads them."""
    fr = ctx.frames(chunk)
    tr = capi.Tracker(fr, 1, 8, K)
    tr.set_source(0, RW, RH, 3)
    tr.set_undistort(0, *maps)
    out = np.empty((len(frames), synth.H, synth.W), np.uint8)
    for k0 in range(0, len(frames), chunk):
        part = frames[k0:k0 + chunk]
        tr.upload_stream(0, 0, part)
        for k in range(len(part)):
            out[k0 + k] = fr.download_level(k, 0)
    tr.close()
    fr.close()
    return out


def run(ctx, data, window, raw, burst=8):
    """One engine per run, created outside the timed region, every stream of the HD format and lens (raw) or the default
    format (pre).  Returns (seconds, lost results, trajectory)."""
    S, n = len(data), len(data[0][0])
    kw = dict(lenses=[(RAW_K, DIST)] * S, frame_formats=[(RW, RH, 3)] * S) if raw else {}
    eng = vo_native.Engine(ctx, S, window=window, **kw, **POLICY)
    ctx.synchronize()
    t0 = time.perf_counter()
    for k0 in range(0, n, burst):
        for s in range(S):
            for k in range(k0, min(n, k0 + burst)):
                eng.push(s, data[s][0][k], data[s][1] if k == 0 else None)
        eng.step()
    eng.flush()
    sec = time.perf_counter() - t0
    res = eng.poll()
    eng.close()
    assert len(res) == S * n
    traj = np.zeros((S, n, 12))
    traj[res["stream"], res["frame"]] = res["T_cw"]
    return sec, int((res["status"] == 2).sum()), traj


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--window", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    ctx = Context(0)
    S, n = a.streams, a.frames
    maps = capi.undistort_map(synth.W, synth.H, RAW_K, DIST, K)
    raw = [(raw_frames(f), d) for f, d, _ in (synth.shift_stream(s, n) for s in range(S))]
    pre = [(resample(ctx, f, maps), d) for f, d in raw]
    legs = {"pre": lambda: run(ctx, pre, a.window, False), "raw": lambda: run(ctx, raw, a.window, True)}
    refs = {k: fn() for k, fn in legs.items()}   # warm-up, and the trajectories every run must reproduce
    assert np.array_equal(refs["pre"][2], refs["raw"][2])
    fps = {k: [] for k in legs}
    for _ in range(a.repeats):
        for k, fn in legs.items():
            sec, _, traj = fn()
            assert np.array_equal(traj, refs[k][2]), k
            fps[k].append(S * n / sec)
    gpu = gpu_name_and_power()
    us = remap_us(legs["raw"]) / (S * n)
    print(json.dumps(dict(metric="tracked frames/s", gpu=gpu, streams=S, frames=n, window=a.window, repeats=a.repeats,
                          raw=f"{RW}x{RH}x3", median_fps={k: float(np.median(v)) for k, v in fps.items()},
                          lost={k: r[1] for k, r in refs.items()}, remap_us_per_tracked_frame=us,
                          runs={k: [round(x, 1) for x in v] for k, v in fps.items()})))
    ctx.close()


if __name__ == "__main__":
    main()
