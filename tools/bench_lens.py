"""Cost of per-stream lenses in the streaming engine (ygz_vo_set_lens) at bench.py's C5 shape: 8 streams on one engine,
window 8, bench.py's key-frame policy, 8 frames per stream pushed before each ygz_vo_step.  Two runs, alternated
`--repeats` times:
- on:  raw frames of TUM fr2's lens (synth.LENS_TUM_FR2, raw camera = the engine's camera): synth.shift_stream's frames
       distorted on the host once, before any run; every stream has the lens, so the engine remaps every upload;
- off: the same raw frames undistorted before the run (by a frame pool's undistorting upload, which
       tests/test_gpu_undistort.py pins to cv2) and pushed without a lens -- what a caller without lenses in the engine
       does, minus the host's own undistortion.  Both legs track the same frames and must give the same trajectories.
Host clock from the first push to the end of the flush gives tracked frames/s; a separate torch.profiler run of the lens
leg gives the device time of remap_gray_kernel per tracked frame (speculative frames are uploaded again, so a frame may be
remapped more than once).  Prints one JSON line of medians with the GPU's name and power limit, read in the same run."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import numpy as np  # noqa: E402

from ygz_slam_b200 import Context, synth, vo_native  # noqa: E402

POLICY = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)   # bench.py's KF_POLICY
K = (synth.FX, synth.FY, synth.CX, synth.CY)


def gpu_name_and_power():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def distort(frames):
    """The raw frames of a lens with coefficients LENS_TUM_FR2 whose undistorted view is `frames`: every raw pixel takes
    the bilinear sample of the undistorted frame at its ray (synth.undistort_rays)."""
    u, v = np.meshgrid(np.arange(synth.W, dtype=np.float64), np.arange(synth.H, dtype=np.float64))
    x, y = synth.undistort_rays(u, v, synth.LENS_TUM_FR2)
    px, py = x * K[0] + K[2], y * K[1] + K[3]
    inside = (px >= 0) & (px <= synth.W - 1) & (py >= 0) & (py <= synth.H - 1)
    x0 = np.clip(np.floor(px), 0, synth.W - 2).astype(np.int64)
    y0 = np.clip(np.floor(py), 0, synth.H - 2).astype(np.int64)
    ax, ay = (px - x0).astype(np.float32), (py - y0).astype(np.float32)
    i00 = y0 * synth.W + x0
    out = np.empty_like(frames)
    for k, f in enumerate(frames):
        g = f.reshape(-1).astype(np.float32)
        val = (1 - ay) * ((1 - ax) * g[i00] + ax * g[i00 + 1]) + ay * ((1 - ax) * g[i00 + synth.W] + ax * g[i00 + synth.W + 1])
        out[k] = np.where(inside, np.clip(np.rint(val), 0, 255), 0).astype(np.uint8)
    return out


def undistort(ctx, frames):
    """The frames undistorted by a frame pool with the lens's maps (level 0 of each slot)."""
    from ygz_slam_b200 import capi
    fr = ctx.frames(len(frames))
    fr.set_undistort(*capi.undistort_map(synth.W, synth.H, K, synth.LENS_TUM_FR2))
    fr.upload(frames)
    out = np.stack([fr.download_level(k, 0) for k in range(len(frames))])
    fr.close()
    return out


def run(ctx, data, lens, window, burst=8):
    """One engine per run, created outside the timed region.  Returns (seconds, lost results, trajectory)."""
    S, n = len(data), len(data[0][0])
    eng = vo_native.Engine(ctx, S, window=window, lenses=[lens] * S, **POLICY)
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


def remap_us(fn):
    """Device time of remap_gray_kernel over one run under torch.profiler, in microseconds."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return float(sum(e.self_device_time_total for e in prof.key_averages()
                     if e.device_type.name == "CUDA" and "remap_gray_kernel" in e.key))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--frames", type=int, default=240)
    ap.add_argument("--window", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    ctx = Context(0)
    S, n = a.streams, a.frames
    on = [(distort(f), d) for f, d, _ in (synth.shift_stream(s, n) for s in range(S))]
    off = [(undistort(ctx, f), d) for f, d in on]
    legs = {"off": lambda: run(ctx, off, None, a.window), "on": lambda: run(ctx, on, (K, synth.LENS_TUM_FR2), a.window)}
    refs = {k: fn() for k, fn in legs.items()}   # warm-up, and the trajectories every run must reproduce
    assert np.array_equal(refs["off"][2], refs["on"][2])
    fps = {k: [] for k in legs}
    for _ in range(a.repeats):
        for k, fn in legs.items():
            sec, _, traj = fn()
            assert np.array_equal(traj, refs[k][2]), k
            fps[k].append(S * n / sec)
    gpu = gpu_name_and_power()
    us = remap_us(legs["on"]) / (S * n)
    print(json.dumps(dict(metric="tracked frames/s", gpu=gpu, streams=S, frames=n, window=a.window, repeats=a.repeats,
                          median_fps={k: float(np.median(v)) for k, v in fps.items()}, lost={k: r[1] for k, r in refs.items()},
                          remap_us_per_tracked_frame=us, runs={k: [round(x, 1) for x in v] for k, v in fps.items()})))
    ctx.close()


if __name__ == "__main__":
    main()
