"""Cost of per-stream cameras in the streaming engine (ygz_vo_set_camera) at bench.py's C5 shape: 8 streams on one engine,
window 8, bench.py's key-frame policy, 8 frames per stream pushed before each ygz_vo_step.  Two runs, alternated
`--repeats` times:
- one:   every stream on the context's camera (synth.shift_stream);
- eight: eight cameras, one per stream: crops of one render at eight offsets, each with its own principal point.
Host clock from the first push to the end of the flush gives tracked frames/s; the context's launch counter gives kernel
launches per frame; a separate torch.profiler run of each gives the device time of all kernels per frame.  Prints one
JSON line of medians with the GPU's name and power limit, read in the same run."""
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


def gpu_name_and_power():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def crop_stream(s, n):
    """synth.shift_stream's motion over a render of stream s's texture, cropped at an offset of its own: (frames, depth, K)."""
    tex = synth.texture(0x59475A00 + s, 2048)
    bw, bh = synth.W + 256, synth.H + 128
    base, _ = synth.render_plane(tex, np.eye(4)[:3], w=bw, h=bh, cx=bw / 2, cy=bh / 2)
    x0, y0 = 64 + 16 * s, 32 + 8 * s
    offs = [(x0 + int(round(40 * np.sin(2 * np.pi * k / 240))), y0 + int(round(20 * np.sin(2 * np.pi * k / 170)))) for k in range(n)]
    rng = np.random.default_rng(s)
    frames = np.stack([np.clip(base[oy:oy + synth.H, ox:ox + synth.W].astype(np.int16)
                               + np.rint(rng.normal(0, 2.0, (synth.H, synth.W))).astype(np.int16), 0, 255).astype(np.uint8) for ox, oy in offs])
    return frames, np.full((synth.H, synth.W), 2.0), (synth.FX, synth.FY, bw / 2 - offs[0][0], bh / 2 - offs[0][1])


def run(ctx, data, cameras, window, burst=8):
    """One engine per run, created outside the timed region.  Returns (seconds, launches, trajectory)."""
    S, n = len(data), len(data[0][0])
    eng = vo_native.Engine(ctx, S, window=window, cameras=cameras, **POLICY)
    ctx.synchronize()
    l0 = ctx.launch_count
    t0 = time.perf_counter()
    for k0 in range(0, n, burst):
        for s in range(S):
            for k in range(k0, min(n, k0 + burst)):
                eng.push(s, data[s][0][k], data[s][1] if k == 0 else None)
        eng.step()
    eng.flush()
    sec = time.perf_counter() - t0
    launches = ctx.launch_count - l0
    res = eng.poll()
    eng.close()
    assert len(res) == S * n and not (res["status"] == 2).any()
    traj = np.zeros((S, n, 12))
    traj[res["stream"], res["frame"]] = res["T_cw"]
    return sec, launches, traj


def kernel_us(fn):
    """Device time of all kernels of one run under torch.profiler, in microseconds."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return float(sum(e.self_device_time_total for e in prof.key_averages() if e.device_type.name == "CUDA"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--frames", type=int, default=240)
    ap.add_argument("--window", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    ctx = Context(0)
    S, n = a.streams, a.frames
    one = [tuple(synth.shift_stream(s, n)[:2]) for s in range(S)]
    crops = [crop_stream(s, n) for s in range(S)]
    eight = [(f, d) for f, d, _ in crops]
    cams = [K for _, _, K in crops]
    assert len(set(cams)) == S
    legs = {"one": lambda: run(ctx, one, None, a.window), "eight": lambda: run(ctx, eight, cams, a.window)}
    refs = {k: fn()[2] for k, fn in legs.items()}   # warm-up, and the trajectories every run must reproduce
    fps, lpf = {k: [] for k in legs}, {}
    for _ in range(a.repeats):
        for k, fn in legs.items():
            sec, launches, traj = fn()
            assert np.array_equal(traj, refs[k]), k
            fps[k].append(S * n / sec)
            lpf[k] = launches / (S * n)
    kus = {k: kernel_us(fn) / (S * n) for k, fn in legs.items()}
    print(json.dumps(dict(metric="tracked frames/s", gpu=gpu_name_and_power(), streams=S, frames=n, window=a.window, repeats=a.repeats,
                          median_fps={k: float(np.median(v)) for k, v in fps.items()}, launches_per_frame=lpf,
                          kernel_us_per_frame=kus, runs={k: [round(x, 1) for x in v] for k, v in fps.items()})))
    ctx.close()


if __name__ == "__main__":
    main()
