"""Cost of the pose information records of the streaming API (ygz_vo_set_information / ygz_vo_poll_ex) on the legs of
tools/bench_stream.py: 8 synthetic streams (shift_stream) of 240 frames at bench.py's key-frame policy, window 8,
- stream: one frame per stream pushed (with its depth map), then ygz_vo_step and a poll, frame after frame, then a flush;
- burst:  8 frames per stream pushed before each step.
Each leg runs with information off (ygz_vo_poll) and on (ygz_vo_poll_ex into a reused host buffer), the four runs
alternated `--repeats` times; host clock from the first push to the end of the flush.  Both give the same trajectory bit
for bit.  A separate torch.profiler run of the burst leg with information on gives the device time of the kernel that
builds the records (track_info_kernel) per launch and per frame.  Prints one JSON line of medians (tracked frames/s over
all streams) with the GPU's name and power limit, read in the same run."""
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
from ygz_slam_b200.capi import INFO_DTYPE, pinned_empty  # noqa: E402

POLICY = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)   # bench.py's KF_POLICY


def gpu_name_and_power():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def stream_run(ctx, images, depths, window, burst, information, info_buf):
    """One engine per run, created outside the timed region.  Returns (seconds, trajectory, records of all results)."""
    lib = vo_native._lib()
    S, n = len(images), len(images[0])
    eng = vo_native.Engine(ctx, S, window=window, information=information, **POLICY)
    out = np.zeros(S * n, vo_native.RESULT_DTYPE)
    got = C.c_int(0)
    n_out = 0

    def poll():
        nonlocal n_out
        if information:
            ctx.check(lib.ygz_vo_poll_ex(eng.h, out[n_out:].ctypes.data, len(out) - n_out, C.byref(got), info_buf[n_out:].ctypes.data, None,
                                         0, None), "ygz_vo_poll_ex")
        else:
            ctx.check(lib.ygz_vo_poll(eng.h, out[n_out:].ctypes.data, len(out) - n_out, C.byref(got)), "ygz_vo_poll")
        n_out += got.value

    ctx.synchronize()
    t0 = time.perf_counter()
    for k0 in range(0, n, burst):
        for s in range(S):
            for k in range(k0, min(n, k0 + burst)):
                ctx.check(lib.ygz_vo_push(eng.h, s, images[s][k], depths[s], k), "ygz_vo_push")
        ctx.check(lib.ygz_vo_step(eng.h), "ygz_vo_step")
        poll()
    ctx.check(lib.ygz_vo_flush(eng.h), "ygz_vo_flush")
    poll()
    sec = time.perf_counter() - t0
    eng.close()
    assert n_out == S * n
    traj = np.zeros((S, n, 12))
    traj[out["stream"], out["frame"]] = out["T_cw"]
    order = np.lexsort((out["frame"], out["stream"]))
    return sec, traj.reshape(S, n, 3, 4), info_buf[order].tobytes() if information else None


def info_kernel_time(run):
    """Device time of track_info_kernel in one run under torch.profiler: (us per launch, launches, total us)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    us = [e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total for e in prof.events() if "track_info_kernel" in e.name]
    if not us:
        raise RuntimeError("the profiler recorded no track_info_kernel launch")
    return float(np.median(us)), len(us), float(np.sum(us))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--frames", type=int, default=240)
    ap.add_argument("--window", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=7)
    a = ap.parse_args()
    ctx = Context(0)
    S, n = a.streams, a.frames
    data = [synth.shift_stream(s, n) for s in range(S)]
    separate = [[pinned_empty(data[s][0][k].shape, np.uint8) for k in range(n)] for s in range(S)]
    for s in range(S):
        for k in range(n):
            separate[s][k][...] = data[s][0][k]
    pinned_depths = []
    for d in data:
        p = pinned_empty(d[1].shape, np.float64)
        p[...] = d[1]
        pinned_depths.append(p)
    images = [[f.ctypes.data for f in row] for row in separate]
    depths = [d.ctypes.data for d in pinned_depths]
    info_buf = np.zeros(S * n, INFO_DTYPE)   # every result's record
    legs = {f"{leg}_{'on' if on else 'off'}": (lambda burst=burst, on=on: stream_run(ctx, images, depths, a.window, burst, on, info_buf))
            for leg, burst in (("stream", 1), ("burst", 8)) for on in (False, True)}
    ref = legs["burst_off"]()[1]   # warm-up, and the trajectory every run must reproduce
    for fn in legs.values():
        fn()
    fps, records = {k: [] for k in legs}, None
    for _ in range(a.repeats):
        for name, fn in legs.items():
            sec, traj, r = fn()
            assert np.array_equal(traj, ref), name
            fps[name].append(S * n / sec)
            if name.endswith("_on"):   # the records do not depend on the pacing
                assert records is None or records == r
                records = r
    med = {k: float(np.median(v)) for k, v in fps.items()}
    kernel_us, launches, kernel_total_us = info_kernel_time(legs["burst_on"])
    print(json.dumps(dict(metric="tracked frames/s", gpu=gpu_name_and_power(), streams=S, frames=n, window=a.window, repeats=a.repeats,
                          median_fps=med, cost_of_information={leg: 1 - med[f"{leg}_on"] / med[f"{leg}_off"] for leg in ("stream", "burst")},
                          bytes_per_frame=INFO_DTYPE.itemsize,
                          info_kernel=dict(us_per_launch_median=kernel_us, launches=launches, us_per_frame=kernel_total_us / (S * n)),
                          runs={k: [round(x, 1) for x in v] for k, v in fps.items()})))
    ctx.close()


if __name__ == "__main__":
    main()
