"""Cost of the map updates of the streaming API (ygz_vo_set_map_updates / ygz_vo_poll_map_updates) on the legs of
tools/bench_stream.py: 8 synthetic streams (shift_stream) of 240 frames at bench.py's key-frame policy, window 8,
- stream: one frame per stream pushed (with its depth map), then ygz_vo_step and a poll, frame after frame, then a flush;
- burst:  8 frames per stream pushed before each step.
Each leg runs with map updates off (ygz_vo_poll) and on (ygz_vo_poll, then ygz_vo_poll_map_updates into reused host
buffers), the four runs alternated `--repeats` times; host clock from the first push to the end of the flush.  All give
the same trajectory bit for bit, and the runs with updates on the same updates.  A separate torch.profiler run of the
burst leg with updates on gives the device time of the kernel that writes the rows (kf_points_kernel) per launch (one
launch per round with key-frame insertions) and per insertion.  Prints one JSON line of medians (tracked frames/s over all
streams) with the GPU's name and power limit, read in the same run."""
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
from ygz_slam_b200.capi import MAP_POINT_DTYPE, pinned_empty  # noqa: E402

POLICY = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)   # bench.py's KF_POLICY


def gpu_name_and_power():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def stream_run(ctx, images, depths, window, burst, updates, upd_buf, row_buf):
    """One engine per run, created outside the timed region.  Returns (seconds, trajectory, update count, rows, bytes of
    the updates and rows)."""
    lib = vo_native._lib()
    S, n = len(images), len(images[0])
    eng = vo_native.Engine(ctx, S, window=window, map_updates=updates, **POLICY)
    out = np.zeros(S * n, vo_native.RESULT_DTYPE)
    got, got_rows = C.c_int(0), C.c_size_t(0)
    n_out = n_upd = n_rows = 0

    def poll():
        nonlocal n_out, n_upd, n_rows
        ctx.check(lib.ygz_vo_poll(eng.h, out[n_out:].ctypes.data, len(out) - n_out, C.byref(got)), "ygz_vo_poll")
        n_out += got.value
        if updates:
            ctx.check(lib.ygz_vo_poll_map_updates(eng.h, upd_buf[n_upd:].ctypes.data, len(upd_buf) - n_upd, C.byref(got),
                                                  row_buf[n_rows:].ctypes.data, len(row_buf) - n_rows, C.byref(got_rows)),
                      "ygz_vo_poll_map_updates")
            n_upd += got.value
            n_rows += got_rows.value

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
    if not updates:
        return sec, traj.reshape(S, n, 3, 4), 0, 0, None
    u = upd_buf[:n_upd]
    assert n_upd == (out["status"] == 1).sum() and int((u["n_moved"].astype(np.int64) + u["n_new"]).sum()) == n_rows
    # updates of different streams may interleave differently with the pacing: compare them per stream
    ends = np.concatenate([[0], np.cumsum(u["n_moved"].astype(np.int64) + u["n_new"])])
    per = sorted((int(x["stream"]), int(x["frame"]), x.tobytes(), row_buf[ends[i]:ends[i + 1]].tobytes()) for i, x in enumerate(u))
    return sec, traj.reshape(S, n, 3, 4), n_upd, n_rows, hash(tuple(per))


def kernel_time(run, name="kf_points_kernel"):
    """Device time of `name` in one run under torch.profiler: (us per launch, launches, total us)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    us = [e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total for e in prof.events() if name in e.name]
    if not us:
        raise RuntimeError(f"the profiler recorded no {name} launch")
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
    # every update of a run, with room for its most rows: a stream inserts at most one key-frame per kf_min_frames frames
    max_updates = S * (n // POLICY["kf_min_frames"] + 2)
    upd_buf = np.zeros(max_updates, vo_native.MAP_UPDATE_DTYPE)
    row_buf = np.zeros(max_updates * 4 * ctx.n_cells, MAP_POINT_DTYPE)
    legs = {f"{leg}_{'on' if on else 'off'}": (lambda burst=burst, on=on: stream_run(ctx, images, depths, a.window, burst, on, upd_buf, row_buf))
            for leg, burst in (("stream", 1), ("burst", 8)) for on in (False, True)}
    ref = legs["burst_off"]()[1]   # warm-up, and the trajectory every run must reproduce
    for fn in legs.values():
        fn()
    fps, digest, counts = {k: [] for k in legs}, None, None
    for _ in range(a.repeats):
        for name, fn in legs.items():
            sec, traj, n_upd, n_rows, h = fn()
            assert np.array_equal(traj, ref), name
            fps[name].append(S * n / sec)
            if name.endswith("_on"):   # the updates do not depend on the pacing
                assert digest is None or digest == h
                digest, counts = h, (n_upd, n_rows)
    med = {k: float(np.median(v)) for k, v in fps.items()}
    kernel_us, launches, kernel_total_us = kernel_time(legs["burst_on"])
    n_upd, n_rows = counts
    print(json.dumps(dict(metric="tracked frames/s", gpu=gpu_name_and_power(), streams=S, frames=n, window=a.window, repeats=a.repeats,
                          median_fps=med, cost_of_map_updates={leg: 1 - med[f"{leg}_on"] / med[f"{leg}_off"] for leg in ("stream", "burst")},
                          updates=n_upd, rows_per_update=n_rows / n_upd,
                          bytes_per_update=(n_upd * vo_native.MAP_UPDATE_DTYPE.itemsize + n_rows * MAP_POINT_DTYPE.itemsize) / n_upd,
                          kf_points_kernel=dict(us_per_launch_median=kernel_us, launches=launches, us_per_insertion=kernel_total_us / n_upd),
                          runs={k: [round(x, 1) for x in v] for k, v in fps.items()})))
    ctx.close()


if __name__ == "__main__":
    main()
