"""Time a stream record's save and load (ygz_vo_save_stream / ygz_vo_load_stream) and report its size.  Setting of
tools/bench_handoff.py: 8 synthetic streams (shift_stream, key-frames every >= 5 frames at 0.03), pushed in lock step with
their depth maps to frame --cut (mid-sequence) and flushed, in both reference modes.

- Save: per repetition every stream is saved (ygz_vo_save_stream into a buffer allocated once); each call synchronises the
  context.  Load: every record is loaded (ygz_vo_load_stream) into the same stream of a second engine, then its context is
  synchronised.  Time = host clock around the 8 C calls (and the synchronisation) / streams, medians and ranges over
  --reps repetitions after --warmup.
- Every load is checked: the loaded stream saves the same bytes again.
Prints one JSON line (ms, bytes) with the GPU's name and power limit, read in the same run."""
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

POLICY = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)


def gpu_name_and_power():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def measure(ctx, data, mode, cut, window, reps, warmup):
    S = len(data)
    with vo_native.Engine(ctx, S, window=window, ref_mode=mode, **POLICY) as src, \
            vo_native.Engine(ctx, S, window=window, ref_mode=mode, **POLICY) as dst:
        for k in range(cut):
            for s in range(S):
                src.push(s, data[s][0][k], data[s][1])
        src.flush()
        src.poll()
        # the C calls themselves, into and out of buffers allocated once (the Python wrappers copy the record to bytes)
        lib, bound = src.lib, src.stream_record_bound()
        bufs, sizes = [np.empty(bound, np.uint8) for _ in range(S)], [C.c_size_t(0) for _ in range(S)]
        save_ms, load_ms = [], []
        for r in range(warmup + reps):
            t0 = time.perf_counter()
            for s in range(S):
                ctx.check(lib.ygz_vo_save_stream(src.h, s, bufs[s].ctypes.data, bound, C.byref(sizes[s])), "ygz_vo_save_stream")
            t1 = time.perf_counter()
            for s in range(S):
                ctx.check(lib.ygz_vo_load_stream(dst.h, s, bufs[s].ctypes.data, sizes[s].value), "ygz_vo_load_stream")
            ctx.synchronize()
            t2 = time.perf_counter()
            if r >= warmup:
                save_ms.append((t1 - t0) * 1e3 / S)
                load_ms.append((t2 - t1) * 1e3 / S)
        sizes = [sz.value for sz in sizes]
        for s in range(S):
            assert dst.save_stream(s) == bufs[s][:sizes[s]].tobytes(), s
        return dict(record_bytes=sizes, record_bound=bound, save_ms_per_stream=float(np.median(save_ms)),
                    load_ms_per_stream=float(np.median(load_ms)), save_ms_range=[min(save_ms), max(save_ms)],
                    load_ms_range=[min(load_ms), max(load_ms)], save_ms_runs=save_ms, load_ms_runs=load_ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--cut", type=int, default=20)
    ap.add_argument("--window", type=int, default=8)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    assert 0 < a.cut <= a.frames
    ctx = Context(0)
    data = [synth.shift_stream(s, a.frames) for s in range(a.streams)]
    out = {mode: measure(ctx, data, mode, a.cut, a.window, a.reps, a.warmup) for mode in ("keyframe", "previous")}
    print(json.dumps(dict(metric="stream record ms per stream", gpu=gpu_name_and_power(), streams=a.streams, cut=a.cut,
                          window=a.window, cells=ctx.n_cells, modes=out)))
    ctx.close()


if __name__ == "__main__":
    main()
