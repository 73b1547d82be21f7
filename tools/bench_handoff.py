"""Time a stream's hand-over to a new tracker: per stream, the export + import of its map record, the export + import of its
reference record (previous-frame mode), and the engine's whole hand-over (ygz_vo_run_handoff_ex) in either mode.  Setting
of tools/bench_ref_modes.py: 8 synthetic streams (shift_stream, key-frames every >= 5 frames at 0.03).

- Records: the maps and references the engine exports at frame --handoff are imported into a fresh previous-mode tracker;
  then, per repetition, every stream's record is exported into a second buffer and imported again, and the context is
  synchronised.  Time = host clock around the repetition / streams.
- Hand-over: `seconds` of the engine covers frames [warm, n_frames) and ends in a synchronisation.  With warm = handoff the
  hand-over falls inside that region, so a run with the hand-over minus the run split at the same frame without one is
  the hand-over's cost (tear-down, a new context, frame pool and tracker, the record copies).  The two runs alternate.
Prints one JSON line of medians (ms) with the GPU's name and power limit, read in the same run."""
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
from ygz_slam_b200.capi import TRACK_RING, MapBuffers, ReferenceBuffers  # noqa: E402

POLICY = (5, 0.03, 0.03)


def gpu_name_and_power():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def time_records(ctx, maps, refs, reps, warmup):
    """Median ms per stream of a map export + import and of a reference export + import, on a fresh previous-mode tracker."""
    S = len(maps)
    lib = ctx.lib
    fr = ctx.frames(S * TRACK_RING + S)
    tr = fr.tracker(S, 8, maps[0].header["K"])
    tr.set_reference_mode("previous", S * TRACK_RING + np.arange(S))
    entries, slots = [], []
    for s in range(S):
        n = maps[s].rec.n_keyframes
        entries.append(np.ascontiguousarray(maps[s].a["entry"][:n], np.int32))
        slots.append(np.ascontiguousarray(s * TRACK_RING + entries[s], np.int32))
        tr.import_(s, entries[s], slots[s], maps[s])
        tr.import_reference(s, refs[s])
    map_out = [MapBuffers(TRACK_RING, 640, 480, ctx.n_cells) for _ in range(S)]
    ref_out = [ReferenceBuffers(640, 480, ctx.n_cells) for _ in range(S)]

    def map_round():
        for s in range(S):
            e = entries[s].ctypes.data_as(C.c_void_p)
            ctx.check(lib.ygzb_tracker_export(tr.h, s, len(entries[s]), e, C.byref(map_out[s].rec)), "ygzb_tracker_export")
            ctx.check(lib.ygzb_tracker_import(tr.h, s, e, slots[s].ctypes.data_as(C.c_void_p), C.byref(maps[s].rec)), "ygzb_tracker_import")

    def ref_round():
        for s in range(S):
            ctx.check(lib.ygzb_tracker_export_reference(tr.h, s, C.byref(ref_out[s].rec)), "ygzb_tracker_export_reference")
            ctx.check(lib.ygzb_tracker_import_reference(tr.h, s, C.byref(refs[s].rec)), "ygzb_tracker_import_reference")

    out = {}
    for name, fn in (("map_export_import", map_round), ("reference_export_import", ref_round)):
        times = []
        for r in range(warmup + reps):
            ctx.synchronize()
            t0 = time.perf_counter()
            fn()
            ctx.synchronize()
            if r >= warmup:
                times.append((time.perf_counter() - t0) * 1e3 / S)
        out[name] = times
    # the exports of the last repetition are the records that went in
    for s in range(S):
        assert np.array_equal(ref_out[s].a["px"], refs[s].a["px"]) and np.array_equal(ref_out[s].a["image"], refs[s].a["image"])
        assert np.array_equal(map_out[s].a["pw"], maps[s].a["pw"])
    tr.close()
    fr.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--handoff", type=int, default=20)
    ap.add_argument("--window", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=10, help="alternating pairs of engine runs per mode")
    ap.add_argument("--record-reps", type=int, default=50)
    ap.add_argument("--record-warmup", type=int, default=5)
    a = ap.parse_args()
    assert 0 < a.handoff < a.frames
    ctx = Context(0)
    data = [synth.shift_stream(s, a.frames) for s in range(a.streams)]
    frames = vo_native.stack_pinned([d[0] for d in data])
    depths = [d[1] for d in data]
    kw = dict(warm=a.handoff, window=a.window)
    *_, maps, refs = vo_native.run(ctx, frames, depths, *POLICY, handoff=a.handoff, return_maps=True, ref_mode="previous", **kw)
    records = time_records(ctx, maps, refs, a.record_reps, a.record_warmup)
    handover = {}
    for mode in ("keyframe", "previous"):
        vo_native.run(ctx, frames, depths, *POLICY, handoff=a.handoff, ref_mode=mode, **kw)   # warm-up
        split, handed = [], []
        for _ in range(a.repeats):
            traj_a, stats_a, sec_a = vo_native.run(ctx, frames, depths, *POLICY, ref_mode=mode, **kw)
            traj_b, stats_b, sec_b = vo_native.run(ctx, frames, depths, *POLICY, handoff=a.handoff, ref_mode=mode, **kw)
            assert np.array_equal(traj_a, traj_b) and stats_a == stats_b, mode
            split.append(sec_a * 1e3)
            handed.append(sec_b * 1e3)
        diff = [b - s for s, b in zip(split, handed)]
        handover[mode] = dict(split_run_ms=float(np.median(split)), handoff_run_ms=float(np.median(handed)),
                              handover_ms=float(np.median(diff)), handover_ms_per_stream=float(np.median(diff)) / a.streams,
                              handover_ms_runs=diff)
    print(json.dumps(dict(metric="hand-over ms", gpu=gpu_name_and_power(), streams=a.streams, frames=a.frames, handoff=a.handoff,
                          window=a.window, ms_per_stream={k: float(np.median(v)) for k, v in records.items()},
                          record_runs={k: [float(x) for x in v] for k, v in records.items()}, engine=handover)))
    ctx.close()


if __name__ == "__main__":
    main()
