"""Tracked frames/s of the device-resident engine with the key-frame reference and with the previous-frame reference
(ygz_vo_run_ex), at windows 1 and 8, in one run: BASELINE config C5's shape of 8 independent synthetic streams on one GPU
(shift_stream, key-frames every >= 5 frames at 0.03).  Prints one JSON line; the GPU's name and power limit go with it."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import numpy as np  # noqa: E402

from ygz_slam_b200 import Context, synth, vo_native  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warm", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    ctx = Context(0)
    data = [synth.shift_stream(s, a.frames) for s in range(a.streams)]
    frames = vo_native.stack_pinned([d[0] for d in data])
    depths = [d[1] for d in data]
    out = {}
    for rep in range(a.repeats):   # modes and windows alternate inside every repeat
        for mode in ("keyframe", "previous"):
            for w in (1, 8):
                traj, stats, sec = vo_native.run(ctx, frames, depths, 5, 0.03, 0.03, warm=a.warm, window=w, ref_mode=mode)
                assert not any(s["lost"] for s in stats), (mode, w)
                out.setdefault(f"{mode}_w{w}", []).append(a.streams * (a.frames - a.warm) / sec)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(metric="tracked frames/s", streams=a.streams, frames=a.frames, gpu=gpu,
                          median={k: float(np.median(v)) for k, v in out.items()}, runs=out)))
    ctx.close()


if __name__ == "__main__":
    main()
