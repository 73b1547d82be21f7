"""Time undistortion on upload: upload + pyramid of 8 streams x 10 frames at 640 x 480 with 3 levels, grey and BGR, maps off
and on (TUM fr1 camera), device time between two ygzb_timer_* events around each batch of uploads.  Off and on runs alternate
within one command; medians over --reps.  Next to it, cv2.remap of one grey frame on one host thread (the CPU alternative a
caller would otherwise run before uploading), if cv2 is installed.  Prints one JSON line with the GPU's name and power limit,
read in the same run.  Sources are page-locked host frames (one batched upload of 8 frames per frame index)."""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

import numpy as np  # noqa: E402

import undistort_ref as U  # noqa: E402
from ygz_slam_b200 import Context, capi  # noqa: E402


def gpu_name_and_power():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--reps", type=int, default=9)
    args = ap.parse_args()
    S, N, W, H = args.streams, args.frames, 640, 480
    ctx = Context(0, n_levels=3)
    fr = ctx.frames(S)
    w, h, K, D, _ = U.CASES["tum_fr1"]
    xy, a = capi.undistort_map(W, H, K, D)
    src = {c: capi.pinned_empty((N, S) + ((H, W) if c == 1 else (H, W, 3)), np.uint8) for c in (1, 3)}
    rng = np.random.default_rng(0)
    for c in (1, 3):
        src[c][...] = rng.integers(0, 256, src[c].shape, dtype=np.uint8)
    frame = {c: W * H * c for c in (1, 3)}

    def run(c):
        ctx.check(ctx.lib.ygzb_timer_start(ctx.h), "ygzb_timer_start")
        for k in range(N):
            fr.upload_raw(src[c][k].ctypes.data, S, c, frame[c])
        ms = C.c_double()
        ctx.check(ctx.lib.ygzb_timer_stop(ctx.h, C.byref(ms)), "ygzb_timer_stop")
        return ms.value / (S * N)

    times = {(c, m): [] for c in (1, 3) for m in ("off", "on")}
    for c in (1, 3):   # warm-up: allocations, staging, first launches
        for m in ("off", "on"):
            fr.set_undistort(xy, a) if m == "on" else fr.set_undistort()
            run(c)
    for _ in range(args.reps):
        for c in (1, 3):
            for m in ("off", "on"):
                fr.set_undistort(xy, a) if m == "on" else fr.set_undistort()
                times[(c, m)].append(run(c))
    out = {f"{'grey' if c == 1 else 'bgr'}_maps_{m}_ms_per_frame": float(np.median(v)) for (c, m), v in times.items()}
    try:
        import cv2
        img = src[1][0, 0].copy()
        cv2.setNumThreads(1)
        t = []
        for _ in range(50):
            t0 = time.perf_counter()
            cv2.remap(img, xy, a, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
            t.append(time.perf_counter() - t0)
        out["host_cv2_remap_ms_per_frame_1_thread"] = float(np.median(t) * 1e3)
    except ImportError:
        out["host_cv2_remap_ms_per_frame_1_thread"] = None
    out.update(streams=S, frames=N, size=f"{W}x{H}", levels=3, reps=args.reps, gpu=gpu_name_and_power())
    print(json.dumps(out))
    fr.close()
    ctx.close()


if __name__ == "__main__":
    main()
