"""The streaming API of libygz_vo.so (include/ygz_vo.h, vo_native.Engine): the device-resident engine fed frame by frame.
Pushed in lock step it must reproduce the batch entry point (ygz_vo_run_ex) bit for bit, at any window and in both
reference modes; pushed at any pace it must give every stream the trajectory of its own frames; each key-frame must
take its map points from its own depth map; the camera comes from the context."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from ygz_slam_b200 import se3, synth

ROOT = Path(__file__).resolve().parent.parent
LIBDIR = ROOT / "ygz_slam_b200"
POLICY = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)   # test_vo._run's key-frame policy
ERR_INVALID = -1


def declared_stream_symbols():
    text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "ygz_vo.h").read_text(), flags=re.S)
    return sorted(set(re.findall(r"\b(ygz_vo_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from ygz_slam_b200 import build
    build.build()
    lib = C.CDLL(str(build.VO_LIB))
    syms = declared_stream_symbols()
    assert len(syms) >= 8
    missing = [s_ for s_ in syms if not hasattr(lib, s_)]
    assert not missing, missing


def test_header_is_plain_c_and_links(tmp_path):
    """include/ygz_vo.h compiles as pedantic C99 and every entry point it declares links against libygz_vo.so."""
    syms = declared_stream_symbols()
    src = tmp_path / "vo.c"
    body = "\n".join(f"    p[{i}] = (fn)&{s_};" for i, s_ in enumerate(syms))
    src.write_text('#include "ygz_vo.h"\n#include <stdio.h>\ntypedef void (*fn)(void);\nint main(void) {\n    fn p[%d];\n%s\n'
                   '    ygz_vo_result r;\n    ygz_vo_config c;\n    printf("%%d %%d %%d\\n", (int)(sizeof p / sizeof p[0]), (int)sizeof r, (int)sizeof c);\n'
                   '    return p[0] == 0;\n}\n' % (len(syms), body))
    exe = tmp_path / "vo"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", f"-I{ROOT / 'include'}", str(src), "-o", str(exe), f"-L{LIBDIR}",
                    "-lygz_vo", "-lygz_b200", f"-Wl,-rpath,{LIBDIR}"], check=True, capture_output=True, text=True)
    n, size_result, size_config = map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split())
    from ygz_slam_b200 import vo_native
    assert n == len(syms)
    assert size_result == vo_native.RESULT_DTYPE.itemsize and size_config == C.sizeof(vo_native.VoConfig)


# ---- GPU ---------------------------------------------------------------------------------------------------------------

N_FRAMES = 30


@pytest.fixture(scope="module")
def shift_data():
    return [synth.shift_stream(s_, N_FRAMES) for s_ in range(4)]


_BATCH = {}


def batch(ctx, data, n_streams, window, ref_mode):
    """vo_native.run (ygz_vo_run_ex) on the first n_streams shift streams: (trajectory (S, n, 3, 4), stats rows)."""
    key = (n_streams, window, ref_mode)
    if key not in _BATCH:
        from ygz_slam_b200 import vo_native
        traj, stats, _ = vo_native.run(ctx, [d[0] for d in data[:n_streams]], [d[1] for d in data[:n_streams]], window=window,
                                       ref_mode=ref_mode, **POLICY)
        _BATCH[key] = (traj, stats)
    return _BATCH[key]


def collect(results, lengths):
    """Per-stream trajectories (S, n, 3, 4) from polled results; checks per-stream frame order and each tag exactly once."""
    traj = [np.full((n, 3, 4), np.nan) for n in lengths]
    status = [np.full(n, -1) for n in lengths]
    seen = [[] for _ in lengths]
    for r in results:
        s_, f = int(r["stream"]), int(r["frame"])
        seen[s_].append(int(r["tag"]))
        assert f == len(seen[s_]) - 1, "results out of frame order"
        traj[s_][f] = r["T_cw"].reshape(3, 4)
        status[s_][f] = r["status"]
    for s_, n in enumerate(lengths):
        assert seen[s_] == [1000 * s_ + k for k in range(n)], s_   # every tag exactly once, in frame order
    return traj, status


@pytest.mark.gpu
@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
@pytest.mark.parametrize("window", [1, 8])
def test_lock_step_matches_batch(ctx3, shift_data, window, ref_mode):
    """3 shift streams pushed in lock step (every frame with its depth map), then flush: trajectories and the 16 counters
    bit-identical to ygz_vo_run_ex on the same data."""
    from ygz_slam_b200 import vo_native
    S = 3
    ref_traj, ref_stats = batch(ctx3, shift_data, S, window, ref_mode)
    with vo_native.Engine(ctx3, S, window=window, ref_mode=ref_mode, **POLICY) as eng:
        for k in range(N_FRAMES):
            for s_ in range(S):
                assert eng.push(s_, shift_data[s_][0][k], shift_data[s_][1], tag=1000 * s_ + k) == k
        eng.flush()
        traj, status = collect(eng.poll(), [N_FRAMES] * S)
        stats = [eng.stats(s_) for s_ in range(S)]
        assert len(eng._alive) == 0   # every pushed array has been released
    for s_ in range(S):
        assert np.array_equal(traj[s_], ref_traj[s_]), s_
        assert stats[s_] == ref_stats[s_], s_
        assert stats[s_]["keyframes"] >= 3 and stats[s_]["ba"] >= 2 and stats[s_]["lost"] == 0
        assert (status[s_] == 1).sum() == stats[s_]["keyframes"] and status[s_][0] == 1 and (status[s_] == 2).sum() == 0


@pytest.mark.gpu
def test_arbitrary_pacing(ctx3, shift_data):
    """4 streams of different lengths (stream 1 starts 7 steps late, stream 3 ends early), seeded random pushes interleaved
    with steps at window 8: each stream's trajectory is that of the lock-step batch run over its frames."""
    from ygz_slam_b200 import vo_native
    lengths = [N_FRAMES, N_FRAMES - 3, N_FRAMES, 17]
    ref_traj, _ = batch(ctx3, shift_data, 4, 8, "keyframe")
    rng = np.random.default_rng(7)
    results = []
    with vo_native.Engine(ctx3, 4, window=8, **POLICY) as eng:
        pushed, steps = [0] * 4, 0
        while any(p < n for p, n in zip(pushed, lengths)):
            if rng.random() < 0.3:
                eng.step()
                steps += 1
                if rng.random() < 0.5:
                    results.append(eng.poll())
                continue
            s_ = int(rng.integers(4))
            if pushed[s_] >= lengths[s_] or (s_ == 1 and steps < 7):
                continue
            for _ in range(int(rng.integers(1, 4))):   # one to three frames of that stream at once
                if pushed[s_] < lengths[s_]:
                    k = pushed[s_]
                    eng.push(s_, shift_data[s_][0][k], shift_data[s_][1] if k == 0 or rng.random() < 0.5 else None, tag=1000 * s_ + k)
                    pushed[s_] += 1
        eng.flush()
        results.append(eng.poll())
        assert eng.poll().size == 0
    traj, status = collect(np.concatenate(results), lengths)
    for s_, n in enumerate(lengths):
        assert np.array_equal(traj[s_], ref_traj[s_][:n]), s_
        assert (status[s_] == 2).sum() == 0


@pytest.mark.gpu
def test_per_keyframe_depth(ctx3):
    """The rotating synth.stream_frame camera, whose depth changes from frame to frame: the streaming engine against the
    Python loop on the GPU backend (which uses each key-frame's own depth map), and every key-frame's map points from the
    depth map of the frame it was made from."""
    from ygz_slam_b200 import vo, vo_native
    S, n, step = 2, 20, 2
    frames = [[synth.stream_frame(step * k, stream=s_) for k in range(n)] for s_ in range(S)]
    be = vo.GpuBackend(ctx3, S * vo.VisualOdometry.SLOTS_PER_STREAM)
    V = vo.VisualOdometry(be, S, **POLICY)
    for k in range(n):
        V.add_frames([frames[s_][k][0] for s_ in range(S)], [frames[s_][k][1] for s_ in range(S)], k)
    be.fr.close()
    with vo_native.Engine(ctx3, S, window=8, **POLICY) as eng:
        for k in range(n):
            for s_ in range(S):
                eng.push(s_, frames[s_][k][0], frames[s_][k][1], tag=1000 * s_ + k)
            eng.step()
        eng.flush()
        traj, status = collect(eng.poll(), [n] * S)
        stats = [eng.stats(s_) for s_ in range(S)]
        maps = [eng.export_map(s_) for s_ in range(S)]
    for s_ in range(S):
        st = V.streams[s_]
        assert not st.lost and stats[s_]["lost"] == 0
        assert stats[s_]["keyframes"] == st.stats["keyframes"] >= 3 and stats[s_]["ba"] == st.stats["ba"] >= 2
        for key in ("candidates", "projected", "inliers"):
            assert abs(stats[s_][key] - st.stats[key]) <= 1e-3 * st.stats[key], key
        T0 = frames[s_][0][2]
        for k in range(n):
            assert np.linalg.norm(se3.se3_log(se3.mul(traj[s_][k], se3.inv(st.trajectory[k])))) < 1e-4, (s_, k)
            gt = se3.mul(frames[s_][k][2], se3.inv(T0))
            assert np.linalg.norm(se3.se3_log(se3.mul(traj[s_][k], se3.inv(gt)))) < 3e-3, (s_, k)
        # the ring holds the newest key-frames, oldest first: the last ones the results reported
        kf_frames = np.flatnonzero(status[s_] == 1)
        kfs = maps[s_].keyframes()
        assert 2 <= len(kfs) <= len(kf_frames)
        changed = 0
        assert np.array_equal(kfs[-1]["T_cw"], traj[s_][kf_frames[-1]])   # older ones moved in later local BAs
        for kf, f in zip(kfs, kf_frames[-len(kfs):]):
            px = kf["px"].astype(np.int64)
            own = frames[s_][f][1][px[:, 1], px[:, 0]]
            assert kf["depth"].size > 500 and np.array_equal(kf["depth"], own), (s_, f)
            changed += f > 0 and not np.array_equal(own, frames[s_][0][1][px[:, 1], px[:, 0]])
        assert changed >= 1   # the key-frames' own maps differ from the first frame's: the test sees the difference


def sliding_crops(n, w, h, plane_z=2.0, noise_sigma=2.0):
    """synth.shift_stream at another geometry: w x h crops sliding over one render of the stream-0 texture.  Returns frames,
    the constant depth, ground-truth poses and the crops' camera (fx, fy, cx, cy)."""
    tex = synth.texture(0x59475A00, 2048)
    bw, bh = w + 256, h + 128
    base, _ = synth.render_plane(tex, np.eye(4)[:3], plane_z=plane_z, w=bw, h=bh, cx=bw / 2, cy=bh / 2)
    rng = np.random.default_rng(2000)
    offs = [(int(round(128 + 110 * np.sin(2 * np.pi * k / 240))), int(round(64 + 50 * np.sin(2 * np.pi * k / 170)))) for k in range(n)]
    frames, poses = [], []
    for ox, oy in offs:
        crop = base[oy:oy + h, ox:ox + w].astype(np.int16) + np.rint(rng.normal(0, noise_sigma, (h, w))).astype(np.int16)
        frames.append(np.clip(crop, 0, 255).astype(np.uint8))
        T = np.eye(4)[:3].copy()
        T[0, 3] = -(ox - offs[0][0]) * plane_z / synth.FX
        T[1, 3] = -(oy - offs[0][1]) * plane_z / synth.FY
        poses.append(T)
    K = (synth.FX, synth.FY, bw / 2 - offs[0][0], bh / 2 - offs[0][1])
    return frames, np.full((h, w), plane_z), poses, K


@pytest.mark.gpu
def test_camera_from_context():
    """A 752 x 480 context with the crops' own principal point: the engine takes the image size from the context and K from
    its configuration, and tracks the ground truth."""
    from ygz_slam_b200 import Context, vo_native
    w, h, n = 752, 480, 30
    frames, depth, poses, K = sliding_crops(n, w, h)
    ctx = Context(0, image_width=w, image_height=h, fx=K[0], fy=K[1], cx=K[2], cy=K[3])
    try:
        with vo_native.Engine(ctx, 1, window=8, **POLICY) as eng:
            assert tuple(eng.cfg.K) == K   # the shortest decimals of the context's floats
            for k in range(n):
                eng.push(0, frames[k], depth, tag=k)
                if k % 3 == 2:
                    eng.step()
            eng.flush()
            res = eng.poll()
            stats = eng.stats(0)
        assert res["frame"].tolist() == list(range(n)) and stats["lost"] == 0 and stats["keyframes"] >= 3
        for k in range(n):
            T = res["T_cw"][k].reshape(3, 4)
            assert np.linalg.norm(se3.se3_log(se3.mul(T, se3.inv(poses[k])))) < 3e-3, k
    finally:
        ctx.close()


@pytest.mark.gpu
def test_invalid_input(ctx3, shift_data):
    """Every invalid input returns YGZB_ERR_INVALID and changes nothing: the valid pushes that follow give the results of
    the lock-step run."""
    from ygz_slam_b200 import vo_native
    lib = vo_native._lib()
    good = vo_native.VoConfig(3, 8, 0, POLICY["kf_min_frames"], POLICY["kf_min_rot"], POLICY["kf_min_trans"], 30,
                              (C.c_double * 4)(synth.FX, synth.FY, synth.CX, synth.CY))
    h = C.c_void_p()
    for field, value in (("n_streams", 0), ("window", 0), ("ref_mode", 2), ("min_inliers", -1)):
        bad = vo_native.VoConfig.from_buffer_copy(good)
        setattr(bad, field, value)
        assert lib.ygz_vo_create(ctx3.h, C.byref(bad), C.byref(h)) == ERR_INVALID and not h.value, field
    bad = vo_native.VoConfig.from_buffer_copy(good)
    bad.K[2] = synth.CX + 1e-3   # a camera that is not the context's
    assert lib.ygz_vo_create(ctx3.h, C.byref(bad), C.byref(h)) == ERR_INVALID and not h.value
    assert lib.ygz_vo_create(None, C.byref(good), C.byref(h)) == ERR_INVALID

    S = 3
    ref_traj, ref_stats = batch(ctx3, shift_data, S, 8, "keyframe")
    with vo_native.Engine(ctx3, S, window=8, **POLICY) as eng:
        img, dep = shift_data[0][0][0], shift_data[0][1]
        for stream in (-1, S):
            assert lib.ygz_vo_push(eng.h, stream, img.ctypes.data, dep.ctypes.data, 0) == ERR_INVALID
        assert lib.ygz_vo_push(eng.h, 0, None, dep.ctypes.data, 0) == ERR_INVALID
        assert lib.ygz_vo_push(eng.h, 0, img.ctypes.data, None, 0) == ERR_INVALID   # no depth map yet
        eng.step()
        assert eng.poll().size == 0
        for k in range(N_FRAMES):
            for s_ in range(S):
                eng.push(s_, shift_data[s_][0][k], shift_data[s_][1] if k == 0 else None, tag=1000 * s_ + k)
            if k == 0:   # the stream has a depth map now, but an image is still required
                assert lib.ygz_vo_push(eng.h, 0, None, None, 0) == ERR_INVALID
        eng.flush()
        traj, _ = collect(eng.poll(), [N_FRAMES] * S)
        for s_ in range(S):
            assert np.array_equal(traj[s_], ref_traj[s_]) and eng.stats(s_) == ref_stats[s_], s_
