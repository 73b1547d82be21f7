"""GPU suite: undistorting uploads (ygzb_frames_set_undistort) give every pyramid level bit for bit equal to
tools/undistort_ref.py's remap (pinned to cv2 by tests/test_undistort.py) followed by the oracle's pyramid, through every upload
entry point; without maps nothing changes, and images re-uploaded from the tracker's records are not warped twice."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import undistort_ref as U  # noqa: E402

pytestmark = pytest.mark.gpu

# (width, height, levels, camera case of undistort_ref.CASES)
GEOMS = [(640, 480, 3, "tum_fr1"), (640, 480, 8, "tum_fr2"), (752, 480, 3, "euroc_cam0"), (321, 241, 3, "odd_321x241"),
         (640, 480, 3, "saturating")]


def _ctx(w, h, L):
    from ygz_slam_b200 import Context
    return Context(0, image_width=w, image_height=h, n_levels=L)


def _maps(name):
    w, h, K, D, newK = U.CASES[name]
    return U.undistort_map(w, h, K, D, None if isinstance(newK, str) else newK)


def _check_pyramids(oracle, fr, slots, raw, xy, a, what):
    w, h, L = fr.lw[0], fr.lh[0], len(fr.lw)
    for s, img in zip(slots, raw):
        want = oracle.build_pyramid(U.undistort_image(img, xy, a), L)
        for lv in range(L):
            got = fr.download_level(int(s), lv)
            n = int((got != oracle.level_view(want, w, h, L, lv)).sum())
            assert n == 0, f"{what}: slot {s} level {lv}: {n} pixels differ"


@pytest.mark.parametrize("geom", GEOMS, ids=lambda g: f"{g[0]}x{g[1]}x{g[2]}")
@pytest.mark.parametrize("channels", [1, 3])
@pytest.mark.parametrize("n", [1, 17])
def test_upload_bit_exact(oracle, geom, channels, n):
    w, h, L, case = geom
    ctx = _ctx(w, h, L)
    fr = ctx.frames(n + 2)
    xy, a = _maps(case)
    fr.set_undistort(xy, a)
    raw = [U.seeded_image(1000 + 31 * k + channels, h, w, channels) for k in range(n)]
    fr.upload(np.stack(raw), first=2)
    _check_pyramids(oracle, fr, range(2, n + 2), raw, xy, a, f"{case} C={channels} n={n}")
    fr.close()
    ctx.close()


@pytest.mark.parametrize("channels", [1, 3])
def test_device_source_and_long_stride(oracle, channels):
    """Sources in device memory and in host memory with a frame_stride larger than one image."""
    import torch
    w, h, L = 640, 480, 3
    ctx = _ctx(w, h, L)
    n = 17
    fr = ctx.frames(n)
    xy, a = _maps("tum_fr1")
    fr.set_undistort(xy, a)
    frame = w * h * channels
    stride = frame + 4096 + 3
    raw = [U.seeded_image(7 + k, h, w, channels) for k in range(n)]
    host = np.zeros((n, stride), np.uint8)
    for k in range(n):
        host[k, :frame] = raw[k].reshape(-1)
    fr.upload_raw(host.ctypes.data, n, channels, stride)
    _check_pyramids(oracle, fr, range(n), raw, xy, a, "host, long stride")
    dev = torch.from_numpy(host).cuda()
    torch.cuda.synchronize()
    fr.upload_raw(dev.data_ptr(), n, channels, stride)
    _check_pyramids(oracle, fr, range(n), raw, xy, a, "device source")
    fr.close()
    ctx.close()


def test_identity_clear_and_invalid(oracle):
    from ygz_slam_b200 import YgzbError
    w, h, L = 640, 480, 3
    ctx = _ctx(w, h, L)
    fr = ctx.frames(4)
    grey = U.seeded_image(5, h, w)
    bgr = U.seeded_image(6, h, w, 3)

    def levels(slot):
        return [fr.download_level(slot, lv) for lv in range(L)]

    fr.upload(grey[None], first=0)
    fr.upload(bgr[None], first=1)
    plain = [levels(0), levels(1)]
    # identity maps (D = 0, newK = K): bit-identical to an upload without maps
    ixy, ia = _maps("zero")
    gy, gx = np.mgrid[0:h, 0:w]
    assert (ia == 0).all() and (ixy[..., 0] == gx).all() and (ixy[..., 1] == gy).all()
    fr.set_undistort(ixy, ia)
    fr.upload(grey[None], first=2)
    fr.upload(bgr[None], first=3)
    for got, want in zip([levels(2), levels(3)], plain):
        assert all(np.array_equal(g, x) for g, x in zip(got, want))
    # invalid maps: YGZB_ERR_INVALID, the previous maps stay
    xy, a = _maps("tum_fr1")
    fr.set_undistort(xy, a)
    bad = a.copy()
    bad[100, 200] = 1024
    with pytest.raises(YgzbError, match="rc=-1"):
        fr.set_undistort(xy, bad)
    with pytest.raises(YgzbError, match="rc=-1"):
        ctx.check(ctx.lib.ygzb_frames_set_undistort(fr.h, xy.ctypes.data, None), "ygzb_frames_set_undistort")
    fr.upload(grey[None], first=2)
    _check_pyramids(oracle, fr, [2], [grey], xy, a, "after a rejected map")
    # clearing restores the plain path
    fr.set_undistort()
    fr.upload(grey[None], first=2)
    assert all(np.array_equal(g, x) for g, x in zip(levels(2), plain[0]))
    # ygzb_frames_build_pyramid starts from level 0 as it is, maps or not
    fr.set_undistort(xy, a)
    fr.build_pyramid(0, 1)
    assert all(np.array_equal(g, x) for g, x in zip(levels(0), plain[0]))
    fr.close()
    ctx.close()


def test_launch_counts():
    """Without maps an upload launches what it did before; with maps the remap replaces bgr2gray, or adds one launch for grey."""
    w, h, L = 640, 480, 3
    ctx = _ctx(w, h, L)
    fr = ctx.frames(8)
    grey = np.stack([U.seeded_image(k, h, w) for k in range(8)])
    bgr = np.stack([U.seeded_image(k, h, w, 3) for k in range(8)])

    def count(imgs):
        c0 = ctx.launch_count
        fr.upload(imgs)
        ctx.synchronize()
        return ctx.launch_count - c0

    plain_grey, plain_bgr = count(grey), count(bgr)
    assert (plain_grey, plain_bgr) == (2, 3)    # two pyrDown launches at 640 x 480 x 3 levels, plus bgr2gray
    fr.set_undistort(*_maps("tum_fr1"))
    assert (count(grey), count(bgr)) == (plain_grey + 1, plain_bgr)
    fr.set_undistort()
    assert (count(grey), count(bgr)) == (plain_grey, plain_bgr)
    fr.close()
    ctx.close()


def test_tracker_upload_equals_frames_upload(oracle):
    from ygz_slam_b200 import capi
    w, h, L = 640, 480, 3
    ctx = _ctx(w, h, L)
    xy, a = _maps("tum_fr2")
    fa, fb = ctx.frames(6), ctx.frames(6)
    fa.set_undistort(xy, a)
    fb.set_undistort(xy, a)
    K = U.CASES["tum_fr2"][2]
    t = capi.Tracker(fb, 2, 4, K)
    raw = np.stack([U.seeded_image(40 + k, h, w) for k in range(5)])
    fa.upload(raw, first=1)
    t.upload(1, raw)
    for s in range(1, 6):
        for lv in range(L):
            assert np.array_equal(fa.download_level(s, lv), fb.download_level(s, lv)), (s, lv)
    _check_pyramids(oracle, fb, range(1, 6), list(raw), xy, a, "tracker upload")
    t.close()
    fa.close()
    fb.close()
    ctx.close()


def test_record_imports_are_not_undistorted_again(oracle):
    """ygzb_tracker_import and ygzb_tracker_import_reference put the record's image into level 0 as it is, with maps set on the
    destination pool, and a second export returns the same bytes."""
    from ygz_slam_b200 import capi
    w, h, L = 640, 480, 3
    ctx = _ctx(w, h, L)
    xy, a = _maps("tum_fr1")
    K = U.CASES["tum_fr1"][2]
    fr = ctx.frames(8)
    fr.set_undistort(xy, a)
    t = capi.Tracker(fr, 1, 4, K)
    t.set_reference_mode("previous", [7])
    img = U.undistort_image(U.seeded_image(77, h, w), xy, a)   # an undistorted key-frame image
    rec = t.export(0, [0])
    rec.a["image"][0] = img
    t.import_(0, [0], [3], rec)
    want = oracle.build_pyramid(img, L)
    for lv in range(L):
        assert np.array_equal(fr.download_level(3, lv), oracle.level_view(want, w, h, L, lv)), lv
    again = t.export(0, [0])
    assert np.array_equal(again.a["image"][0], img)
    ref = capi.ReferenceBuffers(w, h, ctx.n_cells)
    r = ref.rec
    r.width, r.height, r.cells, r.n_levels = w, h, ctx.n_cells, L
    r.K[:] = list(K)
    r.capacity, r.n = capi.REF_FEATURES_PER_CELL * ctx.n_cells, 0
    r.T_cw[:] = list(np.eye(4)[:3].reshape(-1))
    ref.a["image"][...] = img
    t.import_reference(0, ref)
    for lv in range(L):
        assert np.array_equal(fr.download_level(7, lv), oracle.level_view(want, w, h, L, lv)), lv
    out = t.export_reference(0)
    assert np.array_equal(out.a["image"], img)
    t.close()
    fr.close()
    ctx.close()


# ---- the tracking loop on lens-rendered streams (4 streams) -------------------------------------------------------------
def test_gpu_loop_on_lens_streams(oracle, ctx3):
    """GPU loop with maps: within 1e-4 of the oracle loop with maps, bit-identical to the GPU loop without maps on frames
    undistorted by the restatement, and within the ground-truth bound measured on the CPU oracle (test_undistort.py)."""
    from oracle.vo_backend import OracleBackend
    from test_undistort import LENS_LOOP_BOUND, lens_frames, lens_maps, run_loop
    from ygz_slam_b200 import se3, vo
    S, n = 4, 12
    frames, depths, gts = lens_frames(S, n)
    xy, a = lens_maps()
    V, traj, errs = run_loop(vo.GpuBackend(ctx3, S * vo.VisualOdometry.SLOTS_PER_STREAM, undistort=(xy, a)), frames, depths, gts)
    Vo, traj_o, _ = run_loop(U.UndistortingBackend(OracleBackend(oracle), xy, a), frames, depths, gts)
    und = [[U.undistort_image(f, xy, a) for f in fs] for fs in frames]
    Vp, traj_p, _ = run_loop(vo.GpuBackend(ctx3, S * vo.VisualOdometry.SLOTS_PER_STREAM), und, depths, gts)
    Vr, _, raw_errs = run_loop(vo.GpuBackend(ctx3, S * vo.VisualOdometry.SLOTS_PER_STREAM), frames, depths, gts)
    for s in range(S):
        assert not V.streams[s].lost and V.streams[s].stats["keyframes"] == Vo.streams[s].stats["keyframes"]
    worst = max(float(np.linalg.norm(se3.se3_log(se3.mul(traj[s, k], se3.inv(traj_o[s, k])))))
                for s in range(S) for k in range(n))
    assert worst < 1e-4, worst
    assert np.array_equal(traj, traj_p)
    print(f"ground-truth error, worst over {S} streams: {np.nanmax(errs):.3e} with maps, {np.nanmax(raw_errs):.3e} without")
    assert np.nanmax(errs) < LENS_LOOP_BOUND


# ---- the C++ shim -------------------------------------------------------------------------------------------------------
def test_shim_camera_with_distortion(oracle, tmp_path):
    """PinholeCamera with k1 k2 p1 p2 + b200::Runtime::SetUndistortion, then Frame::InitFrame and FeatureDetector::Detect on a
    raw frame: the features of the oracle's detection on the undistorted frame."""
    import subprocess
    from ygz_slam_b200 import capi, synth
    capi.load_library()
    exe = tmp_path / "cpp_undistort_test"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-o", str(exe), str(ROOT / "tests" / "cpp_undistort_test.cpp"),
                    f"-L{ROOT / 'ygz_slam_b200'}", "-lygz_b200", f"-Wl,-rpath,{ROOT / 'ygz_slam_b200'}"], check=True, capture_output=True)
    raw, _, _ = synth.lens_stream_frame(3)
    cam = np.array([synth.FX, synth.FY, synth.CX, synth.CY] + list(synth.LENS_TUM_FR2[:4]), np.float32)
    blob = tmp_path / "in.bin"
    blob.write_bytes(raw.tobytes() + cam.tobytes())
    lines = subprocess.run([str(exe), str(blob)], capture_output=True, text=True, check=True).stdout.strip().splitlines()
    # the shim builds the maps from the float camera, k3 = 0 (Camera.h's model)
    xy, a = U.undistort_map(640, 480, tuple(float(v) for v in cam[:4]), tuple(float(v) for v in cam[4:]) + (0.0,))
    want = oracle.detect(oracle.build_pyramid(U.undistort_image(raw, xy, a), 3))
    assert lines[0] == f"features {want['n']}" and want["n"] > 500
    got = np.array([[float(t) for t in ln.split()[:3]] for ln in lines[1:]])
    assert np.array_equal(got[:, 0], want["px"]) and np.array_equal(got[:, 1], want["py"]) and np.array_equal(got[:, 2], want["level"])
    h = [int(ln.split()[3]) for ln in lines[1:]]
    wh = []
    for d in want["desc"]:
        v = 0
        for b in d:
            v = (v * 31 + int(b)) & 0xFFFFFFFFFFFFFFFF
        wh.append(v)
    assert h == wh
