"""Raw frames of each stream's own size and colour (ygz_vo_set_frame_format, ygzb_tracker_set_source): a stream pushed raw
frames of another size, or BGR, must give, byte for byte, what a default-format stream gives when it is pushed the frames
resampled in numpy by tools/undistort_ref.py -- maps of the pipeline's size built from the raw camera's K, then
cv::remap(cvtColor(raw)) -- which tests/golden/cv2_raw_frames.npz pins to OpenCV (tools/make_raw_frame_fixture.py)."""
import ctypes as C
import hashlib
import sys
from pathlib import Path

import numpy as np
import pytest

from ygz_slam_b200 import synth

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import make_raw_frame_fixture as FX  # noqa: E402  (its cases; it imports cv2 only to compute them)
import undistort_ref as U  # noqa: E402

POLICY = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)
ERR_INVALID = -1
W, H, N = 640, 480, 24
CAM = (synth.FX, synth.FY, synth.CX, synth.CY)
# raw cameras whose resampling with newK = CAM gives the synthetic streams' pinhole camera at 640 x 480: (width, height,
# K_raw, dist, channels)
RAW_CROP = (752, 480, (synth.FX, synth.FY, synth.CX + 56.0, synth.CY), U.EUROC_CAM0[1], 1)        # EuRoC's size, cropped
RAW_SCALE = (1280, 720, (780.0, 780.0, 639.5, 359.5), (0.05, -0.1, 0.0005, -0.0003, 0.0), 3)       # HD colour, 1.5x down
RAW_UP = (320, 240, (260.45, 260.5, 162.55, 124.85), synth.LENS_TUM_FR2, 1)                       # half size, 2x up
RAW_BGR = (W, H, None, None, 3)                                                                     # colour, no lens


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(ROOT / "tests" / "golden" / "cv2_raw_frames.npz"))


def colourise(grey):
    """A BGR frame whose cvtColor(BGR2GRAY) keeps the grey frame's texture, with three different channels."""
    g = grey.astype(np.int32)
    return np.stack([g, np.clip(g * 3 // 4 + 40, 0, 255), 255 - g // 2], -1).astype(np.uint8)


def _maps(raw):
    w, h, K, dist, _ = raw
    return U.undistort_map(W, H, K, dist, CAM)


def _resample(frames, raw):
    """What a default-format stream is pushed: level 0 of the raw frames, resampled in numpy."""
    if raw[2] is None:
        return [U.bgr2gray(f) if f.ndim == 3 else f for f in frames]
    xy, a = _maps(raw)
    return [U.undistort_image(f, xy, a) for f in frames]


# ---- without a GPU ---------------------------------------------------------------------------------------------------
def test_reference_maps_and_remaps_match_golden(golden):
    """undistort_ref's maps of the pipeline's size from the raw camera, and its remaps of raw frames of another size, equal
    OpenCV's: the digests of the full cases, the small cases entry for entry."""
    for name, (rw, rh, K, D, newK) in FX.CASES.items():
        xy, a = U.undistort_map(*FX.OUT, K, D, newK)
        grey = U.seeded_image(FX.GREY_SEED, rh, rw)
        bgr = U.seeded_image(FX.BGR_SEED, rh, rw, 3)
        got = [_sha(xy), _sha(a), _sha(U.undistort_image(grey, xy, a)), _sha(U.undistort_image(bgr, xy, a))]
        assert got == list(golden[f"{name}/sha"]), name
    for name, (size, (rw, rh, K, D, newK)) in FX.SMALL.items():
        xy, a = U.undistort_map(*size, K, D, newK)
        assert np.array_equal(xy, golden[f"{name}/map_xy"]) and np.array_equal(a, golden[f"{name}/map_a"]), name
        assert np.array_equal(U.undistort_image(U.seeded_image(FX.GREY_SEED, rh, rw), xy, a), golden[f"{name}/remap_grey"]), name
        assert np.array_equal(U.undistort_image(U.seeded_image(FX.BGR_SEED, rh, rw, 3), xy, a), golden[f"{name}/remap_bgr"]), name


def test_library_maps_match_golden(golden):
    """ygzb_undistort_map (host code: no device needed) builds the same maps from a raw camera of another size."""
    from ygz_slam_b200 import capi
    for name, (rw, rh, K, D, newK) in FX.CASES.items():
        xy, a = capi.undistort_map(*FX.OUT, K, D, newK)
        assert [_sha(xy), _sha(a)] == list(golden[f"{name}/sha"][:2]), name
    for name, (size, (rw, rh, K, D, newK)) in FX.SMALL.items():
        xy, a = capi.undistort_map(*size, K, D, newK)
        assert np.array_equal(xy, golden[f"{name}/map_xy"]) and np.array_equal(a, golden[f"{name}/map_a"]), name


def test_reference_matches_cv2_live():
    cv2 = pytest.importorskip("cv2")
    for name, case in FX.CASES.items():
        m1, m2, rg, rb = FX.cv2_case(FX.OUT, *case)
        rw, rh, K, D, newK = case
        xy, a = U.undistort_map(*FX.OUT, K, D, newK)
        assert np.array_equal(xy, m1) and np.array_equal(a, m2), name
        assert np.array_equal(U.undistort_image(U.seeded_image(FX.GREY_SEED, rh, rw), xy, a), rg), name
        assert np.array_equal(U.undistort_image(U.seeded_image(FX.BGR_SEED, rh, rw, 3), xy, a), rb), name
    assert cv2.__version__


def _raw_seq(stream, raw, n=N, step=1):
    """(raw frames of the raw camera `raw`, depth of CAM at 640 x 480, poses) of synthetic stream `stream`."""
    w, h, K, dist, ch = raw
    if K is None:
        fr = [synth.stream_frame(step * k, stream=stream) for k in range(n)]
    else:
        fr = [synth.lens_stream_frame(step * k, stream=stream, dist=dist, raw=(w, h, K)) for k in range(n)]
    frames = [colourise(f[0]) if ch == 3 else f[0] for f in fr]
    return frames, [f[1] for f in fr], [f[2] for f in fr]


def test_synth_raw_camera():
    """The raw camera's frame has its own size; the depth map stays that of CAM at 640 x 480; the defaults are unchanged."""
    g, d, T = synth.lens_stream_frame(4, raw=(1280, 720, RAW_SCALE[2]))
    g0, d0, T0 = synth.lens_stream_frame(4)
    assert g.shape == (720, 1280) and d.shape == (H, W) and np.array_equal(d, d0) and np.array_equal(T, T0)
    assert np.array_equal(synth.lens_stream_frame(4, raw=(W, H, CAM))[0], g0)


def test_oracle_loop_on_raw_hd_bgr_frames(oracle):
    """The Python loop on the CPU oracle, fed raw 1280 x 720 BGR frames through undistort_ref's backend wrapper, tracks
    the synthetic ground truth."""
    from oracle.vo_backend import OracleBackend
    from test_undistort import LENS_LOOP_BOUND, run_loop
    frames, depths, gts = _raw_seq(0, RAW_SCALE, 16, 2)
    V, _, errs = run_loop(U.UndistortingBackend(OracleBackend(oracle), *_maps(RAW_SCALE)), [frames], [depths], [gts])
    worst = float(np.nanmax(errs))
    print(f"worst ground-truth error on raw HD BGR frames: {worst:.3e}")
    assert not V.streams[0].lost and V.streams[0].stats["keyframes"] >= 2
    assert worst < LENS_LOOP_BOUND


# ---- the tracker, on the GPU -----------------------------------------------------------------------------------------
def _ctx():
    from ygz_slam_b200 import Context
    return Context(0, image_width=W, image_height=H)


@pytest.mark.gpu
def test_tracker_uploads_each_format(oracle):
    """ygzb_tracker_upload_stream in each stream's format gives every pyramid level of the oracle on the numpy-resampled
    frame: grey and BGR, raw sizes larger, smaller and odd, maps reaching outside the raw frame, host and device
    sources, a strided batch and single frames.  Refusals leave the stream's format as it was."""
    import torch
    from ygz_slam_b200 import capi
    ctx = _ctx()
    fr = ctx.frames(16)
    L = len(fr.lw)
    tr = capi.Tracker(fr, 6, 8, CAM)
    lib = fr.lib
    odd = FX.CASES["odd_753x481"]
    narrow = FX.CASES["narrow_400x300_outside"]
    # stream -> (width, height, channels, maps or None)
    fmts = {0: (1280, 720, 3, _maps(RAW_SCALE)), 1: (752, 480, 1, _maps(RAW_CROP)), 2: (320, 240, 1, _maps(RAW_UP)),
            3: (W, H, 3, None), 4: (753, 481, 3, U.undistort_map(W, H, odd[2], odd[3], odd[4])),
            5: (400, 300, 1, U.undistort_map(W, H, narrow[2], narrow[3], narrow[4]))}
    raws, want = {}, {}
    for s, (w, h, ch, maps) in fmts.items():
        tr.set_source(s, w, h, ch)
        if maps is not None:
            tr.set_undistort(s, *maps)
        raws[s] = [U.seeded_image(500 + 10 * s + k, h, w, ch) for k in range(2)]
    slot = 0
    for s, (w, h, ch, maps) in fmts.items():
        fb = w * h * ch
        a, b = raws[s]
        if s in (0, 4):    # one strided batch from host memory, rows of the batch padded past one frame
            stride = fb + 80
            buf = np.zeros((2, stride), np.uint8)
            buf[0, :fb], buf[1, :fb] = a.reshape(-1), b.reshape(-1)
            assert lib.ygzb_tracker_upload_stream(tr.h, s, slot, 2, buf.ctypes.data, stride) == 0
        elif s == 2:       # device memory
            dev = torch.from_numpy(np.stack([a, b])).cuda()
            torch.cuda.synchronize()
            assert lib.ygzb_tracker_upload_stream(tr.h, s, slot, 2, dev.data_ptr(), fb) == 0
            torch.cuda.synchronize()
        else:              # frame by frame
            tr.upload_stream(s, slot, a[None])
            tr.upload_stream(s, slot + 1, b[None])
        for k, img in enumerate((a, b)):
            want[slot + k] = (U.bgr2gray(img) if ch == 3 else img) if maps is None else U.undistort_image(img, *maps)
        slot += 2
    ctx.synchronize()

    def check(slots):
        for sl in slots:
            pyr = oracle.build_pyramid(want[sl], L)
            for lv in range(L):
                assert np.array_equal(fr.download_level(sl, lv), oracle.level_view(pyr, W, H, L, lv)), (sl, lv)
    check(range(slot))
    # refusals, each leaving stream 1 at 752 x 480 grey
    for args in ((1, 0, 480, 1), (1, 752, 0, 1), (1, 32768, 480, 1), (1, 752, 32768, 1), (1, 752, 480, 2), (1, 752, 480, 4),
                 (-1, 752, 480, 1), (6, 752, 480, 1)):
        assert lib.ygzb_tracker_set_source(tr.h, *args) == ERR_INVALID, args
    assert lib.ygzb_tracker_set_source(None, 1, 752, 480, 1) == ERR_INVALID
    img = U.seeded_image(900, 480, 752)
    assert lib.ygzb_tracker_upload_stream(tr.h, 1, 12, 1, img.ctypes.data, 752 * 480 - 1) == ERR_INVALID   # stride < frame
    tr.upload_stream(1, 12, img[None])
    want[12] = U.undistort_image(img, *fmts[1][3])
    # a size other than the context's needs the stream's maps; the largest size the maps can address is accepted
    assert lib.ygzb_tracker_set_source(tr.h, 2, 32767, 1, 1) == 0
    tr.set_undistort(2)
    small = U.seeded_image(901, 240, 320)
    tr.set_source(2, 320, 240, 1)
    assert lib.ygzb_tracker_upload_stream(tr.h, 2, 13, 1, small.ctypes.data, small.size) == ERR_INVALID
    # back to the default: exactly the plain upload
    tr.set_source(2, W, H, 1)
    plain = U.seeded_image(902, H, W)
    tr.upload_stream(2, 13, plain[None])
    want[13] = plain
    ctx.synchronize()
    check((12, 13))
    tr.close()
    fr.close()
    ctx.close()


# ---- the engine, on the GPU ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def streams():
    """(raw frames, depth, raw camera) of four streams: 752 x 480 grey cropped, 1280 x 720 BGR scaled, 320 x 240 grey
    upsampled, 640 x 480 BGR without a lens."""
    out = []
    for s, raw in enumerate((RAW_CROP, RAW_SCALE, RAW_UP, RAW_BGR)):
        frames, depths, _ = _raw_seq(s, raw)
        out.append((frames, depths[0], raw))
    return out


def _engine_kw(raws):
    return dict(cameras=[CAM] * len(raws), lenses=[None if r[2] is None else (r[2], r[3]) for r in raws],
                frame_formats=[(r[0], r[1], r[4]) for r in raws])


def _cols(a, names):
    return b"".join(np.ascontiguousarray(a[n]).tobytes() for n in names)


def _run(eng, data, pacing):
    for k in range(N):
        for s, (frames, depth) in enumerate(data):
            eng.push(s, frames[k], depth if k == 0 or k % 7 == 0 else None)
        if pacing == "each":
            eng.step()
    eng.flush()
    res, rows, info = eng.poll()
    upd, urows = eng.poll_map_updates()
    out = []
    for s in range(len(data)):
        m, u = res["stream"] == s, upd["stream"] == s
        mp = eng.export_map(s)
        out.append(dict(res=_cols(res[m], ["frame", "status", "n_inliers", "T_cw"]), rows=b"".join(rows[k].tobytes() for k in np.flatnonzero(m)),
                        info=info[m].tobytes(), upd=_cols(upd[u], [n for n in upd.dtype.names if n != "stream"]),
                        urows=b"".join(urows[k].tobytes() for k in np.flatnonzero(u)), K=tuple(mp.rec.K),
                        map=b"".join(np.asarray(v).tobytes() for v in mp.a.values()), status=res["status"][m].copy()))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
@pytest.mark.parametrize("window", [1, 4, 8])
@pytest.mark.parametrize("pacing", ["each", "flush"])
def test_raw_streams_match_resampled_streams(streams, ref_mode, window, pacing):
    from ygz_slam_b200 import vo_native
    opts = dict(window=window, ref_mode=ref_mode, observations=True, information=True, map_updates=True, **POLICY)
    raws = [s[2] for s in streams]
    ctx = _ctx()
    try:
        with vo_native.Engine(ctx, 4, **_engine_kw(raws), **opts) as eng:
            assert [eng.frame_format(s) for s in range(4)] == [(r[0], r[1], r[4]) for r in raws]
            got = _run(eng, [(s[0], s[1]) for s in streams], pacing)
        for s, (frames, depth, raw) in enumerate(streams):
            with vo_native.Engine(ctx, 1, cameras=[CAM], **opts) as ref:
                want = _run(ref, [(_resample(frames, raw), depth)], pacing)[0]
            for key in ("res", "rows", "info", "upd", "urows", "K", "map"):
                assert got[s][key] == want[key], (s, key)
            assert (got[s]["status"] != 2).all(), s
    finally:
        ctx.close()


@pytest.mark.gpu
def test_format_change_across_a_restart(streams):
    """One stream: HD BGR with a lens, restart, 320 x 240 grey with another lens, restart, the default format without a
    lens -- pushed with no step or flush in between, so the old frames are still queued when the format changes.  Every
    sequence equals a fresh default-format engine pushed its frames resampled."""
    from ygz_slam_b200 import vo_native
    n = 12
    plain, pd, _ = _raw_seq(3, (W, H, None, None, 1), n)
    seqs = [(streams[1][0][:n], streams[1][1], RAW_SCALE), (streams[2][0][:n], streams[2][1], RAW_UP), (plain, pd[0], (W, H, None, None, 1))]
    ctx = _ctx()
    try:
        with vo_native.Engine(ctx, 1, window=4, cameras=[CAM], **POLICY) as eng:
            for q, (frames, depth, raw) in enumerate(seqs):
                if q:
                    eng.restart(0)
                eng.set_frame_format(0, raw[0], raw[1], raw[4])
                eng.set_lens(0, *(() if raw[2] is None else (raw[2], raw[3])))
                for k, f in enumerate(frames):
                    eng.push(0, f, depth if k == 0 else None)
            assert eng.frame_format(0) == (W, H, 1)
            eng.flush()
            got = eng.poll()
        wants = []
        for frames, depth, raw in seqs:
            with vo_native.Engine(ctx, 1, window=4, cameras=[CAM], **POLICY) as ref:
                for k, f in enumerate(_resample(frames, raw)):
                    ref.push(0, f, depth if k == 0 else None)
                ref.flush()
                wants.append(ref.poll())
    finally:
        ctx.close()
    cols = ["status", "n_inliers", "T_cw"]
    k0 = 0
    for q, want in enumerate(wants):
        assert _cols(got[k0:k0 + len(want)], cols) == _cols(want, cols), q
        k0 += len(want)
    assert k0 == len(got)


def _load(eng, s, rec):
    return eng.lib.ygz_vo_load_stream(eng.h, s, np.frombuffer(rec, np.uint8).ctypes.data, len(rec))


@pytest.mark.gpu
@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
def test_stream_records_carry_the_format(streams, ref_mode):
    """A formatted stream's record is version 3 with the format block (and the lens block when it has a lens), round-trips
    byte for byte and continues bit for bit in a stream of the same format; streams of another format, and version 1 and
    2 records into a formatted stream, are refused with the stream untouched."""
    from ygz_slam_b200 import vo_native
    frames, depth, raw = streams[1]            # HD BGR with a lens
    fb, db, rawb = streams[3]                  # 640 x 480 BGR without a lens
    fp, dp, _ = _raw_seq(2, (W, H, None, None, 1))
    lens = (raw[2], raw[3])
    lens3 = (CAM, synth.LENS_TUM_FR2)
    opts = dict(window=4, ref_mode=ref_mode, **POLICY)
    half = N // 2
    ctx = _ctx()
    try:
        with vo_native.Engine(ctx, 4, lenses=[lens, None, None, lens3], frame_formats=[raw[:2] + (3,), (W, H, 3), None, None],
                              **opts) as src:
            for k in range(N):
                src.push(0, frames[k], depth if k == 0 else None)
                src.push(1, fb[k], db if k == 0 else None)
                src.push(2, fp[k], dp[0] if k == 0 else None)
                src.push(3, fp[k], dp[0] if k == 0 else None)
                if k == half - 1:
                    src.flush()
                    rec, rec_bgr, rec_v1, rec_v2 = (src.save_stream(s) for s in range(4))
            src.flush()
            res = src.poll()
            want = _cols(res[(res["stream"] == 0) & (res["frame"] >= half)], ["frame", "status", "n_inliers", "T_cw"])
            bound = src.stream_record_bound()
        with vo_native.Engine(ctx, 1, **opts) as other:
            plain_bound = other.stream_record_bound()
        with vo_native.Engine(ctx, 1, frame_formats=[(W, H, 3)], **opts) as other:
            fmt_bound = other.stream_record_bound()
        assert bound == plain_bound + 16 + 72 and fmt_bound == plain_bound + 16
        p = vo_native.parse_stream_record(rec)
        assert p["version"][1] == 3 and p["end"][0] == len(rec) == p["size"][1]
        assert (p["format.width"][1], p["format.height"][1], p["format.channels"][1], p["format.has_lens"][1]) == (1280, 720, 3, 1)
        assert tuple(p["lens.K"][1]) == lens[0] and tuple(p["lens.dist"][1]) == tuple(lens[1])
        assert vo_native.stream_record_next_frame(np.frombuffer(rec, np.uint8)) == half
        q = vo_native.parse_stream_record(rec_bgr)
        assert q["version"][1] == 3 and q["format.has_lens"][1] == 0 and "lens.K" not in q and q["end"][0] == len(rec_bgr)
        assert vo_native.stream_record_next_frame(np.frombuffer(rec_bgr, np.uint8)) == half
        assert vo_native.parse_stream_record(rec_v1)["version"][1] == 1
        assert vo_native.parse_stream_record(rec_v2)["version"][1] == 2
        # refusals: another channel count, no format, another format; version 2 and 1 records into formatted streams of
        # the same lens (or none)
        with vo_native.Engine(ctx, 5, lenses=[lens, lens, None, lens3, None],
                              frame_formats=[(1280, 720, 1), (1280, 720, 3), None, (W, H, 3), (W, H, 3)], **opts) as dst:
            for s, r in ((0, rec), (2, rec), (0, rec_bgr), (3, rec_v2), (4, rec_v1)):
                before = dst.save_stream(s)
                assert _load(dst, s, r) == ERR_INVALID, s
                assert dst.save_stream(s) == before
            dst.load_stream(1, rec)
            assert dst.save_stream(1) == rec           # the round trip is byte for byte
            for k in range(half, N):
                dst.push(1, frames[k], None)
            dst.flush()
            got = dst.poll()
            got = _cols(got[(got["stream"] == 1) & (got["frame"] >= half)], ["frame", "status", "n_inliers", "T_cw"])
        assert got == want
    finally:
        ctx.close()


@pytest.mark.gpu
def test_invalid_frame_formats(streams):
    """Every refusal returns YGZB_ERR_INVALID and changes neither ygz_vo_get_frame_format nor what is queued."""
    from ygz_slam_b200 import vo_native
    frames, depth, raw = streams[0]            # 752 x 480 grey, with a lens
    ctx = _ctx()
    try:
        with vo_native.Engine(ctx, 2, window=4, cameras=[CAM, CAM], **POLICY) as eng:
            lib, h = eng.lib, eng.h
            eng.set_frame_format(0, 752, 480, 1)
            for args in ((0, 0, 480, 1), (0, 752, -1, 1), (0, 32768, 480, 1), (0, 752, 40000, 1), (0, 752, 480, 0), (0, 752, 480, 4),
                         (-1, 752, 480, 1), (2, 752, 480, 1)):
                assert lib.ygz_vo_set_frame_format(h, *args) == ERR_INVALID, args
            assert lib.ygz_vo_set_frame_format(None, 0, 752, 480, 1) == ERR_INVALID
            w = C.c_int(0)
            assert lib.ygz_vo_get_frame_format(h, 0, C.byref(w), None, C.byref(w)) == ERR_INVALID
            assert lib.ygz_vo_get_frame_format(h, 2, C.byref(w), C.byref(w), C.byref(w)) == ERR_INVALID
            assert eng.frame_format(0) == (752, 480, 1) and eng.frame_format(1) == (W, H, 1)
            # another size without a lens: the sequence's first push is refused, nothing queued
            assert lib.ygz_vo_push(h, 0, frames[0].ctypes.data, depth.ctypes.data, 0) == ERR_INVALID
            with pytest.raises(ValueError):
                eng.push(0, frames[0][:, :W], depth)    # the wrong shape for the stream's format
            with pytest.raises(ValueError):
                eng.push(1, np.zeros((H, W, 3), np.uint8), depth)
            eng.set_lens(0, raw[2], raw[3])
            for k in range(10):
                eng.push(0, frames[k], depth if k == 0 else None)
            assert lib.ygz_vo_set_frame_format(h, 0, W, H, 1) == ERR_INVALID   # mid-sequence
            assert eng.frame_format(0) == (752, 480, 1)
            eng.flush()
            got = _cols(eng.poll(), ["frame", "status", "n_inliers", "T_cw"])
        with vo_native.Engine(ctx, 1, window=4, cameras=[CAM], **POLICY) as ref:
            for k, f in enumerate(_resample(frames[:10], raw)):
                ref.push(0, f, depth if k == 0 else None)
            ref.flush()
            want = _cols(ref.poll(), ["frame", "status", "n_inliers", "T_cw"])
    finally:
        ctx.close()
    assert got == want


@pytest.mark.gpu
def test_no_cost_for_default_streams(streams):
    """Streams given the default format explicitly launch exactly what the engine launched before formats existed (the
    launch counts of test_vo_lenses); a BGR stream without a lens adds one conversion per upload."""
    from test_vo_lenses import LAUNCHES_BATCH, LAUNCHES_STREAM, _plain_seq
    from ygz_slam_b200 import vo_native
    fr = [_plain_seq(s, 16) for s in range(2)]
    ctx = _ctx()
    try:
        _, _, _, det = vo_native.run(ctx, [f[0] for f in fr], [f[1] for f in fr], window=4, details=True, **POLICY)
        assert det["gpu_launches"] == LAUNCHES_BATCH

        def streaming(formats, colour):
            c0 = ctx.launch_count
            with vo_native.Engine(ctx, 2, window=1, frame_formats=formats, **POLICY) as eng:
                for k in range(16):
                    for s in range(2):
                        img = colourise(fr[s][0][k]) if s in colour else fr[s][0][k]
                        eng.push(s, img, fr[s][1] if k == 0 else None)
                    eng.step()
                eng.flush()
                ctx.synchronize()
                return ctx.launch_count - c0
        assert streaming(None, ()) == LAUNCHES_STREAM
        assert streaming([(W, H, 1), (W, H, 1)], ()) == LAUNCHES_STREAM
        assert streaming([(W, H, 3), None], (0,)) == LAUNCHES_STREAM + 16
    finally:
        ctx.close()
