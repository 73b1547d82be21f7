"""A lens per stream of the streaming engine (ygz_vo_set_lens, ygzb_tracker_set_undistort, ygzb_tracker_upload_stream): a
stream pushed raw frames of its lens must give, byte for byte, what a stream without a lens gives when it is pushed the
frames tools/undistort_ref.py undistorts in numpy (pinned to cv2 by tests/test_undistort.py) -- results, observation rows,
information records, map updates and the exported map -- across reference modes, windows, pacings and sequence
changes; the tracker's per-stream maps give the oracle's pyramids; stream records carry the lens."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

from ygz_slam_b200 import se3, synth

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import undistort_ref as U  # noqa: E402

pytestmark = pytest.mark.gpu

POLICY = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)
ERR_INVALID = -1
W, H, N = 640, 480, 24
CAM_A = (synth.FX, synth.FY, synth.CX, synth.CY)
CAM_B = (synth.FX, synth.FY, 337.6, 241.2)   # another principal point: newK != the raw K
L_FR2 = (CAM_A, synth.LENS_TUM_FR2)
L_FR1 = (CAM_A, U.TUM_FR1[1])
SAT = U.CASES["saturating"]                  # a polynomial that explodes inside a wide view: most samples saturate
L_SAT, CAM_SAT = (SAT[2], SAT[3]), SAT[4]


def _maps(lens, newK):
    K, dist = lens
    return U.undistort_map(W, H, K, dist, newK)


def _und(frames, lens, newK):
    xy, a = _maps(lens, newK)
    return [U.undistort_image(f, xy, a) for f in frames]


def _lens_seq(stream, dist, n=N, step=1):
    fr = [synth.lens_stream_frame(step * k, stream=stream, dist=dist) for k in range(n)]
    return [f[0] for f in fr], fr[0][1], [f[2] for f in fr]


def _plain_seq(stream, n=N, step=1):
    fr = [synth.stream_frame(step * k, stream=stream) for k in range(n)]
    return [f[0] for f in fr], fr[0][1], [f[2] for f in fr]


@pytest.fixture(scope="module")
def streams():
    """(raw frames, depth, lens or None, camera) of four streams: TUM fr2's lens, TUM fr1's coefficients seen through
    camera B, the saturating lens, and a stream without a lens."""
    f0, d0, _ = _lens_seq(0, synth.LENS_TUM_FR2)
    f1, d1, _ = _lens_seq(1, U.TUM_FR1[1])
    f2, d2, _ = _plain_seq(2)
    f3, d3, _ = _plain_seq(3)
    return [(f0, d0, L_FR2, CAM_A), (f1, d1, L_FR1, CAM_B), (f2, d2, L_SAT, CAM_SAT), (f3, d3, None, CAM_A)]


def _ctx():
    from ygz_slam_b200 import Context
    return Context(0, image_width=W, image_height=H)


def _cols(a, names):
    return b"".join(np.ascontiguousarray(a[n]).tobytes() for n in names)


def _feed(eng, data, pacing):
    """data[s] = (frames, depth) of engine stream s; pacing 'each': a step after every lock-step push, 'flush': push
    everything, then flush."""
    for k in range(N):
        for s, (frames, depth) in enumerate(data):
            eng.push(s, frames[k], depth if k == 0 or k % 7 == 0 else None)
        if pacing == "each":
            eng.step()
    eng.flush()


def _run(eng, data, pacing):
    _feed(eng, data, pacing)
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


def test_engine_maps_are_the_restatement(streams):
    """The engine builds its maps with ygzb_undistort_map: for these lenses and cameras they are undistort_ref's."""
    from ygz_slam_b200 import capi
    for _, _, lens, cam in streams[:3]:
        xy, a = capi.undistort_map(W, H, lens[0], lens[1], cam)
        rxy, ra = _maps(lens, cam)
        assert np.array_equal(xy, rxy) and np.array_equal(a, ra)


@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
@pytest.mark.parametrize("window", [1, 4, 8])
@pytest.mark.parametrize("pacing", ["each", "flush"])
def test_lens_streams_match_undistorted_streams(streams, ref_mode, window, pacing):
    from ygz_slam_b200 import vo_native
    opts = dict(window=window, ref_mode=ref_mode, observations=True, information=True, map_updates=True, **POLICY)
    ctx = _ctx()
    try:
        with vo_native.Engine(ctx, 4, cameras=[s[3] for s in streams], lenses=[s[2] for s in streams], **opts) as eng:
            for s, (_, _, lens, cam) in enumerate(streams):
                got_lens = eng.lens(s)
                assert (got_lens is None) if lens is None else (tuple(got_lens[0]) == tuple(lens[0]) and tuple(got_lens[1]) == tuple(lens[1]))
                assert tuple(eng.camera(s)) == cam
            got = _run(eng, [(s[0], s[1]) for s in streams], pacing)
        for s, (frames, depth, lens, cam) in enumerate(streams):
            und = frames if lens is None else _und(frames, lens, cam)
            with vo_native.Engine(ctx, 1, cameras=[cam], **opts) as ref:
                want = _run(ref, [(und, depth)], pacing)[0]
            for key in ("res", "rows", "info", "upd", "urows", "K", "map"):
                assert got[s][key] == want[key], (s, key)
        # the lenses that keep their texture track without loss
        for s in (0, 1, 3):
            assert (got[s]["status"] != 2).all(), s
    finally:
        ctx.close()


def test_lens_tracks_ground_truth():
    """On lens-rendered frames the lens-on stream stays within the loop tests' ground-truth bound; the same raw frames
    tracked without the lens are clearly worse."""
    from test_undistort import LENS_KW, LENS_LOOP_BOUND
    from ygz_slam_b200 import vo_native
    n = 12
    fr = [synth.lens_stream_frame(2 * k, stream=0) for k in range(n)]
    ctx = _ctx()
    try:
        with vo_native.Engine(ctx, 2, window=4, lenses=[L_FR2, None], **LENS_KW) as eng:
            for k, (frame, depth, _) in enumerate(fr):   # every frame brings its depth map, as the loop tests feed it
                for s in range(2):
                    eng.push(s, frame, depth)
            eng.flush()
            res = eng.poll()
    finally:
        ctx.close()
    errs = []
    for s in range(2):
        r = res[res["stream"] == s]
        assert r["frame"].tolist() == list(range(n))
        # the sequence starts at the identity: the error against the ground truth relative to frame 0; a lost frame's is inf
        e = [np.inf if r["status"][k] == 2 else
             float(np.linalg.norm(se3.se3_log(se3.mul(r["T_cw"][k].reshape(3, 4), se3.inv(se3.mul(fr[k][2], se3.inv(fr[0][2])))))))
             for k in range(n)]
        errs.append(max(e))
    print(f"ground-truth error over {n} frames: {errs[0]:.3e} with the lens, {errs[1]:.3e} without")
    assert errs[0] < LENS_LOOP_BOUND
    assert errs[1] > 2 * errs[0]


def _segments(seqs, window=4):
    """One stream fed sequence after sequence (frames, depth, lens, camera) with a restart and set_camera / set_lens
    between them and no flush or step anywhere: the old sequence's frames are all still queued when the lens changes."""
    from ygz_slam_b200 import vo_native
    ctx = _ctx()
    try:
        with vo_native.Engine(ctx, 1, window=window, **POLICY) as eng:
            for q, (frames, depth, lens, cam) in enumerate(seqs):
                if q:
                    eng.restart(0)
                eng.set_camera(0, cam)
                eng.set_lens(0, *(lens or ()))
                for k, f in enumerate(frames):
                    eng.push(0, f, depth if k == 0 else None)
            eng.flush()
            got = eng.poll()
        wants = []
        for frames, depth, lens, cam in seqs:
            with vo_native.Engine(ctx, 1, window=window, cameras=[cam], **POLICY) as ref:
                for k, f in enumerate(frames if lens is None else _und(frames, lens, cam)):
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


def test_sequence_barrier(streams):
    """A with lens L1, restart, camera B and L2, then B; then L2 -> no lens and no lens -> L2: every sequence equals a
    fresh engine of its own lens and camera."""
    n = 12
    fa, da = streams[0][0][:n], streams[0][1]
    fb, db = streams[1][0][:n], streams[1][1]
    fc, dc = streams[3][0][:n], streams[3][1]
    _segments([(fa, da, L_FR2, CAM_A), (fb, db, L_FR1, CAM_B), (fc, dc, None, CAM_A), (fb, db, L_FR1, CAM_B)])


def test_tracker_streams_with_their_maps(oracle):
    """ygzb_tracker_upload_stream: two streams with different maps and one without, in one go and with the maps changed
    between uploads of the same stream, give every pyramid level of the oracle on undistort_ref's remap; a pool with maps
    and a stream with maps are refused together."""
    import torch
    from ygz_slam_b200 import capi
    ctx = _ctx()
    fr = ctx.frames(10)
    L = len(fr.lw)
    tr = capi.Tracker(fr, 3, 8, CAM_A)
    lib = fr.lib
    raw = [U.seeded_image(300 + k, H, W) for k in range(9)]
    m0, m1 = _maps(L_FR2, CAM_A), _maps(L_FR1, CAM_B)
    tr.set_undistort(0, *m0)
    tr.set_undistort(1, *m1)
    tr.upload_stream(0, 0, np.stack(raw[0:2]))
    tr.upload_stream(1, 2, np.stack(raw[2:4]))
    tr.upload_stream(2, 4, np.stack(raw[4:6]))   # no maps: the plain upload
    tr.set_undistort(0, *m1)                    # in order behind the uploads enqueued before
    tr.upload_stream(0, 6, raw[6])
    tr.set_undistort(0)
    tr.upload_stream(0, 7, raw[7])
    torch.cuda.synchronize()
    want = {0: m0, 1: m0, 2: m1, 3: m1, 4: None, 5: None, 6: m1, 7: None}
    for slot, maps in want.items():
        img = raw[slot] if maps is None else U.undistort_image(raw[slot], *maps)
        pyr = oracle.build_pyramid(img, L)
        for lv in range(L):
            assert np.array_equal(fr.download_level(slot, lv), oracle.level_view(pyr, W, H, L, lv)), (slot, lv)
    # refusals: only one map, an out-of-range fraction, a stream out of range; a pool with maps
    xy, a = m0
    bad = a.copy()
    bad[5, 7] = 1024
    assert lib.ygzb_tracker_set_undistort(tr.h, 0, xy.ctypes.data, None) == ERR_INVALID
    assert lib.ygzb_tracker_set_undistort(tr.h, 0, xy.ctypes.data, bad.ctypes.data) == ERR_INVALID
    assert lib.ygzb_tracker_set_undistort(tr.h, 3, xy.ctypes.data, a.ctypes.data) == ERR_INVALID
    assert lib.ygzb_tracker_set_undistort(None, 0, xy.ctypes.data, a.ctypes.data) == ERR_INVALID
    assert lib.ygzb_tracker_upload_stream(tr.h, -1, 0, 1, raw[0].ctypes.data, W * H) == ERR_INVALID
    fr.set_undistort(*m0)
    assert lib.ygzb_tracker_upload_stream(tr.h, 1, 8, 1, raw[8].ctypes.data, W * H) == ERR_INVALID   # stream 1 has maps
    assert lib.ygzb_tracker_set_undistort(tr.h, 2, xy.ctypes.data, a.ctypes.data) == ERR_INVALID
    tr.upload_stream(2, 8, raw[8])   # a stream without maps: the pool's maps, as ygzb_tracker_upload
    torch.cuda.synchronize()
    pyr = oracle.build_pyramid(U.undistort_image(raw[8], *m0), L)
    for lv in range(L):
        assert np.array_equal(fr.download_level(8, lv), oracle.level_view(pyr, W, H, L, lv)), lv
    tr.close()
    fr.close()
    ctx.close()


@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
def test_stream_records_carry_the_lens(streams, ref_mode):
    """A lens stream's record is version 2 with the lens block and continues bit for bit in a stream with the same lens;
    streams with another lens or none refuse it and stay as they were; a lens-free stream's record is version 1 of
    today's size."""
    from ygz_slam_b200 import vo_native
    frames, depth, _, _ = streams[0]
    fc, dc = streams[3][0], streams[3][1]
    opts = dict(window=4, ref_mode=ref_mode, **POLICY)
    half = N // 2
    ctx = _ctx()
    try:
        with vo_native.Engine(ctx, 2, lenses=[None, L_FR2], **opts) as src:
            for k in range(N):
                src.push(1, frames[k], depth if k == 0 else None)
                src.push(0, fc[k], dc if k == 0 else None)
                if k == half - 1:
                    src.flush()
                    rec = src.save_stream(1)
                    plain = src.save_stream(0)
            src.flush()
            want = src.poll()
            want = _cols(want[(want["stream"] == 1) & (want["frame"] >= half)], ["frame", "status", "n_inliers", "T_cw"])
            bound = src.stream_record_bound()
        with vo_native.Engine(ctx, 1, **opts) as other:
            plain_bound = other.stream_record_bound()
        assert bound == plain_bound + 72
        p = vo_native.parse_stream_record(rec)
        assert p["version"][1] == 2 and p["end"][0] == len(rec)
        assert tuple(p["lens.K"][1]) == L_FR2[0] and tuple(p["lens.dist"][1]) == tuple(L_FR2[1])
        assert vo_native.stream_record_next_frame(np.frombuffer(rec, np.uint8)) == half
        # the lens-free record: version 1, its sections ending exactly at its size
        q = vo_native.parse_stream_record(plain)
        assert q["version"][1] == 1 and "lens.K" not in q and q["end"][0] == len(plain) == q["size"][1]
        with vo_native.Engine(ctx, 3, lenses=[None, L_FR1, L_FR2], **opts) as dst:
            for s in (0, 1):
                before = dst.save_stream(s)
                assert dst.lib.ygz_vo_load_stream(dst.h, s, np.frombuffer(rec, np.uint8).ctypes.data, len(rec)) == ERR_INVALID, s
                assert dst.save_stream(s) == before
            before = dst.save_stream(2)
            assert dst.lib.ygz_vo_load_stream(dst.h, 2, np.frombuffer(plain, np.uint8).ctypes.data, len(plain)) == ERR_INVALID
            assert dst.save_stream(2) == before
            dst.load_stream(2, rec)
            for k in range(half, N):
                dst.push(2, frames[k], None)
            dst.flush()
            got = dst.poll()
            got = _cols(got[(got["stream"] == 2) & (got["frame"] >= half)], ["frame", "status", "n_inliers", "T_cw"])
        assert got == want
        # hand-over into a stream that has tracked without a lens: flush, restart, set camera, set lens, load
        with vo_native.Engine(ctx, 1, **opts) as dst:
            for k in range(6):
                dst.push(0, fc[k], dc if k == 0 else None)
            dst.flush()
            dst.restart(0)
            dst.set_camera(0, CAM_A)
            dst.set_lens(0, *L_FR2)
            dst.load_stream(0, rec)
            for k in range(half, N):
                dst.push(0, frames[k], None)
            dst.flush()
            got = dst.poll()
            got = _cols(got[got["frame"] >= half], ["frame", "status", "n_inliers", "T_cw"])
        assert got == want
    finally:
        ctx.close()


def test_invalid_lenses(streams):
    """Every refusal returns YGZB_ERR_INVALID and changes neither ygz_vo_get_lens nor the results."""
    from ygz_slam_b200 import vo_native
    frames, depth, _, _ = streams[0]
    K, dist = np.array(L_FR2[0], np.float64), np.array(L_FR2[1], np.float64)
    ctx = _ctx()
    try:
        with vo_native.Engine(ctx, 2, window=4, **POLICY) as eng:
            lib, h = eng.lib, eng.h
            eng.set_lens(0, *L_FR2)
            assert lib.ygz_vo_set_lens(None, 0, K.ctypes.data, dist.ctypes.data) == ERR_INVALID
            assert lib.ygz_vo_set_lens(h, 0, K.ctypes.data, None) == ERR_INVALID
            assert lib.ygz_vo_set_lens(h, 0, None, dist.ctypes.data) == ERR_INVALID
            for s in (-1, 2):
                assert lib.ygz_vo_set_lens(h, s, K.ctypes.data, dist.ctypes.data) == ERR_INVALID
            for arr, k, v in ((K, 0, np.nan), (K, 2, np.inf), (dist, 4, np.nan), (dist, 1, -np.inf), (K, 0, 0.0), (K, 1, -1.0)):
                bad_K, bad_d = K.copy(), dist.copy()
                (bad_K if arr is K else bad_d)[k] = v
                assert lib.ygz_vo_set_lens(h, 0, bad_K.ctypes.data, bad_d.ctypes.data) == ERR_INVALID
            has = C.c_int(0)
            assert lib.ygz_vo_get_lens(h, 0, None, K.ctypes.data, dist.ctypes.data) == ERR_INVALID
            assert lib.ygz_vo_get_lens(h, 2, C.byref(has), K.ctypes.data, dist.ctypes.data) == ERR_INVALID
            got_K, got_d = eng.lens(0)
            assert tuple(got_K) == L_FR2[0] and tuple(got_d) == tuple(L_FR2[1]) and eng.lens(1) is None
            for k in range(10):
                eng.push(0, frames[k], depth if k == 0 else None)
            assert lib.ygz_vo_set_lens(h, 0, None, None) == ERR_INVALID   # mid-sequence
            assert lib.ygz_vo_set_lens(h, 0, K.ctypes.data, dist.ctypes.data) == ERR_INVALID
            got_K, got_d = eng.lens(0)
            assert tuple(got_K) == L_FR2[0] and tuple(got_d) == tuple(L_FR2[1])
            eng.flush()
            got = _cols(eng.poll(), ["status", "n_inliers", "T_cw"])
        with vo_native.Engine(ctx, 1, window=4, **POLICY) as ref:
            for k, f in enumerate(_und(frames[:10], L_FR2, CAM_A)):
                ref.push(0, f, depth if k == 0 else None)
            ref.flush()
            want = _cols(ref.poll(), ["status", "n_inliers", "T_cw"])
    finally:
        ctx.close()
    assert got == want


# kernel launches of the two runs of _launches, as the engine made them before lenses existed (measured on an H100 with the
# parent build); a run without a lens must launch exactly these
LAUNCHES_BATCH, LAUNCHES_STREAM = 107, 203


def _launches(lenses=None):
    """Launches of a ygz_vo_run of 2 streams x 16 frames at window 4, and of a streaming run of the same frames (window 1,
    a step per lock-step push) with the given lenses."""
    from ygz_slam_b200 import vo_native
    fr = [_plain_seq(s, 16) for s in range(2)]
    ctx = _ctx()
    try:
        _, _, _, det = vo_native.run(ctx, [f[0] for f in fr], [f[1] for f in fr], window=4, details=True, **POLICY)
        c0 = ctx.launch_count
        with vo_native.Engine(ctx, 2, window=1, lenses=lenses, **POLICY) as eng:
            for k in range(16):
                for s in range(2):
                    eng.push(s, fr[s][0][k], fr[s][1] if k == 0 else None)
                eng.step()
            eng.flush()
            ctx.synchronize()
        return det["gpu_launches"], ctx.launch_count - c0
    finally:
        ctx.close()


def test_no_cost_without_a_lens():
    """Without a lens the engine launches what it launched before lenses existed; with a lens on one stream, one remap per
    upload of that stream (one upload per frame at window 1) and nothing else."""
    batch, stream = _launches()
    print(f"launches: ygz_vo_run {batch}, streaming {stream}")
    assert (batch, stream) == (LAUNCHES_BATCH, LAUNCHES_STREAM)
    _, with_lens = _launches([L_FR2, None])
    assert with_lens == stream + 16
