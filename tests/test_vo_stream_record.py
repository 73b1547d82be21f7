"""Stream records of the streaming engine (ygz_vo_save_stream / ygz_vo_load_stream, vo_native.Engine.save_stream /
load_stream): a live stream saved as bytes and loaded into another stream of another engine -- other n_streams, other
window, another context or device -- continues exactly as the saved one would have: the same results bit for bit, the same
16 counters and the same local map.  The sequences give their key-frames different depth maps and push most frames
without one, so the depth map a stream carries decides the map points of later key-frames."""
import ctypes as C

import numpy as np
import pytest

from ygz_slam_b200 import synth

POLICY = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)   # test_vo_stream's key-frame policy
N_FRAMES = 30
ERR_INVALID, ERR_CAPACITY = -1, -4
TRACKED, KEYFRAME, LOST = 0, 1, 2
SRC, DST = 1, 0   # the saved stream of engine A, the stream of engine B that continues it


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_header_declares_stream_records():
    from test_abi import declared_symbols
    from test_vo_stream import declared_stream_symbols
    from ygz_slam_b200 import capi
    assert {"ygz_vo_stream_record_bound", "ygz_vo_save_stream", "ygz_vo_load_stream"} <= set(declared_stream_symbols())
    assert "ygzb_tracker_get_depth" in declared_symbols() and "ygzb_tracker_get_depth" in capi.EXPORTS


def test_parser_rejects_a_short_record():
    from ygz_slam_b200 import vo_native
    with pytest.raises(ValueError):
        vo_native.parse_stream_record(b"YGZS" + bytes(20))


# ---- GPU --------------------------------------------------------------------------------------------------------------
MODES = pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
WINDOWS = pytest.mark.parametrize("window", [1, 8])


@pytest.fixture(scope="module")
def shift_data():
    return [synth.shift_stream(s_, N_FRAMES) for s_ in range(4)]


class Seq:
    """Frames of one stream with the ygz_vo_restart calls before some of them (frame -> T_cw).  Frame k brings the depth
    map base * (1 + 1e-3 k) when k is a multiple of 3, starts a sequence, or is the first; every other frame brings none."""

    def __init__(self, frames, base, gts, restarts=None):
        self.frames, self.base, self.gts, self.restarts = frames, base, gts, dict(restarts or {})

    def has_depth(self, k):
        return k % 3 == 0 or k in self.restarts

    def depth_map(self, k):
        return self.base * (1 + 1e-3 * k)

    def depth(self, k):
        return self.depth_map(k) if self.has_depth(k) else None


def feed(eng, stream, seq, lo, hi, restart_at_lo=True):
    """Frames [lo, hi) of seq into `stream` (tag 100 + frame), each behind its restart; the one of frame lo only with
    restart_at_lo (a restart issued before a save travels in the record)."""
    for k in range(lo, hi):
        if k in seq.restarts and (k > lo or restart_at_lo):
            eng.restart(stream, seq.restarts[k])
        assert eng.push(stream, seq.frames[k], seq.depth(k), tag=100 + k) == k


def neighbour(eng, stream, data, lo, hi):
    """Frames [lo, hi) of a shift stream, every one with its depth map, into another stream of the engine."""
    for k in range(lo, hi):
        eng.push(stream, data[0][k], data[1], tag=5000 + k)


def of(res, stream):
    r = res[res["stream"] == stream]
    assert r["frame"].tolist() == sorted(r["frame"].tolist())
    return r


def same_results(got, want):
    for key in ("frame", "tag", "status", "n_inliers"):
        assert np.array_equal(got[key], want[key]), key
    assert np.array_equal(got["T_cw"].view(np.uint64), want["T_cw"].view(np.uint64))   # bit for bit


def same_map(got, want):
    from ygz_slam_b200 import capi
    assert got.header == want.header
    for key in capi._MAP_ARRAYS:
        assert np.array_equal(got.a[key], want.a[key]), key


def save(eng, stream):
    """The stream's record, checked against the layout of include/ygz_vo.h and the engine's bound."""
    from ygz_slam_b200 import vo_native
    rec = eng.save_stream(stream)
    f = vo_native.parse_stream_record(rec)
    assert f["end"][0] == len(rec) == f["size"][1] and bytes(f["magic"][1]) == b"YGZS"
    assert vo_native.stream_record_next_frame(np.frombuffer(rec, np.uint8)) == f["next_frame"][1]
    assert len(rec) <= eng.stream_record_bound()
    return rec


def engine(ctx, n_streams, window, ref_mode, **kw):
    from ygz_slam_b200 import vo_native
    return vo_native.Engine(ctx, n_streams, window=window, ref_mode=ref_mode, **POLICY, **kw)


_REF = {}


def reference(ctx, shift_data, seq, key, window, ref_mode):
    """One uninterrupted run of seq on stream SRC of a 2-stream engine (stream 0: shift stream 2): SRC's results, its 16
    counters and its final map."""
    k = (key, window, ref_mode)
    if k not in _REF:
        with engine(ctx, 2, window, ref_mode) as eng:
            neighbour(eng, 0, shift_data[2], 0, N_FRAMES)
            feed(eng, SRC, seq, 0, N_FRAMES)
            eng.flush()
            _REF[k] = (of(eng.poll(), SRC), eng._stat_row(SRC), eng.export_map(SRC))
    return _REF[k]


def scenario(shift_data, name, window, ref_mode, ctx):
    """(seq, cut): the stream is saved once frames [0, cut) have their results."""
    frames, base, gts = shift_data[0]
    if name == "lost":   # frame 8 of another texture loses the stream; a restart at frame 16 resumes it
        frames = frames.copy()
        frames[8] = shift_data[1][0][8]
        return Seq(frames, base, gts, {16: gts[16]}), 11
    if name == "restart_pending":   # the restart is issued after the flush, before the save
        return Seq(frames, base, gts, {14: gts[14]}), 14
    if name == "after_restart":
        return Seq(frames, base, gts, {10: gts[10]}), 17
    seq = Seq(frames, base, gts)
    if name == "first_keyframe":
        return seq, 1
    status = reference(ctx, shift_data, seq, "plain", window, ref_mode)[0]["status"]
    kfs = np.flatnonzero(status == KEYFRAME)
    assert len(kfs) >= 4 and (status != LOST).all()
    if name == "after_keyframe":
        return seq, int(kfs[2]) + 1
    assert name == "between"
    cut = next(c for c in range(kfs[1] + 3, N_FRAMES) if status[c - 1] == TRACKED and status[c - 2] == TRACKED)
    return seq, cut


SCENARIOS = ["first_keyframe", "between", "after_keyframe", "lost", "restart_pending", "after_restart"]


def split_run(ctx_b, shift_data, seq, cut, window, ref_mode, ctx_a, through=None):
    """Engine A runs seq to `cut` on stream SRC (its stream 0 has two frames still queued at the save), saves SRC and goes
    on; engine B (3 streams, the other window) loads the record into stream DST (through(rec): the bytes B gets) and
    runs the rest beside shift stream 3 on its stream 2.  Returns the record, A's and B's results of the stream, their
    counters and their final maps."""
    with engine(ctx_a, 2, window, ref_mode) as A, engine(ctx_b, 3, 9 - window, ref_mode) as B:
        neighbour(A, 0, shift_data[2], 0, cut)
        feed(A, SRC, seq, 0, cut)
        A.flush()
        neighbour(A, 0, shift_data[2], cut, cut + 2)
        if cut in seq.restarts:
            A.restart(SRC, seq.restarts[cut])
        rec = save(A, SRC)
        neighbour(B, 2, shift_data[3], 0, 4)
        B.load_stream(DST, rec if through is None else through(rec))
        assert save(B, DST) == rec   # round trip
        neighbour(B, 2, shift_data[3], 4, N_FRAMES)
        feed(B, DST, seq, cut, N_FRAMES, restart_at_lo=False)
        feed(A, SRC, seq, cut, N_FRAMES, restart_at_lo=False)   # the source goes on: a fork
        neighbour(A, 0, shift_data[2], cut + 2, N_FRAMES)
        A.flush()
        B.flush()
        ra, rb = of(A.poll(), SRC), of(B.poll(), DST)
        return rec, ra, rb, (A._stat_row(SRC), B._stat_row(DST)), (A.export_map(SRC), B.export_map(DST))


@pytest.mark.gpu
@MODES
@WINDOWS
@pytest.mark.parametrize("name", SCENARIOS)
def test_continuation_is_bit_identical(ctx3, shift_data, name, window, ref_mode):
    """The saved stream continued in another engine gives the results, counters and map of the uninterrupted run, and so
    does the source, which goes on tracking after the save (two identical forks)."""
    seq, cut = scenario(shift_data, name, window, ref_mode, ctx3)
    want, want_stats, want_map = reference(ctx3, shift_data, seq, name if seq.restarts or name == "lost" else "plain", window, ref_mode)
    if name == "lost":
        assert (want["status"][8:16] == LOST).all() and (want["status"][16:] != LOST).all() and want["status"][16] == KEYFRAME
    elif name in ("restart_pending", "after_restart"):
        r = min(seq.restarts)
        assert want["status"][r] == KEYFRAME and (want["status"] != LOST).all()
    rec, ra, rb, stats, maps = split_run(ctx3, shift_data, seq, cut, window, ref_mode, ctx3)
    assert rb["frame"].tolist() == list(range(cut, N_FRAMES))
    same_results(np.concatenate([ra[ra["frame"] < cut], rb]), want)
    same_results(ra, want)
    for s_, m in zip(stats, maps):
        assert np.array_equal(s_, want_stats)
        same_map(m, want_map)


@pytest.mark.gpu
@MODES
def test_depth_map_travels(ctx3, shift_data, ref_mode):
    """Cut right before a key-frame whose frame brings no depth map: the record carries the map of the last key-frame that
    brought one, and the continuation's map equals the uninterrupted one's.  A control record whose depth map is scaled
    gives that key-frame other depths: test_continuation_is_bit_identical would see a missing depth map."""
    from ygz_slam_b200 import vo_native
    frames, base, gts = shift_data[0]
    seq = Seq(frames, base, gts)
    want, _, want_map = reference(ctx3, shift_data, seq, "plain", 8, ref_mode)
    kfs = np.flatnonzero(want["status"] == KEYFRAME)
    f = next(int(k) for k in kfs[1:] if not seq.has_depth(k))
    carried = max(int(k) for k in kfs if k < f and seq.has_depth(k))
    rec, _, _, _, maps = split_run(ctx3, shift_data, seq, f, 8, ref_mode, ctx3)
    fields = vo_native.parse_stream_record(rec)
    assert np.array_equal(fields["depth_map"][1], seq.depth_map(carried).reshape(-1))
    same_map(maps[1], want_map)

    off = fields["depth_map"][0]
    control = bytearray(rec)
    control[off:] = (np.frombuffer(rec, np.float64, offset=off) * 1.01).tobytes()

    def newest_keyframe(data):   # frame f alone after the load: it becomes a key-frame
        with engine(ctx3, 3, 8, ref_mode) as B:
            B.load_stream(DST, data)
            feed(B, DST, seq, f, f + 1)
            B.flush()
            assert B.poll()["status"].tolist() == [KEYFRAME]
            return B.export_map(DST).keyframes()[-1]
    kf, kf_control = newest_keyframe(rec), newest_keyframe(bytes(control))
    px = kf["px"].astype(np.int64)
    assert kf["depth"].size > 500 and np.array_equal(kf["depth"], seq.depth_map(carried)[px[:, 1], px[:, 0]])
    assert not np.array_equal(kf_control["depth"], kf["depth"])


@pytest.mark.gpu
@MODES
def test_never_pushed_stream_round_trips(ctx3, shift_data, ref_mode):
    """A stream that was never pushed, with and without a start pose, round-trips byte for byte and then tracks as the
    stream it was saved from."""
    T0 = np.concatenate([synth.so3_exp(np.array([0.1, -0.25, 0.15])), np.array([[0.6], [-0.5], [0.7]])], 1)
    seq = Seq(*shift_data[1])
    for start in (None, T0):
        with engine(ctx3, 2, 8, ref_mode) as A, engine(ctx3, 3, 1, ref_mode) as B:
            if start is not None:
                A.restart(SRC, start)
            rec = save(A, SRC)
            B.load_stream(2, rec)
            assert save(B, 2) == rec
            feed(A, SRC, seq, 0, N_FRAMES)
            feed(B, 2, seq, 0, N_FRAMES)
            A.flush()
            B.flush()
            ra, rb = of(A.poll(), SRC), of(B.poll(), 2)
            same_results(rb, ra)
            assert np.array_equal(A._stat_row(SRC), B._stat_row(2))
            assert ra["status"][0] == KEYFRAME and (ra["status"] != LOST).all()
            if start is not None:
                assert np.array_equal(ra["T_cw"][0].reshape(3, 4), T0)


@pytest.mark.gpu
def test_get_depth_and_record_bound(ctx3):
    """ygzb_tracker_get_depth reads back what ygzb_tracker_set_depth wrote and rejects bad arguments; the record bound is
    the documented layout with a full ring, a full reference and a depth map."""
    fr = ctx3.frames(4)
    tr = fr.tracker(2, 4, (synth.FX, synth.FY, synth.CX, synth.CY))
    lib = tr.lib
    d = np.random.default_rng(3).uniform(1.5, 3.0, (480, 640))
    tr.set_depth(1, d)
    assert np.array_equal(tr.get_depth(1), d)
    out = np.zeros((480, 640))
    assert lib.ygzb_tracker_get_depth(None, 0, out.ctypes.data) == ERR_INVALID
    assert lib.ygzb_tracker_get_depth(tr.h, 0, None) == ERR_INVALID
    for stream in (-1, 2):
        assert lib.ygzb_tracker_get_depth(tr.h, stream, out.ctypes.data) == ERR_INVALID
    tr.close()
    fr.close()
    R, cells, WH = 4, ctx3.n_cells, 640 * 480
    want = (68 + 4 + R * 116 + 2 * 96 + 4 + 16 + 12 * 8 + 4 + R * (116 + WH) + R * cells * 49 + R * 4 * cells * 24 + 4 + 96
            + 5 * cells * 24 + WH + 8 * WH)
    for mode in ("keyframe", "previous"):
        with engine(ctx3, 1, 8, mode) as eng:
            assert eng.stream_record_bound() == want


def _device_count():
    import torch
    return torch.cuda.device_count()


@pytest.mark.gpu
@MODES
def test_across_contexts_through_a_file(ctx3, shift_data, ref_mode, tmp_path):
    """The record goes through a file and into an engine on a second context of the same device."""
    from ygz_slam_b200 import Context
    seq, cut = scenario(shift_data, "between", 8, ref_mode, ctx3)
    want, want_stats, want_map = reference(ctx3, shift_data, seq, "plain", 8, ref_mode)
    path = tmp_path / "stream.rec"

    def through_file(rec):
        path.write_bytes(rec)
        return path.read_bytes()
    ctx = Context(0)
    try:
        _, ra, rb, stats, maps = split_run(ctx, shift_data, seq, cut, 8, ref_mode, ctx3, through=through_file)
    finally:
        ctx.close()
    same_results(np.concatenate([ra[ra["frame"] < cut], rb]), want)
    assert np.array_equal(stats[1], want_stats)
    same_map(maps[1], want_map)


@pytest.mark.gpu
def test_across_devices(ctx3, shift_data):
    """With a second device visible, the record moves to it (previous-frame mode)."""
    if _device_count() < 2:
        pytest.skip("one device visible")
    from ygz_slam_b200 import Context
    seq, cut = scenario(shift_data, "after_keyframe", 8, "previous", ctx3)
    want, want_stats, want_map = reference(ctx3, shift_data, seq, "plain", 8, "previous")
    ctx = Context(1)
    try:
        _, ra, rb, stats, maps = split_run(ctx, shift_data, seq, cut, 8, "previous", ctx3)
    finally:
        ctx.close()
    same_results(np.concatenate([ra[ra["frame"] < cut], rb]), want)
    assert np.array_equal(stats[1], want_stats)
    same_map(maps[1], want_map)


def _mutator(rec):
    """(fields of rec, mutated(*(field, value, dtype)) -> a copy of rec with those fields overwritten)."""
    from ygz_slam_b200 import vo_native
    f = vo_native.parse_stream_record(rec)

    def mutated(*changes):
        b = bytearray(rec)
        for name, value, dtype in changes:
            b[f[name][0]:f[name][0] + np.dtype(dtype).itemsize * np.size(value)] = np.array(value, dtype).tobytes()
        return bytes(b)
    return f, mutated


def _mutations(rec, blank, cells, n_levels):
    """Records that must be rejected, by name: `rec` (a stream with a full ring) or `blank` (a stream never pushed) with one
    thing wrong.  Where the layout allows it, a record keeps its size and every row offset, so that only the check it is
    named after can reject it."""
    f, mutated = _mutator(rec)
    n_kf = int(f["n_kf"][1])
    assert n_kf == 4
    n = [int(f[f"kf[{k}].n"][1]) for k in range(n_kf)]
    last = int(f[f"kf[{n_kf - 1}].frame_id"][1])
    # one key-frame with cells + 1 features; the others give up as many rows, so the rows keep their total and offsets
    target = int(np.argmax(n[:-1]))
    changes, left = [(f"kf[{target}].n", cells + 1, "<i4"), (f"map[{target}].n_features", cells + 1, "<i4")], cells + 1 - n[target]
    for k in sorted(set(range(n_kf)) - {target}, key=lambda k: k == n_kf - 1):   # the newest key-frame last
        give = min(left, n[k])
        changes += [(f"kf[{k}].n", n[k] - give, "<i4"), (f"map[{k}].n_features", n[k] - give, "<i4")]
        left -= give
    assert left == 0
    K = f["K"][1].copy()
    K[0] = np.nextafter(K[0], np.inf)   # one ulp off
    out = dict(magic=mutated(("magic", [ord("X"), ord("G"), ord("Z"), ord("S")], "u1")), version=mutated(("version", 2, "<u4")),
               size=mutated(("size", len(rec) + 1, "<u8")), truncated=rec[:-1], truncated_header=rec[:40], oversized=rec + b"\0",
               width=mutated(("width", f["width"][1] + 1, "<i4")), height=mutated(("height", f["height"][1] - 1, "<i4")),
               cells=mutated(("cells", cells + 1, "<i4")), levels=mutated(("n_levels", n_levels + 1, "<i4")), K_ulp=mutated(("K", K, "<f8")),
               ref_mode=mutated(("ref_mode", 1 - f["ref_mode"][1], "<i4")),
               n_keyframes=mutated(("n_kf", 5, "<i4"), ("n_keyframes", 5, "<i4")),
               duplicate_entry=mutated(("kf[1].entry", f["kf[0].entry"][1], "<i4"), ("map[1].entry", f["map[0].entry"][1], "<i4")),
               n_features=mutated(*changes),
               level=mutated(("level", np.r_[n_levels, f["level"][1][1:]], "u1")),
               flag=mutated(("lost", 2, "u1")),
               # host states no saved stream has
               next_frame_zero=mutated(("next_frame", 0, "<i4")),
               next_frame_at_keyframe=mutated(("next_frame", last, "<i4")),
               keyframe_order=mutated(("kf[1].frame_id", f["kf[0].frame_id"][1], "<i4")),
               frames_since_kf=mutated(("frames_since_kf", int(f["next_frame"][1]) - last, "<i4")),
               next_mp=mutated(("next_mp", int(f["next_mp"][1]) + 1, "<i8")),
               no_pose=mutated(("has_pose", 0, "u1")), no_depth=mutated(("has_depth", 0, "u1")))
    fb, mutated_blank = _mutator(blank)
    assert int(fb["n_kf"][1]) == 0 and int(fb["next_frame"][1]) == 0
    out.update(blank_next_frame=mutated_blank(("next_frame", 5, "<i4")), blank_restart_pending=mutated_blank(("restart_pending", 1, "u1")),
               blank_lost=mutated_blank(("lost", 1, "u1")), blank_has_pose=mutated_blank(("has_pose", 1, "u1")),
               blank_frames_since_kf=mutated_blank(("frames_since_kf", 1, "<i4")), blank_next_mp=mutated_blank(("next_mp", 3, "<i8")))
    return out


@pytest.mark.gpu
@MODES
def test_rejections_change_nothing(ctx3, shift_data, ref_mode):
    """Saves of a stream with queued frames or a pending insertion and a save one byte short; loads into a stream with
    queued frames and loads of damaged records: each returns its error, and both engines then track exactly as engines that
    never saw the calls.  The undamaged record loads."""
    from ygz_slam_b200 import vo_native
    lib = vo_native._lib()
    seq = Seq(*shift_data[0])
    live = Seq(*shift_data[2])
    want, want_stats, _ = reference(ctx3, shift_data, seq, "plain", 1, ref_mode)
    with engine(ctx3, 1, 1, ref_mode) as solo:   # what B's stream 0 gives without any of the calls
        feed(solo, 0, live, 0, N_FRAMES)
        solo.flush()
        want_live, want_live_stats = of(solo.poll(), 0), solo._stat_row(0)
    with engine(ctx3, 2, 1, ref_mode) as A, engine(ctx3, 2, 8, ref_mode) as B:
        cut = 15
        neighbour(A, 0, shift_data[2], 0, cut)
        feed(A, SRC, seq, 0, cut)
        A.flush()
        buf = np.zeros(A.stream_record_bound(), np.uint8)
        n = C.c_size_t(0)
        results, pending = [A.poll()], 0
        for k in range(cut, N_FRAMES):   # window 1, one push and one step at a time
            A.push(SRC, seq.frames[k], seq.depth(k), tag=100 + k)
            if k == cut:   # a queued frame
                assert lib.ygz_vo_save_stream(A.h, SRC, buf.ctypes.data, buf.size, C.byref(n)) == ERR_INVALID
            A.step()
            results.append(A.poll())
            if sum(int((r["stream"] == SRC).sum()) for r in results) == k:   # frame k is neither queued nor final
                assert lib.ygz_vo_save_stream(A.h, SRC, buf.ctypes.data, buf.size, C.byref(n)) == ERR_INVALID
                pending += 1
        assert pending >= 1
        A.flush()
        results.append(A.poll())
        rec = save(A, SRC)
        assert lib.ygz_vo_save_stream(A.h, SRC, buf.ctypes.data, len(rec) - 1, C.byref(n)) == ERR_CAPACITY and n.value == len(rec)
        assert lib.ygz_vo_save_stream(A.h, SRC, None, 0, C.byref(n)) == ERR_CAPACITY and n.value == len(rec)
        for stream in (-1, 2):
            assert lib.ygz_vo_save_stream(A.h, stream, buf.ctypes.data, buf.size, C.byref(n)) == ERR_INVALID
        same_results(of(np.concatenate(results), SRC), want)
        assert np.array_equal(A._stat_row(SRC), want_stats)

        blank = save(B, 1)   # never pushed
        feed(B, 0, live, 0, 12)
        B.flush()
        res = [B.poll()]
        cells, n_levels = ctx3.n_cells, ctx3.params.n_levels

        def last_error():
            return ctx3.lib.ygzb_last_error(ctx3.h)
        # the tracker's checks leave a message on the context; the record's are made before any tracker call and leave the
        # message of this rejected restart in place
        sheared = np.eye(4)[:3].copy()
        sheared[0, 1] = 1e-3
        assert lib.ygz_vo_restart(B.h, 0, sheared.ctypes.data) == ERR_INVALID
        marker = last_error()
        assert b"orthonormal" in marker
        for name, bad in _mutations(rec, blank, cells, n_levels).items():
            data = np.frombuffer(bad, np.uint8)
            assert lib.ygz_vo_load_stream(B.h, 0, data.ctypes.data, data.size) == ERR_INVALID, name
            assert last_error() == marker, name
        f, mutated = _mutator(rec)
        start = f["start"][1].copy()
        start[3] = np.nan   # a start pose the tracker refuses, as ygz_vo_restart does
        data = np.frombuffer(mutated(("start", start, "<f8")), np.uint8)
        assert lib.ygz_vo_load_stream(B.h, 0, data.ctypes.data, data.size) == ERR_INVALID and b"not finite" in last_error()
        good = np.frombuffer(rec, np.uint8)
        for stream in (-1, 2):
            assert lib.ygz_vo_load_stream(B.h, stream, good.ctypes.data, good.size) == ERR_INVALID
        assert lib.ygz_vo_load_stream(B.h, 0, None, good.size) == ERR_INVALID
        feed(B, 0, live, 12, 13)   # a queued frame
        assert lib.ygz_vo_load_stream(B.h, 0, good.ctypes.data, good.size) == ERR_INVALID
        feed(B, 0, live, 13, N_FRAMES)
        B.flush()
        res.append(B.poll())
        same_results(of(np.concatenate(res), 0), want_live)
        assert np.array_equal(B._stat_row(0), want_live_stats)
        B.load_stream(1, blank)   # the undamaged records
        assert save(B, 1) == blank
        B.load_stream(1, rec)
        assert save(B, 1) == rec
