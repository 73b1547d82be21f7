"""Observation rows: the map points each tracked frame's pose rests on (ygzb_observation, ygzb_tracker_set_observations,
ygz_vo_set_observations / ygz_vo_poll_observations, vo_native.Engine(observations=True)).

Tracker: on imported maps, a job's rows must be, bit for bit, the pose-only inliers ygzb_tracker_debug_job shows (ids from
c_src and the ring's mp0, px from c_px, pw from c_pw), exactly n_inliers of them, in both reference modes, whatever the
batch around the job; turning the rows on must not change a result.  Engine: on shift streams the rows must not depend on
the window or the pacing, must be those the key-frames take over, and must not change any result; against the Python loop
(vo.VisualOdometry, which agrees on poses to 1e-4, not bit for bit) the agreement is measured and bounded."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from ygz_slam_b200 import synth

ROOT = Path(__file__).resolve().parent.parent
W, H = synth.W, synth.H
K = (synth.FX, synth.FY, synth.CX, synth.CY)
ERR_INVALID, ERR_CAPACITY = -1, -4
POLICY = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)


def test_observation_row_layout_matches_the_header(tmp_path):
    """ygzb_observation is 48 bytes, laid out as vo_native.OBS_DTYPE, in plain C99."""
    from ygz_slam_b200 import vo_native
    src = tmp_path / "obs.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "ygz_vo.h"\nint main(void) {\n'
                   '    printf("%d %d %d %d\\n", (int)sizeof(ygzb_observation), (int)offsetof(ygzb_observation, id),\n'
                   '           (int)offsetof(ygzb_observation, px), (int)offsetof(ygzb_observation, pw));\n    return 0;\n}\n')
    exe = tmp_path / "obs"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", f"-I{ROOT / 'include'}", str(src), "-o", str(exe)], check=True,
                   capture_output=True, text=True)
    got = list(map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()))
    dt = vo_native.OBS_DTYPE
    assert got == [48, dt.fields["id"][1], dt.fields["px"][1], dt.fields["pw"][1]] == [48, 0, 8, 24]
    assert dt.itemsize == 48


def test_null_handles_are_rejected_without_a_device():
    """The argument checks that come before any device work."""
    from ygz_slam_b200 import build, capi, vo_native
    build.build()
    lib = capi.load_library()
    lib.ygzb_tracker_set_observations.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    assert lib.ygzb_tracker_set_observations(None, None, 0) == ERR_INVALID
    vl = vo_native._lib()
    n, n_obs = C.c_int(7), C.c_size_t(7)
    assert vl.ygz_vo_set_observations(None, 1) == ERR_INVALID
    assert vl.ygz_vo_poll_observations(None, None, 0, C.byref(n), None, 0, C.byref(n_obs)) == ERR_INVALID


# ---- tracker -----------------------------------------------------------------------------------------------------------
KF_FRAMES = (0, 4, 8)
MP0 = (0, 10000, 20000)
KF_SLOT0 = 8


@pytest.fixture(scope="module")
def frames():
    out = {k: dict(zip(("gray", "depth", "T"), synth.stream_frame(k))) for k in KF_FRAMES + (10, 11, 12)}
    T = out[8]["T"].copy()   # 0.3 m closer to the plane than key-frame 8: the alignment's motion fails the 0.2 rule
    T[2, 3] -= 0.3
    g, d = synth.render_plane(synth.texture(0x59475A00, 2048), T, noise_sigma=2.0, seed=5)
    out["far"] = dict(gray=g, depth=d, T=T)
    return out


def _backproject(T, px, d):
    Ti = np.linalg.inv(np.vstack([T, [0, 0, 0, 1]]))
    pc = np.stack([(px[:, 0] - K[2]) * d / K[0], (px[:, 1] - K[3]) * d / K[1], d], 1)
    return pc @ Ti[:3, :3].T + Ti[:3, 3]


def _filled(fr, cells, mp0, seed, behind=False):
    """A key-frame with a feature in every grid cell; behind=True puts its map points behind the camera (it still serves as
    the alignment's reference, but nothing of it projects)."""
    px, d = synth.pixel_features(fr["depth"], cells, seed=seed, margin=12)
    pw = _backproject(fr["T"], px, d)
    if behind:
        pw = _backproject(fr["T"], px, -d)
    return dict(gray=fr["gray"], T=fr["T"], px=px, level=np.random.default_rng(seed).integers(0, 3, cells), depth=d, pw=pw, mp0=mp0)


def _record(kfs, cells):
    from ygz_slam_b200 import capi
    rec = capi.MapBuffers(capi.TRACK_RING, W, H, cells)
    r, a = rec.rec, rec.a
    r.width, r.height, r.cells, r.n_levels, r.n_keyframes = W, H, cells, 3, len(kfs)
    r.K[:] = list(K)
    f0 = 0
    for k, kf in enumerate(kfs):
        n = len(kf["depth"])
        a["entry"][k], a["T_cw"][k], a["mp0"][k], a["n_features"][k], a["n_obs"][k] = k, kf["T"].reshape(-1), kf["mp0"], n, 0
        a["image"][k] = kf["gray"]
        a["px"][f0:f0 + n], a["level"][f0:f0 + n], a["depth"][f0:f0 + n], a["pw"][f0:f0 + n] = kf["px"], kf["level"], kf["depth"], kf["pw"]
        f0 += n
    return rec


def _obs_buffer(rows):
    from ygz_slam_b200 import capi, vo_native
    return _sentinel(capi.pinned_empty(rows, vo_native.OBS_DTYPE))


def _sentinel(buf):
    buf["id"] = -7
    buf["px"] = np.nan
    buf["pw"] = np.nan
    return buf


def _set_obs(tr, buf, capacity=None):
    return tr.set_observations(buf, capacity)


def _want_rows(dbg, mp0_of_local, cells):
    """The rows a job must give: its inliers in candidate order, ids from c_src and the ring's mp0."""
    src = dbg["c_src"][dbg["inlier"]]
    return (np.asarray(mp0_of_local)[src // cells] + src % cells, dbg["c_px"][dbg["inlier"]], dbg["c_pw"][dbg["inlier"]])


def _check_rows(buf, j, stride, res, dbg, mp0_of_local, cells):
    n = res["n_inliers"]
    rows = buf[j * stride:(j + 1) * stride]
    ids, px, pw = _want_rows(dbg, mp0_of_local, cells)
    if not dbg["aligned"]:
        ids, px, pw = ids[:0], px[:0], pw[:0]
    assert len(ids) == n == (dbg["n_inliers"] if dbg["aligned"] else 0)
    assert np.array_equal(rows["id"][:n], ids) and np.array_equal(rows["px"][:n], px) and np.array_equal(rows["pw"][:n], pw)
    assert (rows["id"][n:] == -7).all() and np.isnan(rows["px"][n:]).all()   # exactly n rows written


def _same_bytes(a, b):
    """Rows equal bit for bit, the NaN sentinels of unwritten rows included."""
    return a.tobytes() == b.tobytes()


def _same_debug(a, b):
    for k in ("T_aligned", "rel", "n_meas", "aligned", "n_candidates", "n_projected", "n_inliers", "cand_ok", "c_src", "c_px", "c_pw", "inlier"):
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.gpu
def test_tracker_rows_are_the_pose_only_inliers(ctx3, frames):
    """Key-frame mode on imported maps of 3 streams (key-frames with a feature in every one of the 3,072 cells: the scan
    runs over up to 12 chunks of 1,024): a job with 3, 2 and 1 local key-frames, a job the alignment loses (0 rows), a
    job with nothing projected; one batch, the reversed batch and one job per batch give the same rows.  Results and
    debug views are bit-identical with and without the rows; after NULL a sentinel-filled buffer stays untouched;
    pageable memory and a short capacity are rejected with the previous buffer still in use."""
    cells = ctx3.n_cells
    fr = ctx3.frames(KF_SLOT0 + 4 * 3)
    tr = fr.tracker(3, 8, K)
    maps = [[_filled(frames[k], cells, MP0[i], seed=3 + i) for i, k in enumerate(KF_FRAMES)],
            [_filled(frames[k], cells, MP0[i], seed=7 + i) for i, k in enumerate(KF_FRAMES)],
            [_filled(frames[4], cells, MP0[0], seed=11), _filled(frames[8], cells, MP0[1], seed=12, behind=True)]]
    for s, kfs in enumerate(maps):
        e = np.arange(len(kfs), dtype=np.int32)
        tr.import_(s, e, KF_SLOT0 + 4 * s + e, _record(kfs, cells))
    tr.upload(0, np.stack([frames[k]["gray"] for k in (10, 11, 12, "far")]))
    jobs = [(0, 0, [0, 1, 2]), (1, 1, [0, 1, 2]), (1, 2, [1, 2]), (0, 3, [0, 1, 2]), (2, 0, [1]), (2, 1, [0, 1]), (0, 1, [2])]
    mp0 = [[maps[s][e]["mp0"] for e in local] for s, _, local in jobs]
    stride = 4 * cells
    plain = tr.track(jobs)
    plain_dbg = [tr.debug_job(j) for j in range(len(jobs))]
    buf = _obs_buffer(8 * stride)
    assert _set_obs(tr, buf) == 0
    res = tr.track(jobs)
    for j in range(len(jobs)):
        dbg = tr.debug_job(j)
        _same_debug(dbg, plain_dbg[j])
        assert all(np.array_equal(res[j][k], plain[j][k]) for k in res[j]), j
        _check_rows(buf, j, stride, res[j], dbg, mp0[j], cells)
    n_inl = [r["n_inliers"] for r in res]
    print("rows per job:", n_inl)
    assert res[3]["aligned"] == 0 and n_inl[3] == 0                       # lost by the alignment
    assert res[4]["aligned"] == 1 and res[4]["n_candidates"] == 0 and n_inl[4] == 0   # nothing projected
    assert res[0]["n_projected"] > 3 * 1024 and min(n_inl[k] for k in (0, 1, 5)) > 1000   # several scan chunks
    first = buf.copy()
    rev = _obs_buffer(8 * stride)
    assert _set_obs(tr, rev) == 0
    tr.track(jobs[::-1])
    for j in range(len(jobs)):
        r = len(jobs) - 1 - j
        assert _same_bytes(rev[r * stride:(r + 1) * stride], first[j * stride:(j + 1) * stride]), j
    one = _obs_buffer(8 * stride)
    assert _set_obs(tr, one) == 0
    for j in range(len(jobs)):
        _sentinel(one)
        tr.track([jobs[j]])
        assert _same_bytes(one[:stride], first[j * stride:(j + 1) * stride]), j
    # rejected calls keep the buffer in use
    assert _set_obs(tr, np.zeros(8 * stride, vo_native_obs())) == ERR_INVALID                  # pageable
    assert _set_obs(tr, _obs_buffer(8 * stride - 1)) == ERR_INVALID                             # short
    assert _set_obs(tr, buf, capacity=8 * stride - 1) == ERR_INVALID
    _sentinel(one)
    tr.track([jobs[0]])
    assert _same_bytes(one[:stride], first[:stride])
    # NULL: nothing written from the next batch on
    assert _set_obs(tr, None, 0) == 0
    _sentinel(one)
    again = tr.track(jobs)
    assert (one["id"] == -7).all() and np.isnan(one["px"]).all()
    assert all(np.array_equal(again[j][k], plain[j][k]) for j in range(len(jobs)) for k in plain[j])
    tr.close()
    fr.close()


def vo_native_obs():
    from ygz_slam_b200 import vo_native
    return vo_native.OBS_DTYPE


@pytest.mark.gpu
def test_tracker_rows_in_previous_frame_mode(ctx3):
    """Previous-frame mode: 2 streams after their first key-frame track 3 and 2 frames in one interleaved batch (3 waves,
    jobs reordered on the device): each caller job's rows are its debug view's inliers; the key-frame made from the last
    job takes over exactly those rows."""
    cells = ctx3.n_cells
    data = [synth.shift_stream(s, 4) for s in range(2)]
    fr = ctx3.frames(16)
    tr = fr.tracker(2, 8, K)
    tr.set_reference_mode("previous", [14, 15])
    for s in range(2):
        tr.set_depth(s, data[s][1])
        tr.upload(s * 4, data[s][0][0])
    kres = tr.make_keyframes([dict(stream=s, frame_slot=s * 4, kf_slot=8 + s * 4, entry=0, track_job=-1, local_entry=[0]) for s in range(2)])
    for s in range(2):
        tr.upload(s * 4, data[s][0][1:4])
    stride = 4 * cells
    buf = _obs_buffer(8 * stride)
    assert _set_obs(tr, buf) == 0
    jobs = [(0, 0, [0]), (1, 4, [0]), (0, 1, [0]), (1, 5, [0]), (0, 2, [0])]
    res = tr.track(jobs)
    for j in range(len(jobs)):
        assert res[j]["aligned"] and res[j]["n_inliers"] > 100, j
        _check_rows(buf, j, stride, res[j], tr.debug_job(j), [0], cells)
    tr.make_keyframes([dict(stream=0, frame_slot=2, kf_slot=9, entry=1, track_job=4, local_entry=[0, 1], mp0=kres[0]["n_features"])])
    new = tr.export(0, [1]).keyframes()[0]
    n = res[4]["n_inliers"]
    assert np.array_equal(new["obs_id"], buf["id"][4 * stride:4 * stride + n])
    assert np.array_equal(new["obs_px"], buf["px"][4 * stride:4 * stride + n])
    tr.close()
    fr.close()


# ---- engine ------------------------------------------------------------------------------------------------------------
N_FRAMES = 30
S = 3


@pytest.fixture(scope="module")
def shift_data():
    return [synth.shift_stream(s_, N_FRAMES) for s_ in range(4)]


def _engine(ctx, window, ref_mode, observations=True, **kw):
    from ygz_slam_b200 import vo_native
    return vo_native.Engine(ctx, S, window=window, ref_mode=ref_mode, observations=observations, **dict(POLICY, **kw))


def _per_frame(res, rows):
    """{(stream, frame): (result, rows)}; checks every result carries exactly n_inliers rows."""
    out = {}
    for r, o in zip(res, rows):
        assert len(o) == r["n_inliers"]
        out[(int(r["stream"]), int(r["frame"]))] = (r, o)
    return out


def _lock_step(ctx, data, window, ref_mode, observations=True, pace=None):
    with _engine(ctx, window, ref_mode, observations) as eng:
        for k in range(N_FRAMES):
            for s_ in range(S):
                eng.push(s_, data[s_][0][k], data[s_][1], tag=k)
            if pace and k % pace == pace - 1:
                eng.step()
        eng.flush()
        got = eng.poll()
        stats = [eng.stats(s_) for s_ in range(S)]
        maps = [eng.export_map(s_).keyframes() for s_ in range(S)]
    return got, stats, maps


_RUNS = {}


def lock_step(ctx, data, window, ref_mode, pace=None):
    key = (window, ref_mode, pace)
    if key not in _RUNS:
        _RUNS[key] = _lock_step(ctx, data, window, ref_mode, pace=pace)
    return _RUNS[key]


def _by_frame(res):
    return res[np.lexsort((res["frame"], res["stream"]))]


def _same_rows(a, b):
    assert a.keys() == b.keys()
    for key in a:
        assert np.array_equal(a[key][1], b[key][1]), key


@pytest.mark.gpu
@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
def test_engine_rows_across_windows_and_pacing(ctx3, shift_data, ref_mode):
    """Windows 1, 4 and 8, lock step and a step every 3 pushes: the rows are bit-identical everywhere; results and stats
    are those of an engine without observations; every result has n_inliers rows; a key-frame's rows are its map
    record's obs_id / obs_px; a tracked frame's ids lie in its local key-frames' [mp0, mp0 + n)."""
    (plain, plain_stats, _) = _lock_step(ctx3, shift_data, 8, ref_mode, observations=False)
    base = None
    for window, pace in ((1, None), (4, None), (8, None), (8, 3)):
        (res, rows), stats, maps = lock_step(ctx3, shift_data, window, ref_mode, pace)
        assert np.array_equal(_by_frame(res), _by_frame(plain)), window
        assert stats == plain_stats
        per = _per_frame(res, rows)
        if base is None:
            base = per
        _same_rows(per, base)
    (res, rows), stats, maps = lock_step(ctx3, shift_data, 8, ref_mode)
    per = _per_frame(res, rows)
    for s_ in range(S):
        assert stats[s_]["keyframes"] >= 3 and stats[s_]["lost"] == 0
        status = {f: int(r["status"]) for (ss, f), (r, _) in per.items() if ss == s_}
        assert status[0] == 1 and len(per[(s_, 0)][1]) == 0
        kf_frames = [f for f in sorted(status) if status[f] == 1]
        # the key-frames still in the ring, newest last: their observations are the rows of their results
        for kf, f in zip(maps[s_], kf_frames[-len(maps[s_]):]):
            o = per[(s_, f)][1]
            assert np.array_equal(kf["obs_id"], o["id"]) and np.array_equal(kf["obs_px"], o["px"]), (s_, f)
        # ids of a tracked frame lie in [mp0, mp0 + n) of its local key-frames: the 3 newest of the ring for the frames
        # after the newest key-frame, the 3 before it for the newest key-frame of a full ring
        ring, kf_in_ring = maps[s_], kf_frames[-len(maps[s_]):]
        assert len(ring) == 4
        checks = [(f, ring[-3:]) for f in sorted(status) if f > kf_in_ring[-1]] + [(kf_in_ring[3], ring[:3])]
        for f, local in checks:
            o = per[(s_, f)][1]
            ok = np.zeros(len(o), bool)
            for kf in local:
                ok |= (o["id"] >= kf["mp0"]) & (o["id"] < kf["mp0"] + len(kf["depth"]))
            assert len(o) > 0 and ok.all(), (s_, f)


@pytest.mark.gpu
@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
def test_engine_rows_after_restart_and_record(ctx3, shift_data, ref_mode):
    """A stream restarted for a new sequence gives the rows of a fresh engine on that sequence; a stream saved at frame 20
    and loaded into another engine with observations on gives the rows of the uninterrupted run."""
    (res, rows), _, _ = lock_step(ctx3, shift_data, 8, ref_mode)
    full = _per_frame(res, rows)
    # record: frames [0, 20) in engine A, the rest in engine B
    with _engine(ctx3, 8, ref_mode) as a, _engine(ctx3, 8, ref_mode) as b:
        for k in range(20):
            a.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        a.flush()
        ra, oa = a.poll()
        b.load_stream(0, a.save_stream(0))
        for k in range(20, N_FRAMES):
            b.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        b.flush()
        rb, ob = b.poll()
    for r, o in list(zip(ra, oa)) + list(zip(rb, ob)):
        assert int(r["stream"]) == 0
        assert np.array_equal(o, full[(0, int(r["frame"]))][1]), int(r["frame"])
    assert len(ra) + len(rb) == N_FRAMES
    # restart: stream 0 runs stream 3's frames after 12 frames of its own; they get a fresh engine's rows
    with _engine(ctx3, 8, ref_mode) as e:
        for k in range(12):
            e.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        e.restart(0)
        for k in range(N_FRAMES):
            e.push(0, shift_data[3][0][k], shift_data[3][1], tag=100 + k)
        e.flush()
        r2, o2 = e.poll()
    with _engine(ctx3, 8, ref_mode) as f:
        for k in range(N_FRAMES):
            f.push(0, shift_data[3][0][k], shift_data[3][1], tag=100 + k)
        f.flush()
        r3, o3 = f.poll()
    assert [int(t) for t in r2["tag"][12:]] == [int(t) for t in r3["tag"]]
    for o, want in zip(o2[12:], o3):
        assert np.array_equal(o, want)
    for r, o in zip(r2[:12], o2[:12]):
        assert np.array_equal(o, full[(0, int(r["frame"]))][1])


@pytest.mark.gpu
@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
def test_engine_rows_of_a_lost_stream(ctx3, shift_data, ref_mode):
    """min_inliers above any count: the first tracked frame is LOST by pose-only with its n_inliers > 0 rows, every later
    frame LOST with none.  A frame of another texture loses a stream too: n_inliers rows on it, none after."""
    from ygz_slam_b200 import vo_native
    with vo_native.Engine(ctx3, 1, window=8, ref_mode=ref_mode, observations=True, **POLICY, min_inliers=10 ** 6) as e:
        for k in range(8):
            e.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        e.flush()
        res, rows = e.poll()
    assert list(res["status"]) == [1] + [2] * 7
    assert res["n_inliers"][1] > 100 and len(rows[1]) == res["n_inliers"][1]
    assert all(len(o) == 0 for o in rows[2:]) and (res["n_inliers"][2:] == 0).all()
    frames = shift_data[0][0].copy()
    frames[8] = shift_data[1][0][8]
    with vo_native.Engine(ctx3, 1, window=8, ref_mode=ref_mode, observations=True, **POLICY) as e:
        for k in range(12):
            e.push(0, frames[k], shift_data[0][1], tag=k)
        e.flush()
        res, rows = e.poll()
    assert (res["status"][8:] == 2).all() and (res["status"][:8] != 2).all()
    assert len(rows[8]) == res["n_inliers"][8] and all(len(o) == 0 for o in rows[9:])
    print(f"{ref_mode}: the injected frame is LOST with {res['n_inliers'][8]} rows")


@pytest.mark.gpu
def test_engine_observation_calls_check_their_state(ctx3, shift_data):
    """set_observations while frames are queued, while a key-frame insertion is pending or while results wait is rejected
    and changes nothing; an undersized poll moves nothing and says how many rows the first result needs; a poll with
    observations off is rejected."""
    from ygz_slam_b200 import vo_native
    with vo_native.Engine(ctx3, 1, window=8, **POLICY) as e:
        lib, h = e.lib, e.h
        out = np.zeros(64, vo_native.RESULT_DTYPE)
        obs = np.zeros(16, vo_native.OBS_DTYPE)
        n, n_obs = C.c_int(0), C.c_size_t(0)
        assert lib.ygz_vo_poll_observations(h, out.ctypes.data, 64, C.byref(n), obs.ctypes.data, 16, C.byref(n_obs)) == ERR_INVALID
        e.push(0, shift_data[0][0][0], shift_data[0][1])
        assert lib.ygz_vo_set_observations(h, 1) == ERR_INVALID           # queued
        e.flush()
        assert lib.ygz_vo_set_observations(h, 1) == ERR_INVALID           # a result waits
        e.poll()
        e.set_observations(True)
        for k in range(1, 8):
            e.push(0, shift_data[0][0][k], shift_data[0][1])
        e.step()
        e.step()
        assert lib.ygz_vo_set_observations(h, 0) == ERR_INVALID
        e.flush()
        # room for 16 rows: the first waiting result (frame 1, tracked) does not fit, and nothing moves
        rc = lib.ygz_vo_poll_observations(h, out.ctypes.data, 64, C.byref(n), obs.ctypes.data, 16, C.byref(n_obs))
        assert rc == ERR_CAPACITY and n.value == 0 and n_obs.value > 16
        res, rows = e.poll()
        assert list(res["frame"]) == list(range(1, 8))
        assert res["n_inliers"][0] == n_obs.value == len(rows[0])
        assert all(len(o) == r["n_inliers"] for r, o in zip(res, rows))
        # capacity 0 moves nothing and is not an error; off again, a poll with rows is rejected
        assert lib.ygz_vo_poll_observations(h, None, 0, C.byref(n), None, 0, C.byref(n_obs)) == 0 and n.value == 0
        e.set_observations(False)
        assert lib.ygz_vo_poll_observations(h, out.ctypes.data, 64, C.byref(n), obs.ctypes.data, 16, C.byref(n_obs)) == ERR_INVALID


@pytest.mark.gpu
def test_engine_rows_agree_with_the_python_loop(ctx3, shift_data):
    """vo.VisualOdometry on the GPU backend (its last_obs after every tracked frame) against the engine's rows.  The two
    loops agree on poses to 1e-4, not bit for bit, so the id lists may differ at the threshold of the 20-pixel border or of
    pose-only's inlier test, and FindDirectProjection's result follows the pose it starts from; measured and bounded: the
    share of ids in one list only, and the pixel difference of ids in both.  Measured on an H100 80GB HBM3 (700 W): 67 of
    75 tracked frames with identical id sets, at most 3 ids (8.8e-4 of the union) in one list only, shared ids' pixels
    within 0.21 px."""
    from ygz_slam_b200 import se3, vo
    n = 26
    be = vo.GpuBackend(ctx3, S * vo.VisualOdometry.SLOTS_PER_STREAM)
    V = vo.VisualOdometry(be, S, **POLICY)
    loop = {}
    for k in range(n):
        V.add_frames([shift_data[s_][0][k] for s_ in range(S)], [shift_data[s_][1] for s_ in range(S)], k)
        if k > 0:
            for s_ in range(S):
                loop[(s_, k)] = V.streams[s_].last_obs
    be.fr.close()
    (res, rows), _, _ = lock_step(ctx3, shift_data, 8, "keyframe")
    per = _per_frame(res, rows)
    same = worst_sym = 0
    worst_px = worst_share = 0.0
    for (s_, k), (ids, px) in loop.items():
        r, o = per[(s_, k)]
        T_loop = V.streams[s_].trajectory[k]
        if np.array_equal(r["T_cw"].reshape(3, 4), T_loop):
            assert np.array_equal(o["id"], ids)
        a, b = set(o["id"].tolist()), set(np.asarray(ids).tolist())
        sym = len(a ^ b)
        same += sym == 0
        worst_sym = max(worst_sym, sym)
        worst_share = max(worst_share, sym / max(1, len(a | b)))
        _, ia, ib = np.intersect1d(o["id"], ids, return_indices=True)
        if len(ia):
            worst_px = max(worst_px, float(np.abs(o["px"][ia] - np.asarray(px)[ib]).max()))
        assert np.linalg.norm(se3.se3_log(se3.mul(r["T_cw"].reshape(3, 4), se3.inv(T_loop)))) < 1e-4
    print(f"{same} of {len(loop)} tracked frames with identical id sets; at most {worst_sym} ids ({worst_share:.2e} of the union) "
          f"in one list only; shared ids' pixels differ by at most {worst_px:.2e} px")
    assert worst_share < 5e-3 and worst_px < 0.5
