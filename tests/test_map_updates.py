"""Map updates: the local map as each key-frame insertion leaves it (ygzb_map_point, ygzb_tracker_set_map_updates,
ygz_vo_set_map_updates / ygz_vo_poll_map_updates, vo_native.Engine(map_updates=True)).

Tracker: on imported maps, an insertion's rows must be the local BA's points -- restated here in numpy from the map record
exported before it: the points of the older local key-frames that at least two local key-frames observe, in dense order
-- then the new key-frame's points, each with the position the ring holds afterwards, bit for bit.  Engine: a mirror
folded from the updates alone must equal ygz_vo_export_map bit for bit at every flush, and the updates must not depend on
the window, the pacing, a restart or a stream record cut; turning them on must not change a result."""
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


def test_map_update_layouts_match_the_headers(tmp_path):
    """ygzb_map_point (32 bytes) and ygz_vo_map_update (432 bytes) are laid out as capi.MAP_POINT_DTYPE and
    vo_native.MAP_UPDATE_DTYPE, in plain C99."""
    from ygz_slam_b200 import capi, vo_native
    fields = ["stream", "frame", "sequence", "n_local", "retired_frame", "local_frame", "n_moved", "n_new", "T_cw"]
    src = tmp_path / "upd.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "ygz_vo.h"\nint main(void) {\n'
                   '    printf("%d %d %d\\n", (int)sizeof(ygzb_map_point), (int)offsetof(ygzb_map_point, id), (int)offsetof(ygzb_map_point, pw));\n'
                   '    printf("%d", (int)sizeof(ygz_vo_map_update));\n'
                   + "".join(f'    printf(" %d", (int)offsetof(ygz_vo_map_update, {f}));\n' for f in fields)
                   + '    printf(" %d\\n", YGZB_TRACK_RING);\n    return 0;\n}\n')
    exe = tmp_path / "upd"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", f"-I{ROOT / 'include'}", str(src), "-o", str(exe)], check=True,
                   capture_output=True, text=True)
    got = list(map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()))
    pt, up = capi.MAP_POINT_DTYPE, vo_native.MAP_UPDATE_DTYPE
    assert got[:3] == [pt.itemsize, pt.fields["id"][1], pt.fields["pw"][1]] == [32, 0, 8]
    assert got[3:-1] == [up.itemsize] + [up.fields[f][1] for f in fields]
    assert got[3] == 432 and got[-1] == capi.TRACK_RING == up.fields["local_frame"][0].shape[0] == up.fields["T_cw"][0].shape[0]


def test_null_handles_are_rejected_without_a_device():
    """The argument checks that come before any device work."""
    from ygz_slam_b200 import build, capi, vo_native
    build.build()
    lib = capi.load_library()
    assert "ygzb_tracker_set_map_updates" in capi.EXPORTS
    lib.ygzb_tracker_set_map_updates.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    assert lib.ygzb_tracker_set_map_updates(None, None, 0) == ERR_INVALID
    vl = vo_native._lib()
    n, n_rows = C.c_int(7), C.c_size_t(7)
    assert vl.ygz_vo_set_map_updates(None, 1) == ERR_INVALID
    assert vl.ygz_vo_poll_map_updates(None, None, 0, C.byref(n), None, 0, C.byref(n_rows)) == ERR_INVALID


# ---- tracker -----------------------------------------------------------------------------------------------------------
KF_SLOT0 = 8
# per stream: the frames of its two imported key-frames and its current frame; stream 2 starts with a first key-frame
STREAMS = (((0, 4), 8), ((4, 8), 11))
FIRST_FRAME = 12
MP0 = ((0, 10000), (50000, 60000))


def _backproject(T, px, d):
    Ti = np.linalg.inv(np.vstack([T, [0, 0, 0, 1]]))
    pc = np.stack([(px[:, 0] - K[2]) * d / K[0], (px[:, 1] - K[3]) * d / K[1], d], 1)
    return pc @ Ti[:3, :3].T + Ti[:3, 3]


def _project(T, pw):
    pc = pw @ T[:3, :3].T + T[:3, 3]
    return np.stack([K[0] * pc[:, 0] / pc[:, 2] + K[2], K[1] * pc[:, 1] / pc[:, 2] + K[3]], 1), pc[:, 2]


def _scene(cells, s):
    """Two key-frames with a feature in every grid cell; the second observes every other point of the first, at its
    projection."""
    kfs = []
    for k, f in enumerate(STREAMS[s][0]):
        gray, depth, T = synth.stream_frame(f)
        px, d = synth.pixel_features(depth, cells, seed=31 + 2 * s + k, margin=12)
        kfs.append(dict(gray=gray, T=T, px=px, level=np.random.default_rng(5 + k).integers(0, 3, cells), depth=d, pw=_backproject(T, px, d),
                        mp0=MP0[s][k], obs_id=np.zeros(0, np.int64), obs_px=np.zeros((0, 2))))
    uv, z = _project(kfs[1]["T"], kfs[0]["pw"])
    sel = np.flatnonzero((np.arange(cells) % 2 == 0) & (z > 0) & (uv[:, 0] > 0) & (uv[:, 0] < W) & (uv[:, 1] > 0) & (uv[:, 1] < H))
    kfs[1]["obs_id"], kfs[1]["obs_px"] = kfs[0]["mp0"] + sel, uv[sel]
    return kfs


def _record(kfs, cells):
    from ygz_slam_b200 import capi
    rec = capi.MapBuffers(capi.TRACK_RING, W, H, cells)
    r, a = rec.rec, rec.a
    r.width, r.height, r.cells, r.n_levels, r.n_keyframes = W, H, cells, 3, len(kfs)
    r.K[:] = list(K)
    f0 = o0 = 0
    for k, kf in enumerate(kfs):
        n, no = len(kf["depth"]), len(kf["obs_id"])
        a["entry"][k], a["T_cw"][k], a["mp0"][k], a["n_features"][k], a["n_obs"][k] = k, kf["T"].reshape(-1), kf["mp0"], n, no
        a["image"][k] = kf["gray"]
        a["px"][f0:f0 + n], a["level"][f0:f0 + n], a["depth"][f0:f0 + n], a["pw"][f0:f0 + n] = kf["px"], kf["level"], kf["depth"], kf["pw"]
        a["obs_id"][o0:o0 + no], a["obs_px"][o0:o0 + no] = kf["obs_id"], kf["obs_px"]
        f0 += n
        o0 += no
    return rec


def _sentinel(buf):
    buf["id"] = -7
    buf["pw"] = np.nan
    return buf


def _rows_buffer(n):
    from ygz_slam_b200 import capi
    return _sentinel(capi.pinned_empty(n, capi.MAP_POINT_DTYPE))


def _ba_ids(before, new_obs_id):
    """The local BA's points of an insertion, restated from the map before it: the points of the older local key-frames
    (the record's key-frames) that at least two local key-frames observe -- a key-frame observes its own points and the
    ids in its observations -- in dense order (key-frame, then feature)."""
    observed = [set(kf["obs_id"].tolist()) for kf in before] + [set(np.asarray(new_obs_id).tolist())]
    ids = []
    for kf in before:
        own = kf["mp0"] + np.arange(len(kf["depth"]))
        deg = 1 + np.array([sum(int(i) in o for o in observed) for i in own])
        ids.append(own[deg >= 2])
    return np.concatenate(ids)


def _insert(ctx, cells, frames, scenes, buf=None, after_set=None, order=(0, 1, 2)):
    """A fresh 3-stream tracker: streams 0 and 1 on imported maps track their current frame and insert it as a key-frame
    with a local BA over 3 key-frames; stream 2 inserts its first key-frame.  The key-frame jobs go in `order`.  buf:
    the map rows' buffer, set before the insertion; after_set: a callable run on the tracker right after that (rejected
    calls, switching off).  Returns (key-frame results in job order, maps before, maps after, track results)."""
    fr = ctx.frames(KF_SLOT0 + 4 * 3)
    tr = fr.tracker(3, 8, K)
    try:
        for s in range(2):
            e = np.arange(2, dtype=np.int32)
            tr.import_(s, e, KF_SLOT0 + 4 * s + e, _record(scenes[s], cells))
        cur = [STREAMS[0][1], STREAMS[1][1], FIRST_FRAME]
        tr.upload(0, np.stack([frames[f][0] for f in cur]))
        for s in range(3):
            tr.set_depth(s, frames[cur[s]][1])
        tres = tr.track([(0, 0, [0, 1]), (1, 1, [0, 1])])
        before = [tr.export(s, [0, 1]).keyframes() for s in range(2)]
        if buf is not None:
            assert tr.set_map_updates(buf) == 0
        if after_set is not None:
            after_set(tr)
        jobs = [dict(stream=s, frame_slot=s, kf_slot=KF_SLOT0 + 4 * s + 2, entry=2, track_job=s, local_entry=[0, 1, 2], run_ba=1,
                     mp0=MP0[s][1] + 10000) for s in range(2)]
        jobs.append(dict(stream=2, frame_slot=2, kf_slot=KF_SLOT0 + 8, entry=0, track_job=-1, local_entry=[0], mp0=0))
        kres = tr.make_keyframes([jobs[j] for j in order])
        after = [tr.export(s, [0, 1, 2]).keyframes() for s in range(2)] + [tr.export(2, [0]).keyframes()]
    finally:
        tr.close()
        fr.close()
    return kres, before, after, tres


@pytest.fixture(scope="module")
def tracker_scene(ctx3):
    cells = ctx3.n_cells
    frames = {f: synth.stream_frame(f) for f in (STREAMS[0][1], STREAMS[1][1], FIRST_FRAME)}
    scenes = [_scene(cells, s) for s in range(2)]
    return cells, frames, scenes


def _same_maps(a, b):
    for ma, mb in zip(a, b):
        for ka, kb in zip(ma, mb):
            for k in ka:
                assert np.array_equal(ka[k], kb[k]), k


@pytest.mark.gpu
def test_tracker_rows_are_the_ba_points_then_the_new_points(ctx3, tracker_scene):
    """Two insertions with a local BA over 3 key-frames (each with a feature in every one of the 3,072 cells) and a first
    key-frame in one batch.  Each job's rows sit at its own stride: the BA's points (ids restated from the map before
    the insertion), then the new key-frame's points; every pw is the ring's after the insertion, bit for bit; nothing past
    them is written.  Results and maps are bit-identical without rows, and the reversed batch moves the rows with the jobs."""
    cells, frames, scenes = tracker_scene
    stride = 4 * cells
    plain, _, plain_after, plain_tres = _insert(ctx3, cells, frames, scenes)
    buf = _rows_buffer(3 * stride)
    kres, before, after, tres = _insert(ctx3, cells, frames, scenes, buf=buf)
    assert all(np.array_equal(a[k], b[k]) for a, b in zip(kres, plain) for k in a)
    assert all(np.array_equal(a[k], b[k]) for a, b in zip(tres, plain_tres) for k in a)
    _same_maps(after, plain_after)
    for j in range(3):
        rows = buf[j * stride:(j + 1) * stride]
        n_moved, n_new = kres[j]["ba_points"], kres[j]["n_features"]
        new = after[j][-1]
        assert n_new == len(new["depth"]) > 0
        if j < 2:
            want = _ba_ids(before[j], new["obs_id"])
            assert n_moved == len(want) > 1000, (j, n_moved)
            assert np.array_equal(rows["id"][:n_moved], want)
        else:
            assert n_moved == 0
        assert np.array_equal(rows["id"][n_moved:n_moved + n_new], new["mp0"] + np.arange(n_new))
        pw = {}
        for kf in after[j]:
            for i, p in zip(kf["mp0"] + np.arange(len(kf["depth"])), kf["pw"]):
                pw[int(i)] = p
        got = rows[:n_moved + n_new]
        assert np.array_equal(got["pw"], np.array([pw[int(i)] for i in got["id"]]))
        assert (rows["id"][n_moved + n_new:] == -7).all() and np.isnan(rows["pw"][n_moved + n_new:]).all()
        if j < 2:   # the BA moved the points it refined
            moved_before = {int(i): p for kf in before[j] for i, p in zip(kf["mp0"] + np.arange(len(kf["depth"])), kf["pw"])}
            assert any(not np.array_equal(p["pw"], moved_before[int(p["id"])]) for p in got[:n_moved])
    print("rows per job (moved, new):", [(int(r["ba_points"]), int(r["n_features"])) for r in kres])
    first = buf.copy()
    rev = _rows_buffer(3 * stride)
    kres_rev, _, after_rev, _ = _insert(ctx3, cells, frames, scenes, buf=rev, order=(2, 1, 0))
    _same_maps(after_rev, after)
    for j in range(3):
        assert rev[(2 - j) * stride:(3 - j) * stride].tobytes() == first[j * stride:(j + 1) * stride].tobytes(), j


@pytest.mark.gpu
def test_tracker_rows_switched_off_and_bad_buffers(ctx3, tracker_scene):
    """After NULL a sentinel-filled buffer stays untouched and the results are unchanged; pageable memory and a short
    capacity are rejected with the previous buffer still in use."""
    from ygz_slam_b200 import capi
    cells, frames, scenes = tracker_scene
    stride = 4 * cells
    plain, _, plain_after, _ = _insert(ctx3, cells, frames, scenes)
    off = _rows_buffer(3 * stride)
    kres, _, after, _ = _insert(ctx3, cells, frames, scenes, buf=off, after_set=lambda tr: tr.set_map_updates(None))
    assert (off["id"] == -7).all() and np.isnan(off["pw"]).all()
    assert all(np.array_equal(a[k], b[k]) for a, b in zip(kres, plain) for k in a)
    _same_maps(after, plain_after)

    def reject(tr):
        assert tr.set_map_updates(np.zeros(3 * stride, capi.MAP_POINT_DTYPE)) == ERR_INVALID   # pageable
        assert tr.set_map_updates(_rows_buffer(3 * stride - 1)) == ERR_INVALID                # short
        assert tr.set_map_updates(kept, capacity=3 * stride - 1) == ERR_INVALID
    kept = _rows_buffer(3 * stride)
    ref = _rows_buffer(3 * stride)
    _insert(ctx3, cells, frames, scenes, buf=ref)
    kres, _, _, _ = _insert(ctx3, cells, frames, scenes, buf=kept, after_set=reject)
    assert kept.tobytes() == ref.tobytes()


# ---- engine ------------------------------------------------------------------------------------------------------------
N_FRAMES = 30
S = 3


@pytest.fixture(scope="module")
def shift_data():
    return [synth.shift_stream(s_, N_FRAMES) for s_ in range(4)]


class Mirror:
    """The map a caller holds from the updates alone: poses by (stream, sequence, frame), points by (stream, sequence,
    id), plus the bookkeeping the checks need."""

    def __init__(self):
        self.pose, self.point, self.retired, self.mp0 = {}, {}, {}, {}
        self.frames = {}   # (stream, sequence) -> key-frame frame indices in insertion order

    def fold(self, updates, rows):
        for u, r in zip(updates, rows):
            s_, q = int(u["stream"]), int(u["sequence"])
            nl, nm, nn = int(u["n_local"]), int(u["n_moved"]), int(u["n_new"])
            assert len(r) == nm + nn and 1 <= nl <= 3
            assert int(u["local_frame"][nl - 1]) == int(u["frame"]) and (u["local_frame"][nl:] == -1).all()
            assert not u["T_cw"][nl:].any()
            kfs = self.frames.setdefault((s_, q), [])
            assert list(u["local_frame"][:nl]) == (kfs + [int(u["frame"])])[-nl:]
            kfs.append(int(u["frame"]))
            if u["retired_frame"] >= 0:
                f = int(u["retired_frame"])
                assert f not in self.retired.get((s_, q), {}) and f in kfs[:-3]
                self.retired.setdefault((s_, q), {})[f] = (self.pose[(s_, q, f)].copy(), self.mp0[(s_, q, f)])
            else:
                assert len(kfs) <= 3
            new_ids = r["id"][nm:]
            assert np.array_equal(new_ids, new_ids[0] + np.arange(nn)) if nn else True
            assert not np.isin(r["id"][:nm], new_ids).any()
            self.mp0[(s_, q, int(u["frame"]))] = (int(new_ids[0]) if nn else 0, nn)
            for k in range(nl):
                self.pose[(s_, q, int(u["local_frame"][k]))] = u["T_cw"][k].copy()
            for p in r:
                self.point[(s_, q, int(p["id"]))] = p["pw"].copy()
            # nothing a retired key-frame holds moves again
            for f, (T, (m0, n)) in self.retired.get((s_, q), {}).items():
                assert np.array_equal(self.pose[(s_, q, f)], T)
                assert not ((r["id"] >= m0) & (r["id"] < m0 + n)).any()

    def check(self, eng, sequences):
        """Every ring key-frame's pose and every live point of export_map equal the mirror's, bit for bit."""
        for s_ in range(eng.n_streams):
            q = sequences[s_]
            ring = eng.export_map(s_).keyframes()
            kfs = self.frames[(s_, q)][-len(ring):]
            assert len(kfs) == len(ring)
            for f, kf in zip(kfs, ring):
                assert np.array_equal(self.pose[(s_, q, f)], kf["T_cw"].reshape(-1)), (s_, f)
                assert self.mp0[(s_, q, f)] == (kf["mp0"], len(kf["depth"]))
                got = np.array([self.point[(s_, q, kf["mp0"] + g)] for g in range(len(kf["depth"]))])
                assert np.array_equal(got, kf["pw"]), (s_, f)


def _engine(ctx, window, ref_mode, map_updates=True, n_streams=S, **kw):
    from ygz_slam_b200 import vo_native
    return vo_native.Engine(ctx, n_streams, window=window, ref_mode=ref_mode, map_updates=map_updates, **dict(POLICY, **kw))


def _by_frame(a):
    return a[np.lexsort((a["frame"], a["stream"]))]


def _run(ctx, data, window, ref_mode, pacing="flush", map_updates=True):
    """Streams 0..S-1 of `data`, all N_FRAMES frames.  pacing "flush": push everything, flush; "checkpoints": flush and
    poll after frames 10, 20 and 30, checking the mirror against export_map each time; "step": push one frame per
    stream, step, poll.  Returns (results, updates, rows, mirror)."""
    res, upd, rows = [], [], []
    mirror = Mirror()
    with _engine(ctx, window, ref_mode, map_updates) as eng:
        def poll():
            res.append(eng.poll())
            if map_updates:
                u, r = eng.poll_map_updates()
                mirror.fold(u, r)
                upd.append(u)
                rows.extend(r)
        for k in range(N_FRAMES):
            for s_ in range(S):
                eng.push(s_, data[s_][0][k], data[s_][1], tag=k)
            if pacing == "step":
                eng.step()
                poll()
            if pacing == "checkpoints" and k % 10 == 9:
                eng.flush()
                poll()
                mirror.check(eng, [0] * S)
        eng.flush()
        poll()
        if map_updates:
            mirror.check(eng, [0] * S)
    res = np.concatenate(res)
    if not map_updates:
        return res, None, None, None
    upd = np.concatenate(upd)
    return res, upd, rows, mirror


_RUNS = {}


def run(ctx, data, window, ref_mode, pacing="flush"):
    key = (window, ref_mode, pacing)
    if key not in _RUNS:
        _RUNS[key] = _run(ctx, data, window, ref_mode, pacing)
    return _RUNS[key]


def _keyed(upd, rows):
    return {(int(u["stream"]), int(u["frame"])): (u.tobytes(), r.tobytes()) for u, r in zip(upd, rows)}


@pytest.mark.gpu
@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
def test_engine_mirror_equals_the_exported_map(ctx3, shift_data, ref_mode):
    """Windows 1, 4 and 8 at checkpoints, push-all-then-flush and push / step / poll: a mirror folded from the updates
    equals export_map at every flush, bit for bit; the updates are identical everywhere; the results are those of an
    engine without updates; each key-frame result's T_cw is its update's newest pose; the BA moves at least one
    key-frame after its result; every key-frame but the newest three of a stream retires exactly once."""
    plain = _by_frame(_run(ctx3, shift_data, 8, ref_mode, map_updates=False)[0])
    base = None
    for window, pacing in ((1, "checkpoints"), (4, "checkpoints"), (8, "checkpoints"), (8, "flush"), (8, "step")):
        res, upd, rows, mirror = run(ctx3, shift_data, window, ref_mode, pacing)
        assert np.array_equal(_by_frame(res), plain), (window, pacing)
        keyed = _keyed(upd, rows)
        assert len(keyed) == len(upd)
        if base is None:
            base = keyed
        assert keyed == base, (window, pacing)
    res, upd, rows, mirror = run(ctx3, shift_data, 8, ref_mode)
    kf_results = {(int(r["stream"]), int(r["frame"])): r for r in res if r["status"] == 1}
    assert set(kf_results) == {(int(u["stream"]), int(u["frame"])) for u in upd}
    moved = 0
    for u in upd:
        r = kf_results[(int(u["stream"]), int(u["frame"]))]
        assert np.array_equal(u["T_cw"][u["n_local"] - 1], r["T_cw"])
        final = mirror.pose[(int(u["stream"]), 0, int(u["frame"]))]
        moved += not np.array_equal(final, r["T_cw"])
    assert moved > 0
    for s_ in range(S):
        kfs = mirror.frames[(s_, 0)]
        assert len(kfs) >= 4 and sorted(mirror.retired[(s_, 0)]) == kfs[:-3]
    assert (upd["sequence"] == 0).all() and (upd["n_moved"][upd["n_local"] > 1] > 0).all() and (upd["n_moved"][upd["n_local"] == 1] == 0).all()
    print(f"{ref_mode}: {len(upd)} updates, {moved} key-frames moved after their result, "
          f"{int(upd['n_moved'].mean())} moved + {int(upd['n_new'].mean())} new rows per update on average")


@pytest.mark.gpu
@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
def test_engine_updates_across_restart_lost_and_record(ctx3, shift_data, ref_mode):
    """A restart starts a new sequence (sequence + 1, n_local 1, ids from 0) whose updates are a fresh engine's; a lost
    stream brings no update until it is restarted; a stream saved at frame 20 and loaded into another engine brings the
    updates of the uninterrupted run after the cut."""
    _, upd, rows, _ = run(ctx3, shift_data, 8, ref_mode)
    full = [(u, r) for u, r in zip(upd, rows) if u["stream"] == 0]
    # record: frames [0, 20) in engine A, the rest in engine B
    with _engine(ctx3, 8, ref_mode, n_streams=1) as a, _engine(ctx3, 8, ref_mode, n_streams=1) as b:
        for k in range(20):
            a.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        a.flush()
        a.poll()
        ua, ra = a.poll_map_updates()
        b.load_stream(0, a.save_stream(0))
        for k in range(20, N_FRAMES):
            b.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        b.flush()
        ub, rb = b.poll_map_updates()
    assert len(ub) > 0 and len(ua) + len(ub) == len(full)
    for (u, r), (uf, rf) in zip(list(zip(ua, ra)) + list(zip(ub, rb)), full):
        assert u.tobytes() == uf.tobytes() and r.tobytes() == rf.tobytes()
    # restart: stream 0 runs stream 3's frames after 12 frames of its own
    with _engine(ctx3, 8, ref_mode, n_streams=1) as e:
        mirror = Mirror()
        for k in range(12):
            e.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        e.restart(0)
        for k in range(N_FRAMES):
            e.push(0, shift_data[3][0][k], shift_data[3][1], tag=100 + k)
        e.flush()
        u2, r2 = e.poll_map_updates()
        mirror.fold(u2, r2)
        mirror.check(e, [1])
    with _engine(ctx3, 8, ref_mode, n_streams=1) as f:
        for k in range(N_FRAMES):
            f.push(0, shift_data[3][0][k], shift_data[3][1], tag=100 + k)
        f.flush()
        u3, r3 = f.poll_map_updates()
    old = u2["sequence"] == 0   # the frames pushed before the restart keep the updates of the uninterrupted run
    assert [(u.tobytes(), r.tobytes()) for u, r, o in zip(u2, r2, old) if o] == [(u.tobytes(), r.tobytes()) for u, r in full if u["frame"] < 12]
    new, new_rows = u2[~old], [r for r, o in zip(r2, old) if not o]
    assert (new["sequence"] == 1).all() and len(new) == len(u3)
    assert new[0]["n_local"] == 1 and new[0]["retired_frame"] == -1 and new[0]["n_moved"] == 0 and new_rows[0]["id"][0] == 0
    for u, r, uf, rf in zip(new, new_rows, u3, r3):
        assert u["frame"] - 12 == uf["frame"] and r.tobytes() == rf.tobytes()
        assert np.array_equal(u["local_frame"][:u["n_local"]] - 12, uf["local_frame"][:uf["n_local"]])
        assert u["retired_frame"] == (uf["retired_frame"] + 12 if uf["retired_frame"] >= 0 else -1)
        for k in ("n_local", "n_moved", "n_new", "T_cw"):
            assert np.array_equal(u[k], uf[k]), k
    # lost: min_inliers above any count loses the stream on its first tracked frame; a restart brings updates back
    with _engine(ctx3, 8, ref_mode, n_streams=1, min_inliers=10 ** 6) as e:
        for k in range(8):
            e.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        e.flush()
        res = e.poll()
        u, _ = e.poll_map_updates()
        assert list(res["status"]) == [1] + [2] * 7
        assert list(u["frame"]) == [0]
        e.restart(0)
        for k in range(8, 12):
            e.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        e.flush()
        e.poll()
        u, r = e.poll_map_updates()
        assert list(u["frame"]) == [8] and u[0]["sequence"] == 1 and r[0]["id"][0] == 0


@pytest.mark.gpu
def test_engine_map_update_calls_check_their_state(ctx3, shift_data):
    """set_map_updates while frames are queued, while a key-frame insertion is pending, while results or updates wait is
    rejected and changes nothing; an undersized poll moves nothing and says how many rows the first update needs; a
    poll with updates off is rejected; ygz_vo_poll leaves the updates queued."""
    from ygz_slam_b200 import capi, vo_native
    with _engine(ctx3, 8, "keyframe", map_updates=False, n_streams=1) as e:
        lib, h = e.lib, e.h
        out = np.zeros(16, vo_native.MAP_UPDATE_DTYPE)
        rows = np.zeros(16, capi.MAP_POINT_DTYPE)
        n, n_rows = C.c_int(0), C.c_size_t(0)
        assert lib.ygz_vo_poll_map_updates(h, out.ctypes.data, 16, C.byref(n), rows.ctypes.data, 16, C.byref(n_rows)) == ERR_INVALID
        e.push(0, shift_data[0][0][0], shift_data[0][1])
        assert lib.ygz_vo_set_map_updates(h, 1) == ERR_INVALID           # queued
        e.flush()
        assert lib.ygz_vo_set_map_updates(h, 1) == ERR_INVALID           # a result waits
        e.poll()
        e.set_map_updates(True)
        for k in range(1, 12):
            e.push(0, shift_data[0][0][k], shift_data[0][1])
        e.step()
        e.step()
        assert lib.ygz_vo_set_map_updates(h, 0) == ERR_INVALID
        e.flush()
        res = e.poll()                                                   # results only: the updates stay queued
        assert (res["status"] == 1).sum() >= 1
        assert lib.ygz_vo_set_map_updates(h, 0) == ERR_INVALID           # an update waits
        rc = lib.ygz_vo_poll_map_updates(h, out.ctypes.data, 16, C.byref(n), rows.ctypes.data, 16, C.byref(n_rows))
        assert rc == ERR_CAPACITY and n.value == 0 and n_rows.value > 16
        need = n_rows.value
        upd, r = e.poll_map_updates()
        assert len(upd) == (res["status"] == 1).sum() and upd[0]["n_moved"] + upd[0]["n_new"] == need == len(r[0])
        assert lib.ygz_vo_poll_map_updates(h, None, 0, C.byref(n), None, 0, C.byref(n_rows)) == 0 and n.value == 0
        e.set_map_updates(False)
        assert lib.ygz_vo_poll_map_updates(h, out.ctypes.data, 16, C.byref(n), rows.ctypes.data, 16, C.byref(n_rows)) == ERR_INVALID
