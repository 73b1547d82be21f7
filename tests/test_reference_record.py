"""Reference records of the previous-frame mode (ygzb_tracker_export_reference / ygzb_tracker_import_reference) and the
engine's hand-over of streams tracked against the previous frame (ygz_vo_run_handoff_ex with YGZB_TRACK_REF_PREVIOUS).

Setting of test_gpu_vo_previous.py: 3 shift_stream streams of 26 frames, key-frame policy 5 / 0.03 / 0.03.  A hand-over at
frame h must give exactly the results of a run split at h; an exported reference must be the tracker's live reference, with
the level 0 of the slot its pyramid is in; a record must survive export -> import -> export bit for bit, and the stream must
then track on exactly as in its source; a bad record must be rejected without touching the tracker."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from ygz_slam_b200 import se3, synth, vo

ROOT = Path(__file__).resolve().parent.parent
N_STREAMS, N_FRAMES = 3, 26
POLICY = (5, 0.03, 0.03)
KW = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)
K = np.array([synth.FX, synth.FY, synth.CX, synth.CY])


def test_reference_record_layout_matches_the_header(tmp_path):
    """capi.ReferenceRecord has the size and field offsets of ygzb_reference_record as a C compiler lays it out, and the
    capacity constant is the header's."""
    from ygz_slam_b200 import capi
    fields = [f for f, _ in capi.ReferenceRecord._fields_]
    src = tmp_path / "layout.c"
    body = "\n".join(f'    printf("%s %%zu\\n", offsetof(ygzb_reference_record, {f}));' % f for f in fields)
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "ygz_b200.h"\nint main(void) {\n'
                   '    printf("sizeof %%zu\\n", sizeof(ygzb_reference_record));\n'
                   '    printf("per_cell %%d\\n", YGZB_TRACK_REF_FEATURES_PER_CELL);\n%s\n    return 0;\n}\n' % body)
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", f"-I{ROOT / 'include'}", str(src), "-o", str(exe)], check=True,
                   capture_output=True, text=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(got["sizeof"]) == C.sizeof(capi.ReferenceRecord)
    assert int(got["per_cell"]) == capi.REF_FEATURES_PER_CELL
    for f in fields:
        assert int(got[f]) == getattr(capi.ReferenceRecord, f).offset, f


def test_previous_mode_with_the_stages_engine_is_still_rejected():
    from ygz_slam_b200 import vo_native
    with pytest.raises(ValueError):
        vo_native.run(None, np.zeros((1, 1, 480, 640), np.uint8), [np.ones((480, 640))], engine="stages", ref_mode="previous")


@pytest.fixture(scope="module")
def streams():
    return [synth.shift_stream(s, N_FRAMES) for s in range(N_STREAMS)]


@pytest.fixture(scope="module")
def keyframe_frames(ctx3, streams):
    """Frames at which stream 0 of the Python loop in previous-frame mode inserts a key-frame."""
    be = vo.GpuBackend(ctx3, N_STREAMS * vo.VisualOdometry.SLOTS_PER_STREAM)
    V = vo.VisualOdometry(be, N_STREAMS, ref_mode="previous", **KW)
    out = []
    for k in range(N_FRAMES):
        n = V.streams[0].stats["keyframes"]
        V.add_frames([streams[s][0][k] for s in range(N_STREAMS)], [streams[s][1] for s in range(N_STREAMS)], k)
        if V.streams[0].stats["keyframes"] > n:
            out.append(k)
    be.fr.close()
    return out


def _run(ctx, streams, **kw):
    from ygz_slam_b200 import vo_native
    return vo_native.run(ctx, [d[0] for d in streams], [d[1] for d in streams], *POLICY, ref_mode="previous", **kw)


def _handoff_frames(keyframe_frames):
    kf = keyframe_frames[2]   # a key-frame after the first local BA
    # h = 1: the reference is the first key-frame, nothing tracked; kf + 1: the key-frame inserted at kf is the reference, its
    # pyramid in a key-frame slot; kf + 3: inside the key-frame interval (5 frames), the previous frame in the reference slot
    return {"first": 1, "after_keyframe": kf + 1, "inside_interval": kf + 3}


def _pose_err(A, B):
    return float(np.linalg.norm(se3.se3_log(se3.mul(A, se3.inv(B)))))


@pytest.mark.gpu
@pytest.mark.parametrize("window", [1, 8])
@pytest.mark.parametrize("where", ["first", "after_keyframe", "inside_interval"])
def test_engine_handoff_in_previous_mode_is_bit_identical_to_a_split_run(ctx3, streams, keyframe_frames, window, where):
    h = _handoff_frames(keyframe_frames)[where]
    assert 0 < h < N_FRAMES - 5
    traj_a, stats_a, _ = _run(ctx3, streams, warm=h, window=window)
    traj_b, stats_b, _, maps, refs = _run(ctx3, streams, warm=h, window=window, handoff=h, return_maps=True)
    assert np.array_equal(traj_a, traj_b)
    assert stats_a == stats_b
    for s in range(N_STREAMS):
        assert not stats_b[s]["lost"] and stats_b[s]["keyframes"] >= 4 and stats_b[s]["ba"] >= 3
        assert _pose_err(traj_b[s, -1], streams[s][2][-1]) < 3e-3
    # the hand-over point is what its name says (stream 0): the pose of the reference, and where its image comes from
    kfs, ref = maps[0].keyframes(), refs[0]
    assert ref.header["n"] > 0 and ref.header["capacity"] == 5 * ctx3.n_cells
    newest = kfs[-1]
    if where == "first":
        assert len(kfs) == 1
    if where in ("first", "after_keyframe"):
        assert np.array_equal(ref.T_cw, newest["T_cw"]) and np.array_equal(ref.a["image"], newest["image"])
        assert np.array_equal(ref.a["image"], streams[0][0][h - 1])
    else:
        assert not np.array_equal(ref.T_cw, newest["T_cw"])
        assert np.array_equal(ref.a["image"], streams[0][0][h - 1])
        assert not np.array_equal(ref.a["image"], newest["image"])
    assert np.array_equal(ref.T_cw, traj_b[0, h - 1])


@pytest.mark.gpu
def test_fast_stream_survives_a_handoff_in_previous_mode(ctx3):
    """Every 4th frame of shift_stream at the reference's key-frame defaults: key-frame mode loses these streams; handed over
    mid-stream in previous mode they are tracked to the end, exactly as in the run split at the same frame."""
    from ygz_slam_b200 import vo_native
    data = [synth.shift_stream(s, 80) for s in range(2)]
    frames, depths = [d[0][::4] for d in data], [d[1] for d in data]
    h = 10
    _, stats_k, _ = vo_native.run(ctx3, frames, depths, window=8)
    traj_a, stats_a, _ = vo_native.run(ctx3, frames, depths, window=8, warm=h, ref_mode="previous")
    traj_b, stats_b, _ = vo_native.run(ctx3, frames, depths, window=8, warm=h, handoff=h, ref_mode="previous")
    assert np.array_equal(traj_a, traj_b) and stats_a == stats_b
    for s in range(2):
        assert stats_k[s]["lost"]
        assert not stats_b[s]["lost"] and stats_b[s]["keyframes"] >= 2
        assert _pose_err(traj_b[s, -1], data[s][2][::4][-1]) < 3e-3


# ---- a previous-mode tracker driven by hand: 3 streams, frame slots s*4 .., key-frame slots 12 + s*4 + entry, reference
#      slots 24 + s
STAGES = ("keyframe0", "tracked", "keyframe1")


def _tracker(ctx3, streams, ref_slots=(24, 25, 26)):
    fr = ctx3.frames(27)
    tr = fr.tracker(N_STREAMS, 12, K)
    tr.set_reference_mode("previous", list(ref_slots))
    for s in range(N_STREAMS):
        tr.set_depth(s, streams[s][1])
    return fr, tr


def _drive(ctx3, streams, stage):
    """A source tracker at `stage`: after the first key-frame of every stream; after three frames tracked in one batch (each
    against the one before); after a second key-frame made from the last of them, with a local BA.  Returns the tracker,
    its frame pool and the ring entries and mp0 of every stream's key-frames."""
    fr, tr = _tracker(ctx3, streams)
    for s in range(N_STREAMS):
        tr.upload(s * 4, streams[s][0][0])
    kres = tr.make_keyframes([dict(stream=s, frame_slot=s * 4, kf_slot=12 + s * 4, entry=0, track_job=-1, local_entry=[0])
                              for s in range(N_STREAMS)])
    info = dict(entries=[0], next_mp=[r["n_features"] for r in kres], next_frame=1)
    if stage == "keyframe0":
        return fr, tr, info
    for s in range(N_STREAMS):
        tr.upload(s * 4, streams[s][0][1:4])
    res = tr.track([(s, s * 4 + t, [0]) for s in range(N_STREAMS) for t in range(3)])
    assert all(r["aligned"] for r in res)
    info["next_frame"] = 4
    if stage == "tracked":
        return fr, tr, info
    kres = tr.make_keyframes([dict(stream=s, frame_slot=s * 4 + 2, kf_slot=12 + s * 4 + 1, entry=1, track_job=3 * s + 2,
                                   local_entry=[0, 1], run_ba=1, mp0=info["next_mp"][s]) for s in range(N_STREAMS)])
    assert all(r["ba_points"] > 0 for r in kres)
    info["entries"] = [0, 1]
    info["next_mp"] = [m + r["n_features"] for m, r in zip(info["next_mp"], kres)]
    return fr, tr, info


def _same_reference(a, b):
    assert a.header == b.header
    assert np.array_equal(np.array(a.rec.T_cw), np.array(b.rec.T_cw))
    for k in ("px", "depth", "image"):
        assert np.array_equal(a.a[k], b.a[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("stage", STAGES)
def test_exported_reference_is_the_live_reference(ctx3, streams, stage):
    fr, tr, info = _drive(ctx3, streams, stage)
    for s in range(N_STREAMS):
        live = tr.debug_reference(s)
        rec = tr.export_reference(s)
        n = rec.header["n"]
        assert rec.header == dict(width=640, height=480, cells=ctx3.n_cells, n_levels=3, K=tuple(K), capacity=5 * ctx3.n_cells, n=n)
        assert n == len(live["depth"]) > 0
        assert np.array_equal(rec.T_cw, live["T_cw"])
        assert np.array_equal(rec.a["px"][:n], live["px"]) and np.array_equal(rec.a["depth"][:n], live["depth"])
        assert not rec.a["px"][n:].any() and not rec.a["depth"][n:].any()
        assert np.array_equal(rec.a["image"], fr.download_level(live["slot"], 0))
        want_slot = {"keyframe0": 12 + s * 4, "tracked": 24 + s, "keyframe1": 12 + s * 4 + 1}[stage]
        want_frame = {"keyframe0": 0, "tracked": 3, "keyframe1": 3}[stage]
        assert live["slot"] == want_slot and np.array_equal(rec.a["image"], streams[s][0][want_frame])
    tr.close()
    fr.close()


def _hand_over(ctx3, streams, tr, info, src, dst, ref_slots=(20, 21, 22)):
    """Stream `src` of tracker `tr` into stream `dst` of a fresh previous-mode tracker (other key-frame and reference slots):
    map, then reference.  Returns the destination, its frame pool, the records and the destination's key-frame slots."""
    fr2, tr2 = _tracker(ctx3, streams, ref_slots)
    tr2.set_depth(dst, streams[src][1])
    entries = np.array(info["entries"], np.int32)
    slots = 16 - entries   # not the source's slots
    rec = tr.export(src, entries)
    ref = tr.export_reference(src)
    tr2.import_(dst, entries, slots, rec)
    tr2.import_reference(dst, ref)
    return fr2, tr2, rec, ref, slots


@pytest.mark.gpu
@pytest.mark.parametrize("stage", STAGES)
def test_round_trip_is_byte_identical(ctx3, streams, stage):
    """Export -> import into stream 2 of another tracker -> export again: the reference record at full capacity, image
    included, is byte-identical; the image now lives in the destination's reference slot; the other streams have none."""
    from ygz_slam_b200 import YgzbError
    fr, tr, info = _drive(ctx3, streams, stage)
    fr2, tr2, rec, ref, _ = _hand_over(ctx3, streams, tr, info, 0, 2)
    again = tr2.export_reference(2)
    _same_reference(ref, again)
    assert tr2.debug_reference(2)["slot"] == 22
    assert np.array_equal(fr2.download_level(22, 0), ref.a["image"])
    _same_reference(ref, tr.export_reference(0))   # the source is unchanged by its exports
    for s in (0, 1):
        with pytest.raises(YgzbError, match=r"rc=-1"):
            tr2.export_reference(s)
    for t in (tr, tr2):
        t.close()
    fr.close()
    fr2.close()


@pytest.mark.gpu
@pytest.mark.parametrize("stage", STAGES)
def test_tracking_continues_identically_after_an_import(ctx3, streams, stage):
    """The same next frames tracked in the source (stream 0) and in the destination (stream 2): identical result records and
    debug_job state, identical next reference; a key-frame made from the last of them: identical key-frame results."""
    fr, tr, info = _drive(ctx3, streams, stage)
    fr2, tr2, *_ = _hand_over(ctx3, streams, tr, info, 0, 2)
    k = info["next_frame"]
    nxt = streams[0][0][k:k + 2]
    tr.upload(0, nxt)
    tr2.upload(8, nxt)
    res_a = tr.track([(0, t, info["entries"]) for t in range(2)])
    res_b = tr2.track([(2, 8 + t, info["entries"]) for t in range(2)])
    for a, b in zip(res_a, res_b):
        assert a.keys() == b.keys()
        for key in a:
            assert np.array_equal(a[key], b[key]), key
    assert all(r["aligned"] and r["n_inliers"] > 100 for r in res_a)
    for j in range(2):
        da, db = tr.debug_job(j), tr2.debug_job(j)
        # (cand_px is written for candidates only: elsewhere it holds what earlier batches of each tracker left there)
        da["cand_px"], db["cand_px"] = da["cand_px"][da["cand_ok"]], db["cand_px"][db["cand_ok"]]
        for key in da:
            assert np.array_equal(da[key], db[key]), (j, key)
    ra, rb = tr.debug_reference(0), tr2.debug_reference(2)
    for key in ("T_cw", "px", "depth"):
        assert np.array_equal(ra[key], rb[key]), key
    # a key-frame from the last frame (entry 2 is free in both rings), with a local BA when there are two local key-frames
    local = info["entries"] + [2]
    job = dict(frame_slot=1, entry=2, track_job=1, local_entry=local, run_ba=1, mp0=info["next_mp"][0])
    ka = tr.make_keyframes([dict(job, stream=0, kf_slot=12 + 2)])
    kb = tr2.make_keyframes([dict(job, stream=2, frame_slot=9, kf_slot=14)])
    for key in ka[0]:
        assert np.array_equal(ka[0][key], kb[0][key]), key
    ra, rb = tr.export_reference(0), tr2.export_reference(2)
    _same_reference(ra, rb)
    for t in (tr, tr2):
        t.close()
    fr.close()
    fr2.close()


def _bad_copy(ref, **changes):
    r = ref.copy()
    for k, v in changes.items():
        v(r) if callable(v) else setattr(r.rec, k, v)
    return r


@pytest.mark.gpu
def test_bad_reference_records_leave_the_tracker_untouched(ctx3, streams):
    from ygz_slam_b200 import YgzbError
    fr, tr, info = _drive(ctx3, streams, "tracked")
    fr2, tr2, rec, ref, slots = _hand_over(ctx3, streams, tr, info, 0, 1)
    before = tr2.debug_reference(1)
    cap = ref.rec.capacity

    def unchanged():
        now = tr2.debug_reference(1)
        assert now["slot"] == before["slot"]
        for key in ("T_cw", "px", "depth"):
            assert np.array_equal(now[key], before[key]), key

    imports = {
        "stream out of range": (3, ref),
        "negative stream": (-1, ref),
        "capacity below the store's": (1, _bad_copy(ref, capacity=cap - 1)),
        "negative n": (1, _bad_copy(ref, n=-1)),
        "n over capacity": (1, _bad_copy(ref, n=cap + 1)),
        "width": (1, _bad_copy(ref, width=641)),
        "height": (1, _bad_copy(ref, height=479)),
        "cells": (1, _bad_copy(ref, cells=ctx3.n_cells + 1)),
        "levels": (1, _bad_copy(ref, n_levels=4)),
        "K": (1, _bad_copy(ref, K=lambda r: r.rec.K.__setitem__(2, synth.CX + 1e-9))),
        "missing px": (1, _bad_copy(ref, px=None)),
        "missing depth": (1, _bad_copy(ref, depth=None)),
        "missing image": (1, _bad_copy(ref, image=None)),
    }
    for name, (stream, r) in imports.items():
        with pytest.raises(YgzbError, match=r"rc=-1"):
            tr2.import_reference(stream, r)
        unchanged()
    from ygz_slam_b200.capi import ReferenceBuffers
    sentinel = ReferenceBuffers(640, 480, ctx3.n_cells)
    exports = {
        "stream out of range": (3, sentinel),
        "no reference yet": (0, sentinel),
        "capacity below the store's": (1, _bad_copy(sentinel, capacity=cap - 1)),
        "missing px": (1, _bad_copy(sentinel, px=None)),
        "missing depth": (1, _bad_copy(sentinel, depth=None)),
        "missing image": (1, _bad_copy(sentinel, image=None)),
    }
    for name, (stream, out) in exports.items():
        with pytest.raises(YgzbError, match=r"rc=-1"):
            tr2.export_reference(stream, out=out)
        assert out.header["width"] == 0 and not out.a["px"].any(), name   # nothing written
        unchanged()
    # a tracker in key-frame mode has no reference store
    fr3 = ctx3.frames(8)
    tr3 = fr3.tracker(N_STREAMS, 8, K)
    with pytest.raises(YgzbError, match=r"rc=-1"):
        tr3.import_reference(1, ref)
    with pytest.raises(YgzbError, match=r"rc=-1"):
        tr3.export_reference(1, out=sentinel)
    tr3.close()
    fr3.close()
    # the destination tracks its next frame exactly as the source does
    k = info["next_frame"]
    tr.upload(0, streams[0][0][k])
    tr2.upload(8, streams[0][0][k])
    a, b = tr.track([(0, 0, info["entries"])])[0], tr2.track([(1, 8, info["entries"])])[0]
    for key in a:
        assert np.array_equal(a[key], b[key]), key
    for t in (tr, tr2):
        t.close()
    fr.close()
    fr2.close()
