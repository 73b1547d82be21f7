"""Restarting a stream of the streaming engine (ygz_vo_restart, vo_native.Engine.restart) and the start pose of a stream's
first key-frame (ygzb_tracker_set_start_pose, vo.VisualOdometry.set_start_pose).  A restart is a barrier: the frames pushed
before it keep their results, the first frame pushed after it becomes a first key-frame at the given pose, and from there
the stream is a fresh one.  A start pose T0 moves the world frame: every pose of the sequence becomes T_cw * T0."""
import ctypes as C

import numpy as np
import pytest

from ygz_slam_b200 import se3, synth, vo

POLICY = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)   # test_vo_stream's key-frame policy
ERR_INVALID = -1
N_FRAMES = 30
# a start pose with a rotation of 0.31 rad and a translation of 1.05 m
T0 = np.concatenate([synth.so3_exp(np.array([0.1, -0.25, 0.15])), np.array([[0.6], [-0.5], [0.7]])], 1)
# A sequence started at T0 is the identity run moved by T0 up to the solvers' convergence, not to the last bit.  The sparse
# alignment works on the motion relative to its reference and is exact (1.7e-16 on the first frame of shift stream 0).  The
# two solvers that see world coordinates are not:
#  - pose-only (Ceres LM, oracle/ba.cpp ora_pose_only / ceres_lm) optimises pose = [t; angle-axis] with ADDITIVE updates,
#    Jacobi scaling and a trust radius; under T_cw -> T_cw * T0 those coordinates and scales change, so the iterations take
#    another path and stop, by the function / parameter tolerances, at another point near the same optimum (pose-only
#    alone: 1.1e-9 on synth.pose_only_scene);
#  - the local BA's pose update is left-multiplicative (exp(delta) * T, world-frame invariant), but computeLambdaInit takes
#    max |diag H| over the point blocks as well, whose diagonals are in world coordinates (oracle/ba.cpp:188-194), so the
#    first damping and the at most 10 LM trials that follow differ;
# and the odd borderline direct projection or pose-only inlier flips with the last bits.  Measured on the oracle loop
# over 20 frames of shift streams 0-3: 2.9e-5, 1.5e-5, 2.2e-6, 2.3e-6; the engine on 3 streams x 30 frames (H100 80GB HBM3
# at 700 W): 3.2e-5 and 4.6e-5 in the two reference modes.
MOVED_TOL = 1e-4


def _pose_err(A, B):
    return float(np.linalg.norm(se3.se3_log(se3.mul(A, se3.inv(B)))))


def _moved(T):
    """T_cw of a frame whose sequence started at the identity, for the same sequence started at T0."""
    return se3.mul(T, T0)


def _bad_poses():
    nan = T0.copy(); nan[1, 3] = np.nan
    inf = T0.copy(); inf[0, 0] = np.inf
    scaled = T0.copy(); scaled[:, :3] *= 1 + 1e-5          # not orthonormal
    mirror = T0.copy(); mirror[:, 0] = -mirror[:, 0]          # orthonormal, det -1
    sheared = T0.copy(); sheared[0, 1] += 1e-5
    return dict(nan=nan, inf=inf, scaled=scaled, mirror=mirror, sheared=sheared)


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_header_declares_restart():
    """ygz_vo_restart and ygzb_tracker_set_start_pose are declared (test_vo_stream / test_abi compile and link every
    declared entry point as pedantic C99) and bound."""
    from test_abi import declared_symbols
    from test_vo_stream import declared_stream_symbols
    from ygz_slam_b200 import capi
    assert "ygz_vo_restart" in declared_stream_symbols()
    assert "ygzb_tracker_set_start_pose" in declared_symbols() and "ygzb_tracker_set_start_pose" in capi.EXPORTS


def test_loop_start_pose_is_checked():
    V = vo.VisualOdometry(None, 2)
    for name, T in _bad_poses().items():
        with pytest.raises(ValueError):
            V.set_start_pose(0, T)
    assert np.array_equal(V.streams[0].start, np.eye(4)[:3])
    V.set_start_pose(1, T0)
    assert np.array_equal(V.streams[1].start, T0) and np.array_equal(V.streams[0].start, np.eye(4)[:3])


def _same_decisions(got, want):
    """Key-frames and local BAs equal; the other counters within 0.1 %: in another world frame the last bits of the
    arithmetic differ, which can flip a borderline direct projection or pose-only inlier (as between the GPU and the
    oracle loop, test_vo.py)."""
    assert got["keyframes"] == want["keyframes"] and got["ba"] == want["ba"]
    for key in ("candidates", "projected", "inliers"):
        assert abs(got[key] - want[key]) <= 1e-3 * want[key], key


def _loop(backend, data, start=None, ref_mode="keyframe"):
    S = len(data)
    V = vo.VisualOdometry(backend, S, ref_mode=ref_mode, **POLICY)
    if start is not None:
        for s_ in range(S):
            V.set_start_pose(s_, start)
    for k in range(len(data[0][0])):
        V.add_frames([d[0][k] for d in data], [d[1] for d in data], k)
    return V


def test_loop_start_pose_on_oracle_moves_the_world_frame(oracle):
    """The Python loop on the CPU oracle, shift stream 0 started at T0: every pose is the identity run's T_cw * T0 within
    MOVED_TOL, with the same key-frames and BAs, and follows the ground truth moved by T0."""
    from oracle.vo_backend import OracleBackend
    data = [synth.shift_stream(0, 20)]
    Vi = _loop(OracleBackend(oracle), data)
    Vt = _loop(OracleBackend(oracle), data, start=T0)
    si, st = Vi.streams[0], Vt.streams[0]
    assert not si.lost and not st.lost and si.stats["keyframes"] >= 3
    _same_decisions(st.stats, si.stats)
    assert np.array_equal(st.trajectory[0], T0)
    worst = max(_pose_err(Tt, _moved(Ti)) for Ti, Tt in zip(si.trajectory, st.trajectory))
    print(f"largest difference to the identity run moved by T0: {worst:.2e}")
    assert worst < MOVED_TOL
    for k, gt in enumerate(data[0][2]):
        assert _pose_err(st.trajectory[k], _moved(gt)) < 3e-3, k


# ---- GPU --------------------------------------------------------------------------------------------------------------
MODES = pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
WINDOWS = pytest.mark.parametrize("window", [1, 8])


@pytest.fixture(scope="module")
def shift_data():
    return [synth.shift_stream(s_, N_FRAMES) for s_ in range(4)]


_BATCH = {}


def batch(ctx, data, n_streams, window, ref_mode):
    """ygz_vo_run_ex on the first n_streams shift streams (no restart): trajectory (S, n, 3, 4) and stats."""
    key = (n_streams, window, ref_mode)
    if key not in _BATCH:
        from ygz_slam_b200 import vo_native
        traj, stats, _ = vo_native.run(ctx, [d[0] for d in data[:n_streams]], [d[1] for d in data[:n_streams]], window=window,
                                       ref_mode=ref_mode, **POLICY)
        _BATCH[key] = (traj, stats)
    return _BATCH[key]


def results_of(res, stream):
    """(poses (n, 3, 4), status, n_inliers, tags) of one stream's results, checked to be in frame order from 0."""
    r = res[res["stream"] == stream]
    assert r["frame"].tolist() == list(range(len(r)))
    return r["T_cw"].reshape(-1, 3, 4), r["status"], r["n_inliers"], r["tag"]


def lock_step(ctx, data, S, window, ref_mode, before=None):
    """S streams pushed in lock step with their depth maps and flushed; `before(eng)` runs before the first push."""
    from ygz_slam_b200 import vo_native
    with vo_native.Engine(ctx, S, window=window, ref_mode=ref_mode, **POLICY) as eng:
        if before:
            before(eng)
        for k in range(N_FRAMES):
            for s_ in range(S):
                eng.push(s_, data[s_][0][k], data[s_][1], tag=1000 * s_ + k)
        eng.flush()
        return eng.poll(), [eng.stats(s_) for s_ in range(S)], [eng.restarts(s_) for s_ in range(S)]


@pytest.mark.gpu
@MODES
@WINDOWS
def test_identity_restart_before_first_push_changes_nothing(ctx3, shift_data, window, ref_mode):
    ref_traj, ref_stats = batch(ctx3, shift_data, 3, window, ref_mode)
    res, stats, restarts = lock_step(ctx3, shift_data, 3, window, ref_mode, before=lambda e: [e.restart(s_) for s_ in range(3)])
    for s_ in range(3):
        T, status, _, _ = results_of(res, s_)
        assert np.array_equal(T, ref_traj[s_]) and stats[s_] == ref_stats[s_] and restarts[s_] == 0, s_
        assert status[0] == 1 and (status == 2).sum() == 0


_LOOP = {}


@pytest.mark.gpu
@MODES
@WINDOWS
def test_start_pose(ctx3, oracle, shift_data, window, ref_mode):
    """3 streams started at T0 (a second restart before the first push wins over the first): against the oracle-driven
    Python loop started at T0 within the loop's tolerance (1e-4; 5e-4 in previous-frame mode, see
    test_vo_ref_modes.PREVIOUS_MODE_POSE_TOL), against the identity run moved by T0 within MOVED_TOL, against the ground
    truth moved by T0 within 3e-3; the same key-frames and BAs as both."""
    from test_vo_ref_modes import PREVIOUS_MODE_POSE_TOL, DepthOracleBackend
    S = 3
    if ref_mode not in _LOOP:
        _LOOP[ref_mode] = _loop(DepthOracleBackend(oracle), shift_data[:S], start=T0, ref_mode=ref_mode)
    V = _LOOP[ref_mode]
    tol_loop = 1e-4 if ref_mode == "keyframe" else PREVIOUS_MODE_POSE_TOL
    ident, ref_stats = batch(ctx3, shift_data, S, window, ref_mode)

    def start(eng):
        for s_ in range(S):
            eng.restart(s_, np.eye(4)[:3] + 0.0)
            eng.restart(s_, T0)
    res, stats, restarts = lock_step(ctx3, shift_data, S, window, ref_mode, before=start)
    worst = 0.0
    for s_ in range(S):
        T, status, _, _ = results_of(res, s_)
        _same_decisions(stats[s_], ref_stats[s_])
        _same_decisions(stats[s_], V.streams[s_].stats)
        assert stats[s_]["lost"] == 0 and restarts[s_] == 0 and (status == 1).sum() == stats[s_]["keyframes"], s_
        assert np.array_equal(T[0], T0)
        for k in range(N_FRAMES):
            worst = max(worst, _pose_err(T[k], _moved(ident[s_][k])))
            assert _pose_err(T[k], V.streams[s_].trajectory[k]) < tol_loop, (s_, k)
            assert _pose_err(T[k], _moved(shift_data[s_][2][k])) < 3e-3, (s_, k)
    print(f"largest difference to the identity run moved by T0: {worst:.2e}")
    assert worst < MOVED_TOL


def _check_new_sequence(ctx, res, stats, restarts, shift_data, window, ref_mode, n_old):
    """stream 0: frames [0, n_old) of shift stream 0, then shift stream 3; streams 1 and 2: shift streams 1 and 2."""
    ref3, _ = batch(ctx, shift_data, 3, window, ref_mode)
    ref4, _ = batch(ctx, shift_data, 4, window, ref_mode)
    T, status, _, tags = results_of(res, 0)
    assert tags.tolist() == list(range(n_old)) + [3000 + k for k in range(N_FRAMES)]   # every tag once, in order
    assert np.array_equal(T[:n_old], ref3[0][:n_old])          # the old sequence keeps its results
    assert np.array_equal(T[n_old:], ref4[3])                  # the new one is a fresh stream fed shift stream 3
    assert status[n_old] == 1 and (status == 2).sum() == 0
    for s_ in (1, 2):
        assert np.array_equal(results_of(res, s_)[0], ref3[s_]), s_
    assert restarts == [1, 0, 0] and stats[0]["lost"] == 0


@pytest.mark.gpu
@MODES
@WINDOWS
def test_new_sequence_on_a_live_stream(ctx3, shift_data, window, ref_mode):
    """Stream 0 runs 15 frames of shift stream 0, is restarted while they are all still queued and runs 30 frames of shift
    stream 3; streams 1 and 2 run undisturbed.  The new sequence is bit-identical to a fresh engine's stream fed shift
    stream 3, the old frames and the other streams to the run without a restart; the export holds the new key-frames only,
    and its import round trip is byte-identical."""
    from ygz_slam_b200 import capi, vo_native
    lib = vo_native._lib()
    n_old = 15
    with vo_native.Engine(ctx3, 3, window=window, ref_mode=ref_mode, **POLICY) as eng:
        for k in range(N_FRAMES):
            for s_ in (1, 2):
                eng.push(s_, shift_data[s_][0][k], shift_data[s_][1], tag=1000 * s_ + k)
            if k < n_old:
                eng.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        eng.restart(0)
        img = shift_data[3][0][0]
        assert lib.ygz_vo_push(eng.h, 0, img.ctypes.data, None, 0) == ERR_INVALID   # a new sequence needs a depth map
        for k in range(N_FRAMES):
            eng.push(0, shift_data[3][0][k], shift_data[3][1] if k == 0 else None, tag=3000 + k)
        eng.flush()
        res = eng.poll()
        stats = [eng.stats(s_) for s_ in range(3)]
        restarts = [eng.restarts(s_) for s_ in range(3)]
        rec = eng.export_map(0)
    _check_new_sequence(ctx3, res, stats, restarts, shift_data, window, ref_mode, n_old)
    # the export: the new sequence's key-frames only -- those of a fresh stream fed shift stream 3
    with vo_native.Engine(ctx3, 1, window=window, ref_mode=ref_mode, **POLICY) as fresh:
        for k in range(N_FRAMES):
            fresh.push(0, shift_data[3][0][k], shift_data[3][1], tag=k)
        fresh.flush()
        fresh.poll()
        want = fresh.export_map(0)
    assert rec.header == want.header
    for key in capi._MAP_ARRAYS:
        assert np.array_equal(rec.a[key], want.a[key]), key   # map-point ids (mp0) included: numbered from 0 again
    # the import round trip of that record
    n = rec.rec.n_keyframes
    entries = rec.a["entry"][:n].copy()
    slots = 19 - np.arange(n)
    fr = ctx3.frames(3 * 4 + 8)
    tr = fr.tracker(3, 8, rec.header["K"])
    tr.import_(2, entries, slots, rec)
    again = tr.export(2, entries)
    assert again.header == rec.header
    for key in capi._MAP_ARRAYS:
        assert np.array_equal(again.a[key], rec.a[key]), key
    tr.close()
    fr.close()


@pytest.mark.gpu
@MODES
def test_new_sequence_at_random_pacing(ctx3, shift_data, ref_mode):
    """The live-stream restart with seeded random pushes and steps at window 8.  The last 3 old frames of stream 0 are pushed
    together and the restart follows with no step in between, so they are still queued when it is issued (the results,
    polled after every step, show at least 3 old frames without a result); the results are those of
    test_new_sequence_on_a_live_stream."""
    from ygz_slam_b200 import vo_native
    n_old, n_last, window = 15, 3, 8
    rng = np.random.default_rng(11)
    seq0 = [(shift_data[0], k, k) for k in range(n_old)] + [(shift_data[3], k, 3000 + k) for k in range(N_FRAMES)]
    with vo_native.Engine(ctx3, 3, window=window, ref_mode=ref_mode, **POLICY) as eng:
        pushed, results, restarted = [0, 0, 0], [], False
        lengths = [len(seq0), N_FRAMES, N_FRAMES]

        def push(s_):
            if s_ == 0:
                d, k, tag = seq0[pushed[0]]
                eng.push(0, d[0][k], d[1] if k == 0 or rng.random() < 0.5 else None, tag=tag)
            else:
                k = pushed[s_]
                eng.push(s_, shift_data[s_][0][k], shift_data[s_][1], tag=1000 * s_ + k)
            pushed[s_] += 1

        while any(p < n for p, n in zip(pushed, lengths)):
            if rng.random() < 0.3:
                eng.step()
                results.append(eng.poll())
                continue
            s_ = int(rng.integers(3))
            for _ in range(int(rng.integers(1, 4))):
                if pushed[s_] >= lengths[s_]:
                    break
                if s_ == 0 and not restarted and pushed[0] >= n_old - n_last:
                    while pushed[0] < n_old:   # the last old frames, then the restart, no step in between
                        push(0)
                    done = sum(int((r["stream"] == 0).sum()) for r in results)
                    assert pushed[0] - done >= n_last, (pushed[0], done)
                    eng.restart(0)
                    restarted = True
                push(s_)
        assert restarted
        eng.flush()
        results.append(eng.poll())
        stats = [eng.stats(s_) for s_ in range(3)]
        restarts = [eng.restarts(s_) for s_ in range(3)]
    _check_new_sequence(ctx3, np.concatenate(results), stats, restarts, shift_data, window, ref_mode, n_old)


@pytest.mark.gpu
@MODES
def test_restart_behind_a_pending_keyframe(ctx3, shift_data, ref_mode):
    """Window 1, one push and one step at a time: stream 0 is restarted right after the step that decided a key-frame, whose
    insertion is still pending.  Its KEYFRAME result comes first, with the pose of the run without a restart; the new
    sequence is that of a fresh stream."""
    from ygz_slam_b200 import vo_native
    ref3, _ = batch(ctx3, shift_data, 3, 1, ref_mode)
    ref4, _ = batch(ctx3, shift_data, 4, 1, ref_mode)
    with vo_native.Engine(ctx3, 1, window=1, ref_mode=ref_mode, **POLICY) as eng:
        old = []
        for k in range(N_FRAMES):
            eng.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
            eng.step()
            old.append(eng.poll())
            if k > 0 and sum(len(r) for r in old) == k:   # frame k is neither final nor queued: its key-frame insertion is pending
                break
        kf = k
        assert 0 < kf < N_FRAMES - 1
        eng.restart(0)
        for j in range(N_FRAMES):
            eng.push(0, shift_data[3][0][j], shift_data[3][1], tag=3000 + j)
        eng.flush()
        res = np.concatenate(old + [eng.poll()])
    T, status, _, tags = results_of(res, 0)
    assert tags.tolist() == list(range(kf + 1)) + [3000 + j for j in range(N_FRAMES)]
    assert status[kf] == 1 and np.array_equal(T[:kf + 1], ref3[0][:kf + 1])   # the pending key-frame completes first
    assert status[kf + 1] == 1 and np.array_equal(T[kf + 1:], ref4[3])
    assert status[0] == 1 and (status[1:kf] == 0).all()


def _injected(shift_data, k_bad):
    """shift stream 0 with frame k_bad replaced by frame k_bad of shift stream 1 (another texture)."""
    frames = shift_data[0][0].copy()
    frames[k_bad] = shift_data[1][0][k_bad]
    return frames


@pytest.mark.gpu
@MODES
@WINDOWS
@pytest.mark.parametrize("n_lost_queued", [0, 3])
def test_recovery_after_lost(ctx3, shift_data, window, ref_mode, n_lost_queued):
    """One frame of another texture loses a stream; it is restarted at the ground-truth pose of the first frame pushed after
    the restart.  With n_lost_queued = 0 the loss has been flushed before the restart; with 3, three more frames of the old
    sequence are pushed behind the bad one and the restart follows with no step at all, so the loss is found with those
    frames queued ahead of the restart: they come back LOST with the last pose.  The old frames get the results of the old
    sequence alone; later results are not LOST, are bit-identical to a fresh engine started at that pose on the same frames
    and follow the ground truth; the counters are those of the two segments added up, with lost = 0 and one restart."""
    from ygz_slam_b200 import vo_native
    k_bad = 8
    k_new = k_bad + 1 + n_lost_queued
    frames, depth, gts = _injected(shift_data, k_bad), shift_data[0][1], shift_data[0][2]
    T_next = gts[k_new]

    def engine():
        return vo_native.Engine(ctx3, 1, window=window, ref_mode=ref_mode, **POLICY)
    with engine() as seg:   # the old sequence alone
        for k in range(k_new):
            seg.push(0, frames[k], depth, tag=k)
        seg.flush()
        want_old = seg.poll()
        lost_stats = seg.stats(0)
    status = want_old["status"]
    assert lost_stats["lost"] == 1 and (status[:k_bad] != 2).all() and (status[k_bad:] == 2).all()
    assert (want_old["T_cw"][k_bad:] == want_old["T_cw"][k_bad - 1]).all()   # LOST keeps the last pose
    with engine() as eng:
        for k in range(k_new):
            eng.push(0, frames[k], depth, tag=k)
        if n_lost_queued == 0:
            eng.flush()
        eng.restart(0, T_next)
        for k in range(k_new, N_FRAMES):
            eng.push(0, frames[k], depth, tag=k)
        eng.flush()
        res = eng.poll()
        stats, restarts = eng.stats(0), eng.restarts(0)
    with engine() as fresh:
        fresh.restart(0, T_next)
        for k in range(k_new, N_FRAMES):
            fresh.push(0, frames[k], depth, tag=k)
        fresh.flush()
        want = fresh.poll()
        want_stats = fresh.stats(0)
    assert res["frame"].tolist() == list(range(N_FRAMES)) and res["tag"].tolist() == list(range(N_FRAMES))
    before, after = res[:k_new], res[k_new:]
    for key in ("T_cw", "status", "n_inliers"):
        assert np.array_equal(before[key], want_old[key]), key
        assert np.array_equal(after[key], want[key]), key
    assert (after["status"] != 2).all() and after["status"][0] == 1
    for k, T in zip(after["frame"], after["T_cw"]):
        assert _pose_err(T.reshape(3, 4), gts[k]) < 3e-3, k
    assert stats["lost"] == 0 and restarts == 1
    for key in stats:
        if key == "lost":
            continue
        # the BA FLOP model is a double sum reported truncated: the two segments' truncations may add up to one less
        assert abs(stats[key] - (lost_stats[key] + want_stats[key])) <= (1 if key == "ba_flops" else 0), key


@pytest.mark.gpu
def test_start_pose_set_twice_keeps_the_enqueued_one(ctx3, shift_data):
    """ygzb_tracker_set_start_pose after an insertion is enqueued and before the context is synchronised: the insertion
    keeps the pose it was enqueued with, and the next one takes the new pose.  Every invalid pose is rejected and changes
    nothing."""
    from ygz_slam_b200 import capi
    fr = ctx3.frames(4)
    tr = fr.tracker(2, 4, (synth.FX, synth.FY, synth.CX, synth.CY))
    lib = tr.lib
    img, depth = shift_data[0][0][0], shift_data[0][1]
    tr.upload(0, img)
    tr.set_depth(0, depth)
    T1 = T0.copy()
    T2 = np.concatenate([synth.so3_exp(np.array([-0.2, 0.05, 0.1])), np.array([[-0.3], [0.2], [0.4]])], 1)
    ba = capi.BAParams()
    lib.ygzb_default_ba_params(C.byref(ba))
    results = []   # the insertions copy their result records back asynchronously

    def insert(entry, kf_slot):
        job = (capi.KeyframeJob * 1)()
        job[0].stream, job[0].frame_slot, job[0].kf_slot, job[0].entry, job[0].track_job = 0, 0, kf_slot, entry, -1
        job[0].n_local = 1
        job[0].local_entry[0] = entry
        results.append(capi.pinned_empty((C.sizeof(capi.KeyframeResult),), np.uint8))
        assert lib.ygzb_tracker_make_keyframes(tr.h, 1, job, C.byref(ba), results[-1].ctypes.data) == 0

    # invalid input: NULL tracker or pose, stream out of range, non-finite, not a rotation
    p = T1.reshape(12).copy()
    assert lib.ygzb_tracker_set_start_pose(None, 0, p.ctypes.data) == ERR_INVALID
    assert lib.ygzb_tracker_set_start_pose(tr.h, 0, None) == ERR_INVALID
    for stream in (-1, 2):
        assert lib.ygzb_tracker_set_start_pose(tr.h, stream, p.ctypes.data) == ERR_INVALID
    for name, T in _bad_poses().items():
        q = np.ascontiguousarray(T, np.float64).reshape(12)
        assert lib.ygzb_tracker_set_start_pose(tr.h, 0, q.ctypes.data) == ERR_INVALID, name
    tr.set_start_pose(0, T1)
    insert(0, 1)
    tr.set_start_pose(0, T2)          # before any synchronisation
    for name, T in _bad_poses().items():
        q = np.ascontiguousarray(T, np.float64).reshape(12)
        assert lib.ygzb_tracker_set_start_pose(tr.h, 0, q.ctypes.data) == ERR_INVALID, name
    ctx3.synchronize()
    insert(1, 2)
    ctx3.synchronize()
    kfs = tr.export(0, [0, 1]).keyframes()
    for kf, T in zip(kfs, (T1, T2)):
        assert np.array_equal(kf["T_cw"], T)
        pc = (T[:, :3] @ kf["pw"].T).T + T[:, 3]   # the map points sit at their depth in front of the key-frame
        assert kf["depth"].size > 500 and np.abs(pc[:, 2] - kf["depth"]).max() < 1e-12
    tr.close()
    fr.close()


@pytest.mark.gpu
@MODES
@WINDOWS
def test_invalid_restart_changes_nothing(ctx3, shift_data, window, ref_mode):
    """Every invalid ygz_vo_restart returns YGZB_ERR_INVALID, before the first push and in the middle of the run; the results
    are those of the run without the calls."""
    from ygz_slam_b200 import vo_native
    lib = vo_native._lib()
    ref_traj, ref_stats = batch(ctx3, shift_data, 3, window, ref_mode)

    def bad_calls(eng):
        p = T0.reshape(12).copy()
        assert lib.ygz_vo_restart(None, 0, p.ctypes.data) == ERR_INVALID
        for stream in (-1, 3):
            assert lib.ygz_vo_restart(eng.h, stream, p.ctypes.data) == ERR_INVALID
        for name, T in _bad_poses().items():
            q = np.ascontiguousarray(T, np.float64).reshape(12)
            assert lib.ygz_vo_restart(eng.h, 0, q.ctypes.data) == ERR_INVALID, name

    with vo_native.Engine(ctx3, 3, window=window, ref_mode=ref_mode, **POLICY) as eng:
        bad_calls(eng)
        for k in range(N_FRAMES):
            for s_ in range(3):
                eng.push(s_, shift_data[s_][0][k], shift_data[s_][1] if k == 0 else None, tag=1000 * s_ + k)
            if k in (0, 12):
                bad_calls(eng)
                eng.step()
        eng.flush()
        res = eng.poll()
        stats = [eng.stats(s_) for s_ in range(3)]
        restarts = [eng.restarts(s_) for s_ in range(3)]
    for s_ in range(3):
        assert np.array_equal(results_of(res, s_)[0], ref_traj[s_]) and stats[s_] == ref_stats[s_] and restarts[s_] == 0, s_
