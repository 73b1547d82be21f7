"""The previous-frame reference on the device (ygzb_tracker_set_reference_mode(YGZB_TRACK_REF_PREVIOUS), ygz_vo_run_ex):
the engine against the same rule in the Python loop on the same GPU backend, window invariance, the reference the tracker
keeps after a tracked frame and after a key-frame, and the rejected configurations."""
import numpy as np
import pytest

from ygz_slam_b200 import YgzbError, se3, synth, vo

from test_vo_ref_modes import PREVIOUS_MODE_POSE_TOL

KW = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)
K = np.array([synth.FX, synth.FY, synth.CX, synth.CY])


def _pose_err(A, B):
    return float(np.linalg.norm(se3.se3_log(se3.mul(A, se3.inv(B)))))


@pytest.mark.gpu
def test_engine_previous_mode_matches_python_loop_and_is_window_invariant(ctx3):
    from ygz_slam_b200 import vo_native
    n_streams, n_frames = 3, 26
    data = [synth.shift_stream(s, n_frames) for s in range(n_streams)]
    be = vo.GpuBackend(ctx3, n_streams * vo.VisualOdometry.SLOTS_PER_STREAM)
    V = vo.VisualOdometry(be, n_streams, ref_mode="previous", **KW)
    for k in range(n_frames):
        V.add_frames([data[s][0][k] for s in range(n_streams)], [data[s][1] for s in range(n_streams)], k)
    be.fr.close()
    runs = {w: vo_native.run(ctx3, [d[0] for d in data], [d[1] for d in data], 5, 0.03, 0.03, window=w, ref_mode="previous")
            for w in (1, 4, 8)}
    worst = 0.0
    for w, (traj, stats, sec) in runs.items():
        for s in range(n_streams):
            st = V.streams[s]
            assert not st.lost and stats[s]["lost"] == 0, w
            assert stats[s]["keyframes"] == st.stats["keyframes"] and stats[s]["ba"] == st.stats["ba"], w
            for k in range(n_frames):
                worst = max(worst, _pose_err(traj[s, k], st.trajectory[k]))
            assert _pose_err(traj[s, -1], data[s][2][-1]) < 3e-3
    # a window only changes how many frames are in flight, never a result
    assert np.array_equal(runs[1][0], runs[4][0]) and np.array_equal(runs[1][0], runs[8][0])
    # the engine and the Python loop differ in the summation order of pose-only and the local BA; along the chain of
    # previous-frame references these last-bit differences accumulate (measured on an H100: 1.2e-4 after 26 frames)
    assert worst < PREVIOUS_MODE_POSE_TOL, worst
    # and the key-frame mode of the same engine is a different trajectory
    kf = vo_native.run(ctx3, [d[0] for d in data], [d[1] for d in data], 5, 0.03, 0.03, window=8)
    assert not np.array_equal(kf[0], runs[8][0])


@pytest.mark.gpu
def test_engine_previous_mode_tracks_a_fast_stream_at_the_reference_defaults(ctx3):
    from ygz_slam_b200 import vo_native
    data = [synth.shift_stream(s, 80) for s in range(2)]
    frames = [d[0][::4] for d in data]
    traj_k, stats_k, _ = vo_native.run(ctx3, frames, [d[1] for d in data], window=8)
    traj_p, stats_p, _ = vo_native.run(ctx3, frames, [d[1] for d in data], window=8, ref_mode="previous")
    for s in range(2):
        assert stats_k[s]["lost"] and stats_k[s]["keyframes"] == 1
        assert not stats_p[s]["lost"] and stats_p[s]["keyframes"] >= 2
        assert _pose_err(traj_p[s, -1], data[s][2][::4][-1]) < 3e-3


def _tracker(ctx3, n_streams=1):
    fr = ctx3.frames(8 * n_streams)
    return fr, fr.tracker(n_streams, 8, K)


@pytest.mark.gpu
def test_tracker_reference_after_key_frame_and_after_frame(ctx3):
    """The tracker's reference against the rule: after the first key-frame its features at their depth-image depth; after a
    tracked frame (and a batch of three frames) the last frame's pose-only pose and projected candidates, inliers at the depth
    of their map point under that pose; after a second key-frame its tracked features followed by its new ones."""
    frames, depth, _ = synth.shift_stream(0, 8)
    fr, tr = _tracker(ctx3)
    tr.set_depth(0, depth)
    tr.set_reference_mode("previous", [7])
    tr.upload(0, frames[0])
    kres = tr.make_keyframes([dict(stream=0, frame_slot=0, kf_slot=4, entry=0, track_job=-1, local_entry=[0])])
    ref = tr.debug_reference(0)
    n0 = kres[0]["n_features"]
    assert ref["slot"] == 4 and len(ref["depth"]) == n0 and np.all(ref["depth"] == depth[0, 0])
    assert np.array_equal(ref["T_cw"], np.eye(4)[:3])
    # one frame
    tr.upload(0, frames[1])
    res = tr.track([(0, 0, [0])])
    dbg = tr.debug_job(0)
    ref = tr.debug_reference(0)
    T = res[0]["T_cw"]
    assert ref["slot"] == 7 and np.array_equal(ref["T_cw"], T)
    assert np.array_equal(ref["px"], dbg["c_px"])
    pw = dbg["c_pw"]
    z = T[2, 0] * pw[:, 0] + T[2, 1] * pw[:, 1] + T[2, 2] * pw[:, 2] + T[2, 3]
    assert np.array_equal(ref["depth"][dbg["inlier"]], z[dbg["inlier"]])
    # three frames in one batch: each against the one before; the reference is the last one
    tr.upload(0, frames[2:5])
    res = tr.track([(0, 0, [0]), (0, 1, [0]), (0, 2, [0])])
    dbg = tr.debug_job(2)
    ref = tr.debug_reference(0)
    assert np.array_equal(ref["T_cw"], res[2]["T_cw"]) and np.array_equal(ref["px"], dbg["c_px"])
    # a key-frame from the last job, with a local BA
    kres = tr.make_keyframes([dict(stream=0, frame_slot=2, kf_slot=5, entry=1, track_job=2, local_entry=[0, 1], run_ba=1, mp0=n0)])
    ref = tr.debug_reference(0)
    n_tr = len(dbg["c_px"])
    assert ref["slot"] == 5 and len(ref["depth"]) == n_tr + kres[0]["n_features"]
    assert np.array_equal(ref["T_cw"], kres[0]["T_cw"][-1])
    assert np.array_equal(ref["px"][:n_tr], dbg["c_px"]) and np.all(ref["depth"][n_tr:] == depth[0, 0])
    assert len(ref["depth"]) > 2488 or n_tr + n0 <= 2488
    fr.close()


@pytest.mark.gpu
def test_tracker_reference_mode_rejections(ctx3):
    fr, tr = _tracker(ctx3, n_streams=2)
    with pytest.raises(YgzbError):
        tr.set_reference_mode("previous")             # no reference slots
    with pytest.raises(YgzbError):
        tr.set_reference_mode("previous", [6, 6])     # shared
    with pytest.raises(YgzbError):
        tr.set_reference_mode("previous", [6, 99])    # out of range
    with pytest.raises(YgzbError):
        tr.set_reference_mode("sideways", [6, 7])
    with pytest.raises(YgzbError):
        tr.debug_reference(0)                         # key-frame mode has no reference store
    tr.set_reference_mode("previous", [6, 7])
    frames, depth, _ = synth.shift_stream(0, 2)
    tr.set_depth(0, depth)
    tr.upload(0, frames[0])
    with pytest.raises(YgzbError):
        tr.track([(0, 0, [0])])                       # stream 0 has no reference yet
    tr.make_keyframes([dict(stream=0, frame_slot=0, kf_slot=4, entry=0, track_job=-1, local_entry=[0])])
    with pytest.raises(YgzbError):
        tr.set_reference_mode("keyframe")             # too late
    tr.upload(0, frames[1])
    assert tr.track([(0, 0, [0])])[0]["aligned"]      # the tracker is untouched and still in previous mode
    fr.close()
