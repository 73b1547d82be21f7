"""The previous-frame reference of the tracking loop (vo.VisualOdometry(ref_mode="previous")): every frame is aligned
against the frame before it, as VisualOdometry::AddFrame does (VisualOdometry.cpp:66, :88-90), instead of against the
newest key-frame.  On the CPU oracle the loop follows the synthetic ground truth, tracks a stream too fast for the
key-frame reference at the reference's key-frame defaults, and passes pose-only outliers (depth -1 and stale depths) on
to the next alignment; on the GPU the same loop reproduces the oracle's trajectory."""
import dataclasses

import numpy as np
import pytest

from ygz_slam_b200 import se3, synth, vo
from oracle.vo_backend import OracleBackend


class DepthOracleBackend(OracleBackend):
    """OracleBackend whose pose_only can also return pose-only's per-point depth, like vo.GpuBackend.pose_only."""

    def pose_only(self, pts_w, obs, T, return_depth=False):
        Ts, inls, cnts, depths = [], [], [], []
        for p, o, t in zip(pts_w, obs, T):
            if len(p) == 0:
                Ts.append(t); inls.append(np.zeros(0, bool)); cnts.append(0); depths.append(np.zeros(0))
                continue
            Tn, inl, d, cnt = self.o.pose_only(p, o, t)
            Ts.append(Tn); inls.append(inl); cnts.append(cnt); depths.append(d)
        return (Ts, inls, np.array(cnts), depths) if return_depth else (Ts, inls, np.array(cnts))


class Recorder:
    """Wraps a backend and keeps the inputs of every sparse alignment and the inputs and outputs of every pose-only call."""

    def __init__(self, be):
        self.be, self.align, self.pose = be, [], []

    def __getattr__(self, name):
        return getattr(self.be, name)

    def sparse_alignment(self, ref_slots, cur_slots, px, depth, T_ref):
        self.align.append(dict(px=[np.array(p) for p in px], depth=[np.array(d) for d in depth], T_ref=[np.array(t) for t in T_ref]))
        return self.be.sparse_alignment(ref_slots, cur_slots, px, depth, T_ref)

    def pose_only(self, pts_w, obs, T, **kw):
        out = self.be.pose_only(pts_w, obs, T, **kw)
        self.pose.append(dict(pts_w=pts_w, obs=obs, T=out[0], inl=out[1], depth=out[3] if len(out) > 3 else None))
        return out


def _pose_err(A, B):
    return float(np.linalg.norm(se3.se3_log(se3.mul(A, se3.inv(B)))))


def _run(backend, frames, depths, gts, mode, **kw):
    """frames[s][k], depths[s][k], gts[s][k]; returns the loop and the per-frame ground-truth error (nan once lost)."""
    S, n = len(frames), len(frames[0])
    V = vo.VisualOdometry(backend, S, ref_mode=mode, **kw)
    errs = np.full((S, n), np.nan)
    for k in range(n):
        V.add_frames([frames[s][k] for s in range(S)], [depths[s][k] for s in range(S)], k)
        for s in range(S):
            if not V.streams[s].lost:
                errs[s, k] = _pose_err(V.streams[s].T_cw, se3.mul(gts[s][k], se3.inv(gts[s][0])))
    return V, errs


def _stream_frames(n_streams, n_frames, step=2):
    fr = [[synth.stream_frame(step * k, stream=s) for k in range(n_frames)] for s in range(n_streams)]
    return [[f[0] for f in x] for x in fr], [[f[1] for f in x] for x in fr], [[f[2] for f in x] for x in fr]


def _shift_frames(n_streams, n_frames, every=1):
    data = [synth.shift_stream(s, n_frames * every) for s in range(n_streams)]
    return ([d[0][::every] for d in data], [[d[1]] * n_frames for d in data], [d[2][::every] for d in data])


def _shifted_region(img, r0, r1, c0, c1, dx):
    out = img.copy()
    out[r0:r1, c0:c1] = img[r0:r1, c0 - dx:c1 - dx]
    return out


def _outlier_scene(n_frames=12, k=7):
    """shift_stream 0 with frame k corrupted: its left part shifted 8 px right, its right part 2 px left.  Direct projection
    follows the moved texture, so pose-only rejects the left part from its first round on (depth -1), and the first round's
    pose, pulled by all points, rejects right-part points that the alignment pose had accepted (stale depths)."""
    frames, depths, gts = _shift_frames(1, n_frames)
    frames[0] = frames[0].copy()
    frames[0][k] = _shifted_region(frames[0][k], 60, 420, 40, 300, 8)
    frames[0][k] = _shifted_region(frames[0][k], 60, 420, 340, 600, -2)
    return frames, depths, gts


KW_FAST = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)


# ---- CPU oracle ------------------------------------------------------------------------------------------------------
def test_ref_mode_is_checked():
    with pytest.raises(ValueError):
        vo.VisualOdometry(None, 1, ref_mode="last")
    assert vo.VisualOdometry(None, 1).ref_mode == "keyframe"


@pytest.mark.parametrize("scene", ["stream_frame", "shift_stream"])
def test_previous_mode_on_oracle_follows_ground_truth(oracle, scene):
    frames, depths, gts = _stream_frames(1, 24) if scene == "stream_frame" else _shift_frames(1, 26)
    V, errs = _run(DepthOracleBackend(oracle), frames, depths, gts, "previous", **KW_FAST)
    st = V.streams[0]
    assert not st.lost
    assert st.stats["keyframes"] >= 3 and st.stats["ba"] >= 2
    assert errs.max() < 3e-3
    assert st.stats["projected"] > 0.9 * st.stats["candidates"]


def test_previous_mode_reference_rule_on_oracle(oracle):
    """The reference of frame k+1 is frame k: its pose-only pose and its projected candidates in candidate order, inliers
    at the depth of their map point under that pose, outliers at pose-only's depth.  After a key-frame: its BA pose, the
    tracked features (inlier depths under the BA's points and pose), then its new features at their depth-image depth."""
    frames, depths, gts = _shift_frames(1, 14)
    be = Recorder(DepthOracleBackend(oracle))
    V = vo.VisualOdometry(be, 1, ref_mode="previous", **KW_FAST)
    refs, kf_frames, kf_snap = [], [], {}
    for k in range(14):
        n_kf = V.streams[0].stats["keyframes"]
        V.add_frames([frames[0][k]], [depths[0][k]], k)
        st = V.streams[0]
        refs.append(st.ref)
        if st.stats["keyframes"] > n_kf:
            kf_frames.append(k)   # the key-frames as the BA left them (a later BA moves them again)
            kf_snap[k] = [dataclasses.replace(kf, T_cw=kf.T_cw.copy(), pw=kf.pw.copy()) for kf in st.keyframes]
    assert not V.streams[0].lost and kf_frames[0] == 0 and len(kf_frames) >= 3
    # alignment of frame k (k >= 1) reads the reference left by frame k-1; pose-only call k-1 belongs to frame k
    for k in range(1, 14):
        a, r = be.align[k - 1], refs[k - 1]
        assert np.array_equal(a["px"][0], r.px) and np.array_equal(a["depth"][0], r.depth)
        assert np.array_equal(a["T_ref"][0], r.T_cw)
    for k in range(1, 14):
        p, r = be.pose[k - 1], refs[k]
        inl, n = np.asarray(p["inl"][0], bool), len(p["inl"][0])
        T = p["T"][0]
        depth = np.array(p["depth"][0])
        if k in kf_frames:
            kfs = kf_snap[k]
            kf = kfs[-1]
            assert np.array_equal(r.T_cw, kf.T_cw) and _pose_err(r.T_cw, T) > 0   # the BA moved the key-frame
            assert len(r.depth) == n + len(kf.depth) and np.array_equal(r.px[:n], p["obs"][0])
            assert np.array_equal(r.px[n:], kf.px) and np.array_equal(r.depth[n:], kf.depth)
            assert np.array_equal(r.depth[:n][~inl], depth[~inl])
            pw = np.concatenate([kf.pw for kf in kfs])[np.searchsorted(np.concatenate([kf.mp_id for kf in kfs]), r.mp_id)]
            T = kf.T_cw
        else:
            assert np.array_equal(r.T_cw, T) and np.array_equal(r.px, p["obs"][0])
            pw = p["pts_w"][0]
        z = T[2, 0] * pw[:, 0] + T[2, 1] * pw[:, 1] + T[2, 2] * pw[:, 2] + T[2, 3]
        assert np.array_equal(r.depth[:n][inl], z[inl]) and np.array_equal(r.depth[:n][~inl], depth[~inl])


def test_previous_mode_passes_pose_only_outliers_to_the_next_alignment(oracle):
    frames, depths, gts = _outlier_scene()
    be = Recorder(DepthOracleBackend(oracle))
    V = vo.VisualOdometry(be, 1, ref_mode="previous", **KW_FAST)
    for k in range(12):
        V.add_frames([frames[0][k]], [depths[0][k]], k)
        assert not V.streams[0].lost, k
    p7 = be.pose[6]                                            # pose-only of frame 7
    inl, d = np.asarray(p7["inl"][0], bool), np.asarray(p7["depth"][0])
    never, stale = ~inl & (d == -1), ~inl & (d != -1)
    assert never.sum() >= 100 and stale.sum() >= 20, (never.sum(), stale.sum())
    a8 = be.align[7]                                           # alignment of frame 8 reads them all
    assert len(a8["depth"][0]) == len(inl)
    assert np.array_equal(a8["depth"][0][never], d[never]) and np.array_equal(a8["depth"][0][stale], d[stale])
    # and the stream recovers from the corrupted frame
    gt8 = se3.mul(gts[0][8], se3.inv(gts[0][0]))
    assert _pose_err(V.streams[0].trajectory[8], gt8) < 3e-3
    assert _pose_err(V.streams[0].T_cw, se3.mul(gts[0][-1], se3.inv(gts[0][0]))) < 3e-3


def test_previous_mode_tracks_where_keyframe_mode_is_lost(oracle):
    """Every 4th frame of shift_stream 0 (0.03-0.055 m per frame at 2 m depth) at the reference's key-frame defaults (10
    frames, 0.1 rad / 0.1 m).  Against the key-frame, the alignment of frame 3 (0.15 of motion, ~35 px) does not converge
    and its estimate fails the 0.2 motion check: the stream is lost long before a key-frame may be taken.  Against the
    previous frame, each alignment covers one step and the stream is tracked."""
    frames, depths, gts = _shift_frames(1, 20, every=4)
    steps = [np.linalg.norm(gts[0][k][:, 3] - gts[0][k - 1][:, 3]) for k in range(1, 6)]
    assert 0.03 < min(steps) and max(steps) < 0.06
    Vk, ek = _run(DepthOracleBackend(oracle), frames, depths, gts, "keyframe")
    assert Vk.streams[0].lost and Vk.streams[0].stats["keyframes"] == 1
    assert np.isnan(ek[0, 9])
    Vp, ep = _run(DepthOracleBackend(oracle), frames, depths, gts, "previous")
    st = Vp.streams[0]
    assert not st.lost and st.stats["keyframes"] >= 2 and st.stats["ba"] >= 1
    assert ep.max() < 3e-3


# ---- GPU: the same loop on the device backend against the oracle loop ---------------------------------------------------
# In "previous" mode every frame starts from the one before it, so the last-bit differences of the FP64 solvers' summation
# order (and the odd borderline candidate or inlier they flip) accumulate along the stream instead of being reset at each
# key-frame.  Measured on an H100: 1e-7 to 2e-6 after the first frames, up to 1.2e-4 after 26 frames of shift_stream
# (GPU loop against the oracle loop, and the device engine against the GPU loop alike), while every single alignment
# agrees with the oracle's to ~1e-14 on the same inputs (test_previous_mode_gpu_alignment_on_oracle_inputs).  The
# trajectories are therefore compared at 5e-4; key-frame counts and BA counts must be equal.
PREVIOUS_MODE_POSE_TOL = 5e-4


def _check_parity(Vg, Vo, n_streams):
    for s in range(n_streams):
        sg, so = Vg.streams[s].stats, Vo.streams[s].stats
        assert Vg.streams[s].lost == Vo.streams[s].lost
        assert sg["frames"] == so["frames"] and sg["keyframes"] == so["keyframes"] and sg["ba"] == so["ba"]
        for key in ("candidates", "projected", "inliers"):
            assert abs(sg[key] - so[key]) <= 1e-3 * so[key], key
        for Tg, Tw in zip(Vg.streams[s].trajectory, Vo.streams[s].trajectory):
            assert _pose_err(Tg, Tw) < PREVIOUS_MODE_POSE_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["stream_frame", "shift_stream", "outliers"])
def test_previous_mode_gpu_matches_oracle_loop(ctx3, oracle, scene):
    if scene == "stream_frame":
        frames, depths, gts = _stream_frames(2, 20)
    elif scene == "shift_stream":
        frames, depths, gts = _shift_frames(3, 26)
    else:
        frames, depths, gts = _outlier_scene()
    S = len(frames)
    Vo, _ = _run(DepthOracleBackend(oracle), frames, depths, gts, "previous", **KW_FAST)
    be = vo.GpuBackend(ctx3, S * vo.VisualOdometry.SLOTS_PER_STREAM)
    Vg, errs = _run(be, frames, depths, gts, "previous", **KW_FAST)
    be.fr.close()
    _check_parity(Vg, Vo, S)
    assert not any(st.lost for st in Vg.streams)
    assert np.nanmax(errs[:, -1]) < 3e-3
    # a key-frame's reference (tracked + new features) exceeds the 2,488 features a 4-CTA cluster keeps in shared memory
    assert max(len(st.ref.depth) for st in Vg.streams) > 2488 or scene == "outliers"


@pytest.mark.gpu
def test_previous_mode_gpu_tracks_where_keyframe_mode_is_lost(ctx3, oracle):
    frames, depths, gts = _shift_frames(2, 20, every=4)
    be = vo.GpuBackend(ctx3, 2 * vo.VisualOdometry.SLOTS_PER_STREAM)
    Vk, _ = _run(be, frames, depths, gts, "keyframe")
    assert all(st.lost and st.stats["keyframes"] == 1 for st in Vk.streams)
    Vg, errs = _run(be, frames, depths, gts, "previous")
    be.fr.close()
    Vo, _ = _run(DepthOracleBackend(oracle), frames, depths, gts, "previous")
    _check_parity(Vg, Vo, 2)
    assert not any(st.lost for st in Vg.streams) and errs.max() < 3e-3


class _ImageRecorder(DepthOracleBackend):
    """Keeps the images behind the slots and the inputs and result of every sparse alignment."""

    def __init__(self, o):
        super().__init__(o)
        self.img, self.calls = {}, []

    def upload(self, slots, images):
        for s, im in zip(slots, images):
            self.img[int(s)] = np.array(im)
        return super().upload(slots, images)

    def sparse_alignment(self, ref_slots, cur_slots, px, depth, T_ref):
        out = super().sparse_alignment(ref_slots, cur_slots, px, depth, T_ref)
        self.calls += [(self.img[int(r)], self.img[int(c)], np.array(p), np.array(d), np.array(t), T)
                       for r, c, p, d, t, T in zip(ref_slots, cur_slots, px, depth, T_ref, out[0])]
        return out


@pytest.mark.gpu
def test_previous_mode_gpu_alignment_on_oracle_inputs(ctx3, oracle):
    """Every alignment of the previous-mode oracle loop on 2 shift_streams, replayed on the GPU backend: references of
    1,000 to 4,800 features (above 2,488 they take the sparse alignment's global staging path) give the oracle's pose."""
    frames, depths, gts = _shift_frames(2, 22)
    ob = _ImageRecorder(oracle)
    V = vo.VisualOdometry(ob, 2, ref_mode="previous", **KW_FAST)
    for k in range(22):
        V.add_frames([frames[s][k] for s in range(2)], [depths[s][k] for s in range(2)], k)
    assert max(len(c[3]) for c in ob.calls) > 2488 and min(len(c[3]) for c in ob.calls) < 2488
    be = vo.GpuBackend(ctx3, 2)
    errs = []
    for ref_img, cur_img, px, depth, T_ref, T_want in ob.calls:
        be.upload([0, 1], [ref_img, cur_img])
        T_got, _ = be.sparse_alignment([0], [1], [px], [depth], [T_ref])
        errs.append(_pose_err(T_got[0], T_want))
    be.fr.close()
    errs = np.array(errs)
    assert errs.max() < 1e-5 and np.mean(errs < 1e-12) > 0.95, np.sort(errs)[-5:]
