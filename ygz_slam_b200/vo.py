"""Host-side tracking loop in the shape of the reference's VisualOdometry / LocalMapping callers, driving the
hot path through a backend (the C ABI on the GPU; the tests plug the CPU oracle into the same loop).

This is CALLER code -- the reference's src/Module/VisualOdometry.cpp:38-107 (AddFrame), :281-302 (TrackRefFrame),
src/Module/LocalMapping.cpp:24-140 (TrackLocalMap: FindCandidates / ProjectMapPoints / OptimizeCurrent) and
VisualOdometry.cpp:182-218 + :304-321 (SetKeyframe / NeedNewKeyFrame) -- restated in Python only to exercise
BASELINE config C5 ("full VO, independent synthetic streams sharded across GPUs").  No image or optimisation
arithmetic happens here: every numeric step is one batched backend call over all streams of the rank.

Differences from the reference callers, all on the input side (SURVEY.md 8f keeps them out of scope):
  * initialisation: the monocular H/F initialiser is replaced by ground-truth depth for the detected features of
    a keyframe (what the reference's own drivers do with TUM depth, test/test_feature_alignment.cpp:72-85);
  * new map points at keyframes come from that depth as well (CreateNewMapPoints is commented out in the
    reference, LocalMapping.cpp:313, so its map never grows);
  * BoW and loop closing are not part of the path.
"""
from __future__ import annotations

import inspect
from dataclasses import dataclass, field

import numpy as np

from . import se3, synth


@dataclass
class Keyframe:
    slot: int
    T_cw: np.ndarray            # 3x4
    frame_id: int
    px: np.ndarray              # (n, 2) full-res pixels of its features
    level: np.ndarray           # (n,)
    depth: np.ndarray           # (n,) ref-camera depth
    pw: np.ndarray              # (n, 3) world points (map points)
    mp_id: np.ndarray           # (n,) ids in the stream's map
    obs_id: np.ndarray = None   # map points of OLDER keyframes tracked into this frame (ids) ...
    obs_px: np.ndarray = None   # ... and their measured pixels (FindDirectProjection results kept by pose-only)


@dataclass
class RefFrame:
    """The frame the next frame of a stream aligns against in "previous" mode (VisualOdometry.cpp:88-90 sets _ref_frame to
    every tracked frame): its slot, its pose, and one feature per successfully projected candidate, in candidate order."""
    slot: int
    T_cw: np.ndarray            # 3x4
    px: np.ndarray              # (n, 2) FindDirectProjection results ...
    depth: np.ndarray           # (n,) ... and their depths (see VisualOdometry._track); -1 for a point never a pose-only inlier
    mp_id: np.ndarray = None    # map points of the tracked features (the first len(mp_id) features) ...
    inlier: np.ndarray = None   # ... and which of them were pose-only inliers


@dataclass
class Stream:
    sid: int
    slots: tuple                # (slot_a, slot_b, ...) ring of device slots: keyframes + current
    ref: Keyframe | RefFrame | None = None
    keyframes: list = field(default_factory=list)
    T_cw: np.ndarray | None = None
    frames_since_kf: int = 0
    lost: bool = False
    trajectory: list = field(default_factory=list)
    next_mp: int = 0
    last_obs: tuple = None      # (ids, px) of the inlier observations of the most recent tracked frame
    start: np.ndarray = field(default_factory=lambda: np.eye(4)[:3].copy())   # T_cw of the first keyframe
    stats: dict = field(default_factory=lambda: dict(frames=0, keyframes=0, candidates=0, projected=0, inliers=0, ba=0))


class VisualOdometry:
    """Lock-step tracking of `n_streams` independent synthetic sequences on one backend (= one GPU)."""

    KF_MIN_FRAMES = 10          # VisualOdometry.cpp:304-321: >= 10 frames since the last keyframe ...
    KF_MIN_ROT = 0.1            # ... and rotation or translation above vo.keyframe.min_rot / min_trans
    KF_MIN_TRANS = 0.1
    MIN_INLIERS = 30            # vo.keyframe.min_features (config/default.yaml:66)
    LOCAL_KEYFRAMES = 3         # LocalMapping.local_keyframes (config/default.yaml:68)
    SLOTS_PER_STREAM = LOCAL_KEYFRAMES + 2

    def __init__(self, backend, n_streams: int, stream_ids=None, kf_min_frames: int | None = None, kf_min_rot: float | None = None,
                 kf_min_trans: float | None = None, ref_mode: str = "keyframe", camera=None):
        """ref_mode: what a frame is aligned against by the sparse alignment.  "previous" is the reference's rule
        (VisualOdometry.cpp:66 and :88-90: the previous tracked frame, or the key-frame it became); "keyframe" aligns every
        frame against the newest key-frame, which makes the frames between two key-frames independent of each other.
        camera: (fx, fy, cx, cy) in double of the candidate projection and the key-frames' map points (default: the TUM
        camera, synth.FX..CY); the backend's solvers use their own camera, which must be this one rounded to float."""
        if ref_mode not in ("keyframe", "previous"):
            raise ValueError(f"ref_mode must be 'keyframe' or 'previous', not {ref_mode!r}")
        params = inspect.signature(backend.pose_only).parameters.values() if ref_mode == "previous" else ()
        if ref_mode == "previous" and not any(p.name == "return_depth" or p.kind is p.VAR_KEYWORD for p in params):
            raise TypeError("ref_mode='previous' needs a backend whose pose_only(..., return_depth=True) returns pose-only's depths")
        self.ref_mode = ref_mode
        self.K = tuple(float(v) for v in (camera if camera is not None else (synth.FX, synth.FY, synth.CX, synth.CY)))
        self.be = backend
        self.streams = [Stream(sid=(stream_ids[i] if stream_ids else i),
                               slots=tuple(range(i * self.SLOTS_PER_STREAM, (i + 1) * self.SLOTS_PER_STREAM)))
                        for i in range(n_streams)]
        if kf_min_frames is not None:
            self.KF_MIN_FRAMES = kf_min_frames
        # vo.keyframe.min_rot / min_trans are YAML parameters (config/default.yaml:64-65); in "keyframe" mode the sparse
        # alignment starts every frame from the key-frame's pose and rejects more than 0.2 of motion since it
        # (Matcher.cpp:482-488), so fast synthetic streams need a tighter keyframe spacing than the 0.1 default there
        if kf_min_rot is not None:
            self.KF_MIN_ROT = kf_min_rot
        if kf_min_trans is not None:
            self.KF_MIN_TRANS = kf_min_trans
        self._slot_use = [0] * n_streams

    def set_start_pose(self, i: int, T_cw):
        """T_cw (3, 4) of stream i's first keyframe (identity by default), to place the sequence in the caller's world frame
        as the reference's drivers do (test/test_feature_alignment.cpp:63); set it before the stream's first frame.  The
        rules of ygzb_tracker_set_start_pose: finite, and a rotation (orthonormal, det +1) within 1e-6."""
        T = np.array(T_cw, np.float64).reshape(3, 4)
        R = T[:, :3]
        if not np.all(np.isfinite(T)) or np.abs(R @ R.T - np.eye(3)).max() > 1e-6 or abs(np.linalg.det(R) - 1) > 1e-6:
            raise ValueError("start pose must be finite with an orthonormal rotation of determinant +1")
        if self.streams[i].keyframes:
            raise RuntimeError(f"stream {i} has started already")
        self.streams[i].start = T

    # ---- slot ring: current frame always goes to the next free slot of the stream -------------------------
    def _next_slot(self, si: int) -> int:
        st = self.streams[si]
        used = {kf.slot for kf in st.keyframes[-self.LOCAL_KEYFRAMES:]}
        if st.ref is not None:
            used.add(st.ref.slot)      # a key-frame in "keyframe" mode; the previous frame may hold the one free slot otherwise
        for s in st.slots:
            if s not in used:
                return s
        raise RuntimeError("slot ring exhausted")

    # ---- one lock-step frame ---------------------------------------------------------------------------------
    def add_frames(self, images, depths, frame_id: int):
        """images[i], depths[i]: grey frame and ground-truth depth map of stream i (depth is only sampled at keyframes)."""
        S = len(self.streams)
        cur_slots = [self._next_slot(i) for i in range(S)]
        self.be.upload(cur_slots, images)
        live = [i for i in range(S) if not self.streams[i].lost]
        # -- first frame: becomes the first keyframe (depth-initialised map)
        boot = [i for i in live if self.streams[i].ref is None]
        if boot:
            for i in boot:
                self.streams[i].T_cw = self.streams[i].start.copy()
            self._make_keyframes(boot, cur_slots, depths, frame_id, fresh=True)
        track = [i for i in live if i not in boot]
        if track:
            self._track(track, cur_slots, depths, frame_id)
        for i in range(S):
            st = self.streams[i]
            st.trajectory.append(None if st.T_cw is None else st.T_cw.copy())
            st.stats["frames"] += 1

    # ---- TrackRefFrame + TrackLocalMap (+ keyframe decision) for the streams in `idx` -------------------------
    def _track(self, idx, cur_slots, depths, frame_id):
        be = self.be
        # TrackRefFrame: Matcher::SparseImageAlignment(ref, curr) with curr._TCW = ref._TCW (VO.cpp:281-302)
        refs = [self.streams[i].ref for i in idx]
        T_list, ok = be.sparse_alignment([kf.slot for kf in refs], [cur_slots[i] for i in idx], [kf.px for kf in refs],
                                         [kf.depth for kf in refs], [kf.T_cw for kf in refs])
        T_cur, alive = {}, []
        for j, i in enumerate(idx):
            if ok[j]:
                T_cur[i] = T_list[j]
                alive.append(i)
            else:
                self.streams[i].lost = True   # the reference keeps the last pose and reports VO_LOST (VO.cpp:84-99)
        idx = alive
        if not idx:
            return
        # TrackLocalMap / FindCandidates: project the local map points, border 20 (LocalMapping.cpp:47-80)
        jobs = []
        for i in idx:
            st = self.streams[i]
            T = T_cur[i]
            kfs = st.keyframes[-self.LOCAL_KEYFRAMES:]
            kf_of, n_of, uu, vv, ids = [], [], [], [], []
            for k, kf in enumerate(kfs):
                pc = (T[:, :3] @ kf.pw.T).T + T[:, 3]
                z = pc[:, 2]
                with np.errstate(divide="ignore", invalid="ignore"):
                    u = self.K[0] * pc[:, 0] / z + self.K[2]
                    v = self.K[1] * pc[:, 1] / z + self.K[3]
                good = np.nonzero((z > 0) & (u >= 20) & (u < synth.W - 20) & (v >= 20) & (v < synth.H - 20))[0]
                kf_of.append(np.full(len(good), k, np.int32)); n_of.append(good.astype(np.int32))
                uu.append(u[good]); vv.append(v[good]); ids.append(kf.mp_id[good])
            kf_of, n_of, uu, vv, ids = (np.concatenate(a) for a in (kf_of, n_of, uu, vv, ids))
            _, first = np.unique(ids, return_index=True)      # a map point is a candidate once
            first.sort()
            jobs.append(dict(stream=i, kfs=kfs, cur_slot=cur_slots[i], T_cur=T, kf=kf_of[first], n=n_of[first],
                             init=np.stack([uu[first], vv[first]], 1)))
            st.stats["candidates"] += len(first)
        # ProjectMapPoints: Matcher::FindDirectProjection per candidate (LocalMapping.cpp:82-111), one batch
        px, okp = be.project(jobs)
        # OptimizeCurrentPoseOnly on the successfully projected points (LocalMapping.cpp:126; BA.cpp:188-264)
        pts_w, obs, obs_ids = [], [], []
        for job, p, o in zip(jobs, px, okp):
            sel = np.nonzero(o)[0]
            pw = np.concatenate([kf.pw for kf in job["kfs"]])
            ids = np.concatenate([kf.mp_id for kf in job["kfs"]])
            base = np.concatenate([[0], np.cumsum([len(kf.pw) for kf in job["kfs"]])])
            flat = base[job["kf"][sel]] + job["n"][sel]
            pts_w.append(pw[flat].reshape(-1, 3))
            obs_ids.append(ids[flat])
            obs.append(p[sel].reshape(-1, 2))
            self.streams[job["stream"]].stats["projected"] += len(sel)
        if self.ref_mode == "previous":
            T_opt, inl, cnt, po_depth = be.pose_only(pts_w, obs, [T_cur[i] for i in idx], return_depth=True)
        else:
            T_opt, inl, cnt = be.pose_only(pts_w, obs, [T_cur[i] for i in idx])
        for j, i in enumerate(idx):
            st = self.streams[i]
            if cnt[j] < self.MIN_INLIERS:
                st.lost = True
                continue
            keep = np.asarray(inl[j], bool)
            st.last_obs = (obs_ids[j][keep], obs[j][keep])
            st.T_cw = T_opt[j]
            st.frames_since_kf += 1
            st.stats["inliers"] += int(cnt[j])
            if self.ref_mode == "previous":
                # OptimizeCurrent (LocalMapping.cpp:130-134) gives an inlier the depth of its map point under the final pose;
                # an outlier keeps what OptimizeCurrentPoseOnly left: the depth of its last inlier round, under that round's
                # starting pose, or -1.  SparseImgAlign tests only _mappoint and the border, not _bad, so the outliers
                # take part in the next alignment as well
                depth = np.array(po_depth[j], np.float64)
                depth[keep] = _depth_under(T_opt[j], pts_w[j][keep])
                st.ref = RefFrame(slot=cur_slots[i], T_cw=T_opt[j].copy(), px=obs[j].copy(), depth=depth, mp_id=obs_ids[j],
                                  inlier=keep)
        # NeedNewKeyFrame (VO.cpp:304-321) -> SetKeyframe (:182-218); measured from the last key-frame in both modes
        need = []
        for i in idx:
            st = self.streams[i]
            if st.lost or st.frames_since_kf < self.KF_MIN_FRAMES:
                continue
            d = se3.se3_log(se3.mul(st.T_cw, se3.inv(st.keyframes[-1].T_cw)))
            if np.linalg.norm(d[3:]) > self.KF_MIN_ROT or np.linalg.norm(d[:3]) > self.KF_MIN_TRANS:
                need.append(i)
        if need:
            self._make_keyframes(need, cur_slots, depths, frame_id, fresh=False)

    # ---- SetKeyframe: Detect (grid FAST + ORB), depth-initialised map points, local BA ---------------------------
    def _make_keyframes(self, idx, cur_slots, depths, frame_id, fresh):
        be = self.be
        feats = be.detect([cur_slots[i] for i in idx])
        ba_jobs = []
        for j, i in enumerate(idx):
            st = self.streams[i]
            f = feats[j]
            px = np.stack([f["px"], f["py"]], 1)
            d = depths[i][f["py"].astype(int), f["px"].astype(int)]
            T = st.T_cw
            Tin = se3.inv(T)
            fx, fy, cx, cy = self.K
            pc = np.stack([(px[:, 0] - cx) * d / fx, (px[:, 1] - cy) * d / fy, d], 1)
            pw = (Tin[:, :3] @ pc.T).T + Tin[:, 3]
            ids = np.arange(st.next_mp, st.next_mp + len(d))
            st.next_mp += len(d)
            kf = Keyframe(slot=cur_slots[i], T_cw=T.copy(), frame_id=frame_id, px=px, level=f["level"].astype(np.int32),
                          depth=d.astype(np.float64), pw=pw, mp_id=ids)
            if not fresh and st.last_obs is not None:
                kf.obs_id, kf.obs_px = st.last_obs
            st.keyframes.append(kf)
            st.keyframes = st.keyframes[-(self.LOCAL_KEYFRAMES + 1):]
            if fresh or self.ref_mode == "keyframe":
                st.ref = kf
            st.frames_since_kf = 0
            st.stats["keyframes"] += 1
            if not fresh and len(st.keyframes) >= 2:
                ba_jobs.append(i)
        if ba_jobs:
            self._local_ba(ba_jobs)
        if self.ref_mode == "previous" and not fresh:
            for i in idx:
                self._keyframe_reference(self.streams[i])

    def _keyframe_reference(self, st):
        """The reference the frame after a new key-frame aligns against in "previous" mode: the key-frame as SetKeyframe and
        LocalBA leave it (VisualOdometry.cpp:182-218, LocalMapping.cpp:192-206) -- its pose after the BA; its tracked
        features, inliers with the depth of their map point after the BA, outliers unchanged; then its own new features
        with their depth-image depths (the engine's stand-in for map points the reference would not have)."""
        kf, tr = st.keyframes[-1], st.ref
        depth = tr.depth.copy()
        depth[tr.inlier] = _depth_under(kf.T_cw, _map_points(st.keyframes, tr.mp_id[tr.inlier]))
        st.ref = RefFrame(slot=kf.slot, T_cw=kf.T_cw.copy(), px=np.concatenate([tr.px, kf.px]).reshape(-1, 2),
                          depth=np.concatenate([depth, kf.depth]), mp_id=tr.mp_id, inlier=tr.inlier)

    # ---- LocalMapping::LocalBA -> ba::LocalBAG2O over the local keyframes and the points they share -------------------
    def _local_ba(self, idx):
        problems, layouts = [], []
        for i in idx:
            st = self.streams[i]
            kfs = st.keyframes[-self.LOCAL_KEYFRAMES:]
            poses = np.array([se3.se3_log(kf.T_cw) for kf in kfs])
            fixed = np.zeros(len(kfs), np.uint8)
            fixed[0] = 1                                   # the oldest local keyframe fixes the gauge (keyframe 0 in the reference)
            lo = np.array([kf.mp_id[0] for kf in kfs]); hi = np.array([kf.mp_id[-1] + 1 for kf in kfs])
            # observations: a keyframe observes its own points (detected pixel) and the older points tracked into it
            o_kf, o_id, o_px = [], [], []
            for k, kf in enumerate(kfs):
                o_kf.append(np.full(len(kf.mp_id), k, np.int32)); o_id.append(kf.mp_id); o_px.append(kf.px)
                if kf.obs_id is not None and len(kf.obs_id):
                    inside = np.zeros(len(kf.obs_id), bool)
                    for a, b in zip(lo, hi):
                        inside |= (kf.obs_id >= a) & (kf.obs_id < b)
                    o_kf.append(np.full(int(inside.sum()), k, np.int32)); o_id.append(kf.obs_id[inside]); o_px.append(kf.obs_px[inside])
            o_kf, o_id, o_px = np.concatenate(o_kf), np.concatenate(o_id), np.concatenate(o_px)
            ids, inv, counts = np.unique(o_id, return_inverse=True, return_counts=True)
            multi = counts[inv] >= 2                       # points seen by a single keyframe do not constrain anything
            ids2, pt_idx = np.unique(o_id[multi], return_inverse=True)
            owner = np.searchsorted(hi, ids2, side="right")
            local = ids2 - lo[owner]
            base = np.concatenate([[0], np.cumsum([len(kf.pw) for kf in kfs])])
            flat = base[owner] + local                     # position of every BA point in the concatenated local map
            pts = np.concatenate([kf.pw for kf in kfs])[flat].reshape(-1, 3)
            problems.append((poses, fixed, pts, o_kf[multi], pt_idx.astype(np.int32), o_px[multi]))
            layouts.append((kfs, base, flat))
        results = self.be.local_ba(problems)
        for i, (P, X), (kfs, base, flat) in zip(idx, results, layouts):
            st = self.streams[i]
            for k, kf in enumerate(kfs):
                kf.T_cw = se3.se3_exp(P[k])
            pw_all = np.concatenate([kf.pw for kf in kfs])
            pw_all[flat] = X
            for k, kf in enumerate(kfs):
                kf.pw[:] = pw_all[base[k]:base[k + 1]]
            st.T_cw = kfs[-1].T_cw.copy()
            st.stats["ba"] += 1


def _depth_under(T, pw):
    """z of world points under T_cw, summed left to right (Camera::World2Camera(p, T)[2])."""
    pw = np.asarray(pw, np.float64).reshape(-1, 3)
    return T[2, 0] * pw[:, 0] + T[2, 1] * pw[:, 1] + T[2, 2] * pw[:, 2] + T[2, 3]


def _map_points(keyframes, ids):
    """World positions of map points `ids`, each owned by one of `keyframes` (mp_id ranges are contiguous per key-frame)."""
    out = np.empty((len(ids), 3))
    found = np.zeros(len(ids), bool)
    for kf in keyframes:
        if not len(kf.mp_id):
            continue
        sel = (ids >= kf.mp_id[0]) & (ids < kf.mp_id[0] + len(kf.mp_id))
        out[sel] = kf.pw[ids[sel] - kf.mp_id[0]]
        found |= sel
    assert found.all(), "a tracked map point outside the stream's key-frames"
    return out


# ---- backends ---------------------------------------------------------------------------------------------------
class GpuBackend:
    """Every call = one batched C-ABI call on the rank's context (ygz_slam_b200.capi)."""

    def __init__(self, ctx, n_slots: int, undistort=None):
        """undistort: (map_xy, map_a) of capi.undistort_map / cv2.initUndistortRectifyMap(.., CV_16SC2), or None.  With maps
        every frame is undistorted on the device as it is uploaded, and the loop's camera is the undistorted one."""
        self.ctx = ctx
        self.fr = ctx.frames(n_slots)
        if undistort is not None:
            self.fr.set_undistort(*undistort)

    def upload(self, slots, images):
        imgs = np.ascontiguousarray(np.stack(images))
        s = np.asarray(slots)
        if np.all(np.diff(s) == s[1] - s[0] if len(s) > 1 else True) and len(s) > 1 and s[1] - s[0] == 1:
            self.fr.upload(imgs, first=int(s[0]))
        else:
            for k, img in zip(slots, imgs):
                self.fr.upload(img[None], first=int(k))

    def detect(self, slots):
        return self.fr.detect(slots)

    def sparse_alignment(self, ref_slots, cur_slots, px, depth, T_ref):
        offs = np.concatenate([[0], np.cumsum([len(d) for d in depth])]).astype(np.int32)
        T = np.stack([t.reshape(-1) for t in T_ref])
        has = np.ones(int(offs[-1]), np.uint8)
        Tc, nm, _ = self.fr.sparse_align(ref_slots, cur_slots, offs, np.concatenate(px), np.concatenate(depth), has, T, T)
        ok = []
        for j in range(len(ref_slots)):  # Matcher::SparseImageAlignment's motion check (Matcher.cpp:482-488)
            ok.append(np.linalg.norm(se3.se3_log(se3.mul(Tc[j], se3.inv(T_ref[j])))) <= 0.2)
        return list(Tc), ok

    def project(self, jobs):
        """jobs: per stream dict(kfs, cur_slot, T_cur, kf (local keyframe index), n (feature index), init (u, v))."""
        # GetWarpAffineMatrix mixes world and reference-camera coordinates (Matcher.cpp:425-430; kept in the kernel for
        # parity), which is only correct for an identity reference pose.  The caller therefore hands over poses
        # relative to the reference keyframe: (T_ref, T_cur) -> (I, T_cur * T_ref^-1), mathematically the same problem.
        poses, rs, cs, rp, cp, rpx, rd, rl, init = [np.eye(4)[:3].reshape(-1)], [], [], [], [], [], [], [], []
        for job in jobs:
            base = len(poses)
            for kf in job["kfs"]:
                poses.append(se3.mul(job["T_cur"], se3.inv(kf.T_cw)).reshape(-1))
            m = len(job["kf"])
            slots = np.array([kf.slot for kf in job["kfs"]], np.int32)
            rs.append(slots[job["kf"]]); cs.append(np.full(m, job["cur_slot"], np.int32))
            rp.append(np.zeros(m, np.int32)); cp.append(base + job["kf"])
            allpx = [kf.px for kf in job["kfs"]]; alld = [kf.depth for kf in job["kfs"]]; alll = [kf.level for kf in job["kfs"]]
            off = np.concatenate([[0], np.cumsum([len(x) for x in alld])])
            flat = off[job["kf"]] + job["n"]
            rpx.append(np.concatenate(allpx)[flat]); rd.append(np.concatenate(alld)[flat]); rl.append(np.concatenate(alll)[flat])
            init.append(job["init"])
        total = sum(len(x) for x in rs)
        if total == 0:
            return [np.zeros((0, 2)) for _ in jobs], [np.zeros(0, bool) for _ in jobs]
        px, lvl, ok = self.fr.project_align(np.concatenate(rs), np.concatenate(cs), np.stack(poses), np.concatenate(rp).astype(np.int32),
                                            np.concatenate(cp).astype(np.int32), np.concatenate(rpx), np.concatenate(rd),
                                            np.concatenate(rl).astype(np.uint8), np.concatenate(init))
        out_px, out_ok, o = [], [], 0
        for x in rs:
            out_px.append(px[o:o + len(x)]); out_ok.append(ok[o:o + len(x)])
            o += len(x)
        return out_px, out_ok

    def pose_only(self, pts_w, obs, T, return_depth=False):
        """return_depth: also return pose-only's per-point depth (that of the point's last inlier round, else -1)."""
        offs = np.concatenate([[0], np.cumsum([len(p) for p in pts_w])]).astype(np.int32)
        Tn, inl, depth, cnt = self.ctx.pose_only(offs, np.concatenate(pts_w) if offs[-1] else np.zeros((0, 3)),
                                                 np.concatenate(obs) if offs[-1] else np.zeros((0, 2)), np.stack([t.reshape(-1) for t in T]))
        out = (list(Tn), [inl[offs[j]:offs[j + 1]] for j in range(len(T))], cnt)
        return out + ([depth[offs[j]:offs[j + 1]] for j in range(len(T))],) if return_depth else out

    def local_ba(self, problems):
        kf_off = np.concatenate([[0], np.cumsum([len(p[0]) for p in problems])]).astype(np.int32)
        pt_off = np.concatenate([[0], np.cumsum([len(p[2]) for p in problems])]).astype(np.int32)
        ob_off = np.concatenate([[0], np.cumsum([len(p[3]) for p in problems])]).astype(np.int32)
        g2o = np.concatenate([np.concatenate([p[0][:, 3:], p[0][:, :3]], 1) for p in problems])
        P, X, _, _ = self.ctx.local_ba(kf_off, pt_off, ob_off, g2o, np.concatenate([p[1] for p in problems]),
                                       np.concatenate([p[2] for p in problems]), np.concatenate([p[3] for p in problems]),
                                       np.concatenate([p[4] for p in problems]), np.concatenate([p[5] for p in problems]))
        out = []
        for j in range(len(problems)):
            Pj = P[kf_off[j]:kf_off[j + 1]]
            out.append((np.concatenate([Pj[:, 3:], Pj[:, :3]], 1), X[pt_off[j]:pt_off[j + 1]]))
        return out
