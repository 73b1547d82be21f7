"""A camera per stream of the streaming engine (ygz_vo_set_camera, ygzb_tracker_set_camera): one engine on a context with
camera A runs streams with cameras A, B, C and D, and every stream must give, byte for byte, what a one-stream engine on a
context whose camera is its own gives -- results, observation rows, information records, map updates and the exported
map.  Cameras come from crops of one render at different offsets (another principal point) and from a render with
another focal length; every value is the shortest decimal of a float, so each camera can also be a context's."""
import ctypes as C

import numpy as np
import pytest

from ygz_slam_b200 import se3, synth

POLICY = dict(kf_min_frames=5, kf_min_rot=0.03, kf_min_trans=0.03)
ERR_INVALID = -1
W, H, N = 640, 480, 24
CAM_A = (synth.FX, synth.FY, synth.CX, synth.CY)


def render(tex, f, w, h, cx, cy, plane_z=2.0, metres_per_texel=0.0025):
    """synth.render_plane at the identity pose with focal lengths f = (fx, fy)."""
    u, v = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    size = tex.shape[0]
    tx = np.clip((u - cx) / f[0] * plane_z / metres_per_texel + size / 2, 0, size - 1.001)
    ty = np.clip((v - cy) / f[1] * plane_z / metres_per_texel + size / 2, 0, size - 1.001)
    x0, y0 = tx.astype(np.int32), ty.astype(np.int32)
    a, b = tx - x0, ty - y0
    t = tex.astype(np.float64)
    val = (1 - b) * ((1 - a) * t[y0, x0] + a * t[y0, x0 + 1]) + b * ((1 - a) * t[y0 + 1, x0] + a * t[y0 + 1, x0 + 1])
    return np.clip(np.rint(val), 0, 255).astype(np.uint8)


def crops(seed, f, x0, y0, n=N, plane_z=2.0):
    """n W x H crops sliding over one render with focal lengths f, starting at (x0, y0) of it: frames, depth, ground-truth
    poses and the crops' camera."""
    tex = synth.texture(seed, 2048)
    bw, bh = W + 256, H + 128
    base = render(tex, f, bw, bh, bw / 2, bh / 2, plane_z)
    rng = np.random.default_rng(seed)
    offs = [(x0 + int(round(60 * np.sin(2 * np.pi * k / 120))), y0 + int(round(30 * np.sin(2 * np.pi * k / 90)))) for k in range(n)]
    frames, poses = [], []
    for ox, oy in offs:
        c = base[oy:oy + H, ox:ox + W].astype(np.int16) + np.rint(rng.normal(0, 2.0, (H, W))).astype(np.int16)
        frames.append(np.clip(c, 0, 255).astype(np.uint8))
        T = np.eye(4)[:3].copy()
        T[0, 3] = -(ox - offs[0][0]) * plane_z / f[0]
        T[1, 3] = -(oy - offs[0][1]) * plane_z / f[1]
        poses.append(T)
    return frames, np.full((H, W), plane_z), poses, (f[0], f[1], bw / 2 - offs[0][0], bh / 2 - offs[0][1])


@pytest.fixture(scope="module")
def sequences():
    """Four streams: camera A (synth.shift_stream), B and C (crops at other offsets: another cx, cy), D (focal 450, 451)."""
    fr, dep, poses = synth.shift_stream(0, N)
    seqs = [(list(fr), dep, poses, CAM_A)]
    seqs.append(crops(0x59475A10, (synth.FX, synth.FY), 70, 64))
    seqs.append(crops(0x59475A20, (synth.FX, synth.FY), 186, 40))
    seqs.append(crops(0x59475A30, (450.0, 451.0), 128, 64))
    for s in seqs:
        assert all(float(str(np.float32(v))) == v for v in s[3])   # the shortest decimal of a float
    assert len({s[3] for s in seqs}) == 4
    return seqs


def _cols(a, names):
    """The bytes of fields `names` of structured array `a` (a multi-field view keeps the other fields' bytes)."""
    return b"".join(np.ascontiguousarray(a[n]).tobytes() for n in names)


def _ctx(K):
    from ygz_slam_b200 import Context
    return Context(0, image_width=W, image_height=H, fx=K[0], fy=K[1], cx=K[2], cy=K[3])


def _feed(eng, streams, data, pacing):
    """Push frames of the given engine streams (data[s] = frames, depth) in lock step; pacing 'each': a step after every
    push round, 'burst': a step every 5 frames."""
    for k in range(N):
        for s in streams:
            eng.push(s, data[s][0][k], data[s][1] if k == 0 or k % 7 == 0 else None)
        if pacing == "each" or k % 5 == 4:
            eng.step()
    eng.flush()


def _run(eng, streams, data, pacing):
    _feed(eng, streams, data, pacing)
    res, rows, info = eng.poll()
    upd, urows = eng.poll_map_updates()
    out = {}
    for s in streams:
        m = res["stream"] == s
        ks = np.flatnonzero(m)
        u = upd["stream"] == s
        mp = eng.export_map(s)
        out[s] = dict(res=_cols(res[m], ["frame", "status", "n_inliers", "T_cw"]), rows=b"".join(rows[k].tobytes() for k in ks),
                      info=info[m].tobytes(), upd=_cols(upd[u], [n for n in upd.dtype.names if n != "stream"]),
                      urows=b"".join(urows[k].tobytes() for k in np.flatnonzero(u)), K=tuple(mp.rec.K),
                      map=b"".join(np.asarray(v).tobytes() for v in mp.a.values()), T=res["T_cw"][m].copy())
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
@pytest.mark.parametrize("window,pacing", [(1, "each"), (4, "burst"), (8, "each"), (8, "burst")])
def test_streams_match_one_camera_engines(sequences, ref_mode, window, pacing):
    from ygz_slam_b200 import vo_native
    data = [(s[0], s[1]) for s in sequences]
    cams = [s[3] for s in sequences]
    opts = dict(window=window, ref_mode=ref_mode, observations=True, information=True, map_updates=True, **POLICY)
    ctx = _ctx(CAM_A)
    try:
        with vo_native.Engine(ctx, 4, cameras=cams, **opts) as eng:
            assert [tuple(eng.camera(s)) for s in range(4)] == cams
            got = _run(eng, range(4), data, pacing)
    finally:
        ctx.close()
    for s, K in enumerate(cams):
        ctx = _ctx(K)
        try:
            with vo_native.Engine(ctx, 1, **opts) as eng:
                want = _run(eng, [0], [data[s]], pacing)[0]
        finally:
            ctx.close()
        for key in ("res", "rows", "info", "upd", "urows", "K", "map"):
            assert got[s][key] == want[key], (s, key)
        assert got[s]["K"] == K
        # and the stream tracks its ground truth
        for k, T in enumerate(got[s]["T"]):
            assert np.linalg.norm(se3.se3_log(se3.mul(T.reshape(3, 4), se3.inv(sequences[s][2][k])))) < 3e-3, (s, k)


@pytest.mark.gpu
def test_restart_with_another_camera(sequences):
    """set_camera while a restart is pending: the frames pushed before keep camera A's results, the new sequence gives
    those of a fresh engine with camera D."""
    from ygz_slam_b200 import vo_native
    fa, da = sequences[0][0], sequences[0][1]
    fd, dd, _, KD = sequences[3]
    ctx = _ctx(CAM_A)
    try:
        with vo_native.Engine(ctx, 1, window=4, **POLICY) as eng:
            for k in range(12):
                eng.push(0, fa[k], da if k == 0 else None)
            assert eng.lib.ygz_vo_set_camera(eng.h, 0, np.array(KD).ctypes.data) == ERR_INVALID   # mid-sequence
            eng.restart(0)
            eng.set_camera(0, KD)
            eng.set_camera(0, (1.0, 1.0, 1.0, 1.0))
            eng.set_camera(0, KD)   # the last one counts
            for k in range(12):
                eng.push(0, fd[k], dd if k == 0 else None)
            eng.flush()
            res = eng.poll()
        with vo_native.Engine(ctx, 1, window=4, **POLICY) as ref_a:
            for k in range(12):
                ref_a.push(0, fa[k], da if k == 0 else None)
            ref_a.flush()
            want_a = ref_a.poll()
    finally:
        ctx.close()
    ctx = _ctx(KD)
    try:
        with vo_native.Engine(ctx, 1, window=4, **POLICY) as ref_d:
            for k in range(12):
                ref_d.push(0, fd[k], dd if k == 0 else None)
            ref_d.flush()
            want_d = ref_d.poll()
    finally:
        ctx.close()
    cols = ["status", "n_inliers", "T_cw"]
    assert _cols(res[:12], cols) == _cols(want_a, cols)
    assert _cols(res[12:], cols) == _cols(want_d, cols)


@pytest.mark.gpu
@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
def test_stream_record_with_its_camera(sequences, ref_mode):
    """A record saved from a stream with camera B loads into a stream set to B of another engine and continues bit for
    bit; a stream still on A refuses it and stays as it was.  Hand-over into a stream that has tracked: flush, restart,
    set_camera, load."""
    from ygz_slam_b200 import vo_native
    fb, db, _, KB = sequences[1]
    fa, da = sequences[0][0], sequences[0][1]
    opts = dict(window=4, ref_mode=ref_mode, **POLICY)
    half = N // 2
    ctx = _ctx(CAM_A)
    try:
        with vo_native.Engine(ctx, 2, cameras=[None, KB], **opts) as src:
            for k in range(N):
                src.push(1, fb[k], db if k == 0 else None)
                if k == half - 1:
                    src.flush()
                    rec = src.save_stream(1)
            src.flush()
            want = src.poll()
            want = _cols(want[want["frame"] >= half], ["frame", "status", "n_inliers", "T_cw"])
        with vo_native.Engine(ctx, 3, **opts) as dst:
            for k in range(6):
                dst.push(2, fa[k], da if k == 0 else None)
            dst.flush()
            before = dst.save_stream(2)
            with pytest.raises(Exception):
                dst.load_stream(2, rec)   # stream 2 is on A
            assert dst.save_stream(2) == before
            assert dst.lib.ygz_vo_load_stream(dst.h, 0, np.frombuffer(rec, np.uint8).ctypes.data, len(rec)) == ERR_INVALID
            dst.restart(2)
            dst.set_camera(2, KB)
            dst.load_stream(2, rec)
            assert tuple(dst.camera(2)) == KB
            for k in range(half, N):
                dst.push(2, fb[k], None)
            dst.flush()
            got = dst.poll()
            got = _cols(got[(got["stream"] == 2) & (got["frame"] >= half)], ["frame", "status", "n_inliers", "T_cw"])
    finally:
        ctx.close()
    assert got == want


@pytest.mark.gpu
def test_invalid_cameras(sequences):
    """Every refusal returns YGZB_ERR_INVALID and changes nothing; the valid pushes that follow give the undisturbed
    results."""
    from ygz_slam_b200 import vo_native
    fb, db, _, KB = sequences[1]
    ctx = _ctx(CAM_A)
    try:
        with vo_native.Engine(ctx, 2, window=4, **POLICY) as eng:
            lib = eng.lib
            good = np.array(KB, np.float64)
            assert lib.ygz_vo_set_camera(eng.h, 2, good.ctypes.data) == ERR_INVALID
            assert lib.ygz_vo_set_camera(eng.h, -1, good.ctypes.data) == ERR_INVALID
            assert lib.ygz_vo_set_camera(None, 0, good.ctypes.data) == ERR_INVALID
            assert lib.ygz_vo_set_camera(eng.h, 0, None) == ERR_INVALID
            assert lib.ygz_vo_get_camera(eng.h, 0, None) == ERR_INVALID
            for k, v in ((0, np.nan), (1, np.inf), (2, -np.inf), (0, 0.0), (1, -1.0)):
                bad = good.copy()
                bad[k] = v
                assert lib.ygz_vo_set_camera(eng.h, 0, bad.ctypes.data) == ERR_INVALID, (k, v)
            assert tuple(eng.camera(0)) == CAM_A
            eng.set_camera(0, KB)
            for k in range(10):
                eng.push(0, fb[k], db if k == 0 else None)
            assert lib.ygz_vo_set_camera(eng.h, 0, np.array(CAM_A).ctypes.data) == ERR_INVALID   # mid-sequence
            assert tuple(eng.camera(0)) == KB
            eng.flush()
            got = _cols(eng.poll(), ["status", "n_inliers", "T_cw"])
        _tracker_invalid(ctx)
    finally:
        ctx.close()
    ctx = _ctx(KB)
    try:
        with vo_native.Engine(ctx, 1, window=4, **POLICY) as ref:
            for k in range(10):
                ref.push(0, fb[k], db if k == 0 else None)
            ref.flush()
            want = _cols(ref.poll(), ["status", "n_inliers", "T_cw"])
    finally:
        ctx.close()
    assert got == want


def _tracker_invalid(ctx):
    """ygzb_tracker_set_camera's refusals leave every stream's camera as it was (the K its map records carry)."""
    from ygz_slam_b200 import capi
    fr = ctx.frames(4)
    tr = capi.Tracker(fr, 2, 4, CAM_A)
    lib = fr.lib
    h = tr.h
    KD = (450.0, 451.0, 320.0, 240.0)
    tr.set_camera(0, KD)
    cams = lambda: [tuple(tr.export(s, [], images=False).rec.K) for s in range(2)]   # noqa: E731
    assert cams() == [KD, CAM_A]
    good = np.array(CAM_A, np.float64)
    assert lib.ygzb_tracker_set_camera(None, 0, good.ctypes.data) == ERR_INVALID
    assert lib.ygzb_tracker_set_camera(h, 0, None) == ERR_INVALID
    assert lib.ygzb_tracker_set_camera(h, 2, good.ctypes.data) == ERR_INVALID
    assert lib.ygzb_tracker_set_camera(h, -1, good.ctypes.data) == ERR_INVALID
    for s in range(2):
        for k, v in ((3, np.nan), (0, 0.0), (1, -2.0), (2, np.inf)):
            bad = good.copy()
            bad[k] = v
            assert lib.ygzb_tracker_set_camera(h, s, bad.ctypes.data) == ERR_INVALID, (s, k, v)
    assert cams() == [KD, CAM_A]
    tr.set_camera(1, KD)
    assert cams() == [KD, KD]
    tr.close()
    fr.close()


# ---- the Python loop (vo.VisualOdometry) on the CPU oracle with a camera of its own --------------------------------------
class _CameraOracle:
    """The oracle with camera K in every call that takes one (the oracle's default is the TUM camera)."""

    def __init__(self, oracle, K):
        from oracle.pyoracle import Camera
        self.o, self.cam = oracle, Camera(*K)

    def __getattr__(self, name):
        f = getattr(self.o, name)
        if name in ("matcher_sparse_alignment", "find_direct_projection", "pose_only", "local_ba"):
            return lambda *a, **kw: f(*a, cam=self.cam, **kw)
        return f


@pytest.mark.gpu
@pytest.mark.parametrize("s", [1, 3])
def test_camera_stream_matches_the_oracle_loop(oracle, sequences, s):
    """A stream with a camera that is not the context's (B: another principal point, D: another focal length) tracks what
    vo.VisualOdometry(camera=K) tracks on the CPU oracle with camera K, within the loop tests' 1e-4, and its ground truth
    within 3e-3."""
    from oracle.vo_backend import OracleBackend
    from ygz_slam_b200 import vo, vo_native
    frames, depth, poses, K = sequences[s]
    V = vo.VisualOdometry(OracleBackend(_CameraOracle(oracle, K)), 1, camera=K, **POLICY)
    for k in range(N):
        V.add_frames([frames[k]], [depth], k)
    want = V.streams[0]
    assert not want.lost
    ctx = _ctx(CAM_A)
    try:
        with vo_native.Engine(ctx, 2, window=8, cameras=[None, K], **POLICY) as eng:
            for k in range(N):
                eng.push(1, frames[k], depth if k == 0 else None)
            eng.flush()
            res = eng.poll()
            stats = eng.stats(1)
    finally:
        ctx.close()
    assert res["frame"].tolist() == list(range(N)) and (res["status"] != 2).all()
    assert stats["keyframes"] == want.stats["keyframes"] and stats["lost"] == 0
    worst = 0.0
    for k in range(N):
        T = res["T_cw"][k].reshape(3, 4)
        worst = max(worst, float(np.linalg.norm(se3.se3_log(se3.mul(T, se3.inv(want.trajectory[k]))))))
        assert np.linalg.norm(se3.se3_log(se3.mul(T, se3.inv(poses[k])))) < 3e-3, k
    assert worst < 1e-4, worst


# ---- the tracker stage by stage, on imported maps -----------------------------------------------------------------------
KF_SLOT0, MP0, LEVELS = 8, (0, 10000, 20000), 3
KF_IDX, CUR_IDX = (0, 4, 8), (10, 11)


def _backproject(T, px, d, K):
    pc = np.stack([(px[:, 0] - K[2]) * d / K[0], (px[:, 1] - K[3]) * d / K[1], d], 1)
    Tin = se3.inv(T)
    return (Tin[:, :3] @ pc.T).T + Tin[:, 3]


def _map(seq, cells, seed):
    """The map record of key-frames KF_IDX of a sequence: a feature in every grid cell at its rendered depth, map points
    back-projected with the sequence's camera under the true pose."""
    from ygz_slam_b200 import capi
    frames, depth, poses, K = seq
    rec = capi.MapBuffers(capi.TRACK_RING, W, H, cells)
    r, a = rec.rec, rec.a
    r.width, r.height, r.cells, r.n_levels, r.n_keyframes = W, H, cells, LEVELS, len(KF_IDX)
    r.K[:] = list(K)
    for k, i in enumerate(KF_IDX):
        px, d = synth.pixel_features(depth, cells, seed=seed + k, margin=12)
        f0 = k * cells
        a["entry"][k], a["T_cw"][k], a["mp0"][k], a["n_features"][k], a["n_obs"][k] = k, poses[i].reshape(-1), MP0[k], cells, 0
        a["image"][k] = frames[i]
        a["px"][f0:f0 + cells], a["depth"][f0:f0 + cells] = px, d
        a["level"][f0:f0 + cells] = np.random.default_rng(seed + k).integers(0, LEVELS, cells)
        a["pw"][f0:f0 + cells] = _backproject(poses[i], px, d, K)
    return rec


def _stages(tr, streams, seqs, maps):
    """Import the maps, track CUR_IDX of every stream in ONE batch, insert a key-frame per stream behind the first job (with
    its local BA) and export the ring: (debug views, results, key-frame results, exported maps)."""
    entries = np.arange(len(KF_IDX), dtype=np.int32)
    for s, m in zip(streams, maps):
        tr.import_(s, entries, KF_SLOT0 + 4 * s + entries, m)
    cur = [seqs[q][0][i] for q in range(len(streams)) for i in CUR_IDX]
    tr.upload(0, np.stack(cur))
    jobs = [(s, 2 * q + t, [0, 1, 2]) for q, s in enumerate(streams) for t in range(len(CUR_IDX))]
    res = tr.track(jobs)
    views = [tr.debug_job(j) for j in range(len(jobs))]
    for q, s in enumerate(streams):
        tr.set_depth(s, seqs[q][1])
    kres = tr.make_keyframes([dict(stream=s, frame_slot=2 * q, kf_slot=KF_SLOT0 + 4 * s + 3, entry=3, track_job=2 * q, local_entry=[1, 2, 3],
                                   run_ba=1, mp0=30000) for q, s in enumerate(streams)])
    maps_out = [tr.export(s, [1, 2, 3]) for s in streams]
    return views, res, kres, maps_out


def _project(T, pw, K):
    x = T[0, 0] * pw[:, 0] + T[0, 1] * pw[:, 1] + T[0, 2] * pw[:, 2] + T[0, 3]
    y = T[1, 0] * pw[:, 0] + T[1, 1] * pw[:, 1] + T[1, 2] * pw[:, 2] + T[1, 3]
    z = T[2, 0] * pw[:, 0] + T[2, 1] * pw[:, 1] + T[2, 2] * pw[:, 2] + T[2, 3]
    with np.errstate(divide="ignore", invalid="ignore"):
        u, v = K[0] * x / z + K[2], K[1] * y / z + K[3]
    return (z > 0) & (u >= 20) & (u < W - 20) & (v >= 20) & (v < H - 20)


def _map_arrays(m):
    return {k: np.asarray(v).copy() for k, v in m.a.items()} | dict(K=tuple(m.rec.K))


@pytest.mark.gpu
def test_tracker_stages_with_three_cameras(sequences):
    """One tracker on a context with camera A, streams with cameras A, B and D (ygzb_tracker_set_camera), one batch: every
    stage of every job -- sparse alignment, rel, candidates (cand_px, cand_ok), compaction, pose-only inliers -- and the
    key-frame insertion behind it -- features, depths, map points, the local BA -- equal, bit for bit, those of a
    one-stream tracker created with the stream's camera on a context whose camera it is."""
    from ygz_slam_b200 import capi
    seqs = [sequences[0], sequences[1], sequences[3]]
    ctx = _ctx(CAM_A)
    try:
        cells = ctx.n_cells
        maps = [_map(q, cells, 100 * i) for i, q in enumerate(seqs)]
        fr = ctx.frames(KF_SLOT0 + 4 * 3)
        tr = capi.Tracker(fr, 3, 8, CAM_A)
        for s in (1, 2):
            tr.set_camera(s, seqs[s][3])
        got = _stages(tr, [0, 1, 2], seqs, maps)
        tr.close()
        fr.close()
    finally:
        ctx.close()
    for q, seq in enumerate(seqs):
        K = seq[3]
        ctx = _ctx(K)
        try:
            fr = ctx.frames(KF_SLOT0 + 4)
            tr = capi.Tracker(fr, 1, 8, K)
            want = _stages(tr, [0], [seq], [maps[q]])
            tr.close()
            fr.close()
        finally:
            ctx.close()
        for t in range(len(CUR_IDX)):
            g, w = got[0][2 * q + t], want[0][t]
            for k in ("T_aligned", "rel", "n_local", "n_meas", "aligned", "n_candidates", "n_projected", "n_inliers", "cand_ok", "c_src",
                      "c_px", "c_pw", "inlier"):
                assert np.array_equal(g[k], w[k]), (q, t, k)
            assert g["aligned"] and g["n_inliers"] > 500, (q, t)
            # every candidate (double-K projection into the border-20 window) has its FindDirectProjection pixel
            cand = np.zeros(len(g["cand_ok"]), bool)
            for k in range(3):
                sl = slice(k * cells, (k + 1) * cells)
                cand[sl] = _project(g["T_aligned"], maps[q].a["pw"][sl], K)
            assert cand.sum() == g["n_candidates"] and not (g["cand_ok"] & ~cand).any(), q
            assert np.array_equal(g["cand_px"][cand], w["cand_px"][cand]), (q, t)
            for k in got[1][2 * q + t]:
                assert np.array_equal(got[1][2 * q + t][k], want[1][t][k]), (q, t, k)
        for k in got[2][q]:
            assert np.array_equal(got[2][q][k], want[2][0][k]), (q, k)
        assert got[2][q]["ba_points"] > 0 and got[2][q]["ba_iters"] > 0
        gm, wm = _map_arrays(got[3][q]), _map_arrays(want[3][0])
        assert gm["K"] == wm["K"] == K
        for k in wm:
            assert np.array_equal(gm[k], wm[k]), (q, k)


@pytest.mark.gpu
def test_tracker_records_carry_the_stream_camera(sequences):
    """Map and reference records: export writes the stream's own camera, an import into a stream with that camera gives
    back the same record byte for byte, and an import into a stream with another camera -- the tracker's creation camera
    included -- is refused and changes nothing."""
    from ygz_slam_b200 import capi
    KB, KD = sequences[1][3], sequences[3][3]
    ctx = _ctx(CAM_A)
    try:
        cells = ctx.n_cells
        fr = ctx.frames(KF_SLOT0 + 4 * 3 + 3)
        tr = capi.Tracker(fr, 3, 8, CAM_A)
        lib = fr.lib
        entries = np.arange(3, dtype=np.int32)
        tr.set_camera(1, KB)
        tr.import_(1, entries, KF_SLOT0 + 4 + entries, _map(sequences[1], cells, 7))
        rec = tr.export(1, entries)
        assert tuple(rec.rec.K) == KB
        # into a stream on A, then on D: refused, the stream's map unchanged
        tr.set_camera(2, KD)
        for s in (0, 2):
            before = _map_arrays(tr.export(s, entries))
            rc = lib.ygzb_tracker_import(tr.h, s, entries.ctypes.data, (KF_SLOT0 + 4 * s + entries).ctypes.data, C.byref(rec.rec))
            assert rc == ERR_INVALID, s
            after = _map_arrays(tr.export(s, entries))
            for k in before:
                assert np.array_equal(before[k], after[k]), (s, k)
        # into stream 2 set to B: the same record back
        tr.set_camera(2, KB)
        tr.import_(2, entries, KF_SLOT0 + 8 + entries, rec)
        back = _map_arrays(tr.export(2, entries))
        for k, v in _map_arrays(rec).items():
            assert np.array_equal(back[k], v), k
        tr.close()
        fr.close()
        # reference records (previous-frame mode)
        fr = ctx.frames(KF_SLOT0 + 4 * 3 + 3)
        tr = capi.Tracker(fr, 3, 8, CAM_A)
        tr.set_reference_mode("previous", [KF_SLOT0 + 12 + s for s in range(3)])
        ref = capi.ReferenceBuffers(W, H, cells)
        r = ref.rec
        r.width, r.height, r.cells, r.n_levels, r.n = W, H, cells, LEVELS, 500
        r.K[:] = list(KB)
        r.T_cw[:] = list(sequences[1][2][3].reshape(-1))
        px, d = synth.pixel_features(sequences[1][1], 500, seed=11, margin=12)
        ref.a["px"][:500], ref.a["depth"][:500], ref.a["image"][:] = px, d, sequences[1][0][3]
        tr.set_camera(1, KB)
        for s in (0, 2):   # stream 0 on A (the creation camera), stream 2 on D: refused
            if s == 2:
                tr.set_camera(2, KD)
            assert lib.ygzb_tracker_import_reference(tr.h, s, C.byref(r)) == ERR_INVALID, s
            assert lib.ygzb_tracker_export_reference(tr.h, s, C.byref(capi.ReferenceBuffers(W, H, cells).rec)) == ERR_INVALID, s   # still none
        tr.import_reference(1, ref)
        out = tr.export_reference(1)
        assert tuple(out.rec.K) == KB and out.rec.n == 500 and np.array_equal(out.T_cw, ref.T_cw)
        for k in ref.a:
            assert np.array_equal(out.a[k], ref.a[k]), k
        tr.set_camera(2, KB)
        tr.import_reference(2, out)
        again = tr.export_reference(2)
        for k in ref.a:
            assert np.array_equal(again.a[k], ref.a[k]), k
        tr.close()
        fr.close()
    finally:
        ctx.close()
