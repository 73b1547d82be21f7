"""The device-resident tracker (ygzb_tracker_*) stage by stage against the oracle, on local maps built on the host and put
into a stream with ygzb_tracker_import.  ygzb_tracker_debug_job reads back what each stage of a tracking job computed, so
every stage is compared with the oracle on the inputs the engine actually used:

  a. sparse alignment + composition   n_meas exactly, the pose within 1e-4 (oracle.sparse_align); aligned = the 0.2 rule;
                                      rel[k] exactly (the 3x4 products of track_motion_kernel restated in numpy)
  b. candidates + direct projection   bit for bit: the candidate test of track_project_kernel restated in numpy (f64, the
                                      kernel's operation order), oracle.find_direct_projection per candidate
  c. compaction                       c_src = flatnonzero(cand_ok), c_px / c_pw copied exactly, c_cnt = n_projected
  d. pose-only                        oracle.pose_only from the aligned pose: inliers and their count identical, the pose
                                      within 1e-4
  e. key-frame insertion              Detect, depth, back-projection and the tracked observations exactly
  f. local BA                         assembly (counts exactly, the initial chi2 to 1e-10 relative), the result within 1e-4
                                      of oracle.local_ba, everything outside the BA untouched; truncated (max_iters 1 and
                                      3, max_trials 1) the same iterations, trials, poses and points as ygzb_local_ba on
                                      the problem the host assembles
  g. batches                          a job's result does not depend on the batch around it

Scenes are rendered frames of synth.stream_frame (the textured plane z = 2 seen along synth.trajectory).  The maps are
made by hand: key-frames with no features, with every grid cell filled, map points placed exactly on both sides of the
20-pixel border, behind the camera and at z = 0, observations outside the local window."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from ygz_slam_b200 import se3, synth

ROOT = Path(__file__).resolve().parent.parent
W, H, LEVELS = synth.W, synth.H, 3
K = (synth.FX, synth.FY, synth.CX, synth.CY)
KF_FRAMES = (0, 4, 8)          # frames of the three imported key-frames (oldest first); the newest is the reference
CUR_FRAMES = (10, 11)          # frames tracked against them
KF_SLOT0 = 16                  # frame slots of the key-frames: KF_SLOT0 + 4 * stream + ring entry
MP0 = (0, 10000, 20000)        # first map point id of each imported key-frame
MP0_NEW = 30000


def test_track_debug_layout_matches_the_header(tmp_path):
    """capi.TrackDebug has the size and field offsets of ygzb_track_debug as a C compiler lays it out."""
    from ygz_slam_b200 import capi
    fields = [f for f, _ in capi.TrackDebug._fields_]
    src = tmp_path / "layout.c"
    body = "\n".join(f'    printf("%s %%zu\\n", offsetof(ygzb_track_debug, {f}));' % f for f in fields)
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "ygz_b200.h"\nint main(void) {\n'
                   '    printf("sizeof %%zu\\n", sizeof(ygzb_track_debug));\n%s\n    return 0;\n}\n' % body)
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", f"-I{ROOT / 'include'}", str(src), "-o", str(exe)], check=True,
                   capture_output=True, text=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(got["sizeof"]) == C.sizeof(capi.TrackDebug)
    for f in fields:
        assert int(got[f]) == getattr(capi.TrackDebug, f).offset, f


# ---- host restatements of the kernels' arithmetic (f64, no contraction: align.cu and track.cu build with -fmad=false) ----
def mat34_mul(A, B):
    """track_motion_kernel's mat34_mul, operation by operation."""
    a, b = np.asarray(A, np.float64).reshape(-1), np.asarray(B, np.float64).reshape(-1)
    C_ = np.empty(12)
    for r in range(3):
        for c in range(3):
            C_[4 * r + c] = a[4 * r] * b[c] + a[4 * r + 1] * b[4 + c] + a[4 * r + 2] * b[8 + c]
        C_[4 * r + 3] = a[4 * r] * b[3] + a[4 * r + 1] * b[7] + a[4 * r + 2] * b[11] + a[4 * r + 3]
    return C_.reshape(3, 4)


def mat34_inv(A):
    a = np.asarray(A, np.float64).reshape(-1)
    C_ = np.empty(12)
    for r in range(3):
        for c in range(3):
            C_[4 * r + c] = a[4 * c + r]
        C_[4 * r + 3] = -(a[r] * a[3] + a[4 + r] * a[7] + a[8 + r] * a[11])
    return C_.reshape(3, 4)


def project(T, pw):
    """The candidate test of track_project_kernel (LocalMapping::FindCandidates): (u, v, mask)."""
    t = np.asarray(T, np.float64).reshape(-1)
    X0, X1, X2 = (np.asarray(pw, np.float64).reshape(-1, 3)[:, i] for i in range(3))
    x = t[0] * X0 + t[1] * X1 + t[2] * X2 + t[3]
    y = t[4] * X0 + t[5] * X1 + t[6] * X2 + t[7]
    z = t[8] * X0 + t[9] * X1 + t[10] * X2 + t[11]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = K[0] * x / z + K[2]
        v = K[1] * y / z + K[3]
    return u, v, (z > 0) & (u >= 20) & (u < W - 20) & (v >= 20) & (v < H - 20)


def backproject(T, px, d):
    """kf_fill_kernel's map point: camera point from the depth, then the inverse pose (mat34_inv), operation by operation."""
    Ti = mat34_inv(T).reshape(-1)
    pc0 = (px[:, 0] - K[2]) * d / K[0]
    pc1 = (px[:, 1] - K[3]) * d / K[1]
    pc2 = d
    return np.stack([Ti[4 * r] * pc0 + Ti[4 * r + 1] * pc1 + Ti[4 * r + 2] * pc2 + Ti[4 * r + 3] for r in range(3)], 1)


def _scalar_z(t, X):
    return t[8] * X[0] + t[9] * X[1] + t[10] * X[2] + t[11]


def _scalar_uv(t, X):
    x = t[0] * X[0] + t[1] * X[1] + t[2] * X[2] + t[3]
    y = t[4] * X[0] + t[5] * X[1] + t[6] * X[2] + t[7]
    z = _scalar_z(t, X)
    return K[0] * x / z + K[2], K[1] * y / z + K[3]


def below(edge, c):
    """The largest value under `edge` that u = fx * x / z + c can take: fx * x / z and c are multiples of the spacing of
    doubles at c (|fx * x / z| is in c's binade at both borders), so the rounded sum lies on the coarser of that grid and
    the grid at the edge (20 - 2^-44 for u = 20, not 20 - 1 ulp)."""
    return edge - max(np.spacing(edge), np.spacing(c), np.spacing(edge - c))


def border_targets():
    """(axis, value) of the border points: u = 20 and the value below it, W - 20 and below, the same for v."""
    return [(axis, t) for axis, c, edges in ((0, K[2], (20.0, float(W - 20))), (1, K[3], (20.0, float(H - 20))))
            for e in edges for t in (e, below(e, c))]


def border_points(T, seed=0):
    """World points whose candidate test under T gives exactly each value of border_targets() (the other coordinate well
    inside), one point with z < 0 and one with z = 0 exactly.  Found by bisection over one world coordinate (u grows with
    x_w, v with y_w for a camera looking along +z)."""
    t = [float(c) for c in np.asarray(T).reshape(-1)]
    R, tr = np.asarray(T)[:, :3], np.asarray(T)[:, 3]
    rng = np.random.default_rng(seed)
    out = []
    for axis, target in border_targets():
        for _ in range(2000):
            z = rng.uniform(1.8, 2.4)
            uv = [rng.uniform(100, W - 100), rng.uniform(100, H - 100)]
            uv[axis] = target
            pc = np.array([(uv[0] - K[2]) / K[0] * z, (uv[1] - K[3]) / K[1] * z, z])
            X = [float(c) for c in R.T @ (pc - tr)]
            lo, hi = X[axis] - 1e-3, X[axis] + 1e-3
            f = lambda c: _scalar_uv(t, X[:axis] + [c] + X[axis + 1:])[axis]   # noqa: E731
            assert f(lo) < target <= f(hi)
            while True:
                mid = lo + (hi - lo) / 2
                if mid <= lo or mid >= hi:
                    break
                if f(mid) >= target:
                    hi = mid
                else:
                    lo = mid
            if f(hi) == target:
                X[axis] = hi
                out.append(X)
                break
        else:
            raise AssertionError(f"no world point lands exactly on {target!r}")
    out.append([float(c) for c in R.T @ (np.array([0.2, -0.1, -1.5]) - tr)])     # behind the camera
    for _ in range(2000):                                                           # in the camera's plane z = 0
        X = [float(c) for c in R.T @ (np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), 0.0]) - tr)]
        c0 = -(t[8] * X[0] + t[9] * X[1] + t[11]) / t[10]
        hit = [c for c in (c0 + k * abs(c0) * 2.0 ** -52 for k in range(-40, 41)) if _scalar_z(t, X[:2] + [c]) == 0.0]
        if hit:
            out.append(X[:2] + [hit[0]])
            break
    else:
        raise AssertionError("no world point with z = 0 exactly")
    return np.array(out)


# ---- scenes ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def frames(oracle):
    """Rendered frames (stream 0) by frame index: gray, depth map, true T_cw and the oracle's pyramid."""
    out = {}
    for k in KF_FRAMES + CUR_FRAMES + (12,):
        g, d, T = synth.stream_frame(k)
        out[k] = dict(gray=g, depth=d, T=T, pyr=oracle.build_pyramid(g, LEVELS))
    # the camera 0.3 m closer to the plane than at the reference key-frame (frame 8): the alignment follows it (to 6e-4 on
    # the oracle) and the motion, 0.30, fails Matcher::SparseImageAlignment's 0.2 rule
    T = out[8]["T"].copy()
    T[2, 3] -= 0.3
    g, d = synth.render_plane(synth.texture(0x59475A00, 2048), T, noise_sigma=2.0, seed=5)
    out["far"] = dict(gray=g, depth=d, T=T, pyr=oracle.build_pyramid(g, LEVELS))
    return out


def _kf(fr, T, px, level, depth, pw, mp0, obs_id=(), obs_px=()):
    return dict(gray=fr["gray"], pyr=fr["pyr"], T=np.asarray(T, np.float64).reshape(3, 4), px=np.asarray(px, np.float64).reshape(-1, 2),
                level=np.asarray(level, np.int32), depth=np.asarray(depth, np.float64), pw=np.asarray(pw, np.float64).reshape(-1, 3),
                mp0=mp0, obs_id=np.asarray(obs_id, np.int64), obs_px=np.asarray(obs_px, np.float64).reshape(-1, 2))


def detected_kf(oracle, fr, mp0, limit=None, **obs):
    """A key-frame as SetKeyframe makes it: the oracle's Detect, the rendered depth, map points under the true pose."""
    f = oracle.detect(fr["pyr"], n_levels=LEVELS)
    n = f["n"] if limit is None else min(limit, f["n"])
    px = np.stack([f["px"], f["py"]], 1)[:n]
    d = fr["depth"][px[:, 1].astype(int), px[:, 0].astype(int)]
    return _kf(fr, fr["T"], px, f["level"][:n], d, backproject(fr["T"], px, d), mp0, **obs)


def filled_kf(fr, cells, mp0, seed=3):
    """A key-frame with a feature in every grid cell: random sub-pixel positions with their rendered depth."""
    px, d = synth.pixel_features(fr["depth"], cells, seed=seed, margin=12)
    level = np.random.default_rng(seed).integers(0, LEVELS, cells)
    return _kf(fr, fr["T"], px, level, d, backproject(fr["T"], px, d), mp0)


def to_record(kfs, cells, entries):
    from ygz_slam_b200 import capi
    rec = capi.MapBuffers(capi.TRACK_RING, W, H, cells)
    r = rec.rec
    r.width, r.height, r.cells, r.n_levels, r.n_keyframes = W, H, cells, LEVELS, len(kfs)
    r.K[:] = list(K)
    f0 = o0 = 0
    for k, kf in enumerate(kfs):
        nf, no = len(kf["depth"]), len(kf["obs_id"])
        a = rec.a
        a["entry"][k], a["T_cw"][k], a["mp0"][k], a["n_features"][k], a["n_obs"][k] = entries[k], kf["T"].reshape(-1), kf["mp0"], nf, no
        a["image"][k] = kf["gray"]
        a["px"][f0:f0 + nf], a["level"][f0:f0 + nf], a["depth"][f0:f0 + nf], a["pw"][f0:f0 + nf] = kf["px"], kf["level"], kf["depth"], kf["pw"]
        a["obs_id"][o0:o0 + no], a["obs_px"][o0:o0 + no] = kf["obs_id"], kf["obs_px"]
        f0, o0 = f0 + nf, o0 + no
    return rec


def new_tracker(ctx3, n_streams=3, max_jobs=8):
    fr = ctx3.frames(KF_SLOT0 + 4 * n_streams)
    return fr, fr.tracker(n_streams, max_jobs, K)


def put_map(tr, stream, kfs):
    entries = np.arange(len(kfs), dtype=np.int32)
    tr.import_(stream, entries, KF_SLOT0 + 4 * stream + entries, to_record(kfs, tr.ctx.n_cells, entries))


def _pose_err(A, B):
    return float(np.linalg.norm(se3.se3_log(se3.mul(A, se3.inv(B)))))


# ---- stage checks ------------------------------------------------------------------------------------------------------
def check_job(oracle, dbg, res, kfs, local, cur, cells, stats):
    """Stages a-d of one tracking job: kfs are the imported key-frames, local the indices of the job's local key-frames
    (oldest first), cur the current frame."""
    ref = kfs[local[-1]]
    # a. sparse alignment against the reference key-frame, from the identity, then the key-frame's pose
    Trel, n_meas, _ = oracle.sparse_align(ref["pyr"], cur["pyr"], W, H, LEVELS, ref["px"], ref["depth"], np.ones(len(ref["depth"]), np.uint8),
                                          np.eye(4)[:3], np.eye(4)[:3])
    motion = float(np.linalg.norm(se3.se3_log(Trel)))
    assert dbg["n_meas"] == res["n_meas"] == n_meas
    assert dbg["n_local"] == len(local)
    T = dbg["T_aligned"]
    err = _pose_err(T, se3.mul(Trel, ref["T"]))
    stats["align"] = max(stats.get("align", 0.0), err)
    assert err < 1e-4
    assert dbg["aligned"] == res["aligned"] == int(np.linalg.norm(se3.se3_log(mat34_mul(T, mat34_inv(ref["T"])))) <= 0.2)
    assert abs(motion - 0.2) > 1e-3          # the scene is not at the rule's threshold
    for k, i in enumerate(local):
        assert np.array_equal(dbg["rel"][k], mat34_mul(T, mat34_inv(kfs[i]["T"]))), k
    if not dbg["aligned"]:
        assert motion > 0.2
        assert dbg["n_candidates"] == res["n_candidates"] == 0 and not dbg["cand_ok"].any()
        assert dbg["n_projected"] == res["n_projected"] == 0 and res["n_inliers"] == 0
        return
    # b. candidates (exact f64 restatement) and FindDirectProjection per candidate (relative to the key-frame: identity, rel[k])
    want_ok = np.zeros(4 * cells, bool)
    n_cand = 0
    for k, i in enumerate(local):
        kf = kfs[i]
        u, v, m = project(T, kf["pw"])
        sel = np.flatnonzero(m)
        n_cand += len(sel)
        if not len(sel):
            continue
        px, _, ok = oracle.find_direct_projection(kf["pyr"], cur["pyr"], W, H, LEVELS, np.eye(4)[:3], dbg["rel"][k], kf["px"][sel],
                                                  kf["depth"][sel], kf["level"][sel], np.stack([u[sel], v[sel]], 1))
        assert np.array_equal(dbg["cand_px"][k * cells + sel], px), k
        want_ok[k * cells + sel] = ok
    assert dbg["n_candidates"] == res["n_candidates"] == n_cand
    assert np.array_equal(dbg["cand_ok"], want_ok)
    # c. ordered compaction
    src = np.flatnonzero(want_ok)
    assert dbg["n_projected"] == res["n_projected"] == len(src)
    assert np.array_equal(dbg["c_src"], src)
    assert np.array_equal(dbg["c_px"], dbg["cand_px"][src])
    pw_all = np.zeros((4 * cells, 3))
    for k, i in enumerate(local):
        pw_all[k * cells:k * cells + len(kfs[i]["pw"])] = kfs[i]["pw"]
    assert np.array_equal(dbg["c_pw"], pw_all[src])
    # d. pose-only from the aligned pose on the compacted points
    Tp, inl, _, cnt = oracle.pose_only(dbg["c_pw"], dbg["c_px"], T)
    assert np.array_equal(dbg["inlier"], inl)
    assert dbg["n_inliers"] == res["n_inliers"] == cnt
    err = _pose_err(res["T_cw"], Tp)
    stats["pose_only"] = max(stats.get("pose_only", 0.0), err)
    assert err < 1e-4
    return dict(n_cand=n_cand, n_proj=len(src), n_inl=int(cnt))


def _stage_scene(oracle, frames, cells, special=None):
    """Stream map of the stage tests: an empty key-frame (frame 0), a detected one (frame 4) that carries the border
    points when `special` is given, and the reference key-frame (frame 8) with a feature in every cell."""
    empty = _kf(frames[0], frames[0]["T"], [], [], [], [], MP0[0])
    border = detected_kf(oracle, frames[4], MP0[1])
    if special is not None:
        T4 = frames[4]["T"]
        pc = (T4[:, :3] @ special.T).T + T4[:, 3]
        z = np.where(pc[:, 2] > 0.5, pc[:, 2], 2.0)
        spx = np.stack([np.clip(K[0] * pc[:, 0] / z + K[2], 12, W - 13), np.clip(K[1] * pc[:, 1] / z + K[3], 12, H - 13)], 1)
        n = min(len(border["depth"]), cells - len(special))
        border = _kf(frames[4], T4, np.r_[border["px"][:n], spx], np.r_[border["level"][:n], np.zeros(len(special), np.int32)],
                     np.r_[border["depth"][:n], z], np.r_[border["pw"][:n], special], MP0[1])
    return [empty, border, filled_kf(frames[8], cells, MP0[2])]


# jobs of the stage test: (cur slot, local key-frames); slot 0 = frame 10, 1 = frame 11, 2 = a frame the alignment cannot follow
STAGE_JOBS = ((0, [0, 1, 2]), (0, [1, 2]), (0, [2]), (1, [0, 1, 2]), (2, [0, 1, 2]))


@pytest.mark.gpu
def test_tracking_stages_match_the_oracle(ctx3, oracle, frames):
    """Stages a-d on one stream with n_local = 3, 2 and 1: local key-frames with 0 features and with all cells filled (the
    dense range spans 9 of the compaction's 1024-chunks), map points exactly on both sides of the four borders, behind the
    camera and at z = 0, and a job the alignment loses (aligned = 0).  Two passes: the border points are placed under the
    first pass's aligned pose, and the second pass must reproduce that pose bit for bit (the alignment reads only the
    reference key-frame)."""
    cells = ctx3.n_cells
    fr, tr = new_tracker(ctx3, n_streams=1)
    cur = [frames[10], frames[11], frames["far"]]
    tr.upload(0, np.stack([c["gray"] for c in cur]))
    jobs = [(0, slot, local) for slot, local in STAGE_JOBS]
    put_map(tr, 0, _stage_scene(oracle, frames, cells))
    tr.track(jobs)
    first = [tr.debug_job(j)["T_aligned"] for j in range(len(jobs))]
    special = border_points(first[0])
    u, v, m = project(first[0], special)
    assert list(u[:4]) + list(v[4:8]) == [t for _, t in border_targets()]
    assert list(m) == [True, False, False, True, True, False, False, True, False, False]
    kfs = _stage_scene(oracle, frames, cells, special)
    assert len(kfs[2]["depth"]) == cells and len(kfs[0]["depth"]) == 0
    put_map(tr, 0, kfs)
    res = tr.track(jobs)
    stats = {}
    for j, (slot, local) in enumerate(STAGE_JOBS):
        dbg = tr.debug_job(j)
        assert np.array_equal(dbg["T_aligned"], first[j]), j
        assert np.array_equal(dbg["T_aligned"], first[0]) == (slot == 0)
        got = check_job(oracle, dbg, res[j], kfs, local, cur[slot], cells, stats)
        assert (got is None) == (slot == 2), j
        if got:
            assert got["n_proj"] > 1500 and got["n_inl"] > 1000, (j, got)
            print(f"job {j}: n_local {len(local)}, {got['n_cand']} candidates, {got['n_proj']} projected, {got['n_inl']} inliers")
        if slot == 0 and 1 in local:   # the border points of key-frame 1 took part exactly as predicted
            k = local.index(1)
            base = k * cells + len(kfs[1]["depth"]) - len(special)
            assert dbg["n_candidates"] == int(sum(project(dbg["T_aligned"], kfs[i]["pw"])[2].sum() for i in local))
            assert np.array_equal(np.isin(np.arange(base, base + len(special)), dbg["c_src"]) | ~m, ~m | dbg["cand_ok"][base:base + len(special)])
    print(f"largest pose differences to the oracle: sparse alignment {stats['align']:.2e}, pose-only {stats['pose_only']:.2e}")
    tr.close()
    fr.close()


def _debug_same(a, b):
    for k in ("T_aligned", "rel", "n_local", "n_meas", "aligned", "n_candidates", "n_projected", "n_inliers", "cand_ok", "c_src", "c_px",
              "c_pw", "inlier"):
        assert np.array_equal(a[k], b[k]), k
    assert np.array_equal(a["cand_px"][a["cand_ok"]], b["cand_px"][b["cand_ok"]])


def _result_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.gpu
def test_a_job_does_not_depend_on_its_batch(ctx3, oracle, frames):
    """Stage g: one batch with jobs of 3 streams, two of them on stream 1 against the same reference key-frame (a window),
    in this order, in the reverse order and one job per batch: every job's debug view and result are bit-identical."""
    cells = ctx3.n_cells
    fr, tr = new_tracker(ctx3, n_streams=3)
    maps = [_stage_scene(oracle, frames, cells),
            [detected_kf(oracle, frames[k], MP0[i]) for i, k in enumerate(KF_FRAMES)],
            [detected_kf(oracle, frames[k], MP0[i]) for i, k in enumerate(KF_FRAMES[1:])]]
    for s, kfs in enumerate(maps):
        put_map(tr, s, kfs)
    cur = [frames[10], frames[10], frames[11], frames[12]]
    tr.upload(0, np.stack([c["gray"] for c in cur]))
    jobs = [(0, 0, [0, 1, 2]), (1, 1, [0, 1, 2]), (1, 2, [1, 2]), (2, 3, [0, 1])]
    res = tr.track(jobs)
    views = [tr.debug_job(j) for j in range(len(jobs))]
    stats = {}
    for j, (s, slot, local) in enumerate(jobs):
        assert check_job(oracle, views[j], res[j], maps[s], local, cur[slot], cells, stats) is not None, j
    rres = tr.track(jobs[::-1])
    for j in range(len(jobs)):
        _debug_same(tr.debug_job(len(jobs) - 1 - j), views[j])
        _result_same(rres[len(jobs) - 1 - j], res[j])
    for j in range(len(jobs)):
        one = tr.track([jobs[j]])
        _debug_same(tr.debug_job(0), views[j])
        _result_same(one[0], res[j])
    tr.close()
    fr.close()


def ba_scene(oracle, frames, seed=9):
    """Map of the key-frame tests: key-frames of frames 0, 4 and 8 as SetKeyframe makes them.  Key-frame 4 has no
    observations; key-frame 8 observes every other point of key-frames 0 and 4 that it sees (projection + 0.7 px of noise)
    and 5 points of a key-frame that has left the ring (ids no entry owns)."""
    rng = np.random.default_rng(seed)
    kfs = [detected_kf(oracle, frames[k], MP0[i]) for i, k in enumerate(KF_FRAMES)]
    ids, pxs = [], []
    for kf in kfs[:2]:
        u, v, m = project(kfs[2]["T"], kf["pw"])
        sel = np.flatnonzero(m)[::2]
        ids.append(kf["mp0"] + sel)
        pxs.append(np.stack([u[sel], v[sel]], 1) + rng.normal(0, 0.7, (len(sel), 2)))
    ids.append(np.arange(90000, 90005))
    pxs.append(rng.uniform(50, 400, (5, 2)))
    kfs[2] = dict(kfs[2], obs_id=np.concatenate(ids), obs_px=np.concatenate(pxs))
    return kfs


def host_ba(oracle, kfs, local, **ba):
    """LocalMapping::LocalBA by the rule of vo.VisualOdometry._local_ba on exported key-frames `kfs` (by ring entry):
    the points at least two of the local key-frames observe (a key-frame observes its own points and the older points
    tracked into it), the oldest local key-frame fixed.  Returns the problem (`problem`: the arguments of local_ba), its
    points' (entry, feature) and the oracle's (poses as T_cw, points, stats); `ba`: oracle.local_ba's solver parameters."""
    lo = np.array([kfs[e]["mp0"] for e in local])
    hi = lo + np.array([len(kfs[e]["depth"]) for e in local])
    o_kf, o_id, o_px = [], [], []
    for k, e in enumerate(local):
        kf = kfs[e]
        o_kf.append(np.full(len(kf["depth"]), k)); o_id.append(kf["mp0"] + np.arange(len(kf["depth"]))); o_px.append(kf["px"])
        inside = ((kf["obs_id"][:, None] >= lo) & (kf["obs_id"][:, None] < hi)).any(1)
        o_kf.append(np.full(int(inside.sum()), k)); o_id.append(kf["obs_id"][inside]); o_px.append(kf["obs_px"][inside])
    o_kf, o_id, o_px = np.concatenate(o_kf).astype(np.int32), np.concatenate(o_id), np.concatenate(o_px)
    _, inv, counts = np.unique(o_id, return_inverse=True, return_counts=True)
    multi = counts[inv] >= 2
    ids, pt_idx = np.unique(o_id[multi], return_inverse=True)
    owner = np.array([int(np.flatnonzero((lo <= i) & (i < hi))[0]) for i in ids], np.int64)
    feat = ids - lo[owner]
    pts = np.array([kfs[local[k]]["pw"][f] for k, f in zip(owner, feat)]).reshape(-1, 3)
    log = np.array([se3.se3_log(kfs[e]["T_cw"]) for e in local])
    fixed = np.zeros(len(local), np.uint8)
    fixed[0] = 1
    problem = (np.concatenate([log[:, 3:], log[:, :3]], 1), fixed, pts, o_kf[multi], pt_idx.astype(np.int32), o_px[multi])
    P, X, _, st = oracle.local_ba(*problem, **ba)
    T = [se3.se3_exp(np.concatenate([p[3:], p[:3]])) for p in P]
    return dict(n_pts=len(ids), n_obs=int(multi.sum()), owner=owner, feat=feat, T=T, X=X, stats=st, problem=problem)


def _same_entry(a, b, skip=()):
    for k in ("T_cw", "mp0", "px", "level", "depth", "pw", "obs_id", "obs_px", "image"):
        if k not in skip:
            assert np.array_equal(a[k], b[k]), k


@pytest.mark.gpu
def test_keyframe_insertion_and_local_ba_match_the_oracle(ctx3, oracle, frames):
    """Stages e and f.  Three streams hold the same imported map and track frame 10 in one batch (identical results).
    Each then inserts frame 10 as a key-frame into ring entry 3: stream 0 without a BA (the state the BA starts from),
    stream 1 with a BA over 3 local key-frames (4, 8 and the new one: key-frame 0 has left the window, key-frame 4 has no
    observations), stream 2 over 2 (8 and the new one: one free pose).  The depth image is random per pixel, not a plane."""
    cells = ctx3.n_cells
    fr, tr = new_tracker(ctx3, n_streams=3)
    kfs = ba_scene(oracle, frames)
    for s in range(3):
        put_map(tr, s, kfs)
    tr.upload(0, np.stack([frames[10]["gray"]] * 3))
    res = tr.track([(s, s, [0, 1, 2]) for s in range(3)])
    dbg = tr.debug_job(0)
    for s in (1, 2):
        _result_same(res[s], res[0])
    assert check_job(oracle, dbg, res[0], kfs, [0, 1, 2], frames[10], cells, {}) is not None
    depth = np.random.default_rng(17).uniform(1.5, 3.0, (H, W))
    for s in range(3):
        tr.set_depth(s, depth)
    locals_ = ([1, 2, 3], [1, 2, 3], [2, 3])
    kres = tr.make_keyframes([dict(stream=s, frame_slot=s, kf_slot=KF_SLOT0 + 4 * s + 3, entry=3, track_job=s, local_entry=locals_[s],
                                   run_ba=int(s > 0), mp0=MP0_NEW) for s in range(3)])
    maps = [tr.export(s, [0, 1, 2, 3]).keyframes() for s in range(3)]
    pre = maps[0]
    # e. the new key-frame (stream 0: no BA after it)
    f = oracle.detect(frames[10]["pyr"], n_levels=LEVELS)
    new = pre[3]
    px = np.stack([f["px"], f["py"]], 1)
    assert kres[0]["n_features"] == f["n"] == len(new["depth"])
    assert np.array_equal(new["px"], px) and np.array_equal(new["level"], f["level"])
    assert np.array_equal(new["depth"], depth[px[:, 1].astype(int), px[:, 0].astype(int)])
    assert np.array_equal(new["T_cw"], res[0]["T_cw"]) and new["mp0"] == MP0_NEW
    assert np.array_equal(new["pw"], backproject(res[0]["T_cw"], px, new["depth"]))
    src = dbg["c_src"][dbg["inlier"]]
    mp0 = np.array([kfs[k]["mp0"] for k in (0, 1, 2)])
    assert np.array_equal(new["obs_id"], mp0[src // cells] + src % cells)
    assert np.array_equal(new["obs_px"], dbg["c_px"][dbg["inlier"]])
    assert len(new["obs_id"]) == res[0]["n_inliers"] > 1000
    assert np.array_equal(new["image"], frames[10]["gray"])
    for e in range(3):
        _same_entry(pre[e], dict(kfs[e], T_cw=kfs[e]["T"], image=kfs[e]["gray"]))
    # f. local BA: assembly, initial chi2, result, and nothing outside the BA touched
    for s in (1, 2):
        local, got, r = locals_[s], maps[s], kres[s]
        _same_entry(got[3], pre[3], skip=("T_cw", "pw"))
        want = host_ba(oracle, pre, local)
        assert (r["ba_points"], r["ba_observations"]) == (want["n_pts"], want["n_obs"]), s
        assert r["ba_points"] > 500 and not (want["owner"] == len(local) - 1).any()   # the new key-frame's own points: one view
        rel = abs(r["chi2_initial"] - want["stats"]["chi2_initial"]) / want["stats"]["chi2_initial"]
        assert rel < 1e-10, (s, rel)
        dT = max(_pose_err(got[e]["T_cw"], T) for e, T in zip(local, want["T"]))
        in_ba = {e: np.zeros(len(got[e]["depth"]), bool) for e in local}
        dX = 0.0
        for k, g, x in zip(want["owner"], want["feat"], want["X"]):
            in_ba[local[k]][g] = True
            dX = max(dX, float(np.abs(got[local[k]]["pw"][g] - x).max()))
        print(f"stream {s}: {r['ba_points']} points, {r['ba_observations']} observations, initial chi2 relative difference {rel:.1e}, "
              f"largest pose difference {dT:.1e}, point difference {dX:.1e} m")
        assert dT < 1e-4 and dX < 1e-4, s
        for e in local:
            assert np.array_equal(got[e]["pw"][~in_ba[e]], pre[e]["pw"][~in_ba[e]]), (s, e)
            _same_entry(got[e], pre[e], skip=("T_cw", "pw"))
            assert np.array_equal(r["T_cw"][local.index(e)], got[e]["T_cw"])
        for e in set(range(4)) - set(local):
            _same_entry(got[e], pre[e])
    tr.close()
    fr.close()


TRACKER_BA_TOL = 1e-13  # T_cw entries and landmark coordinates (absolute), chi2_final (relative): ~100x the measured 8.9e-16


@pytest.mark.gpu
@pytest.mark.parametrize("max_iters,max_trials", [(1, 10), (3, 10), (3, 1)])
def test_truncated_tracker_ba_matches_local_ba(ctx3, oracle, frames, max_iters, max_trials):
    """Stage f with non-default ygzb_ba_params: the tracker's local BA, which hands the solver its own landmark-major lists,
    stops where ygzb_local_ba stops on the problem the host assembles (the same iterations and LM trials as the oracle)
    and leaves the same key-frame poses and points.  Stream 1 runs the 3-key-frame window (two free poses), stream 2
    the 2-key-frame one (one free pose).  Largest differences measured on an H100 80GB HBM3 (700 W): T_cw entries 4.0e-16,
    landmark coordinates 8.9e-16 m."""
    from ygz_slam_b200 import capi
    fr, tr = new_tracker(ctx3, n_streams=3)
    kfs = ba_scene(oracle, frames)
    for s in range(3):
        put_map(tr, s, kfs)
    tr.upload(0, np.stack([frames[10]["gray"]] * 3))
    tr.track([(s, s, [0, 1, 2]) for s in range(3)])
    depth = np.random.default_rng(17).uniform(1.5, 3.0, (H, W))
    for s in range(3):
        tr.set_depth(s, depth)
    prm = capi.BAParams()
    ctx3.lib.ygzb_default_ba_params(C.byref(prm))
    prm.max_iters, prm.max_trials = max_iters, max_trials
    locals_ = ([1, 2, 3], [1, 2, 3], [2, 3])
    kres = tr.make_keyframes([dict(stream=s, frame_slot=s, kf_slot=KF_SLOT0 + 4 * s + 3, entry=3, track_job=s, local_entry=locals_[s],
                                   run_ba=int(s > 0), mp0=MP0_NEW) for s in range(3)], ba=prm)
    maps = [tr.export(s, [0, 1, 2, 3]).keyframes() for s in range(3)]
    for s in (1, 2):
        local, got, r = locals_[s], maps[s], kres[s]
        want = host_ba(oracle, maps[0], local, max_iters=max_iters, max_trials=max_trials)
        n_kf, n_pt, n_obs = len(local), want["n_pts"], want["n_obs"]
        P, X, _, st = ctx3.local_ba([0, n_kf], [0, n_pt], [0, n_obs], *want["problem"], max_iters=max_iters, max_trials=max_trials)
        st = st[0]
        assert (r["ba_points"], r["ba_observations"]) == (n_pt, n_obs), s
        assert (r["ba_iters"], r["ba_trials"]) == (st["iters"], st["lm_trials"]) == (want["stats"]["iters"], want["stats"]["lm_trials"]), s
        assert st["iters"] == (1 if max_trials == 1 else max_iters), s
        dT = max(float(np.abs(got[e]["T_cw"] - se3.se3_exp(np.concatenate([p[3:], p[:3]]))).max()) for e, p in zip(local, P))
        dX = max(float(np.abs(got[local[k]]["pw"][g] - x).max()) for k, g, x in zip(want["owner"], want["feat"], X))
        print(f"stream {s}: {st['iters']} iterations, {st['lm_trials']} trials, pose difference {dT:.1e}, point difference {dX:.1e}")
        assert dT <= TRACKER_BA_TOL and dX <= TRACKER_BA_TOL, (s, dT, dX)
        assert abs(r["chi2_final"] - st["chi2_final"]) <= TRACKER_BA_TOL * st["chi2_final"], s
    tr.close()
    fr.close()

