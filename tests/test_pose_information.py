"""Pose information: how well each tracked frame's pose is determined (ygzb_pose_information, ygzb_sparse_align_fisher,
ygzb_tracker_set_information, ygz_vo_set_information / ygz_vo_poll_ex, vo_native.Engine(information=True)).

align_fisher is SparseImgAlign::getFisherInformation() (SparseImageAlign.cpp:52-57): H_ of the alignment's last
linearisation at min_level over 5e-4 * 255^2.  pose_info is sum J^T J over the frame's observation rows at its returned
pose, J = d pi(exp(delta) T_cw P_w) / d delta at 0.  The reference H_ comes from a numpy restatement of SparseImgAlign::run
(np_sparse_align), itself held to oracle/align.cpp's iterations and poses without a GPU, together with the pose_info
formula against finite differences, the record layout and the argument checks.  On the GPU: the kernel's H_ against the
restatement's on every exit of the Gauss-Newton loop, the tracker's records against the restatement and numpy, and the
engine's records across windows, pacings, restarts and stream records."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from ygz_slam_b200 import se3, synth

ROOT = Path(__file__).resolve().parent.parent
SIGMA_I_SQ = 5e-4 * 255 * 255
ERR_INVALID = -1
# Fisher information against the numpy restatement: relative to the matrix's largest diagonal entry (the sums run in another order);
# measured on an H100 80GB HBM3 (700 W): 9.3e-15 for ygzb_sparse_align_fisher, 8.1e-15 for the tracker
FISHER_TOL = 1e-9


def _full(packed):
    F = np.zeros((6, 6))
    r, c = np.triu_indices(6)
    F[r, c] = packed
    F[c, r] = packed
    return F


def _rel(a, b):
    scale = max(float(np.abs(np.diag(b)).max()), 1e-300)
    return float(np.abs(a - b).max()) / scale


def pose_info(T, pw, fx, fy):
    """sum_i J_i^T J_i, J_i = d pi(exp(delta) T P_w,i) / d delta at delta = 0, delta = [upsilon; omega] (left)."""
    pw = np.asarray(pw, np.float64).reshape(-1, 3)
    pc = pw @ np.asarray(T)[:, :3].T + np.asarray(T)[:, 3]
    x, y, z = pc.T
    zi = 1.0 / z
    u, v = x * zi, y * zi
    o = np.zeros_like(z)
    Ju = np.stack([fx * zi, o, -fx * u * zi, -fx * u * v, fx * (1 + u * u), -fx * v], 1)
    Jv = np.stack([o, fy * zi, -fy * v * zi, -fy * (1 + v * v), fy * u * v, fy * u], 1)
    return Ju.T @ Ju + Jv.T @ Jv


# ---- without a GPU -----------------------------------------------------------------------------------------------------
def test_information_record_layout_matches_the_header(tmp_path):
    """ygzb_pose_information is 336 bytes, laid out as capi.INFO_DTYPE, in plain C99."""
    from ygz_slam_b200 import capi
    src = tmp_path / "info.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "ygz_vo.h"\nint main(void) {\n'
                   '    printf("%d %d %d\\n", (int)sizeof(ygzb_pose_information), (int)offsetof(ygzb_pose_information, align_fisher),\n'
                   '           (int)offsetof(ygzb_pose_information, pose_info));\n    return 0;\n}\n')
    exe = tmp_path / "info"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", f"-I{ROOT / 'include'}", str(src), "-o", str(exe)], check=True,
                   capture_output=True, text=True)
    got = list(map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()))
    dt = capi.INFO_DTYPE
    assert got == [336, dt.fields["align_fisher"][1], dt.fields["pose_info"][1]] == [336, 0, 168]
    assert dt.itemsize == 336
    packed = np.arange(21.0)
    F = capi.unpack_sym6(packed)
    assert np.array_equal(F, F.T) and list(F[0]) == [0, 1, 2, 3, 4, 5] and list(F[1, 1:]) == [6, 7, 8, 9, 10] and F[5, 5] == 20


def test_null_handles_are_rejected_without_a_device():
    from ygz_slam_b200 import build, capi, vo_native
    build.build()
    lib = capi.load_library()
    lib.ygzb_tracker_set_information.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    assert lib.ygzb_tracker_set_information(None, None, 0) == ERR_INVALID
    lib.ygzb_sparse_align_fisher.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 8 + [C.c_int] * 3 + [C.c_double] + [C.c_void_p] * 3
    assert lib.ygzb_sparse_align_fisher(None, 1, *([None] * 8), 2, 0, 30, 1e-6, None, None, None) == ERR_INVALID
    vl = vo_native._lib()
    n = C.c_int(7)
    assert vl.ygz_vo_set_information(None, 1) == ERR_INVALID
    assert vl.ygz_vo_poll_ex(None, None, 0, C.byref(n), None, None, 0, None) == ERR_INVALID


def test_pose_information_formula_against_finite_differences():
    """The analytic J of pose_info against central differences of the pixel residual through se3.se3_exp (left
    perturbation), on points in front of a generic pose: 1e-6 relative."""
    rng = np.random.default_rng(3)
    T = se3.se3_exp(np.array([0.1, -0.2, 0.05, 0.2, -0.1, 0.3]))
    pc = np.stack([rng.uniform(-1, 1, 40), rng.uniform(-1, 1, 40), rng.uniform(1.5, 4, 40)], 1)
    pw = (pc - T[:, 3]) @ T[:, :3]   # T^-1 pc
    fx, fy, cx, cy = (float(np.float32(v)) for v in (synth.FX, synth.FY, synth.CX, synth.CY))

    def proj(Tm):
        q = pw @ Tm[:, :3].T + Tm[:, 3]
        return np.stack([fx * q[:, 0] / q[:, 2] + cx, fy * q[:, 1] / q[:, 2] + cy], 1)
    h = 1e-6
    J = np.zeros((len(pw), 2, 6))
    for k in range(6):
        d = np.zeros(6)
        d[k] = h
        J[:, :, k] = (proj(se3.mul(se3.se3_exp(d), T)) - proj(se3.mul(se3.se3_exp(-d), T))) / (2 * h)
    want = np.einsum("nik,nil->kl", J, J)
    got = pose_info(T, pw, fx, fy)
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max(), np.abs(got - want).max() / np.abs(want).max()


def _ldlt6(H, b):
    """SparseImgAlign's LDL^T solve (Eigen ldlt in NLLSSolver::solve): None when a pivot is not > 0 in magnitude."""
    L, D = np.eye(6), np.zeros(6)
    for j in range(6):
        d = H[j, j] - sum(L[j, k] * L[j, k] * D[k] for k in range(j))
        D[j] = d
        if not abs(d) > 0:
            return None
        for i in range(j + 1, 6):
            L[i, j] = (H[i, j] - sum(L[i, k] * L[j, k] * D[k] for k in range(j))) / d
    y = np.zeros(6)
    for i in range(6):
        y[i] = b[i] - sum(L[i, k] * y[k] for k in range(i))
    y /= D
    x = np.zeros(6)
    for i in range(5, -1, -1):
        x[i] = y[i] - sum(L[k, i] * x[k] for k in range(i + 1, 6))
    return x


def _bilinear(img, r, c, w):
    """w[0] I(r, c) + w[1] I(r, c + 1) + w[2] I(r + 1, c) + w[3] I(r + 1, c + 1) in float, summed left to right (indices
    clipped: rows of features outside the level are masked by the caller)."""
    h, wd = img.shape

    def at(rr, cc):
        return img[np.clip(rr, 0, h - 1), np.clip(cc, 0, wd - 1)]
    return w[0] * at(r, c) + w[1] * at(r, c + 1) + w[2] * at(r + 1, c) + w[3] * at(r + 1, c + 1)


def _weights(su, sv):
    su64, sv64 = su.astype(np.float64), sv.astype(np.float64)
    return [((1.0 - su64) * (1.0 - sv64)).astype(np.float32), (su64 * (1.0 - sv64)).astype(np.float32),
            ((1.0 - su64) * sv64).astype(np.float32), su * sv]


def np_sparse_align(o, s, max_level=2, min_level=0, n_iter=30, eps=1e-6, n_levels=3):
    """numpy restatement of SparseImgAlign::run (SparseImageAlign.cpp:21-223 with NLLSSolver::optimizeGaussNewton,
    NLSSolver_impl.hpp:18-110; use_weights_ false), written from the reference text: chi2 summed in double and rounded
    to float once, as the kernel does.  Returns (T_cw_cur, iterations per level, H_ of the last linearisation at
    min_level -- zeros when there was none)."""
    from oracle.pyoracle import default_camera
    cam = default_camera()
    fx, fy, cx, cy = (np.float32(v) for v in (cam.fx, cam.fy, cam.cx, cam.cy))
    focal = float(np.float32((fx + fy) / np.float32(2)))
    px, depth, has = np.asarray(s["px"], np.float64), np.asarray(s["depth"], np.float64), np.asarray(s["has"]).astype(bool)
    iters = np.zeros(8, np.int32)
    H_last = np.zeros((6, 6))
    T_ref = np.asarray(s["T_ref"], np.float64).reshape(3, 4)
    n = len(depth)
    if n == 0:
        return T_ref.copy(), iters, H_last
    with np.errstate(all="ignore"):
        X, Y, Z = (px[:, 0] - float(cx)) * depth / float(fx), (px[:, 1] - float(cy)) * depth / float(fy), depth
        zi = 1.0 / Z
        J0 = np.stack([-zi, 0 * zi, X * zi * zi, Y * (X * zi * zi), -(1.0 + X * (X * zi * zi)), Y * zi], 1)   # JacobXYZ2Cam
        J1 = np.stack([0 * zi, -zi, Y * zi * zi, 1.0 + Y * (Y * zi * zi), -(Y * (X * zi * zi)), -X * zi], 1)
        xyz = np.stack([X, Y, Z], 1)
        visible = np.zeros(n, bool)          # never reset across levels (the reference's TODO)
        cache = np.zeros((n, 16), np.float32)
        dy4, dx4 = np.divmod(np.arange(16), 4)
        T = se3.mul(np.asarray(s["T_ref"], np.float64).reshape(3, 4), se3.inv(T_ref))   # T_cur_from_ref (cur starts at ref)
        chi2_ = 1e10
        for L in range(max_level, min_level - 1, -1):
            rim = o.level_view(s["p1"], synth.W, synth.H, n_levels, L).astype(np.float32)
            cim = o.level_view(s["p2"], synth.W, synth.H, n_levels, L).astype(np.float32)
            scale = np.float32(1.0) / np.float32(1 << L)
            # precomputeReferencePatches
            u_ref, v_ref = (px[:, 0] * float(scale)).astype(np.float32), (px[:, 1] * float(scale)).astype(np.float32)
            ui, vi = np.floor(u_ref).astype(int), np.floor(v_ref).astype(int)
            ok = has & (ui - 3 >= 0) & (vi - 3 >= 0) & (ui + 3 < rim.shape[1]) & (vi + 3 < rim.shape[0])
            visible |= ok
            w = [x[:, None] for x in _weights(u_ref - ui.astype(np.float32), v_ref - vi.astype(np.float32))]
            r, c = vi[:, None] + dy4 - 2, ui[:, None] + dx4 - 2
            cache = np.where(ok[:, None], _bilinear(rim, r, c, w), cache)
            gx = np.float32(0.5) * (_bilinear(rim, r, c + 1, w) - _bilinear(rim, r, c - 1, w))
            gy = np.float32(0.5) * (_bilinear(rim, r + 1, c, w) - _bilinear(rim, r - 1, c, w))
            jac = (gx.astype(np.float64)[:, :, None] * J0[:, None, :] + gy.astype(np.float64)[:, :, None] * J1[:, None, :]) * (focal / (1 << L))
            jac[~ok] = 0.0

            def linearise(T):
                pc = xyz @ T[:, :3].T + T[:, 3]
                pu, pv = float(fx) * pc[:, 0] / pc[:, 2] + float(cx), float(fy) * pc[:, 1] / pc[:, 2] + float(cy)
                uc, vc = pu.astype(np.float32) * scale, pv.astype(np.float32) * scale
                uci, vci = np.floor(uc).astype(int), np.floor(vc).astype(int)
                inside = visible & (uci >= 0) & (vci >= 0) & (uci - 3 >= 0) & (vci - 3 >= 0) & (uci + 3 < cim.shape[1]) & (vci + 3 < cim.shape[0])
                wc = [x[:, None] for x in _weights(uc - uci.astype(np.float32), vc - vci.astype(np.float32))]
                res = (_bilinear(cim, vci[:, None] + dy4 - 2, uci[:, None] + dx4 - 2, wc) - cache)[inside]
                Jm = jac[inside]
                H = np.einsum("fpa,fpb->ab", Jm, Jm)
                b = -np.einsum("fpa,fp->a", Jm, res.astype(np.float64))
                n_meas = 16 * int(inside.sum())
                chi2 = float(np.float32(np.sum((res * res).astype(np.float64))) / np.float32(n_meas))
                return H, b, chi2

            old = T
            it = 0
            while it < n_iter:
                H, b, new_chi2 = linearise(T)
                if L == min_level:
                    H_last = H
                x = _ldlt6(H, b)
                stop = x is None or np.isnan(x[0])
                if (it > 0 and new_chi2 > chi2_) or stop:
                    T = old
                    break
                old, T = T, se3.mul(T, se3.se3_exp(-x))
                chi2_ = new_chi2
                if np.abs(x).max() <= eps:
                    break
                it += 1
            iters[L] = it
    return se3.mul(T, T_ref), iters, H_last


def _ora_align(s, **kw):
    from test_gpu_tracking_solvers import _ora_align as ora
    return ora(s, **kw)


@pytest.mark.parametrize("case", ["steps", "runs", "exits"])
def test_numpy_restatement_follows_the_oracle(case):
    """The numpy restatement whose last H_ the GPU tests hold the kernel to, against oracle/align.cpp's SparseImgAlign in
    its exact chi2 mode: iterations per level exactly, the pose within 1e-12 in |log(T^-1 T_oracle)|, on the exits the
    GPU tests use -- single levels after 1 to 3 steps at eps = 0, whole runs at eps 1e-2, 1e-6 and 0 (eps exits and
    rollbacks at it > 0), identical frames (eps exit at it = 0), a flat texture (LDL^T failure), a depth-0 feature (NaN),
    n_iter = 0 and no feature (zero H)."""
    from test_gpu_tracking_solvers import _align
    o = _oracle_()

    def same(kw, s):
        T, it, H = np_sparse_align(o, s, **kw)
        wT, _, wit = _ora_align(s, **kw)
        assert np.array_equal(it[:3], wit[:3]), (kw, it, wit)
        assert float(np.linalg.norm(se3.se3_log(se3.mul(se3.inv(T), wT)))) < 1e-12, kw
        return H
    if case == "steps":
        s = _align("stream")
        for L in (0, 1, 2):
            for k in (1, 2, 3):   # (inverse compositional: H changes with the pose only through the features inside the level)
                assert same(dict(min_level=L, max_level=L, n_iter=k, eps=0.0), s)[0, 0] > 0
    elif case == "runs":
        for eps in (1e-2, 1e-6, 0.0):
            for name in ("stream", "stream2"):
                H = same(dict(eps=eps), _align(name))
                assert H[0, 0] > 0 and np.array_equal(H, H.T)
    else:
        for name in ("identical", "flat", "depth0"):
            H = same(dict(eps=0.0), _align(name))
            assert {"identical": H[0, 0] > 0, "flat": not H.any(), "depth0": np.isnan(H).any()}[name], name
        assert not same(dict(n_iter=0), _align("stream")).any()
        s = _align("stream")
        assert not np_sparse_align(o, dict(s, px=s["px"][:0], depth=s["depth"][:0], has=s["has"][:0]))[2].any()


def _oracle_():
    from test_gpu_tracking_solvers import _oracle
    return _oracle()


# ---- GPU: ygzb_sparse_align_fisher -------------------------------------------------------------------------------------
def _gpu_fisher(ctx, probs, **kw):
    from test_gpu_tracking_solvers import _gpu_align
    kw = dict(dict(max_level=2, min_level=0, n_iter=30, eps=1e-6), **kw)
    fr = ctx.frames(2 * len(probs))
    try:
        fr.upload(np.stack([g for s, _ in probs for g in (s["g1"], s["g2"])]))
        sel = [np.arange(len(s["depth"]))[f] for s, f in probs]
        off = np.cumsum([0] + [len(i) for i in sel])
        T, nm, it, F = fr.sparse_align(2 * np.arange(len(probs)), 2 * np.arange(len(probs)) + 1, off,
                                       np.concatenate([s["px"][i] for (s, _), i in zip(probs, sel)]),
                                       np.concatenate([s["depth"][i] for (s, _), i in zip(probs, sel)]),
                                       np.concatenate([s["has"][i] for (s, _), i in zip(probs, sel)]),
                                       np.stack([s["T_ref"].reshape(-1) for s, _ in probs]), np.stack([s["T_ref"].reshape(-1) for s, _ in probs]),
                                       fisher=True, **kw)
    finally:
        fr.close()
    plain = _gpu_align(ctx, probs, **kw)
    for p in range(len(probs)):   # the plain entry point's poses, measurement counts and iterations, bit for bit
        assert np.array_equal(T[p], plain[p][0]) and nm[p] == plain[p][1] and np.array_equal(it[p], plain[p][2]), p
    return F


def _ora_fisher(s, **kw):
    """The restatement's H_ of the last linearisation at min_level, scaled as getFisherInformation scales it."""
    return np_sparse_align(_oracle_(), s, **kw)[2] / SIGMA_I_SQ


WORST = {}


def _check_fisher(F, want, tag):
    if not want.any():
        assert not F.any(), tag
        return
    nan = np.isnan(want)   # a feature of depth 0 puts NaN into H on both sides (the LDL^T then rolls back at it = 0)
    assert np.array_equal(np.isnan(F), nan), tag
    if nan.all():
        return
    F, want = np.where(nan, 0.0, F), np.where(nan, 0.0, want)
    d = _rel(F, want)
    WORST[tag] = max(WORST.get(tag, 0.0), d)
    assert d <= FISHER_TOL, (tag, d)


@pytest.mark.gpu
@pytest.mark.parametrize("cluster", [1, 2, 4, 8])
def test_align_fisher_matches_the_restatement(ctx3, cluster, monkeypatch):
    """At 1, 2, 4 and 8 CTAs per problem: single levels after 1-3 steps, whole runs at eps 1e-2 / 1e-6 / 0 (eps exits
    and rollbacks at it > 0), identical frames (eps exit at it = 0), a flat texture (LDL^T failure at it = 0), a depth-0
    feature (NaN: rollback at it = 0), n_iter = 0 (zeros), a problem without features (zeros) and the 700-feature problem
    on the global staging path; poses, n_meas and iterations bit-identical to ygzb_sparse_align."""
    from test_gpu_tracking_solvers import _align, _sub
    monkeypatch.setenv("YGZB_TRACK_CLUSTER", str(cluster))
    s, s2 = _align("stream"), _align("stream2")
    for L in (0, 1, 2):
        for k in (1, 2, 3):
            kw = dict(min_level=L, max_level=L, n_iter=k, eps=0.0)
            for name, F in zip(("stream", "stream2"), _gpu_fisher(ctx3, [(s, slice(None)), (s2, slice(None))], **kw)):
                _check_fisher(F, _ora_fisher(_align(name), **kw), "steps")
    for eps in (1e-2, 1e-6, 0.0):
        for name, F in zip(("stream", "stream2"), _gpu_fisher(ctx3, [(s, slice(None)), (s2, slice(None))], eps=eps)):
            _check_fisher(F, _ora_fisher(_align(name), eps=eps), "runs")
    names = ["identical", "flat", "depth0", "stream"]
    probs = [(_align(n), slice(None)) for n in names]
    for name, F in zip(names, _gpu_fisher(ctx3, probs, eps=0.0)):
        _check_fisher(F, _ora_fisher(_align(name), eps=0.0), "exits")
    assert not _gpu_fisher(ctx3, probs, n_iter=0).any()
    F = _gpu_fisher(ctx3, [(s, slice(0, 0)), (s, slice(0, 700)), (s, slice(None))])
    assert not F[0].any()
    _check_fisher(F[1], _ora_fisher(_sub(s, slice(0, 700))), "staging")
    _check_fisher(F[2], _ora_fisher(s), "runs")
    print("largest Fisher difference to the restatement, relative to the largest diagonal entry:",
          ", ".join(f"{k} {v:.1e}" for k, v in sorted(WORST.items())))


# ---- GPU: tracker ------------------------------------------------------------------------------------------------------
from test_tracker_stages import frames  # noqa: E402,F401  (module fixture: rendered frames and their pyramids)


def _set_info(tr, buf, capacity=None):
    return tr.set_information(buf, capacity)


def _info_buffer(n):
    from ygz_slam_b200 import capi
    buf = capi.pinned_empty(n, capi.INFO_DTYPE)
    buf["align_fisher"] = np.nan
    buf["pose_info"] = np.nan
    return buf


@pytest.mark.gpu
def test_tracker_information_matches_restatement_and_rows(ctx3, oracle, frames):
    """Key-frame mode on the stage scene (n_local 3, 2 and 1, and a job the 0.2 rule rejects): align_fisher is the restatement's
    alignment Fisher; pose_info is numpy's sum J^T J over the job's observation rows at its result pose, zero for the
    rejected job; records are bit-identical in one batch, the reversed batch and alone; results, rows and debug views
    are bit-identical with the records on and off; bad buffers are rejected and NULL stops the writes."""
    from test_tracker_stages import LEVELS, STAGE_JOBS, _stage_scene, new_tracker, put_map
    from test_vo_observations import _obs_buffer, _same_debug, _set_obs
    cells = ctx3.n_cells
    fx, fy = float(ctx3.params.fx), float(ctx3.params.fy)
    fr, tr = new_tracker(ctx3, n_streams=1)
    cur = [frames[10], frames[11], frames["far"]]
    tr.upload(0, np.stack([c["gray"] for c in cur]))
    kfs = _stage_scene(oracle, frames, cells)
    put_map(tr, 0, kfs)
    jobs = [(0, slot, local) for slot, local in STAGE_JOBS]
    plain = tr.track(jobs)
    plain_dbg = [tr.debug_job(j) for j in range(len(jobs))]
    stride = 4 * cells
    obs = _obs_buffer(8 * stride)
    assert _set_obs(tr, obs) == 0
    tr.track(jobs)
    rows_off = obs.copy()
    info = _info_buffer(8)
    assert _set_info(tr, info) == 0
    res = tr.track(jobs)
    assert obs.tobytes() == rows_off.tobytes()
    worst = 0.0
    for j, (slot, local) in enumerate(STAGE_JOBS):
        dbg = tr.debug_job(j)
        _same_debug(dbg, plain_dbg[j])
        assert all(np.array_equal(res[j][k], plain[j][k]) for k in res[j]), j
        ref = kfs[local[-1]]
        want = np_sparse_align(oracle, dict(p1=ref["pyr"], p2=cur[slot]["pyr"], px=ref["px"], depth=ref["depth"],
                                            has=np.ones(len(ref["depth"]), np.uint8), T_ref=np.eye(4)[:3]), n_levels=LEVELS)[2] / SIGMA_I_SQ
        F = _full(info[j]["align_fisher"])
        worst = max(worst, _rel(F, want))
        assert _rel(F, want) <= FISHER_TOL, (j, _rel(F, want))
        n = res[j]["n_inliers"]
        P = _full(info[j]["pose_info"])
        if not res[j]["aligned"]:
            assert slot == 2 and n == 0 and not P.any()
            continue
        want_p = pose_info(res[j]["T_cw"].reshape(3, 4), obs["pw"][j * stride:j * stride + n], fx, fy)
        assert n > 1000 and _rel(P, want_p) <= 1e-9, (j, _rel(P, want_p))
    print(f"tracker: largest align_fisher difference to the restatement {worst:.1e} (relative to the largest diagonal entry)")
    first = info.copy()
    rev = _info_buffer(8)
    assert _set_info(tr, rev) == 0
    tr.track(jobs[::-1])
    assert rev[:len(jobs)][::-1].tobytes() == first[:len(jobs)].tobytes()
    one = _info_buffer(8)
    assert _set_info(tr, one) == 0
    for j in range(len(jobs)):
        tr.track([jobs[j]])
        assert one[:1].tobytes() == first[j:j + 1].tobytes(), j
    from ygz_slam_b200 import capi
    assert _set_info(tr, np.zeros(8, capi.INFO_DTYPE)) == ERR_INVALID     # pageable
    assert _set_info(tr, _info_buffer(7)) == ERR_INVALID                   # short
    assert _set_info(tr, one, capacity=7) == ERR_INVALID
    assert _set_info(tr, None) == 0
    one = _info_buffer(8)
    again = tr.track(jobs)
    assert np.isnan(one["pose_info"]).all()
    assert all(np.array_equal(again[j][k], plain[j][k]) for j in range(len(jobs)) for k in plain[j])
    tr.close()
    fr.close()


@pytest.mark.gpu
def test_tracker_information_in_previous_frame_mode(ctx3, oracle):
    """Previous-frame mode, 2 streams tracking 3 and 2 frames in one interleaved batch (3 waves): each job's align_fisher
    is a symmetric matrix with a positive diagonal, its pose_info numpy's over its rows."""
    from test_vo_observations import K, _obs_buffer, _set_obs
    cells = ctx3.n_cells
    fx, fy = float(ctx3.params.fx), float(ctx3.params.fy)
    data = [synth.shift_stream(s, 4) for s in range(2)]
    fr = ctx3.frames(16)
    tr = fr.tracker(2, 8, K)
    tr.set_reference_mode("previous", [14, 15])
    for s in range(2):
        tr.set_depth(s, data[s][1])
        tr.upload(s * 4, data[s][0][0])
    tr.make_keyframes([dict(stream=s, frame_slot=s * 4, kf_slot=8 + s * 4, entry=0, track_job=-1, local_entry=[0]) for s in range(2)])
    for s in range(2):
        tr.upload(s * 4, data[s][0][1:4])
    stride = 4 * cells
    obs = _obs_buffer(8 * stride)
    info = _info_buffer(8)
    assert _set_obs(tr, obs) == 0 and _set_info(tr, info) == 0
    jobs = [(0, 0, [0]), (1, 4, [0]), (0, 1, [0]), (1, 5, [0]), (0, 2, [0])]
    res = tr.track(jobs)
    for j in range(len(jobs)):
        n = res[j]["n_inliers"]
        assert res[j]["aligned"] and n > 100
        P = _full(info[j]["pose_info"])
        assert _rel(P, pose_info(res[j]["T_cw"].reshape(3, 4), obs["pw"][j * stride:j * stride + n], fx, fy)) <= 1e-9, j
        dbg = tr.debug_job(j)
        assert dbg["n_meas"] > 0
        F = _full(info[j]["align_fisher"])
        assert F[0, 0] > 0 and np.array_equal(F, F.T), j
    tr.close()
    fr.close()


# ---- GPU: streaming engine ---------------------------------------------------------------------------------------------
N_FRAMES = 30
S = 3


@pytest.fixture(scope="module")
def shift_data():
    return [synth.shift_stream(s_, N_FRAMES) for s_ in range(4)]


def _engine(ctx, window, ref_mode, observations=True, information=True, **kw):
    from test_vo_observations import POLICY
    from ygz_slam_b200 import vo_native
    return vo_native.Engine(ctx, S, window=window, ref_mode=ref_mode, observations=observations, information=information,
                            **dict(POLICY, **kw))


def _run(ctx, data, window, ref_mode, pace=None, observations=True, information=True):
    with _engine(ctx, window, ref_mode, observations, information) as eng:
        for k in range(N_FRAMES):
            for s_ in range(S):
                eng.push(s_, data[s_][0][k], data[s_][1], tag=k)
            if pace and k % pace == pace - 1:
                eng.step()
        eng.flush()
        return eng.poll()


def _keyed(res, *more):
    return {(int(r["stream"]), int(r["frame"])): (r,) + tuple(m[i] for m in more) for i, r in enumerate(res)}


@pytest.mark.gpu
@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
def test_engine_information_across_windows_and_pacing(ctx3, shift_data, ref_mode):
    """Windows 1, 4 and 8, lock step and a step every 3 pushes: records bit-identical everywhere, results those of an
    engine without records; every tracked result's pose_info is numpy's over its own rows at its T_cw; key-frames carry
    a tracked record (non-zero), first key-frames zeros."""
    fx, fy = float(ctx3.params.fx), float(ctx3.params.fy)
    plain = _run(ctx3, shift_data, 8, ref_mode, observations=False, information=False)
    base = None
    for window, pace in ((1, None), (4, None), (8, None), (8, 3)):
        res, rows, info = _run(ctx3, shift_data, window, ref_mode, pace)
        assert np.array_equal(np.sort(res, order=["stream", "frame"]), np.sort(plain, order=["stream", "frame"])), window
        per = _keyed(res, rows, info)
        if base is None:
            base = per
        assert per.keys() == base.keys()
        for key in per:
            assert per[key][2].tobytes() == base[key][2].tobytes(), (window, pace, key)
    n_tracked = 0
    for (s_, f), (r, o, I) in base.items():
        status = int(r["status"])
        if f == 0:
            assert status == 1 and not I.any()
        elif status == 0:
            assert _rel(I[1], pose_info(r["T_cw"].reshape(3, 4), o["pw"], fx, fy)) <= 1e-9, (s_, f)
            assert I[0][0, 0] > 0
            n_tracked += 1
        elif status == 1:
            assert I[1][0, 0] > 0 and I[0][0, 0] > 0 and len(o) == r["n_inliers"]
    assert n_tracked > 40


@pytest.mark.gpu
@pytest.mark.parametrize("ref_mode", ["keyframe", "previous"])
def test_engine_information_after_restart_record_and_loss(ctx3, shift_data, ref_mode):
    """A stream saved at frame 20 and loaded into another engine, and a stream restarted for a new sequence, continue with
    the records of the uninterrupted run (of a fresh engine); LOST results carry zeros; information alone (no rows)
    polls (results, info)."""
    from ygz_slam_b200 import vo_native
    res, rows, info = _run(ctx3, shift_data, 8, ref_mode)
    full = _keyed(res, info)
    with _engine(ctx3, 8, ref_mode, observations=False) as a, _engine(ctx3, 8, ref_mode, observations=False) as b:
        for k in range(20):
            a.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        a.flush()
        ra, ia = a.poll()
        b.load_stream(0, a.save_stream(0))
        for k in range(20, N_FRAMES):
            b.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        b.flush()
        rb, ib = b.poll()
    assert len(ra) + len(rb) == N_FRAMES
    for r, I in list(zip(ra, ia)) + list(zip(rb, ib)):
        assert I.tobytes() == full[(0, int(r["frame"]))][1].tobytes(), int(r["frame"])
    with _engine(ctx3, 8, ref_mode) as e:
        for k in range(12):
            e.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        e.restart(0)
        for k in range(N_FRAMES):
            e.push(0, shift_data[3][0][k], shift_data[3][1], tag=100 + k)
        e.flush()
        r2, _, i2 = e.poll()
    with _engine(ctx3, 8, ref_mode) as f:
        for k in range(N_FRAMES):
            f.push(0, shift_data[3][0][k], shift_data[3][1], tag=100 + k)
        f.flush()
        r3, _, i3 = f.poll()
    assert i2[12:].tobytes() == i3.tobytes()
    for r, I in zip(r2[:12], i2[:12]):
        assert I.tobytes() == full[(0, int(r["frame"]))][1].tobytes()
    from test_vo_observations import POLICY
    with vo_native.Engine(ctx3, 1, window=8, ref_mode=ref_mode, information=True, **POLICY, min_inliers=10 ** 6) as e:
        for k in range(8):
            e.push(0, shift_data[0][0][k], shift_data[0][1], tag=k)
        e.flush()
        res, info = e.poll()
    assert list(res["status"]) == [1] + [2] * 7 and not info.any()


@pytest.mark.gpu
def test_engine_information_calls_check_their_state(ctx3, shift_data):
    """set_information only while idle; poll_ex's info must match the switch; ygz_vo_poll discards the records."""
    from test_vo_observations import POLICY
    from ygz_slam_b200 import capi, vo_native
    with vo_native.Engine(ctx3, 1, window=8, **POLICY) as e:
        lib, h = e.lib, e.h
        out = np.zeros(64, vo_native.RESULT_DTYPE)
        info = np.zeros(64, capi.INFO_DTYPE)
        n = C.c_int(0)
        assert lib.ygz_vo_poll_ex(h, out.ctypes.data, 64, C.byref(n), info.ctypes.data, None, 0, None) == ERR_INVALID
        e.push(0, shift_data[0][0][0], shift_data[0][1])
        assert lib.ygz_vo_set_information(h, 1) == ERR_INVALID
        e.flush()
        e.poll()
        e.set_information(True)
        for k in range(1, 8):
            e.push(0, shift_data[0][0][k], shift_data[0][1])
        e.step()
        assert lib.ygz_vo_set_information(h, 0) == ERR_INVALID
        e.flush()
        assert lib.ygz_vo_poll_ex(h, out.ctypes.data, 64, C.byref(n), None, None, 0, None) == ERR_INVALID
        assert lib.ygz_vo_poll(h, out.ctypes.data, 3, C.byref(n)) == 0 and n.value == 3
        res, full = e.poll()
        assert list(res["frame"]) == list(range(4, 8)) and full.shape == (4, 2, 6, 6) and full[:, 1, 0, 0].all()
        e.set_information(False)
