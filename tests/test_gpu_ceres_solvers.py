"""The Ceres-flavoured solvers of ba.cu step by step against oracle/ba.cpp: local_ba_kernel (ygzb_local_ba_ceres and
ygzb_two_view_ba) truncated after k trials and on every termination path, and pose_only_kernel (ygzb_pose_only, the tracking
loop's refinement) at its frame-size, inlier-count, threshold and behind-the-camera edges.

The tests without the gpu mark check on the oracle alone that every constructed case reaches the branch it is built for, so
that the GPU comparisons keep testing that branch and not merely convergence."""
import ctypes as C
import functools
import math
from fractions import Fraction

import numpy as np
import pytest

from ygz_slam_b200 import se3, synth

gpu = pytest.mark.gpu

# the context's intrinsics as the kernels and the oracle see them: float, widened to double
FX, FY, CX, CY = (float(np.float32(v)) for v in (520.9, 521.0, 325.1, 249.7))
CHI2 = float(np.float32(5.991))     # pose-only inlier threshold: the float chi2Mono of BA.cpp, compared in double
assert 5.991 < CHI2


def _t_aa(v):  # se3 log [upsilon; omega] -> [t; angle-axis] (the pose block of CeresReprojectionError)
    out = []
    for x in np.atleast_2d(v):
        T = se3.se3_exp(x)
        out.append(np.r_[T[:, 3], se3.so3_log(T[:, :3])])
    return np.array(out)


def _fixed(n_kf, *idx):
    f = np.zeros(n_kf, np.uint8)
    f[list(idx) or [0]] = 1
    return f


def _exact_px(sc, poses, pts):
    """Pixels of the points at the poses (se3 logs) with the float intrinsics: normalised residuals at rounding level."""
    out = np.empty((len(sc["kf_idx"]), 2))
    for o, (k, j) in enumerate(zip(sc["kf_idx"], sc["pt_idx"])):
        T = se3.se3_exp(poses[k])
        pc = T[:, :3] @ pts[j] + T[:, 3]
        out[o] = FX * pc[0] / pc[2] + CX, FY * pc[1] / pc[2] + CY
    return out


# ---- ygzb_local_ba_ceres ------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _scene(name):
    """Ceres-twin problems: dict(P0 [t; aa], fixed, X0, kf_idx, pt_idx, px, max_iters, single (ill-posed landmarks))."""
    if name == "c4":
        sc = synth.ba_scene()
        return dict(P0=_t_aa(sc["poses_noisy"]), fixed=_fixed(10), X0=sc["pts_noisy"], kf_idx=sc["kf_idx"], pt_idx=sc["pt_idx"],
                    px=sc["px"], max_iters=50)
    if name == "kf6":
        sc = synth.ba_scene(n_kf=6, n_pt=300, target_obs=1500, seed=12)
        return dict(P0=_t_aa(sc["poses_noisy"]), fixed=_fixed(6), X0=sc["pts_noisy"], kf_idx=sc["kf_idx"], pt_idx=sc["pt_idx"],
                    px=sc["px"], max_iters=50)
    if name == "rejections":
        # poses 0.2 off (every observation still >= 0.8 m in front of its camera; the oracle takes the same trials from a
        # start moved by 1e-10 relative): after 4 accepted steps three trials in a row are rejected
        sc = synth.ba_scene(n_kf=6, n_pt=300, target_obs=1500, seed=13, pose_sigma=0.2)
        return dict(P0=_t_aa(sc["poses_noisy"]), fixed=_fixed(6), X0=sc["pts_noisy"], kf_idx=sc["kf_idx"], pt_idx=sc["pt_idx"],
                    px=sc["px"], max_iters=50)
    if name == "huber":    # ba::OptimizeCurrent's shape: gross outliers under HuberLoss(0.1), the current frame free
        # (down-weighted landmarks have H_kk below 1e-6: their damping is clamped and depends on the Jacobi scaling)
        sc = synth.ba_scene(n_kf=6, n_pt=400, target_obs=2000, seed=21)
        rng = np.random.default_rng(3)
        px = sc["px"].copy()
        bad = rng.choice(len(px), 40, replace=False)
        px[bad] += rng.choice([-1, 1], (40, 2)) * rng.uniform(60, 150, (40, 2))
        P0 = _t_aa(sc["poses_true"])
        P0[5] = _t_aa(sc["poses_noisy"])[5]
        return dict(P0=P0, fixed=_fixed(6, 0, 1, 2, 3, 4), X0=sc["pts_noisy"], kf_idx=sc["kf_idx"], pt_idx=sc["pt_idx"], px=px,
                    max_iters=50, huber=0.1)
    if name in ("exact_start", "exact_small", "exact_small_last_trial"):
        # noise-free pixels: at the true poses and points the gradient is at rounding level (termination 1 before any step);
        # 1e-4 away from them LM converges quadratically and exits on the gradient after 4 steps
        sc = synth.ba_scene(n_kf=6, n_pt=300, target_obs=1500, seed=12)
        px = _exact_px(sc, sc["poses_true"], sc["pts_true"])
        P0, X0 = _t_aa(sc["poses_true"]), sc["pts_true"].copy()
        if name != "exact_start":
            rng = np.random.default_rng(3)
            P0[1:] += rng.normal(0, 1e-4, P0[1:].shape)
            X0 += rng.normal(0, 1e-4, X0.shape)
        return dict(P0=P0, fixed=_fixed(6), X0=X0, kf_idx=sc["kf_idx"], pt_idx=sc["pt_idx"], px=px,
                    max_iters=4 if name == "exact_small_last_trial" else 50)
    if name == "far_restart":
        # the kf6 problem moved 1e5 m away from the world origin and restarted 1e-4 m off its own optimum: the step is then
        # below 1e-8 |x| while the cost still falls by far more than the function tolerance -- the parameter-tolerance exit
        base = _scene("kf6")
        wP, wX, _ = _oracle().local_ba_ceres(base["P0"], base["fixed"], base["X0"], base["kf_idx"], base["pt_idx"], base["px"])
        D = np.array([1e5, -2e4, 3e4])
        P0 = wP.copy()
        for k in range(len(P0)):
            R = se3.so3_exp(P0[k, 3:])
            P0[k, :3] -= R @ D
        rng = np.random.default_rng(4)
        free = base["fixed"] == 0
        P0[free, :3] += rng.normal(0, 1e-4, (int(free.sum()), 3))
        X0 = wX + D + rng.normal(0, 1e-4, wX.shape)
        return dict(base, P0=P0, X0=X0)
    if name == "free16":   # kMaxFreePoses: 17 key-frames, one fixed -> the 96 x 96 reduced system (74.5 KB of shared memory)
        sc = synth.ba_scene(n_kf=17, n_pt=400, target_obs=3200, seed=40)
        return dict(P0=_t_aa(sc["poses_noisy"]), fixed=_fixed(17), X0=sc["pts_noisy"], kf_idx=sc["kf_idx"], pt_idx=sc["pt_idx"],
                    px=sc["px"], max_iters=50)
    if name == "poses64":  # kMaxPoses: 64 key-frames, the 16 that see the most landmarks free
        sc = synth.ba_scene(n_kf=64, n_pt=600, target_obs=6000, seed=44)
        seen = np.bincount(sc["kf_idx"], minlength=64)
        fixed = np.ones(64, np.uint8)
        fixed[np.argsort(-seen, kind="stable")[:16]] = 0
        P0 = _t_aa(sc["poses_noisy"])
        P0[fixed == 1] = _t_aa(sc["poses_true"])[fixed == 1]
        return dict(P0=P0, fixed=fixed, X0=sc["pts_noisy"], kf_idx=sc["kf_idx"], pt_idx=sc["pt_idx"], px=sc["px"], max_iters=50)
    if name == "edge":     # landmarks seen only by fixed key-frames, with one observation, and never observed
        sc = synth.ba_edge_scene()
        n = len(sc["pts_noisy"])
        X0 = np.concatenate([sc["pts_noisy"], sc["pts_noisy"][:5] + 1.0])      # 5 landmarks nobody observes
        return dict(P0=_t_aa(sc["poses_noisy"]), fixed=_fixed(6, 0, 1), X0=X0, kf_idx=sc["kf_idx"], pt_idx=sc["pt_idx"], px=sc["px"],
                    max_iters=50, single=np.r_[sc["single"], np.arange(n, n + 5)])
    if name == "empty":    # no observations at all
        sc = synth.ba_scene(n_kf=3, n_pt=20, seed=42)
        return dict(P0=_t_aa(sc["poses_noisy"]), fixed=_fixed(3), X0=sc["pts_noisy"], kf_idx=np.zeros(0, np.int32),
                    pt_idx=np.zeros(0, np.int32), px=np.zeros((0, 2)), max_iters=50)
    if name == "tiny":     # 10 landmarks: fewer than the CTAs of a 16-CTA cluster
        sc = synth.ba_scene(n_kf=4, n_pt=10, target_obs=40, seed=43)
        return dict(P0=_t_aa(sc["poses_noisy"]), fixed=_fixed(4), X0=sc["pts_noisy"], kf_idx=sc["kf_idx"], pt_idx=sc["pt_idx"],
                    px=sc["px"], max_iters=50)
    raise KeyError(name)


@functools.lru_cache(maxsize=None)
def _oracle():
    from oracle.pyoracle import Oracle
    return Oracle()


def _ora(pb, max_iters=None):
    return _oracle().local_ba_ceres(pb["P0"], pb["fixed"], pb["X0"], pb["kf_idx"], pb["pt_idx"], pb["px"],
                                    max_iters=pb["max_iters"] if max_iters is None else max_iters, huber=pb.get("huber", 0.0))


def _gpu_batch(ctx, pbs, max_iters):
    kf_off = np.cumsum([0] + [len(p["fixed"]) for p in pbs])
    pt_off = np.cumsum([0] + [len(p["X0"]) for p in pbs])
    obs_off = np.cumsum([0] + [len(p["kf_idx"]) for p in pbs])
    P, X, st = ctx.local_ba_ceres(kf_off, pt_off, obs_off, np.concatenate([p["P0"] for p in pbs]), np.concatenate([p["fixed"] for p in pbs]),
                                  np.concatenate([p["X0"] for p in pbs]), np.concatenate([p["kf_idx"] for p in pbs]),
                                  np.concatenate([p["pt_idx"] for p in pbs]), np.concatenate([p["px"] for p in pbs]), max_iters=max_iters,
                                  huber=pbs[0].get("huber", 0.0))
    return [(P[kf_off[i]:kf_off[i + 1]], X[pt_off[i]:pt_off[i + 1]], st[i]) for i in range(len(pbs))]


def _close(a, b, rel):
    """|a - b| <= rel * max(1, |b|) elementwise (absolute below 1)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return bool(np.all(np.abs(a - b) <= rel * np.maximum(1.0, np.abs(b))))


def _check_step(res, want, rel, cost_abs=0.0, skip_pts=()):
    """One run against the oracle after the same trials: the same decisions (trials, accepted steps, exit) and the same
    numbers (parameters, costs, radius) within rel."""
    P, X, st = res
    wP, wX, wst = want
    assert (st["iters"], st["successful_steps"], st["termination"]) == (wst["iters"], wst["successful_steps"], wst["termination"]), (st, wst)
    keep = np.setdiff1d(np.arange(len(wX)), skip_pts)
    assert _close(P, wP, rel), np.abs(P - wP).max()
    assert _close(X[keep], wX[keep], rel), np.abs(X[keep] - wX[keep]).max()
    for k in ("cost_initial", "cost_final", "radius_final"):
        assert abs(st[k] - wst[k]) <= rel * abs(wst[k]) + cost_abs, (k, st[k], wst[k])


def test_ceres_cases_reach_their_branch(oracle):
    """Oracle only: the termination code and trial count each constructed case is meant for (0 max_iters, 1 gradient,
    2 parameter, 3 function tolerance).  Code 4 (radius below 1e-32) needs 15 rejected trials in a row; every rejection
    halves the radius again, so the damped step approaches the steepest-descent step and the model's predicted decrease
    becomes exact -- a finite, smooth cost with gradient above 1e-10 accepts one of them.  It is left to non-finite input."""
    # rejected trials 5, 6 and 7 in a row: each divides the radius by the decrease factor, which doubles (2, 4, 8)
    runs = {k: _ora(_scene("rejections"), k)[2] for k in REJECTION_TRIALS}
    assert [runs[k]["successful_steps"] for k in REJECTION_TRIALS] == [4, 4, 4, 4, 5]
    assert all(runs[k]["termination"] == 0 and runs[k]["iters"] == k for k in REJECTION_TRIALS)
    r4 = runs[4]["radius_final"]
    assert [runs[k]["radius_final"] for k in (5, 6, 7)] == [r4 / 2, r4 / 8, r4 / 64]
    for k in (0, 1, 2, 3, 5, 8):
        _, _, st = _ora(_scene("huber"), k)
        assert st["termination"] == 0 and st["iters"] == k == st["successful_steps"], ("huber", k, st)
    for k in (0, 1, 2, 3, 5):
        for name in ("c4", "kf6"):
            _, _, st = _ora(_scene(name), k)
            assert st["termination"] == 0 and st["iters"] == k == st["successful_steps"], (name, k, st)
            assert (st["cost_final"] == st["cost_initial"]) == (k == 0)
    for name in ("c4", "kf6"):
        _, _, st = _ora(_scene(name), 8)
        assert st["termination"] == 3 and st["iters"] == 7
    _, _, st = _ora(_scene("exact_start"))
    assert st["termination"] == 1 and st["iters"] == 0 and st["cost_initial"] < 1e-25
    _, _, st = _ora(_scene("exact_start"), 0)
    assert st["termination"] == 1 and st["iters"] == 0        # max_iters = 0: evaluated and tested once all the same
    _, _, st = _ora(_scene("exact_small"))
    assert st["termination"] == 1 and st["iters"] == st["successful_steps"] == 4
    _, _, st = _ora(_scene("exact_small_last_trial"))          # the 4th and last allowed trial is followed by the gradient test
    assert st["termination"] == 1 and st["iters"] == 4
    _, _, st = _ora(_scene("far_restart"))
    assert st["termination"] == 2 and st["iters"] == 1 and st["successful_steps"] == 0
    # the step is not taken; the start lies 1e-3 (relative) above the optimum's cost, far outside the function tolerance
    assert st["cost_final"] == st["cost_initial"] > (1 + 1e-4) * _ora(_scene("kf6"))[2]["cost_final"]
    for name in ("free16", "poses64", "edge", "tiny"):
        _, _, st = _ora(_scene(name))
        assert st["termination"] in (1, 2, 3) and 3 <= st["iters"] < 50, (name, st)
    _, _, st = _ora(_scene("empty"))
    assert st["termination"] == 1 and st["iters"] == 0 and st["cost_initial"] == 0


@gpu
@pytest.mark.parametrize("k", [0, 1, 2, 3, 5, 8])
@pytest.mark.parametrize("name", ["c4", "kf6", "huber"])
def test_ceres_truncated_runs(ctx3, name, k):
    """After exactly k trials: the same poses, points, costs, radius, accepted steps and termination as the oracle -- each
    LM step (damping, Jacobi scaling, radius update) pinned, not only the optimum.  k = 0 reports the initial cost."""
    pb = _scene(name)
    (res,) = _gpu_batch(ctx3, [pb], k)
    _check_step(res, _ora(pb, k), 1e-9)


REJECTION_TRIALS = (4, 5, 6, 7, 8)


@gpu
@pytest.mark.parametrize("k", REJECTION_TRIALS)
def test_ceres_rejected_trials(ctx3, k):
    """Across three rejected trials in a row and the accepted one after them: the parameters are restored, the radius is
    divided by 2, 4 and 8 and the next accepted step starts from the shrunk region -- the same as the oracle after k trials."""
    pb = _scene("rejections")
    (res,) = _gpu_batch(ctx3, [pb], k)
    _check_step(res, _ora(pb, k), 1e-9)


@gpu
@pytest.mark.parametrize("name", ["exact_start", "exact_small", "exact_small_last_trial", "far_restart", "c4"])
def test_ceres_termination_codes(ctx3, name):
    """Termination 1 (before any step, after 4 steps, and on the last allowed trial), 2 and 3 with the oracle's trial
    count and accepted steps.  Costs at rounding level (1e-30 .. 1e-18) compare absolutely."""
    pb = _scene(name)
    (res,) = _gpu_batch(ctx3, [pb], pb["max_iters"])
    _check_step(res, _ora(pb), 1e-9, cost_abs=1e-20)


@gpu
def test_ceres_max_iters_zero_gradient_exit(ctx3):
    (res,) = _gpu_batch(ctx3, [_scene("exact_start")], 0)
    want = _ora(_scene("exact_start"), 0)
    assert want[2]["termination"] == 1
    _check_step(res, want, 1e-9, cost_abs=1e-20)


@gpu
@pytest.mark.parametrize("cluster", [1, 2, 4, 8, 16])
def test_ceres_sizes_and_structure(ctx3, cluster, monkeypatch):
    """One batch at every cluster size: 16 free poses (the 96 x 96 system), 64 poses with 16 free, the edge scene (landmarks
    seen only by fixed key-frames, with one observation, never observed), a problem without observations and a 10-landmark
    problem (fewer landmarks than CTAs), each against the oracle.  A landmark with one observation is free along its ray
    (only the damping fixes its step), so for those the check is finiteness."""
    monkeypatch.setenv("YGZB_BA_CLUSTER", str(cluster))
    names = ["free16", "poses64", "edge", "empty", "tiny"]
    pbs = [_scene(n) for n in names]
    for name, pb, res in zip(names, pbs, _gpu_batch(ctx3, pbs, 50)):
        single = pb.get("single", ())
        _check_step(res, _ora(pb), 1e-6, cost_abs=1e-15, skip_pts=single)
        assert np.isfinite(res[1]).all(), name
        assert np.array_equal(res[0][pb["fixed"] == 1], pb["P0"][pb["fixed"] == 1]), name
    e = pbs[names.index("edge")]
    assert np.array_equal(_gpu_batch(ctx3, [e], 50)[0][1][-5:], e["X0"][-5:])     # unobserved landmarks do not move


def _raw_ceres(ctx, kf_off, pt_off, obs_off, poses, fixed, pts, kf_idx, pt_idx, px, max_iters=50, huber=0.0):
    """ygzb_local_ba_ceres on the caller's arrays themselves: (rc, poses, pts, stats as raw tuples)."""
    from ygz_slam_b200 import capi
    P = max(len(kf_off) - 1, 1)
    st = (capi.CeresStats * P)()
    for s in st:
        s.iters, s.successful_steps, s.cost_initial, s.cost_final, s.radius_final, s.termination = -7, -7, -7.0, -7.0, -7.0, -7
    arr = lambda a, t: np.ascontiguousarray(a, t)   # noqa: E731
    rc = ctx.lib.ygzb_local_ba_ceres(ctx.h, len(kf_off) - 1, capi._p(arr(kf_off, np.int32)), capi._p(arr(pt_off, np.int32)),
                                     capi._p(arr(obs_off, np.int32)), capi._p(poses), capi._p(arr(fixed, np.uint8)), capi._p(pts),
                                     capi._p(arr(kf_idx, np.int32)), capi._p(arr(pt_idx, np.int32)), capi._p(arr(px, np.float64)),
                                     max_iters, C.c_double(huber), st)
    return rc, [(s.iters, s.successful_steps, s.cost_initial, s.cost_final, s.radius_final, s.termination) for s in st]


def _with_duplicate(pb, kf):
    """pb with a second observation, by key-frame kf, of the first landmark kf observes."""
    q = int(np.flatnonzero(pb["kf_idx"] == kf)[0])
    return dict(pb, kf_idx=np.insert(pb["kf_idx"], q, kf), pt_idx=np.insert(pb["pt_idx"], q, pb["pt_idx"][q]),
                px=np.insert(pb["px"], q, pb["px"][q] + 0.5, 0))


@gpu
def test_ceres_rejects_invalid_problems(ctx3):
    """17 free poses, 65 poses, 0 poses, an index out of range, max_iters < 0, huber_a < 0 or NaN, and a landmark observed
    twice by one free pose return YGZB_ERR_INVALID (-1) and leave the caller's poses, points and statistics as they were.
    A duplicate on the fixed key-frame is a valid problem (no Schur cross terms) and matches the oracle."""
    sc = synth.ba_scene(n_kf=10, n_pt=300, target_obs=1200, seed=50)
    n_obs = len(sc["kf_idx"])
    base = (sc["kf_idx"], sc["pt_idx"], sc["px"])
    P10 = _t_aa(sc["poses_noisy"])
    bad_idx = sc["kf_idx"].copy()
    bad_idx[7] = 10
    pb = dict(P0=P10, fixed=_fixed(10), X0=sc["pts_noisy"], kf_idx=sc["kf_idx"], pt_idx=sc["pt_idx"], px=sc["px"], max_iters=50)
    dup = _with_duplicate(pb, 3)   # key-frame 3 is free
    cases = {
        "17 free poses": ([0, 18], np.zeros((18, 6)), _fixed(18), base, 50, 0.0),
        "65 poses": ([0, 65], np.zeros((65, 6)), np.ones(65, np.uint8), base, 50, 0.0),
        "0 poses": ([0, 0], np.zeros((0, 6)), np.zeros(0, np.uint8), base, 50, 0.0),
        "index out of range": ([0, 10], P10, _fixed(10), (bad_idx, sc["pt_idx"], sc["px"]), 50, 0.0),
        "max_iters < 0": ([0, 10], P10, _fixed(10), base, -1, 0.0),
        "huber_a < 0": ([0, 10], P10, _fixed(10), base, 50, -0.1),
        "huber_a NaN": ([0, 10], P10, _fixed(10), base, 50, math.nan),
        "duplicate": ([0, 10], P10, _fixed(10), (dup["kf_idx"], dup["pt_idx"], dup["px"]), 50, 0.0),
    }
    for what, (kf_off, P0, fixed, (kf_idx, pt_idx, px), max_iters, huber) in cases.items():
        poses, pts = np.array(P0, np.float64), np.array(sc["pts_noisy"], np.float64)
        rc, st = _raw_ceres(ctx3, kf_off, [0, 300], [0, len(kf_idx)], poses, fixed, pts, kf_idx, pt_idx, px, max_iters, huber)
        assert rc == -1, what
        assert np.array_equal(poses, P0) and np.array_equal(pts, sc["pts_noisy"]), what
        assert st[0] == (-7, -7, -7.0, -7.0, -7.0, -7), what
    assert n_obs + 1 == len(dup["kf_idx"])
    ok = _with_duplicate(pb, 0)                  # key-frame 0 is fixed
    (res,) = _gpu_batch(ctx3, [ok], 50)
    _check_step(res, _ora(ok), 1e-6, cost_abs=1e-15)


# ---- ygzb_pose_only ------------------------------------------------------------------------------------------------------
I12 = np.eye(4)[:3].reshape(-1)


def _front_points(n, seed):
    """n world points in front of the identity camera with their exact pixels (float intrinsics, the kernels' formula)."""
    rng = np.random.default_rng(seed)
    z = rng.uniform(2.0, 5.0, n)
    u, v = rng.uniform(40, 600, n), rng.uniform(40, 440, n)
    pw = np.stack([(u - CX) / FX * z, (v - CY) / FY * z, z], 1)
    px = np.stack([FX * pw[:, 0] / pw[:, 2] + CX, FY * pw[:, 1] / pw[:, 2] + CY], 1)
    return pw, px


def _split_square(target):
    """(dx, dy) whose squared pixel error dx * dx + dy * dy evaluates to `target` exactly in double, with or without an FMA:
    dx = a 2^-24 (26 bits, dx^2 exact), dy = b 2^-45 (a multiple of the ulp of cy, so cy - dy is exact) makes up the rest."""
    a = math.isqrt(int(Fraction(target) * 2 ** 48))
    dx = a * 2.0 ** -24
    b0 = round(math.sqrt(float(Fraction(target) - Fraction(dx) ** 2)) * 2.0 ** 45)
    for b in (b0 + k for k in (0, 1, -1, 2, -2, 3, -3)):
        dy = b * 2.0 ** -45
        plain = float(Fraction(dx) ** 2 + Fraction(dy * dy))   # fl(fl(dx dx) + fl(dy dy)) = fma(dx, dx, fl(dy dy))
        fused = float(Fraction(dx) ** 2 + Fraction(dy) ** 2)   # fma(dy, dy, fl(dx dx))
        if plain == fused == target:
            return dx, dy
    raise AssertionError(target)


THRESHOLD_CASES = {   # round-0 squared error of the probe point -> inlier (count 10: the rounds go on) or not (9: stop)
    "below": (np.nextafter(5.991, 0), True),
    "at_5.991": (5.991, True),
    "between": ((5.991 + CHI2) / 2, True),
    "at_5.991f": (CHI2, True),
    "above": (np.nextafter(CHI2, 10), False),
}


def _pose_frames():
    """name -> (pw, px, T0 (12,)) for one frame each."""
    frames = {}
    sc = synth.pose_only_scene(11, seed=61, pose_sigma=0.0005, pixel_sigma=0.3)
    for n in (0, 1, 9, 10, 11):
        frames[f"n{n}"] = (sc["pw"][:n], sc["px"][:n], sc["T0"].reshape(-1))
    for name, (target, _) in THRESHOLD_CASES.items():
        pw, px = _front_points(9, 62)
        dx, dy = _split_square(target)
        # the probe point on the optical axis: with the identity pose it projects to (cx, cy) exactly
        frames["thr_" + name] = (np.r_[pw, [[0.0, 0.0, 3.0]]], np.r_[px, [[CX - dx, CY - dy]]], I12)
    pw, px = _front_points(12, 63)
    px = px + np.random.default_rng(63).normal(0, 0.5, px.shape)
    T0 = se3.se3_exp(np.array([0.001, -0.001, 0.0015, 0.0004, -0.0003, 0.0002])).reshape(-1)
    # behind the camera at the start pose, projecting far from its pixel: round 0's solve fails, the point becomes an outlier
    frames["behind_outlier"] = (np.r_[pw, [[0.5, 0.2, -3.0]]], np.r_[px, [[320.0, 240.0]]], T0)
    # behind the camera on the ray of a point in front: it projects onto its pixel, is an inlier with negative depth, and
    # every round's solve fails (the pose stays at the input)
    frames["behind_inlier"] = (np.r_[pw, -pw[:1]], np.r_[px, px[:1]], I12)
    frames["z0"] = (np.r_[pw, [[0.4, 0.3, 0.0]]], np.r_[px, [[400.0, 300.0]]], I12)
    pw, px = _front_points(30, 64)
    frames["all_outliers"] = (pw, px + 40.0, I12)
    frames["at_true_pose"] = (pw, px, I12)
    frames["n10_one_outlier"] = (pw[:11], np.r_[px[:10], px[10:11] + 20.0], I12)
    frames["n10_two_outliers"] = (pw[:11], np.r_[px[:9], px[9:11] + 20.0], I12)
    return frames


def test_pose_only_cases_reach_their_branch(oracle):
    """Oracle only: each frame takes the path it is built for."""
    fr = _pose_frames()
    for name, (target, inlier) in THRESHOLD_CASES.items():
        pw, px, T0 = fr["thr_" + name]
        # numpy restatement of the round-0 classification at the identity pose (BA.cpp:231-251)
        u, v = FX * pw[:, 0] / pw[:, 2] + CX, FY * pw[:, 1] / pw[:, 2] + CY
        e2 = (u - px[:, 0]) ** 2 + (v - px[:, 1]) ** 2
        assert e2[-1] == target and (e2[:-1] < 1e-20).all(), name
        T, inl, depth, cnt = oracle.pose_only(pw, px, T0.reshape(3, 4))
        assert inl[-1] == inlier and (depth[-1] > 2.9 if inlier else depth[-1] == -1.0), name
        if inlier:
            assert cnt >= 10 and not np.array_equal(T, T0.reshape(3, 4)), name   # round 0 counted 10: it refined
        else:
            assert cnt == 9 and np.array_equal(T, T0.reshape(3, 4)), name         # 9 < 10: stop with the input pose
    for n in (0, 1, 9):
        T, _, _, cnt = oracle.pose_only(*fr[f"n{n}"][:2], fr[f"n{n}"][2].reshape(3, 4))
        assert cnt == n and np.allclose(T.reshape(-1), fr[f"n{n}"][2], rtol=0, atol=1e-12)
    for n in (10, 11):
        T, _, _, cnt = oracle.pose_only(*fr[f"n{n}"][:2], fr[f"n{n}"][2].reshape(3, 4))
        assert cnt == n and not np.allclose(T.reshape(-1), fr[f"n{n}"][2], rtol=0, atol=1e-6)
    _, inl, _, cnt = oracle.pose_only(*fr["behind_outlier"][:2], fr["behind_outlier"][2].reshape(3, 4))
    assert not inl[-1] and cnt == 12
    T, inl, depth, cnt = oracle.pose_only(*fr["behind_inlier"][:2], I12.reshape(3, 4))
    assert inl[-1] and depth[-1] < 0 and cnt == 13 and np.array_equal(T.reshape(-1), I12)
    _, inl, _, cnt = oracle.pose_only(*fr["z0"][:2], I12.reshape(3, 4))
    assert not inl[-1] and cnt == 12
    T, inl, _, cnt = oracle.pose_only(*fr["all_outliers"][:2], I12.reshape(3, 4))
    assert cnt == 0 and not inl.any() and np.array_equal(T.reshape(-1), I12)
    T, inl, _, cnt = oracle.pose_only(*fr["at_true_pose"][:2], I12.reshape(3, 4))
    assert cnt == 30 and np.allclose(T.reshape(-1), I12, rtol=0, atol=1e-12)
    # 10 of 11 survive round 0, so round 1 runs (and its count, from round 0's outlier-pulled pose, is what it is); 9 stop
    T, _, _, cnt = oracle.pose_only(*fr["n10_one_outlier"][:2], I12.reshape(3, 4))
    assert not np.array_equal(T.reshape(-1), I12)
    T, _, _, cnt = oracle.pose_only(*fr["n10_two_outliers"][:2], I12.reshape(3, 4))
    assert cnt == 9 and np.array_equal(T.reshape(-1), I12)


def _check_pose_only(T, inl, depth, cnt, want, name):
    wT, winl, wdepth, wcnt = want
    assert cnt == wcnt, (name, cnt, wcnt)
    assert np.array_equal(inl, winl), name
    # depths come from the pose of the previous round: bit-equal while it is the input pose, rounding-level after a solve
    assert np.allclose(depth, wdepth, rtol=0, atol=1e-9), name
    assert np.linalg.norm(se3.se3_log(se3.mul(se3.inv(T), wT))) < 1e-4, name


@gpu
def test_pose_only_edges_batched_and_alone(ctx3, oracle):
    """Every frame of _pose_frames in one batch and then alone: n_inlier and the inlier flags exactly as the oracle's, depths
    within 1e-9 and the pose within 1e-4 (frames that stop with the input pose: bit-equal)."""
    fr = _pose_frames()
    names = list(fr)
    offs = np.cumsum([0] + [len(fr[n][0]) for n in names])
    T, inl, depth, cnt = ctx3.pose_only(offs, np.concatenate([fr[n][0] for n in names]).reshape(-1, 3),
                                        np.concatenate([fr[n][1] for n in names]).reshape(-1, 2), np.stack([fr[n][2] for n in names]))
    failed = []
    for p, name in enumerate(names):
        pw, px, T0 = fr[name]
        want = oracle.pose_only(pw, px, T0.reshape(3, 4))
        s = slice(offs[p], offs[p + 1])
        runs = [("batched", (T[p], inl[s], depth[s], cnt[p]))]
        if len(pw):   # (an empty frame alone has no point arrays to pass)
            one = ctx3.pose_only([0, len(pw)], pw, px, T0.reshape(1, 12))
            runs.append(("alone", (one[0][0], one[1], one[2], one[3][0])))
        for how, got in runs:
            try:
                _check_pose_only(*got, want, name)
                if np.array_equal(want[0].reshape(-1), T0):   # stopped (or failed every solve) with the input pose
                    assert np.array_equal(got[0], want[0]), name
            except AssertionError as e:
                failed.append(f"{name} {how}: {e}")
    assert not failed, failed


# ---- ygzb_two_view_ba ----------------------------------------------------------------------------------------------------
def _two_view_pairs():
    pairs = {"scene": synth.two_view_scene(21, 120, 12)}
    s = synth.two_view_scene(23, 1, 0)
    pairs["one_point"] = s
    pairs["empty"] = dict(T_ref=s["T_ref"], T_cur0=se3.se3_exp(np.array([-0.1, 0.02, 0.01, 0.02, -0.01, 0.03])),
                          px_ref=np.zeros((0, 2)), px_cur=np.zeros((0, 2)), inlier=np.zeros(0, np.uint8), X0=np.zeros((0, 3)))
    s = synth.two_view_scene(24, 40, 0)
    pairs["all_non_inliers"] = dict(s, inlier=np.zeros(40, np.uint8))
    # 8 points behind both cameras (consistent pixels: they stay behind) among 40 in front
    s = synth.two_view_scene(25, 48, 0)
    X = s["X"].copy()
    X[40:, 2] *= -1
    pc = (s["T_cur"][:, :3] @ X.T).T + s["T_cur"][:, 3]
    assert (pc[40:, 2] < 0).all()
    s["px_ref"][40:] = np.stack([FX * X[40:, 0] / X[40:, 2] + CX, FY * X[40:, 1] / X[40:, 2] + CY], 1)
    s["px_cur"][40:] = np.stack([FX * pc[40:, 0] / pc[40:, 2] + CX, FY * pc[40:, 1] / pc[40:, 2] + CY], 1)
    s["X0"][40:] = X[40:] + np.random.default_rng(25).normal(0, 0.02, (8, 3))
    pairs["behind"] = s
    return pairs


def test_two_view_cases_reach_their_branch(oracle):
    pr = _two_view_pairs()
    T, inl, X, st, cnt = oracle.two_view_ba(*(pr["empty"][k] for k in ("T_ref", "T_cur0", "px_ref", "px_cur", "inlier", "X0")))
    assert cnt == 0 and st["termination"] == 1 and st["iters"] == 0
    assert np.allclose(T, pr["empty"]["T_cur0"], rtol=0, atol=1e-12)       # the exp / log round trip of the input pose
    T, inl, X, st, cnt = oracle.two_view_ba(*(pr["all_non_inliers"][k] for k in ("T_ref", "T_cur0", "px_ref", "px_cur", "inlier", "X0")))
    assert cnt > 30 and st["iters"] > 3                                       # restarted from (0, 0, 1) and recovered
    T, inl, X, st, cnt = oracle.two_view_ba(*(pr["behind"][k] for k in ("T_ref", "T_cur0", "px_ref", "px_cur", "inlier", "X0")))
    assert not inl[40:].any() and inl[:40].sum() >= 38 and (X[40:, 2] < 0).all()


@gpu
def test_two_view_ba_edges(ctx3, oracle):
    """One batch: a 120-point pair, a 1-point pair, a pair without points (its pose is the input's exp / log round trip),
    a pair whose points all come in as non-inliers (restart from (0, 0, 1) under the Huber loss), and a pair with points
    behind both cameras -- inlier flags, pose, points and statistics against the oracle.  The batch runs in two orders of
    the same size, so that the pair without points sits where the previous call wrote another pair's pose."""
    pr = _two_view_pairs()
    for names in (["scene", "one_point", "all_non_inliers", "behind", "empty"], ["scene", "one_point", "empty", "all_non_inliers", "behind"]):
        _two_view_batch(ctx3, oracle, pr, names)


def _two_view_batch(ctx3, oracle, pr, names):
    keys = ("T_ref", "T_cur0", "px_ref", "px_cur", "inlier", "X0")
    offs = np.cumsum([0] + [len(pr[n]["X0"]) for n in names]).astype(np.int32)
    T, inl, X, st = ctx3.two_view_ba(offs, np.stack([pr[n]["T_ref"] for n in names]), np.stack([pr[n]["T_cur0"] for n in names]),
                                     *(np.concatenate([pr[n][k] for n in names]) for k in ("px_ref", "px_cur", "inlier", "X0")))
    for p, name in enumerate(names):
        wT, winl, wX, wst, _ = oracle.two_view_ba(*(pr[name][k] for k in keys))
        sl = slice(offs[p], offs[p + 1])
        tol = 1e-12 if name == "empty" else 1e-4
        assert np.linalg.norm(se3.se3_log(se3.mul(se3.inv(T[p]), wT))) < tol, name
        assert np.array_equal(inl[sl], winl), name
        if len(wX):
            assert np.abs(X[sl] - wX).max() < 1e-4, name
        assert (st[p]["iters"], st[p]["termination"]) == (wst["iters"], wst["termination"]), (name, st[p], wst)
        assert abs(st[p]["cost_final"] - wst["cost_final"]) < 1e-9 * wst["cost_final"] + 1e-15, name
