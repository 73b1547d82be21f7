"""The tracking loop's two iterative solvers step by step against the oracle: the g2o-flavoured local BA (local_ba2_kernel
behind ygzb_local_ba, oracle/ba.cpp) and the sparse image alignment (sparse_align2_kernel behind ygzb_sparse_align,
oracle/align.cpp).

A converged result cannot see a wrong Hessian term, damping schedule or gain ratio: Gauss-Newton and Levenberg-Marquardt
stop where J^T r = 0 whatever H is.  So every run here is truncated (max_iters, max_trials, n_iter, a single pyramid level)
and compared after exactly k steps: the decisions (iterations, LM trials, rollbacks, outlier flags) exactly, the numbers
(poses, points, costs, lambda) within a relative tolerance.  The tests without the gpu mark check on the oracle alone that
every constructed case reaches the branch it is built for."""
import functools

import numpy as np
import pytest

from ygz_slam_b200 import se3, synth

gpu = pytest.mark.gpu

# Tolerances about 100x above the largest differences measured on an H100 80GB HBM3 (700 W power limit); each test's
# docstring states its own largest difference.
BA_TOL = 1e-9         # local BA after k LM trials: poses, points, chi2_initial, chi2_final, lambda_final -- relative to
#                       values above 1, absolute below (_rel: |a - b| / max(1, |b|)); measured 1.2e-11
ALIGN_TOL = 2.5e-12   # sparse alignment: |se3 log of T_gpu^-1 T_oracle| after k Gauss-Newton steps, an absolute norm
#                       (radians and metres); measured 2.5e-14
FEW_TOL = 5e-10       # the same norm after one step of a problem with 3 to 6 features; measured 6.0e-12


def _g2o(v):
    v = np.asarray(v)
    return np.concatenate([v[..., 3:], v[..., :3]], -1)


def _fixed(n_kf, *idx):
    f = np.zeros(n_kf, np.uint8)
    f[list(idx) or [0]] = 1
    return f


# ---- local BA -----------------------------------------------------------------------------------------------------------
AXIS_DEPTHS = (2.0, 2.5, 3.0, 0.05)     # the last landmark is so near that its diagonal of H is the largest
DELTA2 = 5.991 * 5.991                  # Huber delta^2 as both sides compute it


def _grid(x):
    return float(np.round(x * 2.0 ** 30) / 2.0 ** 30)


def _axis_errors():
    """Errors of the 8 observations of the axis scene: |e|^2 just above and below the Huber delta^2 (1e-9 away), just
    above, on and below the 5.991 outlier threshold, and well inside and outside both."""
    e_hub_hi, e_hub_lo = _grid(np.sqrt(DELTA2 * (1 + 1e-9))), _grid(np.sqrt(DELTA2 * (1 - 1e-9)))
    e_out = _grid(np.sqrt(5.991))
    return np.array([[e_hub_hi, 0], [e_hub_lo, 0], [e_out, 0], [-e_out, 0], [0, 7.0], [1.0, -2.0], [0.5, 0.25], [0, 0]])


@functools.lru_cache(maxsize=None)
def _ba(name):
    """Local-BA problems: dict(P0 (g2o order), fixed, X0, kf_idx, pt_idx, px) plus solver parameters."""
    def from_scene(sc, fixed, **kw):
        return dict(P0=_g2o(sc["poses_noisy"]), fixed=fixed, X0=sc["pts_noisy"], kf_idx=sc["kf_idx"], pt_idx=sc["pt_idx"],
                    px=sc["px"], **kw)
    if name == "c4":
        return from_scene(synth.ba_scene(), _fixed(10))
    if name == "kf6":
        return from_scene(synth.ba_scene(n_kf=6, n_pt=300, target_obs=1500, seed=12), _fixed(6))
    if name == "streak":
        # poses 0.3 off, tau = 1e-8: the first Gauss-Newton steps overshoot (rejection streaks in iterations 1 and 4)
        return from_scene(synth.ba_scene(n_kf=6, n_pt=300, target_obs=1500, seed=14, pose_sigma=0.3), _fixed(6), tau=1e-8)
    if name.startswith("free"):
        # n free poses (the solver path: one lane for 1 and 2, a warp up to 4, the CTA in 6 x 6 blocks up to 11, the
        # scalar CTA factorisation above)
        n = int(name[4:])
        return from_scene(synth.ba_scene(n_kf=n + 1, n_pt=400, target_obs=400 * min(n + 1, 4), seed=20 + n), _fixed(n + 1))
    if name.startswith("unobserved"):
        # tau = 0 and n free key-frames, the last of which observes nothing: its block of the reduced system is exactly zero,
        # the factorisation fails, lambda stays 0 and every trial is rejected (key-frames 0 and 1 are fixed, and every
        # landmark keeps at least two observations, so that its own block stays invertible at lambda = 0)
        n = int(name[10:])
        sc = synth.ba_scene(n_kf=n + 2, n_pt=300, target_obs=300 * min(n + 2, 4), seed=30 + n)
        keep = sc["kf_idx"] != n + 1
        assert np.bincount(sc["pt_idx"][keep]).min() >= 2
        return dict(P0=_g2o(sc["poses_noisy"]), fixed=_fixed(n + 2, 0, 1), X0=sc["pts_noisy"], kf_idx=sc["kf_idx"][keep],
                    pt_idx=sc["pt_idx"][keep], px=sc["px"][keep], tau=0.0)
    if name == "axis":
        return from_scene(synth.ba_axis_scene(AXIS_DEPTHS, _axis_errors()), _fixed(2))
    if name == "still":
        # every error exactly zero: b = 0, the step is exactly zero, the trial's cost equals the current one (rho == 0)
        return from_scene(synth.ba_axis_scene(AXIS_DEPTHS, np.zeros((8, 2))), _fixed(2))
    if name == "duplicate":
        base = _ba("kf6")
        o = int(np.flatnonzero(base["kf_idx"] != 0)[0])    # an observation of a free key-frame, repeated
        return dict(base, kf_idx=np.r_[base["kf_idx"], base["kf_idx"][o]], pt_idx=np.r_[base["pt_idx"], base["pt_idx"][o]],
                    px=np.r_[base["px"], base["px"][o:o + 1]])
    raise KeyError(name)


@functools.lru_cache(maxsize=None)
def _oracle():
    from oracle.pyoracle import Oracle
    return Oracle()


def _kw(pb, **kw):
    out = dict(max_iters=20, huber=5.991, tau=pb.get("tau", 1e-5), max_trials=10, chi2_outlier=5.991)
    out.update(kw)
    return out


def _ora_ba(pb, **kw):
    """(poses, points, outlier flags, stats) of oracle/ba.cpp."""
    return _oracle().local_ba(pb["P0"], pb["fixed"], pb["X0"], pb["kf_idx"], pb["pt_idx"], pb["px"], **_kw(pb, **kw))


def _gpu_ba(ctx, pbs, **kw):
    """The problems in one ygzb_local_ba call: per problem (poses, points, outlier flags, stats)."""
    kf_off = np.cumsum([0] + [len(p["fixed"]) for p in pbs])
    pt_off = np.cumsum([0] + [len(p["X0"]) for p in pbs])
    obs_off = np.cumsum([0] + [len(p["kf_idx"]) for p in pbs])
    P, X, out, st = ctx.local_ba(kf_off, pt_off, obs_off, np.concatenate([p["P0"] for p in pbs]),
                                 np.concatenate([p["fixed"] for p in pbs]), np.concatenate([p["X0"] for p in pbs]),
                                 np.concatenate([p["kf_idx"] for p in pbs]), np.concatenate([p["pt_idx"] for p in pbs]),
                                 np.concatenate([p["px"] for p in pbs]), **_kw(pbs[0], **kw))
    return [(P[kf_off[i]:kf_off[i + 1]], X[pt_off[i]:pt_off[i + 1]], out[obs_off[i]:obs_off[i + 1]], st[i]) for i in range(len(pbs))]


def _rel(a, b):
    """Largest |a - b| / max(1, |b|) (absolute below 1)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(1.0, np.abs(b)), initial=0.0))


def ba_diff(res, want):
    """The largest difference of the numbers of one run (poses, points, chi2_initial, chi2_final, lambda_final; relative
    above 1, absolute below, and the three statistics relative) after asserting that its decisions (iterations, LM trials, outlier flags) are the oracle's."""
    P, X, out, st = res
    wP, wX, wout, wst = want
    assert (st["iters"], st["lm_trials"], st["n_outliers"]) == (wst["iters"], wst["lm_trials"], wst["n_outliers"]), (st, wst)
    assert np.array_equal(out, wout)
    return max(_rel(P, wP), _rel(X, wX), *(abs(st[k] - wst[k]) / max(abs(wst[k]), 1e-300) if wst[k] else abs(st[k])
                                          for k in ("chi2_initial", "chi2_final", "lambda_final")))


def _check_ba(res, want):
    d = ba_diff(res, want)
    assert d <= BA_TOL, d


TRUNCATION = (0, 1, 2, 3, 5, 8)
STREAK_TRIALS = (1, 2, 3, 4, 5, 6, 7, 10)    # max_trials on the streak scene at max_iters = 4


def test_ba_cases_reach_their_branch():
    """Oracle only: each constructed local-BA case takes the path it is built for."""
    for name in ("c4", "kf6"):
        for huber in (5.991, 0.0):
            for k in TRUNCATION:     # one accepted trial per iteration: the runs stop on max_iters
                st = _ora_ba(_ba(name), max_iters=k, huber=huber)[3]
                assert st["iters"] == st["lm_trials"] == k, (name, huber, k, st)
                assert (st["chi2_final"] == st["chi2_initial"]) == (k == 0)
    # the streaks: iteration 1 rejects two trials and accepts the third, iterations 2 and 3 take one trial, iteration 4
    # rejects six and accepts the seventh.  Each rejection multiplies lambda by ni = 2, 4, 8, ... and restores the state;
    # max_trials = q cuts a streak after q trials (qmax == max_trials ends the run, after an accepted trial too)
    pb = _ba("streak")
    P0, X0, _, st0 = _ora_ba(pb, max_iters=0)
    P3, X3, _, st3 = _ora_ba(pb, max_iters=3)
    assert (st3["iters"], st3["lm_trials"]) == (3, 5)
    for q in STREAK_TRIALS:
        P, X, _, st = _ora_ba(pb, max_iters=4, max_trials=q)
        grow = 2.0 ** (q * (q + 1) // 2)
        if q < 3:
            assert (st["iters"], st["lm_trials"]) == (1, q) and st["lambda_final"] == st0["lambda_final"] * grow, (q, st)
            assert st["chi2_final"] == st["chi2_initial"] and np.array_equal(P, P0) and np.array_equal(X, X0)
        elif q == 3:   # accepted after the grown lambda (x 8), scaled by the alpha cap 2/3
            assert (st["iters"], st["lm_trials"]) == (1, 3) and st["chi2_final"] < st["chi2_initial"], st
            assert st["lambda_final"] == pytest.approx(st0["lambda_final"] * 8 * 2 / 3, rel=1e-15)
        elif q < 7:
            assert (st["iters"], st["lm_trials"]) == (4, 5 + q) and st["lambda_final"] == st3["lambda_final"] * grow, (q, st)
            assert st["chi2_final"] == st3["chi2_final"] and np.array_equal(P, P3) and np.array_equal(X, X3)
        else:          # six rejections (lambda x 2^21), then the seventh trial is accepted
            assert (st["iters"], st["lm_trials"]) == (4, 12) and st["chi2_final"] < st3["chi2_final"], (q, st)
            grown = st3["lambda_final"] * 2.0 ** 21
            assert grown / 3 * (1 - 1e-15) <= st["lambda_final"] <= grown * 2 / 3 * (1 + 1e-15)
    # max_trials = 1: the first iteration ends the run even though its trial was accepted
    st = _ora_ba(_ba("kf6"), max_trials=1)[3]
    assert (st["iters"], st["lm_trials"]) == (1, 1) and st["chi2_final"] < st["chi2_initial"]
    # rho == 0: a zero step from a zero-cost state ends the run after one trial, the poses keep their bits
    P, X, _, st = _ora_ba(_ba("still"), max_iters=5)
    assert (st["iters"], st["lm_trials"]) == (1, 1) and st["chi2_initial"] == st["chi2_final"] == 0
    assert st["lambda_final"] == 2 * _ora_ba(_ba("still"), max_iters=0)[3]["lambda_final"] > 0
    assert np.array_equal(P, _ba("still")["P0"]) and np.array_equal(X, _ba("still")["X0"])
    # a failed factorisation: every trial rejected, lambda stays 0, nothing moves
    for n in (1, 2, 3, 6):
        pb = _ba(f"unobserved{n}")
        for q in (1, 3, 10):
            P, X, _, st = _ora_ba(pb, max_trials=q)
            assert (st["iters"], st["lm_trials"], st["lambda_final"]) == (1, q, 0.0), (n, q, st)
            assert st["chi2_final"] == st["chi2_initial"] > 0
            assert np.array_equal(P, pb["P0"]) and np.array_equal(X, pb["X0"])
    # max_iters = 0 reports the initial cost and lambda and returns the input
    pb = _ba("kf6")
    P, X, _, st = _ora_ba(pb, max_iters=0)
    assert st["chi2_initial"] == st["chi2_final"] == _ora_ba(pb, max_iters=1)[3]["chi2_initial"] > 0
    assert st["lambda_final"] == 1e-5 * _ora_ba(pb, max_iters=0, tau=1.0)[3]["lambda_final"] > 0
    assert np.array_equal(P, pb["P0"]) and np.array_equal(X, pb["X0"])


def test_ba_axis_scene_errors_are_exact():
    """Oracle only: the axis scene's errors are what it was built with, so the thresholds below sit where they are meant to
    be -- |e|^2 1e-9 above and below delta^2 and the outlier threshold, and exactly on it."""
    e = _axis_errors()
    e2 = (e ** 2).sum(1)
    assert e2[0] > DELTA2 > e2[1] and abs(e2[0] / DELTA2 - 1) < 2e-9 and abs(e2[1] / DELTA2 - 1) < 2e-9
    assert e2[2] == e2[3] and abs(e2[2] / 5.991 - 1) < 1e-8
    pb = _ba("axis")
    for thr, want in ((e2[2], (0, 0)), (e2[2] * (1 - 1e-9), (1, 1)), (e2[2] * (1 + 1e-9), (0, 0))):
        out = _ora_ba(pb, max_iters=0, chi2_outlier=thr)[2]
        assert tuple(out[2:4]) == want, thr
    st = _ora_ba(pb, max_iters=0, huber=5.991)[3]
    plain = _ora_ba(pb, max_iters=0, huber=0.0)[3]
    big = e2[e2 > DELTA2]
    assert np.isclose(plain["chi2_initial"] - st["chi2_initial"], (big - (2 * np.sqrt(big) * 5.991 - DELTA2)).sum(), rtol=1e-9, atol=0)
    # the near landmark's diagonal is the largest entry of diag H: it sets the initial lambda
    z = AXIS_DEPTHS[-1]
    fx = float(np.float32(synth.FX))
    assert st["lambda_final"] == pytest.approx(1e-5 * 2 * (fx / z) ** 2, rel=1e-3)


@gpu
@pytest.mark.parametrize("huber", [5.991, 0.0], ids=["huber", "plain"])
@pytest.mark.parametrize("k", TRUNCATION)
@pytest.mark.parametrize("name", ["c4", "kf6"])
def test_ba_truncated_runs(ctx3, name, k, huber):
    """After exactly k LM iterations: the oracle's iterations, trials and outlier flags, and its poses, points, costs and
    lambda within BA_TOL.  k = 0 reports the initial cost and lambda and returns the input bits.  Largest difference to the oracle measured on an H100 80GB HBM3 (700 W): 1.1e-13."""
    pb = _ba(name)
    (res,) = _gpu_ba(ctx3, [pb], max_iters=k, huber=huber)
    _check_ba(res, _ora_ba(pb, max_iters=k, huber=huber))
    if k == 0:
        assert np.array_equal(res[0], pb["P0"]) and np.array_equal(res[1], pb["X0"])


@gpu
@pytest.mark.parametrize("q", STREAK_TRIALS)
def test_ba_rejection_streak(ctx3, q):
    """Through the streaks of rejected trials and the accepted one after each (max_trials cuts a streak after q trials):
    the state restored, lambda grown by ni = 2, 4, 8, ..., and the accepted step taken from the grown lambda.  Largest difference to the oracle measured on an H100 80GB HBM3 (700 W): 1.2e-11."""
    pb = _ba("streak")
    (res,) = _gpu_ba(ctx3, [pb], max_iters=4, max_trials=q)
    _check_ba(res, _ora_ba(pb, max_iters=4, max_trials=q))


@gpu
@pytest.mark.parametrize("name", ["c4", "kf6"])
def test_ba_trial_limit_exit(ctx3, name):
    """max_trials = 1: qmax == max_trials ends the run after its first iteration, although that trial was accepted (the
    streak scene cuts runs at 2 to 7 trials).  Largest difference to the oracle measured on an H100 80GB HBM3 (700 W): 6.1e-14."""
    pb = _ba(name)
    (res,) = _gpu_ba(ctx3, [pb], max_trials=1)
    _check_ba(res, _ora_ba(pb, max_trials=1))
    assert res[3]["iters"] == 1


@gpu
def test_ba_rho_zero_exit(ctx3):
    """A zero step from a zero-cost state: rho = 0 / (0 + 1e-3) == 0 ends the run after one trial, lambda doubled, the
    input bits returned.  Largest difference to the oracle measured on an H100 80GB HBM3 (700 W): 0 (bit-identical)."""
    pb = _ba("still")
    (res,) = _gpu_ba(ctx3, [pb], max_iters=5)
    _check_ba(res, _ora_ba(pb, max_iters=5))
    assert res[3]["iters"] == 1 and np.array_equal(res[0], pb["P0"]) and np.array_equal(res[1], pb["X0"])


@gpu
@pytest.mark.parametrize("solver", ["0", "1"])
@pytest.mark.parametrize("n", [1, 2, 3, 6])
def test_ba_failed_factorisation(ctx3, n, solver, monkeypatch):
    """tau = 0 and a free key-frame without observations: the factorisation fails on every solver path (one lane for 1 and
    2 free poses, a warp for 3, the CTA for 6; YGZB_BA_SOLVER=1 the scalar LDL^T), the step of the free poses is zero,
    every trial is rejected and the input comes back bit for bit.  Largest difference to the oracle measured on an H100 80GB HBM3 (700 W): 9.1e-16."""
    monkeypatch.setenv("YGZB_BA_SOLVER", solver)
    pb = _ba(f"unobserved{n}")
    for q in (1, 3, 10):
        (res,) = _gpu_ba(ctx3, [pb], max_trials=q)
        _check_ba(res, _ora_ba(pb, max_trials=q))
        assert np.array_equal(res[0], pb["P0"]) and np.array_equal(res[1], pb["X0"])


@gpu
def test_ba_duplicate_observation_is_rejected(ctx3):
    from ygz_slam_b200 import YgzbError
    with pytest.raises(YgzbError, match="observed twice"):
        _gpu_ba(ctx3, [_ba("duplicate")], max_iters=0)


@gpu
@pytest.mark.parametrize("huber", [5.991, 0.0], ids=["huber", "plain"])
def test_ba_thresholds_at_max_iters_zero(ctx3, huber):
    """max_iters = 0 on the axis scene, whose errors are exact: the outlier flags at thresholds on |e|^2, 1e-9 above and
    below it (plain >, on the plain error, not the Huber cost), chi2_initial with |e|^2 1e-9 on either side of delta^2, and
    the initial lambda set by a landmark's diagonal.  Largest difference to the oracle measured on an H100 80GB HBM3 (700 W): 0 (bit-identical)."""
    pb = _ba("axis")
    e2 = (_axis_errors() ** 2).sum(1)
    for thr in (e2[2], e2[2] * (1 - 1e-9), e2[2] * (1 + 1e-9), DELTA2, DELTA2 * (1 - 1e-9), 1.0, 49.0):
        (res,) = _gpu_ba(ctx3, [pb], max_iters=0, huber=huber, chi2_outlier=thr)
        want = _ora_ba(pb, max_iters=0, huber=huber, chi2_outlier=thr)
        assert np.array_equal(res[2], e2 > thr)
        _check_ba(res, want)


@gpu
@pytest.mark.parametrize("n", [1, 2, 3, 9, 13])
def test_ba_solver_paths_truncated(ctx3, n, monkeypatch):
    """Every factorisation under truncation: one lane (6 and 12), the warp, the CTA in 6 x 6 blocks and the scalar CTA
    version, then YGZB_BA_SOLVER=1, each after 2 and 5 iterations.  Largest difference to the oracle measured on an H100 80GB HBM3 (700 W): 1.1e-13."""
    pb = _ba(f"free{n}")
    for solver in ("0", "1"):
        monkeypatch.setenv("YGZB_BA_SOLVER", solver)
        for k in (2, 5):
            (res,) = _gpu_ba(ctx3, [pb], max_iters=k)
            _check_ba(res, _ora_ba(pb, max_iters=k))


@gpu
@pytest.mark.parametrize("cluster", [1, 16])
def test_ba_cluster_sizes_and_batching(ctx3, cluster, monkeypatch):
    """YGZB_BA_CLUSTER at 1 and 16 under truncation, and a problem batched next to others is bit-identical to the same
    problem alone.  Largest difference to the oracle measured on an H100 80GB HBM3 (700 W): 2.2e-14."""
    monkeypatch.setenv("YGZB_BA_CLUSTER", str(cluster))
    pbs = [_ba("kf6"), _ba("c4"), _ba("free3")]
    batch = _gpu_ba(ctx3, pbs, max_iters=3)
    for pb, res in zip(pbs, batch):
        _check_ba(res, _ora_ba(pb, max_iters=3))
        (alone,) = _gpu_ba(ctx3, [pb], max_iters=3)
        for a, b in zip(res[:3], alone[:3]):
            assert np.array_equal(a, b)
        assert res[3] == alone[3]


# ---- sparse alignment ---------------------------------------------------------------------------------------------------
LEVELS = 3


@functools.lru_cache(maxsize=None)
def _align(name):
    """Sparse-alignment problems: dict(g1, g2 (ref / cur images), p1, p2 (oracle pyramids), px, depth, has, T_ref)."""
    o = _oracle()
    if name in ("stream", "stream2", "identical", "depth0"):
        k0, k1 = {"stream": (1, 4), "stream2": (2, 5), "identical": (1, 1), "depth0": (3, 6)}[name]
        g1, d1, T1 = synth.stream_frame(k0)
        g2, _, _ = synth.stream_frame(k1)
        p1 = o.build_pyramid(g1, LEVELS)
        f = o.detect(p1, n_levels=LEVELS)
        px = np.stack([f["px"], f["py"]], 1)
        depth = d1[f["py"].astype(int), f["px"].astype(int)]
        if name == "depth0":
            depth = depth.copy()
            depth[len(depth) // 2] = 0.0
        has = np.ones(len(depth), np.uint8)
        has[::11] = 0
        return dict(g1=g1, g2=g2, p1=p1, p2=o.build_pyramid(g2, LEVELS), px=px, depth=depth, has=has, T_ref=T1)
    if name == "flat":
        g = np.full((synth.H, synth.W), 128, np.uint8)
        base = _align("stream")
        p = o.build_pyramid(g, LEVELS)
        return dict(base, g1=g, g2=g, p1=p, p2=p)
    raise KeyError(name)


def _ora_align(s, **kw):
    """(T_cw, n_meas, iterations per level) of oracle/align.cpp with the kernel's chi2 accumulation."""
    kw = dict(dict(max_level=2, min_level=0, n_iter=30, eps=1e-6), **kw)
    return _oracle().sparse_align(s["p1"], s["p2"], synth.W, synth.H, LEVELS, s["px"], s["depth"], s["has"], s["T_ref"], s["T_ref"],
                                  exact=True, **kw)


def _gpu_align(ctx, probs, **kw):
    """The problems (scene, feature selection) in one ygzb_sparse_align call: per problem (T_cw, n_meas, iterations)."""
    kw = dict(dict(max_level=2, min_level=0, n_iter=30, eps=1e-6), **kw)
    fr = ctx.frames(2 * len(probs))
    try:
        fr.upload(np.stack([g for s, _ in probs for g in (s["g1"], s["g2"])]))
        sel = [np.arange(len(s["depth"]))[f] for s, f in probs]
        off = np.cumsum([0] + [len(i) for i in sel])
        T, nm, it = fr.sparse_align(2 * np.arange(len(probs)), 2 * np.arange(len(probs)) + 1, off,
                                    np.concatenate([s["px"][i] for (s, _), i in zip(probs, sel)]),
                                    np.concatenate([s["depth"][i] for (s, _), i in zip(probs, sel)]),
                                    np.concatenate([s["has"][i] for (s, _), i in zip(probs, sel)]),
                                    np.stack([s["T_ref"].reshape(-1) for s, _ in probs]), np.stack([s["T_ref"].reshape(-1) for s, _ in probs]),
                                    **kw)
    finally:
        fr.close()
    return [(T[p], int(nm[p]), it[p]) for p in range(len(probs))]


def _sub(s, f):
    return dict(s, px=s["px"][f], depth=s["depth"][f], has=s["has"][f])


def align_diff(res, want):
    """The pose difference of one run (|se3 log of T^-1 T_oracle|, absolute) after asserting that its measurement count and iterations per level are the oracle's."""
    T, nm, it = res
    wT, wn, wit = want
    assert nm == wn and np.array_equal(it, wit), (nm, wn, it, wit)
    return float(np.linalg.norm(se3.se3_log(se3.mul(se3.inv(T), wT))))


def _check_align(res, want):
    d = align_diff(res, want)
    assert d <= ALIGN_TOL, d


def test_align_cases_reach_their_branch():
    """Oracle only: the exits of the Gauss-Newton loop.  eps = 0 never converges on a nonzero step, so a level that stops
    early with eps = 0 stopped on a chi2 increase (rollback at it > 0); identical frames give an exactly zero step (the
    eps test at eps = 0); a flat texture has H = 0 (the LDL^T fails at it = 0: the pose is unchanged, 0 iterations
    everywhere); a feature of depth 0 puts NaN into H (rollback at it = 0)."""
    s = _align("stream")
    T, nm, it = _ora_align(s, eps=0.0)
    assert nm > 0 and ((it[:3] >= 1) & (it[:3] < 30)).all(), it
    T, _, it = _ora_align(_align("identical"), eps=0.0)     # converged at it = 0 on every level: nothing counted
    assert not it.any() and np.allclose(T, _align("identical")["T_ref"], rtol=0, atol=1e-12)
    _, _, it = _ora_align(_align("identical"), eps=-1.0, n_iter=5)   # (and not an LDL^T failure: without the eps exit it runs on)
    assert list(it[:3]) == [5, 5, 5]
    T, nm, it = _ora_align(_align("flat"))
    assert not it.any() and np.allclose(T, _align("flat")["T_ref"], rtol=0, atol=1e-12) and nm > 0
    T, nm, it = _ora_align(_align("depth0"))
    assert not it.any() and np.allclose(T, _align("depth0")["T_ref"], rtol=0, atol=1e-12)
    for n_iter in (1, 2, 3):
        for L in range(LEVELS):
            _, _, it = _ora_align(s, min_level=L, max_level=L, n_iter=n_iter, eps=0.0)
            assert it[L] == n_iter and it.sum() == n_iter, (n_iter, L, it)


@gpu
@pytest.mark.parametrize("n_iter", [1, 2, 3])
@pytest.mark.parametrize("level", [0, 1, 2])
def test_align_single_level_steps(ctx3, level, n_iter):
    """One pyramid level, n_iter Gauss-Newton steps, eps = 0: after one step the pose is T exp(-H^-1 b), so H itself is
    compared.  Patches and gradients are bit for bit the oracle's (align.cu is built without FMA contraction); only the
    summation order of H and b differs.  Largest difference to the oracle measured on an H100 80GB HBM3 (700 W): 2.5e-14."""
    for name in ("stream", "stream2"):
        s = _align(name)
        (res,) = _gpu_align(ctx3, [(s, slice(None))], min_level=level, max_level=level, n_iter=n_iter, eps=0.0)
        _check_align(res, _ora_align(s, min_level=level, max_level=level, n_iter=n_iter, eps=0.0))


@gpu
@pytest.mark.parametrize("eps", [1e-2, 1e-6, 0.0])
def test_align_iterations_per_level(ctx3, eps):
    """The whole coarse-to-fine run: iterations per level (convergence on eps, rollback on a chi2 increase at it > 0, whose
    chi2 comparison carries over from the previous level) and n_meas exactly, two problems in one batch.  Largest difference to the oracle measured on an H100 80GB HBM3 (700 W): 2.1e-14."""
    probs = [(_align("stream"), slice(None)), (_align("stream2"), slice(None))]
    for (s, _), res in zip(probs, _gpu_align(ctx3, probs, eps=eps)):
        _check_align(res, _ora_align(s, eps=eps))


@gpu
@pytest.mark.parametrize("cluster", [1, 2, 4, 8])
def test_align_exits(ctx3, cluster, monkeypatch):
    """In one batch, at 1, 2, 4 and 8 CTAs per problem: identical frames (an exactly zero step converges at eps = 0 at
    it = 0 on every level), a flat texture (LDL^T failure at it = 0), a feature of depth 0 (NaN: rollback at it = 0) next to
    the stream scene, which the NaN neighbour does not disturb, and n_iter = 0 (nothing runs).  Largest difference to the oracle measured on an H100 80GB HBM3 (700 W): 2.0e-14."""
    monkeypatch.setenv("YGZB_TRACK_CLUSTER", str(cluster))
    names = ["identical", "flat", "depth0", "stream"]
    probs = [(_align(n), slice(None)) for n in names]
    for name, res in zip(names, _gpu_align(ctx3, probs, eps=0.0)):
        _check_align(res, _ora_align(_align(name), eps=0.0))
    for name, res in zip(names, _gpu_align(ctx3, probs, n_iter=0)):
        want = _ora_align(_align(name), n_iter=0)
        _check_align(res, want)
        assert np.allclose(res[0], _align(name)["T_ref"], rtol=0, atol=1e-12) and res[1] == 0


@gpu
@pytest.mark.parametrize("cluster", [1, 2, 4, 8])
def test_align_cluster_sizes(ctx3, cluster, monkeypatch):
    """YGZB_TRACK_CLUSTER at 1, 2, 4 and 8, against the oracle and bit-identical across two calls: one batch of problems
    of 1 and 4 to 7 features spread over the frame (fewer than the CTAs: some ranks own none; the first one has no map
    point, so H = 0), compared after one step at level 0, and one batch with a 700-feature problem (at one CTA more than
    shared memory holds: the global staging path) next to the whole stream scene, run to the end.  (Two or three
    features with map points leave H near-singular, and then rounding alone sets the step; later steps of a handful of
    features meet chi2 ties.)  Largest difference to the oracle measured on an H100 80GB HBM3 (700 W): 6.0e-12 (one step of 3 to 6 features), 2.1e-14 (whole runs)."""
    monkeypatch.setenv("YGZB_TRACK_CLUSTER", str(cluster))
    s = _align("stream")
    few = [(s, np.linspace(0, len(s["depth"]) - 1, n).astype(int)) for n in (1, 4, 5, 6, 7)]
    many = [(s, slice(0, 700)), (s, slice(None))]
    step = dict(min_level=0, max_level=0, n_iter=1, eps=0.0)
    for probs, kw, tol in ((few, step, FEW_TOL), (many, {}, ALIGN_TOL)):
        first = _gpu_align(ctx3, probs, **kw)
        for (sc, f), res in zip(probs, first):
            d = align_diff(res, _ora_align(_sub(sc, f), **kw))
            assert d <= tol, d
        second = _gpu_align(ctx3, probs, **kw)
        for a, b in zip(first, second):
            assert np.array_equal(a[0], b[0]) and a[1] == b[1] and np.array_equal(a[2], b[2])
