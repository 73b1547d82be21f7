"""The standalone patch-alignment entry points -- ygzb_align2d (cvutils::Align2D), ygzb_align1d (cvutils::Align1D) and
ygzb_project_align (Matcher::FindDirectProjection) -- bit for bit against the oracle on the parameters test_gpu_align.py
leaves alone: an explicit reference patch, 0 / 1 / 50 iterations, start points on the right and bottom edges, every level
of an 8-level pyramid (including levels smaller than a patch), mixed slots, flat templates, Align1D's chi^2 rollback,
zero and non-unit directions, per-item poses, reference levels 1 and 2, search levels at their cap, warps leaving the
reference image, predicted pixels on the InFrame border and zero depth.

Outputs that are NaN (singular Hessians, zero depth) are compared by position: the device's canonical NaN and the host's
default NaN differ in their bits."""
from types import SimpleNamespace

import numpy as np
import pytest

from oracle.pyoracle import Camera
from ygz_slam_b200 import se3, synth

FRAMES = (1, 4, 2)   # slot 0: reference frame; slots 1 and 2: search frames


def _same(got, want):
    """Equal bit for bit, NaN by position."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want))
    m = ~np.isnan(want)
    assert np.array_equal(got[m].view(np.int64), want[m].view(np.int64))


def _setup(ctx, oracle):
    imgs = [synth.stream_frame(k)[0] for k in FRAMES]
    pyrs = [oracle.build_pyramid(g, ctx.n_levels) for g in imgs]
    fr = ctx.frames(len(imgs))
    fr.upload(np.stack(imgs))
    view = lambda s, L: oracle.level_view(pyrs[s], 640, 480, ctx.n_levels, L)
    return fr, view


def _items(ctx, view, n, seed, one_d=False):
    """Templates cut from the reference frame (random bytes on levels too small to cut from), 1 in 13 of them flat; an
    explicit reference patch that differs from the template's interior; search slots 1 and 2; start points near the
    template's position or on the right / bottom edges: u_r = w - 5 (the last start the window allows) and w - 4 (breaks
    at once), with and without a fraction."""
    rng = np.random.default_rng(seed)
    L = rng.integers(0, ctx.n_levels, n).astype(np.uint8)
    slot = rng.integers(1, 3, n).astype(np.int32)
    rb = np.empty((n, 100), np.uint8)
    uv = np.empty((n, 2))
    for i in range(n):
        img = view(0, int(L[i]))
        h, w = img.shape
        if w >= 12 and h >= 12:
            x, y = int(rng.integers(6, w - 6)), int(rng.integers(6, h - 6))
            rb[i] = img[y - 5:y + 5, x - 5:x + 5].reshape(-1)
        else:
            x, y = rng.uniform(0, w), rng.uniform(0, h)
            rb[i] = rng.integers(0, 256, 100)
        uv[i] = x + rng.uniform(-2.5, 2.5), y + rng.uniform(-2.5, 2.5)
        kind = i % 7
        frac = 0.0 if i % 3 == 0 else rng.uniform(0, 1)
        if kind == 1:
            uv[i, 0] = w - 5 + frac
        elif kind == 2:
            uv[i, 0] = w - 4 + frac
        elif kind == 3:
            uv[i, 1] = h - 5 + frac
        elif kind == 4:
            uv[i, 1] = h - 4 + frac
    rb[::13] = rng.integers(0, 256, (len(rb[::13]), 1))      # flat: singular Hessian, NaN update
    ref = rb.reshape(n, 10, 10)[:, 1:9, 1:9].reshape(n, 64).astype(np.int32)
    ref = np.clip(ref + rng.integers(-25, 26, ref.shape), 0, 255).astype(np.uint8)
    out = dict(level=L, slot=slot, rb=rb, ref=ref, uv=uv)
    if one_d:
        ang = rng.uniform(0, 2 * np.pi, n)
        d = np.stack([np.cos(ang), np.sin(ang)], 1)
        d[1::5] = [1, 0]                                               # horizontal: v moves only on a rollback
        d[2::5] = d[2::5] * rng.choice([0.3, 2.5], (len(d[2::5]), 1))  # non-unit
        d[3::10] = [0, 1]
        d[4::17] = 0                                                   # zero direction: h_inv infinite
        out["dir"] = d.astype(np.float32)
    return out


@pytest.fixture(scope="module", params=[3, 8], ids=["3-levels", "8-levels"])
def setup(request, ctx3, ctx8, oracle):
    ctx = ctx3 if request.param == 3 else ctx8
    fr, view = _setup(ctx, oracle)
    yield ctx, fr, view
    fr.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_iter", [0, 1, 10, 50])
@pytest.mark.parametrize("explicit_ref", [True, False], ids=["ref", "no-ref"])
def test_gpu_align2d_edges(setup, oracle, n_iter, explicit_ref):
    ctx, fr, view = setup
    it = _items(ctx, view, 700, 100 + n_iter)
    ref = it["ref"] if explicit_ref else None
    got_uv, got_ok = fr.align2d(it["slot"], it["level"], it["rb"], ref, it["uv"], n_iter)
    for i in range(len(got_ok)):
        rb = it["rb"][i].reshape(10, 10)
        r = it["ref"][i].reshape(8, 8) if explicit_ref else rb[1:9, 1:9]
        ok, u, v = oracle.align2d(view(int(it["slot"][i]), int(it["level"][i])), rb, r, it["uv"][i, 0], it["uv"][i, 1], n_iter)
        assert ok == got_ok[i], i
        _same(got_uv[i], [u, v])
    if n_iter == 0:
        assert not got_ok.any() and np.array_equal(got_uv, it["uv"].astype(np.float32).astype(np.float64))
    if n_iter >= 10:
        assert got_ok.sum() > 50 and np.isnan(got_uv).any()


@pytest.mark.gpu
@pytest.mark.parametrize("n_iter", [0, 1, 10, 50])
@pytest.mark.parametrize("explicit_ref", [True, False], ids=["ref", "no-ref"])
def test_gpu_align1d_edges(setup, oracle, n_iter, explicit_ref):
    ctx, fr, view = setup
    it = _items(ctx, view, 700, 200 + n_iter, one_d=True)
    ref = it["ref"] if explicit_ref else None
    got_uv, got_ok, got_h = fr.align1d(it["slot"], it["level"], it["dir"], it["rb"], ref, it["uv"], n_iter)
    for i in range(len(got_ok)):
        rb = it["rb"][i].reshape(10, 10)
        r = it["ref"][i].reshape(8, 8) if explicit_ref else rb[1:9, 1:9]
        ok, u, v, hinv = oracle.align1d(view(int(it["slot"][i]), int(it["level"][i])), float(it["dir"][i, 0]), float(it["dir"][i, 1]),
                                        rb, r, it["uv"][i, 0], it["uv"][i, 1], n_iter)
        assert ok == got_ok[i], i
        _same(got_uv[i], [u, v])
        _same(got_h[i], hinv)
    assert np.isinf(got_h).any()


def test_align1d_rollback_is_reached(oracle):
    """With a horizontal direction an Align1D step never moves v; only the chi^2 rollback (`new_chi2 > chi2` after the
    first iteration) does, as it subtracts the mean-difference update from v.  The constructed items reach it."""
    imgs = [synth.stream_frame(k)[0] for k in FRAMES]
    pyrs = [oracle.build_pyramid(g, 3) for g in imgs]

    it = _items(SimpleNamespace(n_levels=3), lambda s, L: oracle.level_view(pyrs[s], 640, 480, 3, L), 700, 250, one_d=True)
    rolled = 0
    for i in range(1, 700, 5):
        rb = it["rb"][i].reshape(10, 10)
        img = oracle.level_view(pyrs[int(it["slot"][i])], 640, 480, 3, int(it["level"][i]))
        _, u, v, _ = oracle.align1d(img, 1.0, 0.0, rb, it["ref"][i].reshape(8, 8), it["uv"][i, 0], it["uv"][i, 1], 50)
        rolled += not np.isnan(v) and v != float(np.float32(it["uv"][i, 1]))
    assert rolled >= 10, rolled


def _proj_items(ctx, seed):
    """Candidates over several poses and slots: reference levels 0..2, random pixels with their rendered depth, points
    close to the principal point seen by a camera moved to 1/200 of their depth (the search level reaches its cap),
    reference pixels within a few pixels of the image border (the warp samples outside the reference level: zero fill),
    zero and negative depths."""
    rng = np.random.default_rng(seed)
    _, d0, T0 = synth.stream_frame(FRAMES[0])
    Ts = [T0] + [synth.stream_frame(k)[2] for k in FRAMES[1:]]
    n = 600
    ref_px = np.stack([rng.uniform(12, 628, n), rng.uniform(12, 468, n)], 1)
    kind = np.arange(n) % 6
    near = kind == 1
    ref_px[near] = [synth.CX, synth.CY] + rng.uniform(-1, 1, (near.sum(), 2))
    edge = kind == 2
    ref_px[edge] = np.where(rng.random((edge.sum(), 2)) < 0.5, rng.uniform(0, 4, (edge.sum(), 2)),
                            [636, 476] + rng.uniform(0, 3.9, (edge.sum(), 2)))
    depth = d0[ref_px[:, 1].astype(int), ref_px[:, 0].astype(int)].astype(np.float64)
    depth[kind == 3] = 0.0
    depth[(kind == 4) & (np.arange(n) % 4 == 0)] = -1.0
    level = rng.integers(0, 3, n).astype(np.uint8)
    cur_slot = rng.integers(1, 3, n).astype(np.int32)
    # poses 0..2: the reference camera at the origin and the search frames relative to it; 3..5: the same frames'
    # world poses, which the reference transforms with its world / ref-camera mix-up; then one pose per zoomed point
    poses = [np.eye(4)[:3]] + [se3.mul(T, se3.inv(T0)) for T in Ts[1:]] + Ts
    ref_pose = np.zeros(n, np.int32)
    cur_pose = cur_slot.copy()
    ref_pose[kind == 5] = 3
    cur_pose[kind == 5] += 3
    for i in np.nonzero(near)[0]:                 # own pose: moved forward to 1/200 of the point's depth
        Tz = np.eye(4)[:3].copy()
        Tz[2, 3] -= depth[i] * (1 - 1 / 200)
        poses.append(Tz)
        cur_pose[i] = len(poses) - 1
    poses = [T.reshape(-1) for T in poses]
    Xc = np.stack([(ref_px[:, 0] - synth.CX) * depth / synth.FX, (ref_px[:, 1] - synth.CY) * depth / synth.FY, depth], 1)
    P = np.stack(poses).reshape(-1, 3, 4)
    Xw = np.einsum("nji,nj->ni", P[ref_pose][:, :, :3], Xc - P[ref_pose][:, :, 3])
    Xn = np.einsum("nij,nj->ni", P[cur_pose][:, :, :3], Xw) + P[cur_pose][:, :, 3]
    with np.errstate(all="ignore"):
        cur_px = np.stack([synth.FX * Xn[:, 0] / Xn[:, 2] + synth.CX, synth.FY * Xn[:, 1] / Xn[:, 2] + synth.CY], 1)
    cur_px = np.where(np.isfinite(cur_px), cur_px, 320.0) + rng.uniform(-2, 2, (n, 2))
    return dict(ref_slot=np.zeros(n, np.int32), cur_slot=cur_slot, poses=np.stack(poses), ref_pose=ref_pose, cur_pose=cur_pose,
                ref_px=ref_px, depth=depth, level=level, cur_px=cur_px)


def _oracle_project(oracle, pyr, n_levels, it, cam=None):
    out_px, out_lvl, out_ok = np.empty_like(it["cur_px"]), np.empty(len(it["depth"]), np.int32), np.empty(len(it["depth"]), bool)
    for i in range(len(it["depth"])):
        s = slice(i, i + 1)
        px, lvl, ok = oracle.find_direct_projection(pyr[int(it["ref_slot"][i])], pyr[int(it["cur_slot"][i])], 640, 480, n_levels,
                                                    it["poses"][it["ref_pose"][i]].reshape(3, 4), it["poses"][it["cur_pose"][i]].reshape(3, 4),
                                                    it["ref_px"][s], it["depth"][s], it["level"][s].astype(np.int32), it["cur_px"][s], cam=cam)
        out_px[i], out_lvl[i], out_ok[i] = px[0], lvl[0], ok[0]
    return out_px, out_lvl, out_ok


@pytest.mark.gpu
def test_gpu_project_align_edges(setup, oracle):
    ctx, fr, _ = setup
    it = _proj_items(ctx, 300 + ctx.n_levels)
    got_px, got_lvl, got_ok = fr.project_align(it["ref_slot"], it["cur_slot"], it["poses"], it["ref_pose"], it["cur_pose"], it["ref_px"],
                                               it["depth"], it["level"], it["cur_px"])
    pyrs = [oracle.build_pyramid(synth.stream_frame(k)[0], ctx.n_levels) for k in FRAMES]
    want_px, want_lvl, want_ok = _oracle_project(oracle, pyrs, ctx.n_levels, it)
    assert np.array_equal(got_lvl, want_lvl)
    assert np.array_equal(got_ok, want_ok)
    _same(got_px, want_px)
    near = np.arange(len(got_ok)) % 6 == 1
    assert (got_lvl[near] == ctx.n_levels - 1).mean() > 0.9          # the search level stops at its cap
    assert got_ok.sum() > 50


def _border_items():
    """Unit camera (fx = fy = 1, cx = cy = 0) and identity poses: the warp is exactly the identity and the template exactly
    the image around the reference pixel.  Searching the same image from the same integer pixel converges at once onto
    it, so the aligned pixel is exactly the predicted one: 10 and W - 10 / H - 10 themselves, the doubles either side
    (which round to the same float), and the floats either side."""
    ref, cur = [], []
    for b, axis in ((10.0, 0), (630.0, 0), (10.0, 1), (470.0, 1)):
        for x in (b, np.nextafter(b, -np.inf), np.nextafter(b, np.inf), float(np.nextafter(np.float32(b), np.float32(0))),
                  float(np.nextafter(np.float32(b), np.float32(1e9)))):
            ref.append((b, 200.0) if axis == 0 else (300.0, b))
            cur.append((x, 200.0) if axis == 0 else (300.0, x))
    n = len(ref)
    return dict(ref_slot=np.zeros(n, np.int32), cur_slot=np.zeros(n, np.int32), poses=np.eye(4)[:3].reshape(1, 12), ref_pose=np.zeros(n, np.int32),
                cur_pose=np.zeros(n, np.int32), ref_px=np.array(ref), depth=np.ones(n), level=np.zeros(n, np.uint8), cur_px=np.array(cur))


UNIT_CAM = (1.0, 1.0, 0.0, 0.0)


def test_inframe_border_cases_are_exact(oracle):
    pyr = [oracle.build_pyramid(synth.stream_frame(FRAMES[0])[0], 3)]
    it = _border_items()
    px, lvl, ok = _oracle_project(oracle, pyr, 3, it, cam=Camera(*UNIT_CAM))
    exact = [k for k in range(len(ok)) if k % 5 < 3]          # the value itself and its double neighbours
    assert np.array_equal(px[exact], it["cur_px"][exact].astype(np.float32).astype(np.float64))
    assert list(ok[exact]) == [True] * 3 + [False] * 3 + [True] * 3 + [False] * 3


@pytest.mark.gpu
def test_gpu_project_align_on_the_inframe_border(oracle):
    from ygz_slam_b200 import Context
    ctx = Context(0, **dict(zip(("fx", "fy", "cx", "cy"), UNIT_CAM)))
    try:
        fr = ctx.frames(1)
        g = synth.stream_frame(FRAMES[0])[0]
        fr.upload(g[None])
        it = _border_items()
        got = fr.project_align(it["ref_slot"], it["cur_slot"], it["poses"], it["ref_pose"], it["cur_pose"], it["ref_px"], it["depth"],
                               it["level"], it["cur_px"])
        want = _oracle_project(oracle, [oracle.build_pyramid(g, 3)], 3, it, cam=Camera(*UNIT_CAM))
        _same(got[0], want[0])
        assert np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
        fr.close()
    finally:
        ctx.close()
