"""Seeded synthetic inputs for the ygz-slam hot path (SURVEY.md 8d).

No dataset ships with the reference (its tests need a TUM sequence, test/test_orb_match.cpp:36-49),
so every test and the benchmark run on these deterministic, numpy-only generators:

* `texture`     : a large procedural grey texture (value noise octaves + random rectangles/discs)
                  that gives FAST plenty of corners.
* `render_plane`: perspective render of that texture lying on a world plane seen from a pinhole
                  camera T_cw (default.yaml intrinsics, config/default.yaml:32-35), with the
                  per-pixel ground-truth depth -- the stand-in for a 640x480 TUM frame.
* `trajectory`  : the smooth camera path of SURVEY.md 8d.
* `ba_scene`    : keyframes x landmarks x observations with the noise recipe of
                  test/test_local_ba.cpp:49-98.

Everything is a pure function of the seed; images are uint8, B=G=R (so BGR2GRAY is the identity).
"""
from __future__ import annotations

import numpy as np

FX, FY, CX, CY = 520.9, 521.0, 325.1, 249.7  # config/default.yaml:32-35 (TUM fr2)
W, H = 640, 480


def texture(seed: int = 0x59475A00, size: int = 2048) -> np.ndarray:
    """size x size uint8 texture: 3 octaves of value noise + hard-edged shapes."""
    rng = np.random.default_rng(seed)
    img = np.zeros((size, size), np.float32)
    for octave, amp in ((16, 40.0), (64, 30.0), (256, 20.0)):
        n = size // octave + 2
        g = rng.random((n, n), dtype=np.float32)
        # bilinear upsample of the coarse grid
        yy = np.arange(size, dtype=np.float32) / octave
        y0 = yy.astype(np.int32)
        fy = (yy - y0)[:, None]
        x0 = y0
        fx = fy.T
        a = g[y0][:, x0]
        b = g[y0][:, x0 + 1]
        c = g[y0 + 1][:, x0]
        d = g[y0 + 1][:, x0 + 1]
        img += amp * ((1 - fy) * ((1 - fx) * a + fx * b) + fy * ((1 - fx) * c + fx * d))
    n_shapes = int(4000 * (size / 4096.0) ** 2 * 4)
    xs = rng.integers(0, size, n_shapes)
    ys = rng.integers(0, size, n_shapes)
    ws = rng.integers(6, 48, n_shapes)
    hs = rng.integers(6, 48, n_shapes)
    vals = rng.integers(0, 256, n_shapes)
    kinds = rng.integers(0, 2, n_shapes)
    for x, y, w, h, v, k in zip(xs, ys, ws, hs, vals, kinds):
        if k == 0:
            img[y:y + h, x:x + w] = v
        else:
            r = w // 2
            y0, y1 = max(0, y - r), min(size, y + r + 1)
            x0, x1 = max(0, x - r), min(size, x + r + 1)
            yy, xx = np.ogrid[y0:y1, x0:x1]
            m = (yy - y) ** 2 + (xx - x) ** 2 <= r * r
            img[y0:y1, x0:x1][m] = v
    return np.clip(img, 0, 255).astype(np.uint8)


def so3_exp(w: np.ndarray) -> np.ndarray:
    th = float(np.linalg.norm(w))
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]], np.float64)
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th**2 * (K @ K)


def trajectory(k: int) -> np.ndarray:
    """T_cw(k) as 3x4 [R|t] (SURVEY.md 8d stream definition)."""
    t = 0.10 * np.array([np.sin(2 * np.pi * k / 150), 0.5 * np.sin(2 * np.pi * k / 90), 0.2 * k / 300])
    w = 0.05 * np.array([np.sin(2 * np.pi * k / 200), np.cos(2 * np.pi * k / 170), 0.0])
    T = np.zeros((3, 4))
    T[:, :3] = so3_exp(w)
    T[:, 3] = t
    return T


def render_plane(tex: np.ndarray, T_cw: np.ndarray, plane_z: float = 2.0, metres_per_texel: float = 0.0025,
                 noise_sigma: float = 0.0, seed: int = 1, w: int = W, h: int = H, cx: float = CX, cy: float = CY):
    """Render the texture lying on the world plane z = plane_z.  Returns (gray uint8 HxW, depth f64 HxW)."""
    R, t = T_cw[:, :3], T_cw[:, 3]
    u, v = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    # ray in camera frame, then world: X_w = R^T (d * ray - t); solve X_w.z = plane_z
    ray = np.stack([(u - cx) / FX, (v - cy) / FY, np.ones_like(u)], -1)  # h,w,3
    rw = ray @ R  # R^T ray
    cw = -R.T @ t
    d = (plane_z - cw[2]) / rw[..., 2]
    Xw = cw + d[..., None] * rw
    size = tex.shape[0]
    tx = Xw[..., 0] / metres_per_texel + size / 2
    ty = Xw[..., 1] / metres_per_texel + size / 2
    tx = np.clip(tx, 0, size - 1.001)
    ty = np.clip(ty, 0, size - 1.001)
    x0 = tx.astype(np.int32)
    y0 = ty.astype(np.int32)
    fx = tx - x0
    fy = ty - y0
    tf = tex.astype(np.float64)
    val = ((1 - fy) * ((1 - fx) * tf[y0, x0] + fx * tf[y0, x0 + 1]) +
           fy * ((1 - fx) * tf[y0 + 1, x0] + fx * tf[y0 + 1, x0 + 1]))
    if noise_sigma > 0:
        val = val + np.random.default_rng(seed).normal(0, noise_sigma, val.shape)
    gray = np.clip(np.rint(val), 0, 255).astype(np.uint8)
    return gray, d  # depth along the optical axis (ray z component is 1)


def undistort_rays(u, v, dist, fx: float = FX, fy: float = FY, cx: float = CX, cy: float = CY, iters: int = 30):
    """Normalised rays (x, y) whose radial-tangential projection (k1, k2, p1, p2, k3) through K is the pixel (u, v):
    fixed-point iteration x = (xd - tangential(x, y)) / radial(x, y), as cv::undistortPoints does."""
    k1, k2, p1, p2, k3 = (tuple(dist) + (0.0,) * 5)[:5]
    xd, yd = (u - cx) / fx, (v - cy) / fy
    x, y = xd.copy(), yd.copy()
    for _ in range(iters):
        r2 = x * x + y * y
        kr = 1 + ((k3 * r2 + k2) * r2 + k1) * r2
        x = (xd - (2 * p1 * x * y + p2 * (r2 + 2 * x * x))) / kr
        y = (yd - (p1 * (r2 + 2 * y * y) + 2 * p2 * x * y)) / kr
    return x, y


def render_plane_lens(tex: np.ndarray, T_cw: np.ndarray, dist, plane_z: float = 2.0, metres_per_texel: float = 0.0025,
                      noise_sigma: float = 0.0, seed: int = 1):
    """render_plane through a lens: the camera K = (FX, FY, CX, CY) with radial-tangential distortion dist = (k1, k2, p1, p2[,
    k3]).  Every distorted pixel is undistorted iteratively to its ray, the ray is intersected with the plane z = plane_z and
    the texture is sampled there.  Returns (raw distorted gray uint8 HxW, depth HxW of the UNDISTORTED pinhole camera with
    the same K -- the depth map a tracker wants once its frame pool undistorts with newK = K)."""
    R, t = T_cw[:, :3], T_cw[:, 3]
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    x, y = undistort_rays(u, v, dist)
    cw = -R.T @ t

    def hit(rx, ry):
        rw = np.stack([rx, ry, np.ones_like(rx)], -1) @ R
        d = (plane_z - cw[2]) / rw[..., 2]
        return cw + d[..., None] * rw, d

    Xw, _ = hit(x, y)
    size = tex.shape[0]
    tx = np.clip(Xw[..., 0] / metres_per_texel + size / 2, 0, size - 1.001)
    ty = np.clip(Xw[..., 1] / metres_per_texel + size / 2, 0, size - 1.001)
    x0, y0 = tx.astype(np.int32), ty.astype(np.int32)
    fx, fy = tx - x0, ty - y0
    tf = tex.astype(np.float64)
    val = ((1 - fy) * ((1 - fx) * tf[y0, x0] + fx * tf[y0, x0 + 1]) + fy * ((1 - fx) * tf[y0 + 1, x0] + fx * tf[y0 + 1, x0 + 1]))
    if noise_sigma > 0:
        val = val + np.random.default_rng(seed).normal(0, noise_sigma, val.shape)
    gray = np.clip(np.rint(val), 0, 255).astype(np.uint8)
    _, depth = hit((u - CX) / FX, (v - CY) / FY)
    return gray, depth


# TUM fr2's coefficients (k1, k2, p1, p2, k3): the lens of the lens-rendered streams
LENS_TUM_FR2 = (0.2312, -0.7849, -0.0033, -0.0001, 0.9172)


def lens_stream_frame(k: int, stream: int = 0, dist=LENS_TUM_FR2, noise_sigma: float = 2.0, tex_size: int = 2048):
    """Frame k of synthetic stream `stream` (the trajectory of stream_frame) seen through the lens `dist`: (raw distorted
    gray, depth of the undistorted camera, T_cw)."""
    key = (stream, tex_size)
    if key not in _TEX_CACHE:
        _TEX_CACHE[key] = texture(0x59475A00 + stream, tex_size)
    T = trajectory(k)
    gray, depth = render_plane_lens(_TEX_CACHE[key], T, dist, noise_sigma=noise_sigma, seed=(stream << 16) + k + 1)
    return gray, depth, T


_TEX_CACHE: dict = {}


def stream_frame(k: int, stream: int = 0, noise_sigma: float = 2.0, tex_size: int = 2048):
    """Frame k of synthetic stream `stream`: (gray, depth, T_cw)."""
    key = (stream, tex_size)
    if key not in _TEX_CACHE:
        _TEX_CACHE[key] = texture(0x59475A00 + stream, tex_size)
    T = trajectory(k)
    gray, depth = render_plane(_TEX_CACHE[key], T, noise_sigma=noise_sigma, seed=(stream << 16) + k + 1)
    return gray, depth, T


def shifted_pair(w: int, h: int, dx: int, dy: int, seed: int = 0, noise: int = 2):
    """Two w x h crops of the stream-0 texture: what is at (x, y) in the first is at (x + dx, y + dy) in the second.
    Each crop gets its own seeded integer noise in [-noise, noise].  For optical flow with a known answer."""
    key = (0, 2048)
    if key not in _TEX_CACHE:
        _TEX_CACHE[key] = texture(0x59475A00, 2048)
    tex = _TEX_CACHE[key]
    x0 = y0 = 128
    n = tex.shape[0]
    if not (0 <= x0 - dx and max(x0, x0 - dx) + w <= n and 0 <= y0 - dy and max(y0, y0 - dy) + h <= n):
        raise ValueError("crop outside the texture")
    rng = np.random.default_rng(seed)
    out = []
    for ys, xs in ((y0, x0), (y0 - dy, x0 - dx)):
        g = tex[ys:ys + h, xs:xs + w].astype(np.int16) + rng.integers(-noise, noise + 1, (h, w))
        out.append(np.clip(g, 0, 255).astype(np.uint8))
    return out[0], out[1]


def to_bgr(gray: np.ndarray) -> np.ndarray:
    return np.repeat(gray[..., None], 3, axis=-1).copy()


def ba_scene(n_kf: int = 10, n_pt: int = 2000, target_obs: int = 8000, seed: int = 11,
             pose_sigma: float = 0.1, point_sigma: float = 0.1, pixel_sigma: float = 1.0):
    """Local-BA problem in the shape of BASELINE config C4, noise recipe of test/test_local_ba.cpp:49-98.

    Returns dict with true/noisy poses (se3 [upsilon; omega] and g2o order [omega; upsilon]), points,
    observations (kf_idx, pt_idx, px)."""
    from .se3 import se3_exp, se3_log  # local import: pure-numpy helpers
    rng = np.random.default_rng(seed)
    poses_true = []
    for i in range(n_kf):
        T = trajectory(15 * i)
        poses_true.append(se3_log(T))
    poses_true = np.array(poses_true)
    # landmarks on the two planes z=2 (75 %) and z=4 (25 %), inside the field of view of pose 0
    z = np.where(rng.random(n_pt) < 0.75, 2.0, 4.0)
    u = rng.uniform(20, W - 20, n_pt)
    v = rng.uniform(20, H - 20, n_pt)
    pts_true = np.stack([(u - CX) / FX * z, (v - CY) / FY * z, z], 1)
    kf_idx, pt_idx, px = [], [], []
    per_pt = max(2, int(round(target_obs / n_pt)))
    for j in range(n_pt):
        kfs = rng.choice(n_kf, size=min(per_pt, n_kf), replace=False)
        for k in sorted(kfs):
            T = se3_exp(poses_true[k])
            pc = T[:, :3] @ pts_true[j] + T[:, 3]
            if pc[2] <= 0.1:
                continue
            uu = FX * pc[0] / pc[2] + CX
            vv = FY * pc[1] / pc[2] + CY
            kf_idx.append(k)
            pt_idx.append(j)
            px.append([uu + rng.normal(0, pixel_sigma), vv + rng.normal(0, pixel_sigma)])
    poses_noisy = poses_true.copy()
    poses_noisy[1:] += rng.normal(0, pose_sigma, (n_kf - 1, 6))
    pts_noisy = pts_true + rng.normal(0, point_sigma, pts_true.shape)
    return dict(poses_true=poses_true, poses_noisy=poses_noisy, pts_true=pts_true, pts_noisy=pts_noisy,
                kf_idx=np.array(kf_idx, np.int32), pt_idx=np.array(pt_idx, np.int32),
                px=np.array(px, np.float64))


def ba_axis_scene(depths, errors):
    """Local-BA problem whose reprojection errors are exact: two key-frames at the identity pose (0 fixed, 1 free) and one
    landmark per depth on the optical axis, seen by both.  A point on the axis projects to (cx, cy) exactly in any
    arithmetic, so observation o, at (cx + errors[o, 0], cy + errors[o, 1]), has exactly that error when the errors lie on
    a 2^-30 grid.  Observations alternate key-frames 0 and 1 per landmark.  Returns ba_scene's keys."""
    depths = np.asarray(depths, np.float64)
    errors = np.asarray(errors, np.float64).reshape(2 * len(depths), 2)
    assert np.array_equal(errors, np.round(errors * 2.0 ** 30) / 2.0 ** 30)
    cx, cy = float(np.float32(CX)), float(np.float32(CY))   # the intrinsics as the solvers see them: float, widened
    pts = np.stack([np.zeros_like(depths), np.zeros_like(depths), depths], 1)
    poses = np.zeros((2, 6))
    return dict(poses_true=poses, poses_noisy=poses.copy(), pts_true=pts, pts_noisy=pts.copy(),
                kf_idx=np.tile(np.array([0, 1], np.int32), len(depths)), pt_idx=np.repeat(np.arange(len(depths), dtype=np.int32), 2),
                px=errors + np.array([cx, cy]))


def two_view_scene(seed=21, n=120, n_bad=12):
    """Two views of points in front of both cameras (the situation after Initializer::TryInitialize): true relative pose,
    noisy triangulated points, pixel noise, and a few points flagged as non-inliers (they restart from (0,0,1))."""
    from .se3 import se3_exp, se3_log
    rng = np.random.default_rng(seed)
    T_ref = np.eye(4)[:3]
    T_cur = se3_exp(np.array([-0.12, 0.03, 0.02, 0.01, -0.02, 0.015]))
    X = np.stack([rng.uniform(-1.2, 1.2, n), rng.uniform(-0.9, 0.9, n), rng.uniform(2.0, 5.0, n)], 1)

    def proj(T):
        pc = (T[:, :3] @ X.T).T + T[:, 3]
        return np.stack([FX * pc[:, 0] / pc[:, 2] + CX, FY * pc[:, 1] / pc[:, 2] + CY], 1)

    px_ref = proj(T_ref) + rng.normal(0, 0.5, (n, 2))
    px_cur = proj(T_cur) + rng.normal(0, 0.5, (n, 2))
    inlier = np.ones(n, np.uint8)
    inlier[rng.choice(n, n_bad, replace=False)] = 0
    T_cur0 = se3_exp(se3_log(T_cur) + rng.normal(0, 0.01, 6))
    return dict(T_ref=T_ref, T_cur=T_cur, T_cur0=T_cur0, X=X, X0=X + rng.normal(0, 0.05, X.shape), px_ref=px_ref, px_cur=px_cur, inlier=inlier)


def pixel_features(depth: np.ndarray, n: int, seed: int, margin: int = 8):
    """n random sub-pixel positions inside a rendered frame and their rendered depth: sparse-alignment features of any
    count (a detector caps the count by the grid)."""
    rng = np.random.default_rng(seed)
    h, w = depth.shape
    px = np.stack([rng.uniform(margin, w - margin, n), rng.uniform(margin, h - margin, n)], 1)
    return px, depth[px[:, 1].astype(int), px[:, 0].astype(int)].astype(np.float64)


def pose_only_scene(n_pts: int, seed: int = 5, pose_sigma: float = 0.002, pixel_sigma: float = 1.0):
    """One frame for the pose-only refinement: n_pts world points on the planes z = 2 and 4 in front of the camera,
    their noisy projections, the true pose T_cw and a start pose perturbed by pose_sigma in se3."""
    from .se3 import se3_exp, se3_log
    rng = np.random.default_rng(seed)
    T = trajectory(30)
    z = np.where(rng.random(n_pts) < 0.75, 2.0, 4.0)
    u, v = rng.uniform(20, W - 20, n_pts), rng.uniform(20, H - 20, n_pts)
    pc = np.stack([(u - CX) / FX * z, (v - CY) / FY * z, z], 1)
    pw = (pc - T[:, 3]) @ T[:, :3]                        # camera -> world: R^T (x - t)
    px = np.stack([u, v], 1) + rng.normal(0, pixel_sigma, (n_pts, 2))
    T0 = se3_exp(se3_log(T) + rng.normal(0, pose_sigma, 6))
    return dict(pw=pw, px=px, T_true=T, T0=T0)


def ba_edge_scene(seed: int = 41):
    """Local-BA problem with the structural corner cases of a sliding window: 6 key-frames (0 and 1 fixed), 300 landmarks
    seen by 4 key-frames, plus 40 landmarks seen only by the two fixed key-frames and 40 landmarks with one observation
    (20 on a free key-frame, 20 on a fixed one).  Returns ba_scene's dict plus `single`: the single-observation landmarks."""
    sc = ba_scene(n_kf=6, n_pt=380, target_obs=1520, seed=seed)
    sc["poses_noisy"][1] = sc["poses_true"][1]            # key-frame 1 is fixed too: at its true pose
    rng = np.random.default_rng(seed)
    keep = sc["pt_idx"] < 300
    kf, pt, px = [sc["kf_idx"][keep]], [sc["pt_idx"][keep]], [sc["px"][keep]]
    from .se3 import se3_exp
    for j in range(300, 380):
        kfs = [0, 1] if j < 340 else [int(rng.integers(2, 6)) if j < 360 else int(rng.integers(0, 2))]
        for k in kfs:
            T = se3_exp(sc["poses_true"][k])
            pc = T[:, :3] @ sc["pts_true"][j] + T[:, 3]
            kf.append(np.array([k], np.int32))
            pt.append(np.array([j], np.int32))
            px.append(np.array([[FX * pc[0] / pc[2] + CX, FY * pc[1] / pc[2] + CY]]) + rng.normal(0, 1, (1, 2)))
    sc.update(kf_idx=np.concatenate(kf).astype(np.int32), pt_idx=np.concatenate(pt).astype(np.int32), px=np.concatenate(px),
              single=np.arange(340, 380))
    return sc


def shift_stream(stream: int, n_frames: int, noise_sigma: float = 2.0, plane_z: float = 2.0):
    """Cheap exact-ground-truth VO stream: a fronto-parallel textured plane seen by a camera that only translates
    parallel to it, i.e. integer-pixel sliding crops of one render.  Returns (frames u8 (n,H,W), depth (H,W) constant,
    T_cw list) -- the pose of frame k relative to frame 0 is a pure translation known exactly."""
    tex = texture(0x59475A00 + stream, 2048)
    bw, bh = W + 256, H + 128
    base, _ = render_plane(tex, np.eye(4)[:3], plane_z=plane_z, w=bw, h=bh, cx=bw / 2, cy=bh / 2)
    rng = np.random.default_rng(1000 + stream)
    frames = np.empty((n_frames, H, W), np.uint8)
    poses = []
    ox0 = oy0 = None
    for k in range(n_frames):
        ox = int(round(128 + 110 * np.sin(2 * np.pi * k / 240 + 0.3 * stream)))
        oy = int(round(64 + 50 * np.sin(2 * np.pi * k / 170 + 0.5 * stream)))
        if ox0 is None:
            ox0, oy0 = ox, oy
        crop = base[oy:oy + H, ox:ox + W].astype(np.int16) + np.rint(rng.normal(0, noise_sigma, (H, W))).astype(np.int16)
        frames[k] = np.clip(crop, 0, 255).astype(np.uint8)
        T = np.eye(4)[:3].copy()
        T[0, 3] = -(ox - ox0) * plane_z / FX
        T[1, 3] = -(oy - oy0) * plane_z / FY
        poses.append(T)
    depth = np.full((H, W), plane_z, np.float64)
    return frames, depth, poses


def make_vocabulary(k: int = 6, L: int = 4, seed: int = 0, scoring: int = 0, weighting: int = 0, stop_fraction: float = 0.1,
                    early_leaf: float = 0.15, wide_node: bool = True) -> bytes:
    """A random vocabulary tree in DBoW3's binary file format (Vocabulary.cpp:1180-1225): header {u32 nb_nodes (root
    included), u32 size_node = 41, i32 k, i32 L, i32 scoring, i32 weighting}, then records {i32 parent, u8 descriptor[32],
    f32 weight, u8 is_leaf} in depth-first creation order like DBoW3's HKmeansStep (a parent precedes its children, the
    children of different parents interleave).  The tree is ragged like vocab/ORBvoc.bin: nodes with 2..k children, leaves
    above level L, zero-weight (stopped) words and, optionally, one node with k + 1 children."""
    rng = np.random.default_rng(seed)
    recs = []   # (parent, desc, weight, leaf)

    def grow(parent_id, parent_desc, level):
        n_ch = int(rng.integers(2, k + 1))
        if wide_node and level == 2 and not grow.widened:
            n_ch = k + 1
            grow.widened = True
        kids = []
        for _ in range(n_ch):
            d = parent_desc.copy()
            flips = rng.integers(0, 256, int(rng.integers(8, 48)))
            for b in flips:
                d[b >> 3] ^= np.uint8(1 << (b & 7))
            leaf = level == L or (level >= 2 and rng.random() < early_leaf)
            w = 0.0 if (leaf and rng.random() < stop_fraction) else float(np.float32(rng.uniform(0.5, 9.0)))
            recs.append([parent_id, d, w if leaf else 0.0, leaf])
            kids.append((len(recs), d, leaf))
        for nid, d, leaf in kids:
            if not leaf:
                grow(nid, d, level + 1)

    grow.widened = False
    grow(0, rng.integers(0, 256, 32, dtype=np.uint8), 1)
    import struct
    out = bytearray(struct.pack("<IIiiii", len(recs) + 1, 41, k, L, scoring, weighting))
    for parent, d, w, leaf in recs:
        out += struct.pack("<i", parent) + d.tobytes() + struct.pack("<f", w) + bytes([1 if leaf else 0])
    return bytes(out)
