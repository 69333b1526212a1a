"""Synthetic indoor-like scenes for the descriptor front end tests / demo (no dataset access in this image): a room corner
(three walls), boxes and spheres, sampled with noise.  Two samplings of the same scene with a known rigid motion make a pair."""
from __future__ import annotations

import numpy as np


def _box(rng, centre, size, n):
    face = rng.integers(0, 6, n)
    u = rng.uniform(-0.5, 0.5, (n, 3))
    axis = face // 2
    u[np.arange(n), axis] = np.where(face % 2 == 0, -0.5, 0.5)
    return centre + u * size


def _sphere(rng, centre, radius, n):
    v = rng.normal(size=(n, 3))
    return centre + radius * v / np.linalg.norm(v, axis=1, keepdims=True)


def scene(n_points: int, seed: int = 0, layout_seed: int = 7, noise: float = 0.002) -> np.ndarray:
    """[n_points,3] float32.  `layout_seed` fixes the geometry, `seed` the sampling."""
    lay = np.random.default_rng(layout_seed)
    rng = np.random.default_rng(seed)
    parts = []
    quota = n_points // 10
    for axis in range(3):                                   # three walls of a 3 m room
        p = rng.uniform(0.0, 3.0, (2 * quota, 3))
        p[:, axis] = 0.0
        parts.append(p)
    for _ in range(5):
        parts.append(_box(rng, lay.uniform(0.5, 2.5, 3), lay.uniform(0.3, 0.9, 3), quota // 2))
    for _ in range(3):
        parts.append(_sphere(rng, lay.uniform(0.5, 2.5, 3), lay.uniform(0.2, 0.5), quota // 2))
    pts = np.concatenate(parts)
    pts = pts + rng.normal(scale=noise, size=pts.shape)
    if len(pts) < n_points:
        pts = np.concatenate([pts, _sphere(rng, np.array([1.5, 1.5, 1.5]), 0.3, n_points - len(pts))])
    return pts[:n_points].astype(np.float32)


def rigid(seed: int = 0, max_angle_deg: float = 40.0, max_shift: float = 0.8):
    rng = np.random.default_rng(seed)
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    a = np.deg2rad(rng.uniform(10.0, max_angle_deg))
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    R = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
    t = rng.uniform(-max_shift, max_shift, 3)
    return R, t


def fragment_sequence(K: int, seed: int = 0, n_points: int = 20000, layout_seed: int = 11, radius: float = 1.6):
    """K overlapping views of one room for the multiway registration: [(points [n_points,3] float32 in the fragment's own frame,
    pose [4,4] float64 that maps the fragment into the room)].  View k is a fresh sampling of the room cropped to a ball of
    `radius` around a camera that moves along three quarters of a circle, turning with it (so consecutive views overlap most and
    the first and last least)."""
    if K < 2:
        raise ValueError("a fragment sequence needs at least two views")
    rng = np.random.default_rng(seed)
    out = []
    for k in range(K):
        world = scene(12 * n_points, seed=1000 * seed + k, layout_seed=layout_seed).astype(np.float64)
        a = 1.5 * np.pi * k / (K - 1)
        c = np.array([1.5 + 0.5 * np.cos(a), 1.5 + 0.5 * np.sin(a), 1.2])
        pick = np.nonzero(np.linalg.norm(world - c, axis=1) < radius)[0]
        pick = rng.choice(pick, n_points, replace=len(pick) < n_points)
        R = np.array([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]])
        pose = np.eye(4)
        pose[:3, :3], pose[:3, 3] = R, c
        out.append((((world[pick] - c) @ R).astype(np.float32), pose))
    return out


def room_shapes(layout_seed: int = 11):
    """The analytic room `render_rgbd` ray-casts: the six faces of [0, 3]^3, two spheres (centre, radius) and one axis-aligned
    box (lo, hi), placed by `layout_seed`."""
    lay = np.random.default_rng(layout_seed)
    spheres = [(lay.uniform(0.8, 2.2, 3), float(lay.uniform(0.2, 0.4))) for _ in range(2)]
    c, h = lay.uniform(0.8, 2.2, 3), lay.uniform(0.15, 0.35, 3)
    return {"room": 3.0, "spheres": spheres, "box": (c - h, c + h)}


def render_rgbd(camera_pose: np.ndarray, width: int, height: int, fx: float, fy: float, cx: float, cy: float,
                layout_seed: int = 11):
    """Ray-cast the room of `room_shapes` from a pinhole camera (x right, y down, z forward; `camera_pose` maps camera to world):
    (depth [H,W] uint16 millimetres of the nearest hit along the optical axis, colour [H,W,3] uint8 of a smooth procedural texture
    of the hit point, so the photometric term has gradients)."""
    shapes = room_shapes(layout_seed)
    v, u = np.meshgrid(np.arange(height, dtype=np.float64), np.arange(width, dtype=np.float64), indexing="ij")
    d_cam = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones_like(u)], -1)          # z = 1: the ray parameter is the depth
    R, o = np.asarray(camera_pose, np.float64)[:3, :3], np.asarray(camera_pose, np.float64)[:3, 3]
    d = d_cam @ R.T
    t = np.full(u.shape, np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        for a in range(3):                                                           # the room's faces from the inside
            for wall in (0.0, shapes["room"]):
                ta = (wall - o[a]) / d[..., a]
                t = np.where((ta > 0) & (ta < t), ta, t)
        for c, r in shapes["spheres"]:
            oc = o - c
            b = d @ oc
            a2 = np.einsum("hwk,hwk->hw", d, d)
            disc = b * b - a2 * (oc @ oc - r * r)
            ts = (-b - np.sqrt(disc)) / a2
            t = np.where((disc >= 0) & (ts > 0) & (ts < t), ts, t)
        lo, hi = shapes["box"]
        t1, t2 = (lo - o) / d, (hi - o) / d
        tn, tf = np.minimum(t1, t2).max(-1), np.maximum(t1, t2).min(-1)
        t = np.where((tn <= tf) & (tn > 0) & (tn < t), tn, t)
    p = o + t[..., None] * d
    depth = np.where(np.isfinite(t), np.round(t * 1000.0), 0).clip(0, 65535).astype(np.uint16)
    tex = np.stack([np.sin(2.1 * p[..., 0] + 1.3 * p[..., 1]), np.sin(1.7 * p[..., 1] + 2.3 * p[..., 2] + 1.0),
                    np.sin(2.9 * p[..., 2] + 1.1 * p[..., 0] + 2.0)], -1)
    color = np.where(np.isfinite(t)[..., None], 128 + 100 * tex, 0).astype(np.uint8)
    return depth, color


def camera_path(n: int, seed: int = 0):
    """n camera poses [n,4,4] float64 inside the room, looking at its centre from a slowly moving point (consecutive frames of an
    RGB-D sequence)."""
    rng = np.random.default_rng(seed)
    a0 = rng.uniform(0, 2 * np.pi)
    out = []
    for k in range(n):
        a = a0 + 0.02 * k
        eye = np.array([1.5 + 0.6 * np.cos(a), 1.5 + 0.6 * np.sin(a), 1.3 + 0.05 * np.sin(0.3 * k)])
        fwd = np.array([1.5, 1.5, 1.2]) - eye + np.array([0.4 * np.cos(a + 1.0), 0.4 * np.sin(a + 1.0), 0.0])
        fwd /= np.linalg.norm(fwd)
        right = np.cross(fwd, [0.0, 0.0, 1.0])
        right /= np.linalg.norm(right)
        down = np.cross(fwd, right)
        pose = np.eye(4)
        pose[:3, :3] = np.stack([right, down, fwd], 1)
        pose[:3, 3] = eye
        out.append(pose)
    return np.stack(out)
