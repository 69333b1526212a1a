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
