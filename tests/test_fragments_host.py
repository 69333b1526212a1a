"""The fragment-volume restatement (oracle/fragments_oracle.py) against its definition on hand-built cases, and the synthetic
RGB-D renderer against ray-plane, ray-sphere and ray-box distances.  No GPU."""
import math

import numpy as np
import pytest

from oracle import fragments_oracle as O
from pointdsc_b200.synth_scene import camera_path, render_rgbd, room_shapes

V = 3.0 / 512
INTR = (525.0 / 8, 525.0 / 8, 319.5 / 8, 239.5 / 8)


def test_depth_conversion_truncates_at_depth_trunc():
    d = O.depth_to_float(np.array([[0, 1, 2999, 3000, 65535]], np.uint16))
    assert d.dtype == np.float32
    assert d.tolist()[0] == [0.0, float(np.float32(1) / np.float32(1000)), float(np.float32(2999) / np.float32(1000)), 0.0, 0.0]


def test_touched_units_span_the_truncation_box():
    depth = np.zeros((8, 8), np.float32)
    depth[0, 0] = 1.0
    pose = np.eye(4)
    pose[:3, 3] = (0.0, 0.0, -1.0 + 0.01)               # the point lands at z = 0.01, x = y = -cx / fx
    units = O.touched_units(depth, pose, (1.0, 1.0, 0.0, 0.0), V, 0.04)
    L = 16 * V
    want = {(x, y, z) for x in range(math.floor(-0.04 / L), math.floor(0.04 / L) + 1)
            for y in range(math.floor(-0.04 / L), math.floor(0.04 / L) + 1)
            for z in range(math.floor((0.01 - 0.04) / L), math.floor((0.01 + 0.04) / L) + 1)}
    assert units == want and len(units) == 8


@pytest.fixture(scope="module")
def two_frames():
    poses = camera_path(12, 3)[[0, 11]]
    fr = [render_rgbd(p, 80, 60, *INTR) for p in poses]
    return np.stack([f[0] for f in fr]), np.stack([f[1] for f in fr]), np.linalg.inv(poses)


def test_unit_not_touched_by_a_frame_keeps_its_values(two_frames):
    dep, col, ext = two_frames
    units = O.integrate(dep, col, ext, INTR, V, 0.04)
    depth = np.stack([O.depth_to_float(d) for d in dep])
    only_first = [u for u, r in units.items() if r[0] == [0]]
    assert only_first
    changed = 0
    for u in only_first:
        _, t, w, c = units[u]
        t0, w0, c0 = O.integrate_unit(u, [0], depth, col, ext, INTR, V, 0.04)
        assert np.array_equal(t, t0) and np.array_equal(w, w0) and np.array_equal(c, c0)
        t1, w1, _ = O.integrate_unit(u, [0, 1], depth, col, ext, INTR, V, 0.04)
        changed += not np.array_equal(w1, w0)
    assert changed > 0, "frame 1 would update none of the units it did not touch: the case does not test the mask"


def test_edge_whose_only_valid_cube_lies_in_the_next_unit():
    z = np.zeros((16, 16, 16), np.float32)
    units = {(-1, 0, 0): [z.copy(), z.copy(), np.zeros((16, 16, 16, 3), np.float32)],
             (0, 0, 0): [z.copy(), z.copy(), np.zeros((16, 16, 16, 3), np.float32)]}
    for x in (-1, 0):                                   # the one cube with all 8 weights: origin (-1, 0, 0)
        for y in (0, 1):
            for zz in (0, 1):
                u = units[(-1 if x < 0 else 0, 0, 0)]
                u[0][x % 16, y, zz] = 0.5
                u[1][x % 16, y, zz] = 1.0
                u[2][x % 16, y, zz] = (255.0, 0.0, 0.0)
    units[(0, 0, 0)][0][0, 0, 0] = -0.25
    units[(0, 0, 0)][2][0, 0, 0] = (0.0, 255.0, 0.0)
    verts, cols = O.extract_vertices(units, V)
    # unit (-1,0,0) owns the x edge from (-1,0,0); unit (0,0,0) the y and z edges from (0,0,0), whose cubes at (0,0,0), (0,-1,0)
    # and (0,0,-1) hold zero weights: only the cube across the unit boundary makes them vertices
    frac = 0.5 / 0.75
    want = [(-0.5 * V + frac * V, 0.5 * V, 0.5 * V), (0.5 * V, 0.5 * V + 0.25 / 0.75 * V, 0.5 * V),
            (0.5 * V, 0.5 * V, 0.5 * V + 0.25 / 0.75 * V)]
    assert verts.shape == (3, 3)
    np.testing.assert_allclose(verts, want, rtol=0, atol=1e-15)
    np.testing.assert_allclose(cols[0], (0.25 * 1.0 / 0.75, 0.5 / 0.75, 0.0), atol=1e-15)


def _ray_depth(o, d, shapes):
    best = math.inf
    for a in range(3):
        for wall in (0.0, shapes["room"]):
            if d[a] != 0:
                t = (wall - o[a]) / d[a]
                if 0 < t < best:
                    best = t
    for c, r in shapes["spheres"]:
        oc = o - c
        A, B, Cc = d @ d, d @ oc, oc @ oc - r * r
        disc = B * B - A * Cc
        if disc >= 0:
            t = (-B - math.sqrt(disc)) / A
            if 0 < t < best:
                best = t
    lo, hi = shapes["box"]
    tn, tf = -math.inf, math.inf
    for a in range(3):
        t1, t2 = (lo[a] - o[a]) / d[a], (hi[a] - o[a]) / d[a]
        tn, tf = max(tn, min(t1, t2)), min(tf, max(t1, t2))
    if tn <= tf and 0 < tn < best:
        best = tn
    return best


def test_renderer_depth_is_the_nearest_analytic_surface():
    pose = camera_path(1, 2)[0]
    W, H = 80, 60
    depth, color = render_rgbd(pose, W, H, *INTR)
    shapes = room_shapes()
    rng = np.random.default_rng(0)
    fx, fy, cx, cy = INTR
    hits = set()
    for _ in range(200):
        u, v = int(rng.integers(W)), int(rng.integers(H))
        d = pose[:3, :3] @ np.array([(u - cx) / fx, (v - cy) / fy, 1.0])
        t = _ray_depth(pose[:3, 3], d, shapes)
        assert depth[v, u] == round(t * 1000.0), (u, v)
        hits.add(round(t, 3))
    assert len(hits) > 50 and color.std() > 10


def test_camera_path_is_rigid_and_inside_the_room():
    poses = camera_path(5, 1)
    for p in poses:
        assert np.allclose(p[:3, :3].T @ p[:3, :3], np.eye(3), atol=1e-12) and np.isclose(np.linalg.det(p[:3, :3]), 1.0)
        assert ((p[:3, 3] > 0) & (p[:3, 3] < 3)).all()


def test_unit_bound_and_device_only():
    import torch

    from pointdsc_b200 import _capi
    from pointdsc_b200.fragments import integrate_packed, unit_bound
    assert unit_bound(2, 8, 8, V, 0.04) == 2 * 4 * 8
    with pytest.raises(_capi.PdscError, match="H100"):
        integrate_packed(torch.zeros(1, 8, 8, dtype=torch.uint16), torch.zeros(1, 8, 8, 3, dtype=torch.uint8), np.eye(4)[None],
                         [0, 1], INTR)
