"""numpy restatement of the fragment volume of multiway/make_fragments.py (open3d 0.9's ScalableTSDFVolume with RGB8 colour and the
vertex half of extract_triangle_mesh), the definition pointdsc_b200/csrc/fragments.cu is held to.

PARITY UNPINNED: open3d is not part of the reference tree or of this image, so the conventions below are recalled, not checked.

Integration is float32, one rounding per operation (numpy float32 arithmetic has no fused multiply-add), in the order written, so
the device is held to it bit for bit.  Touched units are float64.  Vertices are float64.

1. depth = float32(raw) / float32(depth_scale), 0 where depth >= depth_trunc.
2. Touch: the stride-4 pixels (row, col multiples of 4) with depth d > 0 lift to x = (col - cx) d / fx, y = (row - cy) d / fy, z = d
   and to the world by the camera pose P (the extrinsic's inverse): p_r = ((P_r0 x + P_r1 y) + P_r2 z) + P_r3.  Every unit from
   floor((p - trunc) / L) to floor((p + trunc) / L) per axis (L = 16 voxel_length) is touched by the frame.
3. Integrate, for each unit in the order of the frames that touched it: with e = float32(extrinsic), v = float32(voxel_length),
   h = v * 0.5, the voxel (x, y, z) of the unit with origin o = float32(unit * L) starts its column at
   c_r = ((e_r0 bx + e_r1 by) + e_r2 bz) + e_r3 with bx = (h + v x) + o_x, by = (h + v y) + o_y, bz = h + o_z, and steps z by
   adding e_r2 * v.  Where c_2 > 0: u_f = ((c_0 fx) / c_2 + cx) + 0.5 (v_f alike) is kept in [1e-4, W - 1e-4) (H alike), u = int(u_f);
   where d(u, v) > 0 the sdf (d - c_2) * sqrt((xx^2 + yy^2) + 1), xx = (u - cx) * (1 / fx), yy = (v - cy) * (1 / fy), updates the
   voxel when sdf > -trunc: tsdf = min(1, sdf * (1 / trunc)), t <- (t w + tsdf) / (w + 1), each colour channel alike with the pixel's
   0 .. 255 value, then w <- w + 1.  The multiplication by 1 / trunc (not a division by trunc) is open3d's sdf_trunc_inv_f.
4. Vertices: the edge (g, a) of the global voxel grid carries a vertex when tsdf(g) < 0 and tsdf(g + e_a) < 0 differ and one of the
   four cubes sharing it has all 8 corner weights non-zero.  Its position is (g + 0.5) v with f0 v / (f0 + f1) added along a,
   f0 = |tsdf(g)|, f1 = |tsdf(g + e_a)|; its colour (f1 c0 + f0 c1) / (f0 + f1) with c = colour / 255.  Vertices are listed by
   (unit coordinates, x, y, z, a), the unit owning g.
"""
from __future__ import annotations

import numpy as np

RES = 16
F32 = np.float32


def depth_to_float(raw: np.ndarray, depth_scale: float = 1000.0, depth_trunc: float = 3.0) -> np.ndarray:
    d = raw.astype(F32) / F32(depth_scale)
    d[d.astype(np.float64) >= depth_trunc] = F32(0.0)
    return d


def touched_units(depth: np.ndarray, camera_pose: np.ndarray, intrinsic, voxel_length: float, sdf_trunc: float) -> set:
    """Step 2 for one frame: the set of touched unit coordinates (ix, iy, iz)."""
    fx, fy, cx, cy = (float(v) for v in intrinsic)
    H, W = depth.shape
    rows, cols = np.meshgrid(np.arange(0, H, 4), np.arange(0, W, 4), indexing="ij")
    d = depth[rows, cols]
    keep = d > 0
    z = d[keep].astype(np.float64)
    x = (cols[keep].astype(np.float64) - cx) * z / fx
    y = (rows[keep].astype(np.float64) - cy) * z / fy
    P = np.asarray(camera_pose, np.float64)
    L = voxel_length * RES
    lo, hi = [], []
    for r in range(3):
        p = ((P[r, 0] * x + P[r, 1] * y) + P[r, 2] * z) + P[r, 3]
        lo.append(np.floor((p - sdf_trunc) / L).astype(np.int64))
        hi.append(np.floor((p + sdf_trunc) / L).astype(np.int64))
    out = set()
    span = [int((h - l).max()) + 1 if len(l) else 0 for l, h in zip(lo, hi)]
    for dx in range(span[0] if span else 0):
        for dy in range(span[1]):
            for dz in range(span[2]):
                ok = (lo[0] + dx <= hi[0]) & (lo[1] + dy <= hi[1]) & (lo[2] + dz <= hi[2])
                out.update(zip((lo[0] + dx)[ok].tolist(), (lo[1] + dy)[ok].tolist(), (lo[2] + dz)[ok].tolist()))
    return out


def integrate_unit(unit, frames, depth, color, extrinsic, intrinsic, voxel_length: float, sdf_trunc: float, state=None):
    """Step 3 for one unit over the frame indices `frames` (ascending): (tsdf, weight [16,16,16], colour [16,16,16,3]) float32."""
    fx, fy, cx, cy = (F32(v) for v in intrinsic)
    H, W = depth.shape[1:]
    v = F32(voxel_length)
    half = v * F32(0.5)
    trunc = F32(sdf_trunc)
    trunc_inv = F32(1.0) / trunc
    safe_w, safe_h = F32(W) - F32(0.0001), F32(H) - F32(0.0001)
    ffl0, ffl1 = F32(1.0) / fx, F32(1.0) / fy
    L = voxel_length * RES
    o = [F32(float(unit[k]) * L) for k in range(3)]
    xs, ys = np.meshgrid(np.arange(RES), np.arange(RES), indexing="ij")
    bx = (half + v * xs.astype(F32)) + o[0]
    by = (half + v * ys.astype(F32)) + o[1]
    bz = half + o[2]
    if state is None:
        ts = np.zeros((RES, RES, RES), F32)
        w = np.zeros((RES, RES, RES), F32)
        col = np.zeros((RES, RES, RES, 3), F32)
    else:
        ts, w, col = (a.copy() for a in state)
    for j in frames:
        e = np.asarray(extrinsic[j], np.float64).astype(F32)
        p = [((e[r, 0] * bx + e[r, 1] * by) + e[r, 2] * bz) + e[r, 3] for r in range(3)]
        step = [e[r, 2] * v for r in range(3)]
        for z in range(RES):
            with np.errstate(divide="ignore", invalid="ignore"):
                uf = ((p[0] * fx) / p[2] + cx) + F32(0.5)
                vf = ((p[1] * fy) / p[2] + cy) + F32(0.5)
            ok = (p[2] > 0) & (uf >= F32(0.0001)) & (uf < safe_w) & (vf >= F32(0.0001)) & (vf < safe_h)
            u = np.where(ok, uf, 0).astype(np.int64)
            vv = np.where(ok, vf, 0).astype(np.int64)
            d = np.where(ok, depth[j][vv, u], F32(0.0))
            ok &= d > 0
            xx = (u.astype(F32) - cx) * ffl0
            yy = (vv.astype(F32) - cy) * ffl1
            mult = np.sqrt((xx * xx + yy * yy) + F32(1.0))
            sdf = (d - p[2]) * mult
            ok &= sdf > -trunc
            tsdf = np.minimum(F32(1.0), sdf * trunc_inv)
            w0 = w[:, :, z]
            w1 = w0 + F32(1.0)
            ts[:, :, z] = np.where(ok, (ts[:, :, z] * w0 + tsdf) / w1, ts[:, :, z])
            rgb = color[j][vv, u].astype(F32)
            for ch in range(3):
                col[:, :, z, ch] = np.where(ok, (col[:, :, z, ch] * w0 + rgb[..., ch]) / w1, col[:, :, z, ch])
            w[:, :, z] = np.where(ok, w1, w0)
            p = [p[r] + step[r] for r in range(3)]
    return ts, w, col


def integrate(depth_raw, color, extrinsic, intrinsic, voxel_length: float = 3.0 / 512, sdf_trunc: float = 0.04,
              depth_scale: float = 1000.0, depth_trunc: float = 3.0):
    """Steps 1-3 for one fragment's frames: {unit (ix, iy, iz): (frames, tsdf, weight, colour)}, the camera poses being the
    float64 inverses of the extrinsics."""
    depth = np.stack([depth_to_float(d, depth_scale, depth_trunc) for d in depth_raw])
    frames = {}
    for j in range(len(depth)):
        for unit in touched_units(depth[j], np.linalg.inv(np.asarray(extrinsic[j], np.float64)), intrinsic, voxel_length, sdf_trunc):
            frames.setdefault(unit, []).append(j)
    return {unit: (fl,) + integrate_unit(unit, fl, depth, color, extrinsic, intrinsic, voxel_length, sdf_trunc)
            for unit, fl in sorted(frames.items())}


def extract_vertices(units: dict, voxel_length: float):
    """Step 4: {unit: (tsdf [16,16,16], weight, colour [16,16,16,3])} -> (vertices [V,3], colours [V,3]) float64, canonical order."""
    if not units:
        return np.zeros((0, 3)), np.zeros((0, 3))
    keys = np.array(sorted(units), np.int64)
    lo = keys.min(0) - 1
    n = keys.max(0) - lo + 2
    T = np.zeros(tuple(n * RES), np.float32)
    Wt = np.zeros_like(T)
    Cc = np.zeros(tuple(n * RES) + (3,), np.float32)
    for k in keys:
        s = tuple(slice(int(a) * RES, int(a) * RES + RES) for a in (k - lo))
        t, w, c = units[tuple(k.tolist())][-3:]
        T[s], Wt[s], Cc[s] = t, w, c
    verts, cols = [], []
    v = float(voxel_length)
    valid = np.ones(T.shape, bool)                                # cube with origin g: all 8 corner weights non-zero
    for c in range(8):
        valid[:-1, :-1, :-1] &= Wt[c >> 2:T.shape[0] - 1 + (c >> 2), (c >> 1) & 1:T.shape[1] - 1 + ((c >> 1) & 1),
                                   c & 1:T.shape[2] - 1 + (c & 1)] != 0
    valid[-1, :, :] = valid[:, -1, :] = valid[:, :, -1] = False
    for k in keys:
        g0 = (k - lo) * RES
        ax = [np.arange(RES)[:, None, None], np.arange(RES)[None, :, None], np.arange(RES)[None, None, :]]
        gx, gy, gz = (g0[i] + ax[i] for i in range(3))
        gx, gy, gz = np.broadcast_arrays(gx, gy, gz)
        has = np.zeros((RES, RES, RES, 3), bool)
        for a in range(3):
            h = [gx, gy, gz]
            h[a] = h[a] + 1
            diff = (T[gx, gy, gz] < 0) != (T[h[0], h[1], h[2]] < 0)
            b, c2 = (a + 1) % 3, (a + 2) % 3
            cube = np.zeros_like(diff)
            for db in (0, 1):
                for dc in (0, 1):
                    o = [gx, gy, gz]
                    o[b] = o[b] - db
                    o[c2] = o[c2] - dc
                    cube |= valid[o[0], o[1], o[2]]
            has[..., a] = diff & cube
        idx = np.argwhere(has)                                    # (x, y, z, a), row-major: the canonical order
        for x, y, z, a in idx:
            g = np.array([g0[0] + x, g0[1] + y, g0[2] + z])
            h = g.copy()
            h[a] += 1
            f0, f1 = abs(float(T[tuple(g)])), abs(float(T[tuple(h)]))
            gg = (k * RES + np.array([x, y, z])).astype(np.float64)
            p = (gg + 0.5) * v
            p[a] = p[a] + (f0 * v) / (f0 + f1)
            c0 = Cc[tuple(g)].astype(np.float64) / 255.0
            c1 = Cc[tuple(h)].astype(np.float64) / 255.0
            verts.append(p)
            cols.append((f1 * c0 + f0 * c1) / (f0 + f1))
    if not verts:
        return np.zeros((0, 3)), np.zeros((0, 3))
    return np.array(verts), np.array(cols)
