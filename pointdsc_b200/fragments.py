"""Fragment volumes on the device (row f9): the TSDF integration and surface vertices of multiway/make_fragments.py.

The reference builds each fragment of the multiway experiment with open3d 0.9: a ScalableTSDFVolume (voxel 3 / 512, sdf_trunc
0.04, RGB8) integrates the fragment's RGB-D frames at their optimised poses, and the fragment is the vertices and vertex colours of
extract_triangle_mesh() (triangles and normals are discarded).  Here a group of fragments is integrated and extracted on the H100
with one call per stage (csrc/fragments.cu); the conventions are restated in float32 and float64 under oracle/ (PARITY
UNPINNED).

    vol = integrate_packed(depth, color, extrinsics, frame_offsets, (fx, fy, cx, cy))
    vertices, colors, offsets = extract_vertices_packed(vol)

The RGB-D odometry and pose-graph steps of make_fragments.py are not part of this module: the caller supplies each frame's pose.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _capi

MAX_FRAMES = 256            # frames per fragment (a unit's frame mask has 256 bits)
MAX_UNITS = 1 << 20         # units per fragment by default: 2^20 units of 16^3 voxels need 80 GB of volume
_STATUS = {1: "more volume units than max_units: the volume is incomplete", 2: "a point lies beyond 2^20 units of the origin"}


@dataclass
class Volume:
    """The integrated volumes of F fragments: fragment f owns units unit_offsets[f]:unit_offsets[f+1] of unit_keys [U,3] int32
    (unit coordinates, ascending), tsdf / weight [U,16,16,16] float32 and color [U,16,16,16,3] float32 (0 .. 255).  `table` is
    the unit hash the extraction looks neighbours up in."""
    unit_offsets: List[int]
    d_unit_offsets: torch.Tensor
    unit_keys: torch.Tensor
    tsdf: torch.Tensor
    weight: torch.Tensor
    color: torch.Tensor
    table: torch.Tensor
    max_units: int
    voxel_length: float


def unit_bound(frames: int, height: int, width: int, voxel_length: float, sdf_trunc: float) -> int:
    """The most units `frames` frames can touch: every stride-4 pixel touches at most k^3 units, k = floor(2 trunc / L) + 2."""
    k = int(math.floor(2.0 * sdf_trunc / (16.0 * voxel_length))) + 2
    return frames * ((height + 3) // 4) * ((width + 3) // 4) * k ** 3


def _check_status(status: Sequence[int]) -> None:
    for f, s in enumerate(status):
        if s:
            raise _capi.PdscError(f"fragment {f}: " + "; ".join(m for bit, m in _STATUS.items() if s & bit))


@torch.no_grad()
def integrate_packed(depth: torch.Tensor, color: torch.Tensor, extrinsics, frame_offsets: Sequence[int], intrinsic,
                     voxel_length: float = 3.0 / 512, sdf_trunc: float = 0.04, depth_scale: float = 1000.0, depth_trunc: float = 3.0,
                     max_units: Optional[int] = None) -> Volume:
    """ScalableTSDFVolume.integrate of F fragments' frames in order, one call per stage.  depth [NF,H,W] uint16 and color
    [NF,H,W,3] uint8 device tensors; extrinsics [NF,4,4] (world to camera, as open3d's integrate takes them); frame_offsets the
    host list of F + 1 ints (fragment f: frames frame_offsets[f]:frame_offsets[f+1], 1 .. 256 of them); intrinsic (fx, fy, cx, cy).
    One host read: the unit counts, which fix the volume's shape."""
    if depth.device.type != "cuda":
        raise _capi.PdscError("pointdsc_b200.fragments runs on an H100 only: pass CUDA tensors (there is no CPU fallback)")
    dev = depth.device
    if depth.dim() != 3 or depth.dtype != torch.uint16:
        raise ValueError(f"depth must be [NF,H,W] uint16, got {tuple(depth.shape)} {depth.dtype}")
    NF, H, W = (int(s) for s in depth.shape)
    if tuple(color.shape) != (NF, H, W, 3) or color.dtype != torch.uint8 or color.device != dev:
        raise ValueError(f"color must be [{NF},{H},{W},3] uint8 on {dev}, got {tuple(color.shape)} {color.dtype}")
    frame_offsets = [int(o) for o in frame_offsets]
    F = len(frame_offsets) - 1
    if F < 1 or frame_offsets[0] != 0 or frame_offsets[-1] != NF or any(
            not 1 <= b - a <= MAX_FRAMES for a, b in zip(frame_offsets[:-1], frame_offsets[1:])):
        raise ValueError(f"frame_offsets must run from 0 to {NF} with 1 .. {MAX_FRAMES} frames per fragment, got {frame_offsets}")
    ext = np.asarray(extrinsics.cpu() if torch.is_tensor(extrinsics) else extrinsics, np.float64).reshape(NF, 4, 4)
    poses = np.concatenate([ext.reshape(NF, 1, 16), np.linalg.inv(ext).reshape(NF, 1, 16)], 1)
    d_poses = _capi.host_to_device(poses.reshape(-1).tolist(), torch.float64, dev)
    intr = (C.c_double * 4)(*(float(v) for v in intrinsic))
    if max_units is None:
        longest = max(b - a for a, b in zip(frame_offsets[:-1], frame_offsets[1:]))
        max_units = min(unit_bound(longest, H, W, voxel_length, sdf_trunc), MAX_UNITS)
    lib, engine, stream = _capi.device_context(dev)
    h_frames, d_frames = _capi.offsets(frame_offsets, None, dev)
    dep, col = depth.contiguous(), color.contiguous()
    table = _capi.scratch(lib.pdsc_tsdf_table_bytes(F, int(max_units)), dev)
    meta = torch.empty(2, F, dtype=torch.int32, device=dev)            # unit counts, status
    P = C.c_void_p
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_tsdf_touch_packed(engine, F, h_frames, P(d_frames.data_ptr()), H, W, intr, P(dep.data_ptr()),
                                               P(d_poses.data_ptr()), float(depth_scale), float(depth_trunc), float(voxel_length),
                                               float(sdf_trunc), int(max_units), P(meta[0].data_ptr()), P(meta[1].data_ptr()),
                                               P(table.data_ptr()), table.numel(), stream))
    counts, status = meta.tolist()                                     # the one host read: the unit counts fix the shapes
    _check_status(status)
    unit_offsets = [0]
    for n in counts:
        unit_offsets.append(unit_offsets[-1] + n)
    U = unit_offsets[-1]
    h_units, d_units = _capi.offsets(unit_offsets, None, dev)
    keys = torch.empty(U, 3, dtype=torch.int32, device=dev)
    tsdf = torch.empty(U, 16, 16, 16, dtype=torch.float32, device=dev)
    weight = torch.empty(U, 16, 16, 16, dtype=torch.float32, device=dev)
    vcol = torch.empty(U, 16, 16, 16, 3, dtype=torch.float32, device=dev)
    scratch = _capi.scratch(lib.pdsc_tsdf_integrate_scratch_bytes(F, h_units), dev)
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_tsdf_integrate_packed(engine, F, h_frames, P(d_frames.data_ptr()), h_units, P(d_units.data_ptr()), H, W,
                                                   intr, P(dep.data_ptr()), P(col.data_ptr()), P(d_poses.data_ptr()),
                                                   float(depth_scale), float(depth_trunc), float(voxel_length), float(sdf_trunc),
                                                   int(max_units), P(table.data_ptr()), table.numel(), P(keys.data_ptr()),
                                                   P(tsdf.data_ptr()), P(weight.data_ptr()), P(vcol.data_ptr()),
                                                   P(scratch.data_ptr()), scratch.numel(), stream))
    return Volume(unit_offsets, d_units, keys, tsdf, weight, vcol, table, int(max_units), float(voxel_length))


@torch.no_grad()
def extract_vertices_packed(vol: Volume):
    """The vertices of extract_triangle_mesh() for every fragment of `vol`: (vertices [V,3] float64, colours [V,3] float64 in
    0 .. 1, host list of F + 1 vertex offsets), fragment f's rows offsets[f]:offsets[f+1] in the order (unit, x, y, z, edge axis).
    One host read: the vertex counts."""
    dev = vol.tsdf.device
    lib, engine, stream = _capi.device_context(dev)
    F = len(vol.unit_offsets) - 1
    U = vol.unit_offsets[-1]
    h_units = (C.c_int32 * (F + 1))(*vol.unit_offsets)
    ends = torch.empty(max(U, 1), dtype=torch.int64, device=dev)
    offs = torch.empty(F + 1, dtype=torch.int64, device=dev)
    P = C.c_void_p
    common = (engine, F, h_units, P(vol.d_unit_offsets.data_ptr()), vol.max_units, P(vol.table.data_ptr()), vol.table.numel(),
              P(vol.unit_keys.data_ptr()), P(vol.tsdf.data_ptr()), P(vol.weight.data_ptr()))
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_extract_vertices_count_packed(*common, P(ends.data_ptr()), P(offs.data_ptr()), stream))
    offsets = offs.tolist()                                            # the one host read: the vertex counts fix the shapes
    V = offsets[-1]
    verts = torch.empty(V, 3, dtype=torch.float64, device=dev)
    cols = torch.empty(V, 3, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_extract_vertices_packed(*common, P(vol.color.data_ptr()), vol.voxel_length, P(ends.data_ptr()),
                                                     P(verts.data_ptr()), P(cols.data_ptr()), stream))
    return verts, cols, offsets
