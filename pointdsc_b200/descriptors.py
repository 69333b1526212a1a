"""Device-side descriptor front end (SURVEY.md section 8 row f2): PLY reader, voxel down-sampling, normals, FPFH.

Mirrors the open3d 0.9 calls the reference makes before matching (misc/cal_fpfh.py:21-26, demo_registration.py:37-44):

    pcd = orig_pcd.voxel_down_sample(voxel_size)                                   -> voxel_down_sample(points, voxel_size)
    pcd.estimate_normals(KDTreeSearchParamHybrid(radius=2 * voxel, max_nn=30))     -> estimate_normals(keypts, 2 * voxel, 30)
    compute_fpfh_feature(pcd, KDTreeSearchParamHybrid(radius=5 * voxel, max_nn=100)) -> compute_fpfh(keypts, normals, 5 * voxel, 100)

`fpfh_descriptors_many` runs the same chain over a group of clouds of different sizes, one call per stage (what misc/cal_fpfh.py
does cloud by cloud over a data set; `cal_fpfh.py` at the repository root is that script).

open3d itself is not part of the reference tree or of this image: the kernels follow its published algorithms and are checked
against the CPU restatement under oracle/ (parity unpinned, see its header).  Everything runs on the GPU; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence, Tuple

import numpy as np
import torch

from . import _capi

_STATUS = {1: "more than 2^21 voxels along an axis, or a non-finite coordinate",
           2: "a neighbourhood holds more than 4096 points inside the search radius (the search is sized for down-sampled clouds)"}


def _points_device(points: torch.Tensor) -> torch.device:
    """The device of `points`, once it is known to be a CUDA tensor [n,3] with n >= 1."""
    if points.device.type != "cuda":
        raise _capi.PdscError("pointdsc_b200.descriptors runs on an H100 only: pass CUDA tensors (there is no CPU fallback)")
    if points.dim() != 2 or points.shape[1] != 3 or points.shape[0] < 1:
        raise ValueError(f"expected points [n,3] with n >= 1, got {tuple(points.shape)}")
    return points.device


def _raise_status(status: int) -> None:
    if status:
        raise _capi.PdscError("; ".join(msg for bit, msg in _STATUS.items() if status & bit))


def read_ply(path: str) -> np.ndarray:
    """Vertex positions [n,3] float32 of a PLY file (host memory) — `np.asarray(o3d.io.read_point_cloud(path).points)`."""
    lib = _capi.load()
    n = C.c_int64(0)
    _capi.check(lib.pdsc_read_ply(path.encode(), None, 0, C.byref(n)))
    out = np.empty((n.value, 3), np.float32)
    _capi.check(lib.pdsc_read_ply(path.encode(), out.ctypes.data_as(C.c_void_p), n.value, C.byref(n)))
    return out


@torch.no_grad()
def voxel_down_sample(points: torch.Tensor, voxel_size: float) -> torch.Tensor:
    """[n,3] -> [m,3] float32: the mean of the points of every occupied voxel, rows in ascending (ix, iy, iz) order."""
    dev = _points_device(points)
    lib, engine, stream = _capi.device_context(dev)
    pts = points.to(torch.float32).contiguous()
    n = int(pts.shape[0])
    out = torch.empty(n, 3, dtype=torch.float32, device=dev)
    meta = torch.zeros(2, dtype=torch.int32, device=dev)          # [count, status]
    scratch = _capi.scratch(lib.pdsc_voxel_down_sample_scratch_bytes(n), dev)
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_voxel_down_sample(engine, n, C.c_void_p(pts.data_ptr()), float(voxel_size), C.c_void_p(out.data_ptr()),
                                               C.c_void_p(meta.data_ptr()), C.c_void_p(meta.data_ptr() + 4),
                                               C.c_void_p(scratch.data_ptr()), scratch.numel(), stream))
    m, status = (int(v) for v in meta.tolist())                   # the one host read: it fixes the output shape
    _raise_status(status)
    return out[:m].clone()


@torch.no_grad()
def estimate_normals(points: torch.Tensor, radius: float, max_nn: int = 30) -> torch.Tensor:
    """[m,3] -> unit normals [m,3] float64 (largest-magnitude component positive; (0,0,1) below three neighbours)."""
    dev = _points_device(points)
    lib, engine, stream = _capi.device_context(dev)
    pts = points.to(torch.float32).contiguous()
    m = int(pts.shape[0])
    normals = torch.empty(m, 3, dtype=torch.float64, device=dev)
    scratch = _capi.scratch(lib.pdsc_fpfh_scratch_bytes(m, max_nn), dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_estimate_normals(engine, m, C.c_void_p(pts.data_ptr()), float(radius), int(max_nn),
                                              C.c_void_p(normals.data_ptr()), C.c_void_p(status.data_ptr()),
                                              C.c_void_p(scratch.data_ptr()), scratch.numel(), stream))
    _raise_status(int(status.item()))
    return normals


@torch.no_grad()
def compute_fpfh(points: torch.Tensor, normals: torch.Tensor, radius: float, max_nn: int = 100, normalise: bool = False) -> torch.Tensor:
    """[m,3], [m,3] -> FPFH [m,33] float64 (`np.array(fpfh.data).T`); normalise=True applies x / (||x|| + 1e-6) per row."""
    dev = _points_device(points)
    lib, engine, stream = _capi.device_context(dev)
    pts = points.to(torch.float32).contiguous()
    m = int(pts.shape[0])
    if tuple(normals.shape) != (m, 3):
        raise ValueError(f"normals must be [{m},3], got {tuple(normals.shape)}")
    nrm = normals.to(device=dev, dtype=torch.float64).contiguous()
    out = torch.empty(m, 33, dtype=torch.float64, device=dev)
    scratch = _capi.scratch(lib.pdsc_fpfh_scratch_bytes(m, max_nn), dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_compute_fpfh(engine, m, C.c_void_p(pts.data_ptr()), C.c_void_p(nrm.data_ptr()), float(radius), int(max_nn),
                                          1 if normalise else 0, C.c_void_p(out.data_ptr()), C.c_void_p(status.data_ptr()),
                                          C.c_void_p(scratch.data_ptr()), scratch.numel(), stream))
    _raise_status(int(status.item()))
    return out


@torch.no_grad()
def fpfh_descriptors(points: torch.Tensor, voxel_size: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """misc/cal_fpfh.py:21-26 + the row normalisation of demo_registration.py:43: (key points [m,3] float32, FPFH [m,33] float64),
    ready for `pointdsc_b200.frontend.match`."""
    keypts = voxel_down_sample(points, voxel_size)
    normals = estimate_normals(keypts, 2.0 * voxel_size, 30)
    feat = compute_fpfh(keypts, normals, 5.0 * voxel_size, 100, normalise=True)
    return keypts, feat


@torch.no_grad()
def fpfh_descriptors_many(clouds: Sequence[torch.Tensor], voxel_size: float,
                          normalise: bool = True) -> Tuple[torch.Tensor, torch.Tensor, List[int], torch.Tensor]:
    """`fpfh_descriptors` of P clouds of different sizes, one call per stage (pdsc_*_packed).  `clouds`: device [n_p,3] tensors.
    Returns (key points [M,3] float32, FPFH [M,33] float64, offsets (host list of P + 1 ints), d_offsets (the same offsets as a
    device int32 tensor)); cloud p's rows are offsets[p]:offsets[p+1] and bit for bit what `fpfh_descriptors` gives for that
    cloud alone (normalise=False: the raw FPFH, as misc/cal_fpfh.py stores it).  The group makes two host reads: the key-point
    offsets after the down-sampling, which fix the shapes, and the status words at the end."""
    if not clouds:
        raise ValueError("fpfh_descriptors_many needs at least one cloud")
    dev = _points_device(clouds[0])
    lib, engine, stream = _capi.device_context(dev)
    for i, c in enumerate(clouds):
        if c.device != dev or c.dim() != 2 or c.shape[1] != 3 or c.shape[0] < 1:
            raise ValueError(f"cloud {i}: expected a [n,3] tensor on {dev} with n >= 1, got {tuple(c.shape)} on {c.device}")
    P = len(clouds)
    in_off = [0]
    for c in clouds:
        in_off.append(in_off[-1] + int(c.shape[0]))
    pts = (torch.cat([c.to(torch.float32) for c in clouds]) if P > 1 else clouds[0].to(torch.float32)).contiguous()
    h_in, d_in = _capi.offsets(in_off, None, dev)
    out = torch.empty(in_off[-1], 3, dtype=torch.float32, device=dev)
    meta = torch.empty(2 * P + 1, dtype=torch.int32, device=dev)       # [key-point offsets (P + 1), voxel status (P)]
    scratch = _capi.scratch(lib.pdsc_voxel_down_sample_packed_scratch_bytes(P, h_in), dev)
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_voxel_down_sample_packed(engine, P, h_in, C.c_void_p(d_in.data_ptr()), C.c_void_p(pts.data_ptr()),
                                                      float(voxel_size), C.c_void_p(out.data_ptr()), C.c_void_p(meta.data_ptr()),
                                                      C.c_void_p(meta.data_ptr() + 4 * (P + 1)),
                                                      C.c_void_p(scratch.data_ptr()), scratch.numel(), stream))
    h_meta = meta.tolist()                                         # read 1: the key-point offsets fix the shapes
    offsets = h_meta[:P + 1]
    _raise_cloud_status(h_meta[P + 1:])
    h_kp, d_offsets = _capi.offsets(offsets, meta[:P + 1], dev)
    keypts = out[:offsets[-1]].clone()
    del out, scratch
    m = offsets[-1]
    normals = torch.empty(m, 3, dtype=torch.float64, device=dev)
    feat = torch.empty(m, 33, dtype=torch.float64, device=dev)
    status = torch.empty(2, P, dtype=torch.int32, device=dev)
    scratch = _capi.scratch(lib.pdsc_fpfh_packed_scratch_bytes(P, h_kp, 100), dev)
    sc = C.c_void_p(scratch.data_ptr())
    with torch.cuda.device(dev):                                   # the normals' search (max_nn 30) fits the FPFH's scratch
        _capi.check(lib.pdsc_estimate_normals_packed(engine, P, h_kp, C.c_void_p(d_offsets.data_ptr()), C.c_void_p(keypts.data_ptr()),
                                                     2.0 * voxel_size, 30, C.c_void_p(normals.data_ptr()),
                                                     C.c_void_p(status.data_ptr()), sc, scratch.numel(), stream))
        _capi.check(lib.pdsc_compute_fpfh_packed(engine, P, h_kp, C.c_void_p(d_offsets.data_ptr()), C.c_void_p(keypts.data_ptr()),
                                                 C.c_void_p(normals.data_ptr()), 5.0 * voxel_size, 100, 1 if normalise else 0,
                                                 C.c_void_p(feat.data_ptr()), C.c_void_p(status[1].data_ptr()), sc,
                                                 scratch.numel(), stream))
    st = status.cpu()                                              # read 2: the status words
    _raise_cloud_status((st[0] | st[1]).tolist())
    return keypts, feat, offsets, d_offsets


def _raise_cloud_status(status: Sequence[int]) -> None:
    for p, s in enumerate(status):
        if s:
            raise _capi.PdscError(f"cloud {p}: " + "; ".join(msg for bit, msg in _STATUS.items() if s & bit))
