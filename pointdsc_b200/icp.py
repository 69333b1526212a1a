"""Device-side ICP refinement (row f5): the drivers' --use_icp.

Replaces `icp_refine` of evaluation/benchmark_utils.py:40-55, which copies a pair's correspondence key points and `final_trans` to
the host, runs open3d 0.9's point-to-point `registration_icp` (max correspondence distance 0.10, default criteria) and copies the
refined 4x4 back.  Here every set of a group is refined on the H100 in one call (pdsc_icp_packed) and nothing is read back.

    from pointdsc_b200.icp import icp_refine            # evaluation/test_3DMatch.py:79-80, test_KITTI.py:79-80, test_multi.py:53-54
    pred_trans = icp_refine(src_keypts, tgt_keypts, pred_trans)

open3d is not part of the reference tree or of this image: the kernel follows its published algorithm and is checked against the
CPU restatement under oracle/ (parity unpinned, see its header).  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _capi


@torch.no_grad()
def icp_refine_packed(src: torch.Tensor, tgt: torch.Tensor, pred_trans: torch.Tensor, offsets: Sequence[int],
                      d_offsets: Optional[torch.Tensor] = None, max_correspondence_distance: float = 0.10, max_iteration: int = 30,
                      info: bool = False):
    """Point-to-point ICP of B sets in one call.  src / tgt [R,3]: set b's correspondence key points are rows
    offsets[b]:offsets[b+1] (the layout `match_many` and `PointDSC.forward_packed` use); pred_trans [B,4,4] the starting
    transforms; offsets the host list of B + 1 ints, d_offsets the same values as a device int32 tensor (copied from `offsets` when
    None).  Returns the refined [B,4,4] float32; with info=True also {'fitness' [B] float64, 'inlier_rmse' [B] float64, 'iterations'
    [B] int32, 'status' [B] int32}.  A set with status 1 (a non-finite coordinate, or a target spanning 2^21 or more cells of side
    max_correspondence_distance along an axis) keeps its starting transform.  Nothing is read back from the device."""
    if src.device.type != "cuda":
        raise _capi.PdscError("pointdsc_b200.icp runs on an H100 only: pass CUDA tensors (there is no CPU fallback)")
    offsets = [int(o) for o in offsets]
    B = len(offsets) - 1
    if B < 1 or offsets[0] != 0 or any(b <= a for a, b in zip(offsets[:-1], offsets[1:])):
        raise ValueError(f"offsets must start at 0 and increase by at least 1 per set, got {offsets}")
    R = offsets[-1]
    for name, t in (("src", src), ("tgt", tgt)):
        if t.device != src.device or t.dim() != 2 or tuple(t.shape) != (R, 3):
            raise ValueError(f"{name} must be [{R},3] on {src.device}, got {tuple(t.shape)} on {t.device}")
    if tuple(pred_trans.shape) != (B, 4, 4):
        raise ValueError(f"pred_trans must be [{B},4,4], got {tuple(pred_trans.shape)}")
    dev = src.device
    lib, engine, stream = _capi.device_context(dev)
    s = src.to(torch.float32).contiguous()
    t = tgt.to(torch.float32).contiguous()
    init = pred_trans.to(device=dev, dtype=torch.float32).contiguous()
    h_off, d_offsets = _capi.offsets(offsets, d_offsets, dev)
    out = torch.empty(B, 4, 4, dtype=torch.float32, device=dev)
    stats = torch.empty(2, B, dtype=torch.float64, device=dev) if info else None
    ints = torch.empty(2, B, dtype=torch.int32, device=dev) if info else None
    scratch = _capi.scratch(lib.pdsc_icp_packed_scratch_bytes(B, h_off), dev)

    def ptr(x, row=None):
        return C.c_void_p(x[row].data_ptr()) if x is not None else None

    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_icp_packed(engine, B, h_off, C.c_void_p(d_offsets.data_ptr()), C.c_void_p(s.data_ptr()),
                                        C.c_void_p(t.data_ptr()), C.c_void_p(init.data_ptr()), float(max_correspondence_distance),
                                        int(max_iteration), C.c_void_p(out.data_ptr()), ptr(stats, 0), ptr(stats, 1), ptr(ints, 0),
                                        ptr(ints, 1), C.c_void_p(scratch.data_ptr()), scratch.numel(), stream))
    if not info:
        return out
    return out, {"fitness": stats[0], "inlier_rmse": stats[1], "iterations": ints[0], "status": ints[1]}


@torch.no_grad()
def icp_refine(src_keypts: torch.Tensor, tgt_keypts: torch.Tensor, pred_trans: torch.Tensor,
               max_correspondence_distance: float = 0.10) -> torch.Tensor:
    """[B,N,3], [B,N,3], [B,4,4] -> refined [B,4,4] float32: `icp_refine_packed` with offsets b * N.  With B = 1 a drop-in for
    evaluation/benchmark_utils.icp_refine."""
    if src_keypts.dim() != 3 or src_keypts.shape[-1] != 3 or tuple(tgt_keypts.shape) != tuple(src_keypts.shape):
        raise ValueError(f"expected src / tgt key points [B,N,3] of one shape, got {tuple(src_keypts.shape)}, {tuple(tgt_keypts.shape)}")
    B, N = int(src_keypts.shape[0]), int(src_keypts.shape[1])
    return icp_refine_packed(src_keypts.reshape(B * N, 3), tgt_keypts.reshape(B * N, 3), pred_trans, [b * N for b in range(B + 1)],
                             max_correspondence_distance=max_correspondence_distance)
