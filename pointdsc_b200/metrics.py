"""Device-side per-pair evaluation statistics (SURVEY.md section 8 row f3).

Replaces, for a whole batch in one launch and without a host synchronisation, what the evaluation drivers compute per pair
with libs/loss.py:34-63 (TransformationLoss: RE / TE / success / RMSE) and libs/loss.py:94-100 (ClassificationLoss:
precision / recall / F1 through scikit-learn on the host) — evaluation/test_3DMatch.py:83-101.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _capi

COLUMNS = ("success", "re_deg", "te_cm", "gt_inliers", "gt_inlier_ratio", "kept_gt_inliers", "precision", "recall", "f1", "rmse")


@torch.no_grad()
def eval_stats(pred_trans: torch.Tensor, gt_trans: torch.Tensor, src_keypts: torch.Tensor, tgt_keypts: torch.Tensor,
               pred_labels: torch.Tensor, gt_labels: torch.Tensor, re_thre: float = 15.0, te_thre: float = 30.0) -> torch.Tensor:
    """[B,4,4] x2, [B,N,3] x2, [B,N] x2 (device)  ->  [B,10] device tensor, columns = COLUMNS.
    Thresholds as the drivers pass them: 3DMatch 15 deg / 30 cm (test_3DMatch.py), KITTI 5 deg / 60 cm (test_KITTI.py)."""
    if pred_trans.device.type != "cuda":
        raise _capi.PdscError("pointdsc_b200.metrics.eval_stats runs on an H100 only: pass CUDA tensors (there is no CPU fallback)")
    dev = pred_trans.device
    b, n = int(src_keypts.shape[0]), int(src_keypts.shape[1])
    f = lambda x: x.to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
    pt, gt, s, t, pl, gl = f(pred_trans), f(gt_trans), f(src_keypts), f(tgt_keypts), f(pred_labels), f(gt_labels)
    if pt.shape != (b, 4, 4) or gt.shape != (b, 4, 4) or t.shape != (b, n, 3) or pl.shape != (b, n) or gl.shape != (b, n):
        raise ValueError("expected trans [B,4,4], key points [B,N,3], labels [B,N]")
    out = torch.empty(b, 10, dtype=torch.float32, device=dev)
    lib = _capi.load()
    engine = _capi.utility_engine(dev.index if dev.index is not None else torch.cuda.current_device())
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_eval_stats(engine, b, n, C.c_void_p(pt.data_ptr()), C.c_void_p(gt.data_ptr()), C.c_void_p(s.data_ptr()),
                                        C.c_void_p(t.data_ptr()), C.c_void_p(pl.data_ptr()), C.c_void_p(gl.data_ptr()),
                                        float(re_thre), float(te_thre), C.c_void_p(out.data_ptr()),
                                        C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return out


@torch.no_grad()
def eval_stats_packed(pred_trans: torch.Tensor, gt_trans: torch.Tensor, src_keypts: torch.Tensor, tgt_keypts: torch.Tensor,
                      pred_labels: torch.Tensor, gt_labels: torch.Tensor, offsets: Sequence[int],
                      d_offsets: Optional[torch.Tensor] = None, re_thre: float = 15.0, te_thre: float = 30.0) -> torch.Tensor:
    """`eval_stats` over B sets of different sizes packed back to back (pdsc_eval_stats_packed): set b owns rows
    offsets[b]:offsets[b+1] of src_keypts / tgt_keypts [R,3] and the labels [R]; trans [B,4,4].  `offsets`: B + 1 host ints;
    `d_offsets`: the same values as a device int32 tensor (uploaded without a stream synchronisation when omitted).
    -> [B,10] device tensor, columns = COLUMNS, each row bit for bit the one `eval_stats` gives for that set alone."""
    if pred_trans.device.type != "cuda":
        raise _capi.PdscError("pointdsc_b200.metrics.eval_stats runs on an H100 only: pass CUDA tensors (there is no CPU fallback)")
    dev = pred_trans.device
    offsets = [int(x) for x in offsets]
    b, r = len(offsets) - 1, int(src_keypts.shape[0])
    f = lambda x: x.to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
    pt, gt, s, t, pl, gl = f(pred_trans), f(gt_trans), f(src_keypts), f(tgt_keypts), f(pred_labels), f(gt_labels)
    if b < 1 or offsets[-1] != r or pt.shape != (b, 4, 4) or gt.shape != (b, 4, 4) or s.shape != (r, 3) or t.shape != (r, 3) \
            or pl.shape != (r,) or gl.shape != (r,):
        raise ValueError(f"expected B + 1 offsets ending at R, trans [B,4,4], key points [R,3], labels [R] (got {b + 1} offsets, "
                         f"R = {r}, trans {tuple(pt.shape)})")
    if d_offsets is None:
        from .frontend import host_to_device
        d_offsets = host_to_device(offsets, torch.int32, dev)
    if d_offsets.dtype != torch.int32 or d_offsets.device != dev or d_offsets.numel() != b + 1:
        raise ValueError("d_offsets must be a device int32 tensor of B + 1 entries")
    d_off = d_offsets.contiguous()
    h_off = (C.c_int32 * (b + 1))(*offsets)
    out = torch.empty(b, 10, dtype=torch.float32, device=dev)
    lib = _capi.load()
    engine = _capi.utility_engine(dev.index if dev.index is not None else torch.cuda.current_device())
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_eval_stats_packed(engine, b, h_off, C.c_void_p(d_off.data_ptr()), C.c_void_p(pt.data_ptr()),
                                               C.c_void_p(gt.data_ptr()), C.c_void_p(s.data_ptr()), C.c_void_p(t.data_ptr()),
                                               C.c_void_p(pl.data_ptr()), C.c_void_p(gl.data_ptr()), float(re_thre),
                                               float(te_thre), C.c_void_p(out.data_ptr()),
                                               C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return out
