"""Device-side correspondence RANSAC (row f6): the drivers' --solver RANSAC.

Replaces the block of evaluation/test_3DMatch.py:59-77 (and test_KITTI.py:59-77), which copies the correspondences the network
labelled as inliers to the host, runs open3d 0.9's `registration_ransac_based_on_correspondence` (ransac_n 3, 5,000 iterations,
max correspondence distance = the snapshot's inlier threshold) and replaces pred_trans by its transform and pred_labels by its
inliers.  Here every set of a group runs on the H100 in one call (pdsc_ransac_packed_hypotheses, which is pdsc_ransac_packed
with the per-hypothesis transforms as one more optional output) and nothing is read back.

    from pointdsc_b200.ransac import ransac_refine      # evaluation/test_3DMatch.py:59-77, test_KITTI.py:59-77
    pred_trans, pred_labels = ransac_refine(src_keypts, tgt_keypts, pred_labels, config.inlier_threshold)

open3d is not part of the reference tree or of this image: the kernel follows its published algorithm with draws of its own (open3d
seeds rand() from the clock, so its draws cannot be replayed) and is checked against the CPU restatement under oracle/ (parity
unpinned, see its header).  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _capi

DEFAULT_SEED = 51      # the drivers' set_seed() value; a convention only, since open3d's draws never see it


@torch.no_grad()
def ransac_packed(src: torch.Tensor, tgt: torch.Tensor, labels: torch.Tensor, offsets: Sequence[int],
                  d_offsets: Optional[torch.Tensor] = None, max_correspondence_distance: float = 0.10, max_iteration: int = 5000,
                  seed: int = DEFAULT_SEED, info: bool = False, hypotheses: bool = False):
    """RANSAC of B sets in one call.  src / tgt [R,3]: set b's correspondence key points are rows offsets[b]:offsets[b+1] (the
    layout `match_many` and `PointDSC.forward_packed` use); labels [R] the forward's final_labels (rows > 0 are the candidates);
    offsets the host list of B + 1 ints, d_offsets the same values as a device int32 tensor (copied from `offsets` when None).
    Returns (trans [B,4,4] float32, labels [R] float32: 1 on the winner's inliers).  With info=True a third item
    {'fitness' [B] float64, 'inlier_rmse' [B] float64, 'best_iteration' [B] int32 (-1: none), 'status' [B] int32 (1: fewer than 3
    candidates, 2: no hypothesis with an inlier; both give the identity and all-zero labels)}; with hypotheses=True it also holds
    'hyp_good' [B, max_iteration] int32 and 'hyp_rmse' [B, max_iteration] float64, every hypothesis's key, and 'hyp_trans'
    [B, max_iteration, 12] float64, the [R | t] (row-major) each key was scored with (a test output: it solves every hypothesis
    once more).  Nothing is read back from the device."""
    if src.device.type != "cuda":
        raise _capi.PdscError("pointdsc_b200.ransac runs on an H100 only: pass CUDA tensors (there is no CPU fallback)")
    offsets = [int(o) for o in offsets]
    B = len(offsets) - 1
    if B < 1 or offsets[0] != 0 or any(b <= a for a, b in zip(offsets[:-1], offsets[1:])):
        raise ValueError(f"offsets must start at 0 and increase by at least 1 per set, got {offsets}")
    R = offsets[-1]
    for name, t in (("src", src), ("tgt", tgt)):
        if t.device != src.device or t.dim() != 2 or tuple(t.shape) != (R, 3):
            raise ValueError(f"{name} must be [{R},3] on {src.device}, got {tuple(t.shape)} on {t.device}")
    if labels.device != src.device or labels.numel() != R:
        raise ValueError(f"labels must hold {R} values on {src.device}, got {tuple(labels.shape)} on {labels.device}")
    dev = src.device
    lib, engine, stream = _capi.device_context(dev)
    s = src.to(torch.float32).contiguous()
    t = tgt.to(torch.float32).contiguous()
    lab = labels.reshape(R).to(torch.float32).contiguous()
    h_off, d_offsets = _capi.offsets(offsets, d_offsets, dev)
    trans = torch.empty(B, 4, 4, dtype=torch.float32, device=dev)
    out_labels = torch.empty(R, dtype=torch.float32, device=dev)
    want = info or hypotheses
    stats = torch.empty(2, B, dtype=torch.float64, device=dev) if want else None
    ints = torch.empty(2, B, dtype=torch.int32, device=dev) if want else None
    hyp_good = torch.empty(B, max(int(max_iteration), 0), dtype=torch.int32, device=dev) if hypotheses else None
    hyp_rmse = torch.empty(B, max(int(max_iteration), 0), dtype=torch.float64, device=dev) if hypotheses else None
    hyp_trans = torch.empty(B, max(int(max_iteration), 0), 12, dtype=torch.float64, device=dev) if hypotheses else None
    need = lib.pdsc_ransac_packed_scratch_bytes(B, h_off, int(max_iteration)) if max_iteration >= 1 else 0
    scratch = _capi.scratch(need, dev, 16)

    def ptr(x, row=None):
        if x is None:
            return None
        return C.c_void_p((x[row] if row is not None else x).data_ptr())

    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_ransac_packed_hypotheses(
            engine, B, h_off, C.c_void_p(d_offsets.data_ptr()), C.c_void_p(s.data_ptr()), C.c_void_p(t.data_ptr()),
            C.c_void_p(lab.data_ptr()), float(max_correspondence_distance), int(max_iteration), C.c_uint64(int(seed) % (1 << 64)),
            C.c_void_p(trans.data_ptr()), C.c_void_p(out_labels.data_ptr()), ptr(stats, 0), ptr(stats, 1), ptr(ints, 0),
            ptr(ints, 1), ptr(hyp_good), ptr(hyp_rmse), ptr(hyp_trans), C.c_void_p(scratch.data_ptr()), scratch.numel(), stream))
    if not want:
        return trans, out_labels
    extra = {"fitness": stats[0], "inlier_rmse": stats[1], "best_iteration": ints[0], "status": ints[1]}
    if hypotheses:
        extra.update(hyp_good=hyp_good, hyp_rmse=hyp_rmse, hyp_trans=hyp_trans)
    return trans, out_labels, extra


@torch.no_grad()
def ransac_refine(src_keypts: torch.Tensor, tgt_keypts: torch.Tensor, pred_labels: torch.Tensor,
                  max_correspondence_distance: float = 0.10, max_iteration: int = 5000, seed: int = DEFAULT_SEED):
    """[B,N,3], [B,N,3], [B,N] -> (pred_trans [B,4,4] float32, pred_labels [B,N] float32): `ransac_packed` with offsets b * N.
    With B = 1 the drop-in for the drivers' --solver RANSAC block."""
    if src_keypts.dim() != 3 or src_keypts.shape[-1] != 3 or tuple(tgt_keypts.shape) != tuple(src_keypts.shape):
        raise ValueError(f"expected src / tgt key points [B,N,3] of one shape, got {tuple(src_keypts.shape)}, {tuple(tgt_keypts.shape)}")
    B, N = int(src_keypts.shape[0]), int(src_keypts.shape[1])
    if tuple(pred_labels.shape) != (B, N):
        raise ValueError(f"expected pred_labels [{B},{N}], got {tuple(pred_labels.shape)}")
    trans, labels = ransac_packed(src_keypts.reshape(B * N, 3), tgt_keypts.reshape(B * N, 3), pred_labels.reshape(B * N),
                                  [b * N for b in range(B + 1)], max_correspondence_distance=max_correspondence_distance,
                                  max_iteration=max_iteration, seed=seed)
    return trans, labels.view(B, N)
