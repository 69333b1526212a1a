"""Device-side N x N power iteration (SURVEY.md section 8 row f4).

`leading_eigenvector(M)` is `PointDSC.cal_leading_eigenvector(M, method='power')` (reference models/PointDSC.py:338-358) for the
N x N matrices it is applied to outside the testing path: the feature-similarity matrix the non-testing forward returns
(:160-170) and the compatibility matrix of the classical spectral-matching baseline (baseline_scripts/baseline_3DMatch.py:19-44).

`spectral_matching(corr_pos, src_keypts, tgt_keypts, inlier_threshold)` is that baseline as a whole, `SM`
(baseline_scripts/baseline_3DMatch.py:19-53): the compatibility matrix, ten power iterations, the top 10 % of the eigenvector as
inliers and the weighted Kabsch.  It never forms the N x N matrix, and `spectral_matching_packed` runs a group of sets of
different sizes in one call (csrc/spectral_matching.cu).
"""
from __future__ import annotations

import ctypes as C

import torch

from typing import Optional, Sequence

from . import _capi

MAX_ROWS = 16384      # rows per set: the limit of the top-S sort the selection shares with the forward


@torch.no_grad()
def leading_eigenvector(M: torch.Tensor, num_iterations: int = 10, early_exit: bool = True):
    """M [B,N,N] (device, fp32) -> (eigenvector [B,N], iterations run [B] int32).  `early_exit=True` is the module's rule
    (stop when allclose(v, v_prev)), decided per matrix; `False` runs exactly `num_iterations` (the classical baseline)."""
    if M.device.type != "cuda":
        raise _capi.PdscError("pointdsc_b200.spectral.leading_eigenvector runs on an H100 only: pass a CUDA tensor (no CPU fallback)")
    if M.dim() != 3 or M.shape[1] != M.shape[2]:
        raise ValueError(f"expected M [B,N,N], got {tuple(M.shape)}")
    dev = M.device
    m = M.to(torch.float32).contiguous()
    b, n = int(m.shape[0]), int(m.shape[1])
    lib, engine, stream = _capi.device_context(dev)
    v = torch.empty(b, n, dtype=torch.float32, device=dev)
    iters = torch.empty(b, dtype=torch.int32, device=dev)
    scratch = _capi.scratch(lib.pdsc_leading_eigenvector_scratch_bytes(b, n), dev, align=16)
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_leading_eigenvector(engine, b, n, C.c_void_p(m.data_ptr()), int(num_iterations), 1 if early_exit else 0,
                                                 C.c_void_p(v.data_ptr()), C.c_void_p(iters.data_ptr()),
                                                 C.c_void_p(scratch.data_ptr()), scratch.numel(), stream))
    return v, iters


@torch.no_grad()
def spectral_matching_packed(corr_pos: torch.Tensor, src: torch.Tensor, tgt: torch.Tensor, offsets: Sequence[int],
                             d_offsets: Optional[torch.Tensor] = None, inlier_threshold: float = 0.10, eigenvector: bool = False):
    """The spectral-matching baseline of B sets in one call.  corr_pos [R,6], src / tgt [R,3]: set b's rows are
    offsets[b]:offsets[b+1] (the layout `match_many` and `ransac_packed` use), 1 to MAX_ROWS rows each; offsets the host list
    of B + 1 ints, d_offsets the same values as a device int32 tensor (copied from `offsets` when None).  Returns (trans
    [B,4,4] float32, labels [R] float32: 1 on the int(N_b * 0.1) largest eigenvector entries of each set, lowest row first on
    ties), and the eigenvector [R] float32 as a third item with eigenvector=True.  Nothing is read back from the device."""
    if corr_pos.device.type != "cuda":
        raise _capi.PdscError("pointdsc_b200.spectral runs on an H100 only: pass CUDA tensors (there is no CPU fallback)")
    offsets = [int(o) for o in offsets]
    B = len(offsets) - 1
    if B < 1 or offsets[0] != 0 or any(b <= a for a, b in zip(offsets[:-1], offsets[1:])):
        raise ValueError(f"offsets must start at 0 and increase by at least 1 per set, got {offsets}")
    R = offsets[-1]
    dev = corr_pos.device
    for name, t, w in (("corr_pos", corr_pos, 6), ("src", src, 3), ("tgt", tgt, 3)):
        if t.device != dev or t.dim() != 2 or tuple(t.shape) != (R, w):
            raise ValueError(f"{name} must be [{R},{w}] on {dev}, got {tuple(t.shape)} on {t.device}")
    lib, engine, stream = _capi.device_context(dev)
    c = corr_pos.to(torch.float32).contiguous()
    s = src.to(torch.float32).contiguous()
    t = tgt.to(torch.float32).contiguous()
    h_off, d_offsets = _capi.offsets(offsets, d_offsets, dev)
    trans = torch.empty(B, 4, 4, dtype=torch.float32, device=dev)
    labels = torch.empty(R, dtype=torch.float32, device=dev)
    eig = torch.empty(R, dtype=torch.float32, device=dev) if eigenvector else None
    scratch = _capi.scratch(lib.pdsc_spectral_matching_packed_scratch_bytes(B, h_off), dev, 16)
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_spectral_matching_packed(
            engine, B, h_off, C.c_void_p(d_offsets.data_ptr()), C.c_void_p(c.data_ptr()), C.c_void_p(s.data_ptr()),
            C.c_void_p(t.data_ptr()), float(inlier_threshold), C.c_void_p(trans.data_ptr()), C.c_void_p(labels.data_ptr()),
            C.c_void_p(eig.data_ptr()) if eig is not None else None, C.c_void_p(scratch.data_ptr()), scratch.numel(), stream))
    return (trans, labels, eig) if eigenvector else (trans, labels)


@torch.no_grad()
def spectral_matching(corr_pos: torch.Tensor, src_keypts: torch.Tensor, tgt_keypts: torch.Tensor, inlier_threshold: float = 0.10):
    """[bs,N,6], [bs,N,3], [bs,N,3] -> (pred_trans [bs,4,4] float32, pred_labels [bs,N] float32): `spectral_matching_packed`
    with offsets b * N.  With bs = 1 the drop-in for the baseline script's `SM(corr, src_keypts, tgt_keypts, args)`."""
    if corr_pos.dim() != 3 or corr_pos.shape[-1] != 6:
        raise ValueError(f"expected corr_pos [bs,N,6], got {tuple(corr_pos.shape)}")
    B, N = int(corr_pos.shape[0]), int(corr_pos.shape[1])
    for name, t in (("src_keypts", src_keypts), ("tgt_keypts", tgt_keypts)):
        if tuple(t.shape) != (B, N, 3):
            raise ValueError(f"expected {name} [{B},{N},3], got {tuple(t.shape)}")
    trans, labels = spectral_matching_packed(corr_pos.reshape(B * N, 6), src_keypts.reshape(B * N, 3), tgt_keypts.reshape(B * N, 3),
                                             [b * N for b in range(B + 1)], inlier_threshold=inlier_threshold)
    return trans, labels.view(B, N)
