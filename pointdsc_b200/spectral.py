"""Device-side N x N power iteration (SURVEY.md section 8 row f4).

`leading_eigenvector(M)` is `PointDSC.cal_leading_eigenvector(M, method='power')` (reference models/PointDSC.py:338-358) for the
N x N matrices it is applied to outside the testing path: the feature-similarity matrix the non-testing forward returns
(:160-170) and the compatibility matrix of the classical spectral-matching baseline (baseline_scripts/baseline_3DMatch.py:19-44).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _capi


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
