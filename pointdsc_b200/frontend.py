"""Device-side correspondence front end (SURVEY.md section 8 row f1).

Mirrors the lines every caller of `PointDSC.forward` runs first (reference datasets/ThreeDMatch.py:283-291 and :299-308,
datasets/KITTI.py:80-114, demo_registration.py:101-108): nearest neighbour in descriptor space, optional mutual check,
and the centred `corr_pos`.  `match` takes one pair, `match_many` a group of pairs of different sizes in one call; the outputs
are device tensors in the layout the module consumes, so the correspondences never visit the host.  The only read is the
correspondence count with the mutual check, which fixes the shapes; without it every source row is kept.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Sequence, Tuple

import torch

from . import _capi


@torch.no_grad()
def match_many(pairs: Sequence[Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]],
               use_mutual: bool = False) -> Dict[str, object]:
    """Matching and network input of P pairs in one call (pdsc_match_packed).  `pairs`: (src_desc [Ns,D], tgt_desc [Nt,D],
    src_keypts [Ns,3], tgt_keypts [Nt,3]) device tensors, one dtype for every descriptor.  Each pair is matched exactly as
    `match` matches it alone, against its own targets only.  Returns the pairs' kept correspondences packed back to back,
    pair p in rows offsets[p]:offsets[p+1] and centred by its own mean: {'corr' [M,2] int64 (pair-local source, target),
    'corr_pos' [M,6], 'src_keypts' [M,3], 'tgt_keypts' [M,3], 'offsets' (host list of P + 1 ints), 'd_offsets' (the same
    offsets as a device int32 tensor)} — what `PointDSC.forward_packed` takes.  Without the mutual check every source row is
    kept and nothing is read from the device; with it, the P + 1 offsets are read once."""
    if not pairs:
        raise ValueError("match_many needs at least one pair")
    dtype = pairs[0][0].dtype
    dev = pairs[0][0].device
    for i, (sd, td, sk, tk) in enumerate(pairs):
        if sd.device.type != "cuda" or td.device.type != "cuda":
            raise _capi.PdscError("pointdsc_b200.frontend.match runs on an H100 only: pass CUDA tensors (there is no CPU fallback)")
        if sd.device != dev or td.device != dev:
            raise ValueError(f"pair {i}: descriptors on {sd.device}, {td.device}; pair 0 is on {dev}")
        if sd.dtype != td.dtype or sd.dtype not in (torch.float32, torch.float64) or sd.dtype != dtype:
            raise ValueError("descriptors must all be float32 or all float64")
        if sd.dim() != 2 or td.dim() != 2 or sd.shape[1] != td.shape[1] or sd.shape[1] != pairs[0][0].shape[1]:
            raise ValueError(f"pair {i}: expected descriptors [Ns,D] and [Nt,D] of one D, got {tuple(sd.shape)}, {tuple(td.shape)}")
        if tuple(sk.shape) != (sd.shape[0], 3) or tuple(tk.shape) != (td.shape[0], 3):
            raise ValueError("key points must be [Ns,3] and [Nt,3]")
    lib, engine, stream = _capi.device_context(dev)
    P, d = len(pairs), int(pairs[0][0].shape[1])
    src_off, tgt_off = [0], [0]
    for sd, td, _, _ in pairs:
        src_off.append(src_off[-1] + int(sd.shape[0]))
        tgt_off.append(tgt_off[-1] + int(td.shape[0]))
    cat = lambda xs, dt: (torch.cat([x.to(device=dev, dtype=dt) for x in xs]) if len(xs) > 1  # noqa: E731
                          else xs[0].to(device=dev, dtype=dt)).contiguous()
    sd, td = cat([p[0] for p in pairs], dtype), cat([p[1] for p in pairs], dtype)
    sk, tk = cat([p[2] for p in pairs], torch.float32), cat([p[3] for p in pairs], torch.float32)
    d_in = _capi.host_to_device(src_off + tgt_off, torch.int32, dev)
    h_src, h_tgt = (C.c_int32 * (P + 1))(*src_off), (C.c_int32 * (P + 1))(*tgt_off)
    ns = src_off[-1]
    corr = torch.empty(ns, 2, dtype=torch.int32, device=dev)
    d_out = torch.empty(P + 1, dtype=torch.int32, device=dev)
    corr_pos = torch.empty(ns, 6, dtype=torch.float32, device=dev)
    out_src = torch.empty(ns, 3, dtype=torch.float32, device=dev)
    out_tgt = torch.empty(ns, 3, dtype=torch.float32, device=dev)
    scratch = _capi.scratch(lib.pdsc_match_packed_scratch_bytes(P, h_src, h_tgt), dev)
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_match_packed(engine, P, d, h_src, h_tgt, C.c_void_p(d_in.data_ptr()),
                                          C.c_void_p(d_in.data_ptr() + 4 * (P + 1)), C.c_void_p(sd.data_ptr()),
                                          C.c_void_p(td.data_ptr()), 1 if dtype == torch.float64 else 0, C.c_void_p(sk.data_ptr()),
                                          C.c_void_p(tk.data_ptr()), 1 if use_mutual else 0, C.c_void_p(corr.data_ptr()),
                                          C.c_void_p(d_out.data_ptr()), C.c_void_p(corr_pos.data_ptr()),
                                          C.c_void_p(out_src.data_ptr()), C.c_void_p(out_tgt.data_ptr()),
                                          C.c_void_p(scratch.data_ptr()), scratch.numel(), stream))
    offsets = [int(x) for x in d_out.cpu()] if use_mutual else src_off      # the only host read: it fixes the output shapes
    m = offsets[-1]
    return {"corr": corr[:m].long(), "corr_pos": corr_pos[:m], "src_keypts": out_src[:m], "tgt_keypts": out_tgt[:m],
            "offsets": offsets, "d_offsets": d_out}


@torch.no_grad()
def match(src_desc: torch.Tensor, tgt_desc: torch.Tensor, src_keypts: torch.Tensor, tgt_keypts: torch.Tensor,
          use_mutual: bool = False) -> Dict[str, torch.Tensor]:
    """-> {'corr' [M,2] int64 (source, target), 'corr_pos' [1,M,6], 'src_keypts' [1,M,3], 'tgt_keypts' [1,M,3]} on the device.

    Descriptors are L2-normalised rows, float32 (FCGF) or float64 (FPFH); the arithmetic runs in their dtype, as numpy's
    does in the reference.  Ready for `model({'corr_pos': ..., 'src_keypts': ..., 'tgt_keypts': ..., 'testing': True})`.
    `match_many` of one pair."""
    if src_desc.device.type != "cuda":
        raise _capi.PdscError("pointdsc_b200.frontend.match runs on an H100 only: pass CUDA tensors (there is no CPU fallback)")
    if src_desc.dtype != tgt_desc.dtype or src_desc.dtype not in (torch.float32, torch.float64):
        raise ValueError("descriptors must both be float32 or both float64")
    if src_desc.dim() != 2 or tgt_desc.dim() != 2 or src_desc.shape[1] != tgt_desc.shape[1]:
        raise ValueError(f"expected descriptors [Ns,D] and [Nt,D], got {tuple(src_desc.shape)}, {tuple(tgt_desc.shape)}")
    dev = src_desc.device
    sk = src_keypts.to(device=dev, dtype=torch.float32)
    tk = tgt_keypts.to(device=dev, dtype=torch.float32)
    out = match_many([(src_desc, tgt_desc, sk, tk)], use_mutual=use_mutual)
    return {"corr": out["corr"], "corr_pos": out["corr_pos"][None], "src_keypts": out["src_keypts"][None],
            "tgt_keypts": out["tgt_keypts"][None]}
