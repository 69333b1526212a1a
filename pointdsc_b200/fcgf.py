"""FCGF descriptors on the device (SURVEY.md section 8 row f8): the ResUNetBN2C network of the reference's misc/fcgf.py:621-867
and the feature extraction of misc/cal_fcgf.py:11-85, with no MinkowskiEngine.

    model = ResUNetBN2C(1, 32, bn_momentum=0.05, conv1_kernel_size=7, normalize_feature=True)    # cal_fcgf.py:344-350
    model.load_state_dict(load_checkpoint("ResUNetBN2C-feat32-3dmatch-v0.05.pth"))
    xyz_down, features = extract_features(model, xyz, voxel_size=0.05)                          # cal_fcgf.py:11-85

`ResUNetBN2C` only holds the weights, under MinkowskiEngine 0.5's names and shapes, so a released checkpoint loads with no missing
or unexpected key; the network itself runs in csrc/fcgf.cu (pdsc_fcgf_packed).  `fcgf_descriptors_many` describes a group of
clouds of different sizes in one call, as `descriptors.fpfh_descriptors_many` does for FPFH.  The conventions MinkowskiEngine
leaves to its implementation are stated in DESIGN.md row f8 (parity unpinned).  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch
from torch import nn

from . import _capi

CHANNELS = [None, 32, 64, 128, 256]
TR_CHANNELS = [None, 64, 64, 64, 128]
_STATUS = {1: "a non-finite coordinate, or one 2^20 voxels or more from the origin (the point is left out)"}


class _Conv(nn.Module):
    """A MinkowskiConvolution's parameters: `kernel` [K^3, Cin, Cout] ([Cin, Cout] for K = 1), optional `bias` [1, Cout]."""

    def __init__(self, cin: int, cout: int, kernel_size: int, bias: bool = False):
        super().__init__()
        shape = (kernel_size ** 3, cin, cout) if kernel_size > 1 else (cin, cout)
        self.kernel = nn.Parameter(torch.zeros(shape))
        self.bias = nn.Parameter(torch.zeros(1, cout)) if bias else None

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        key = prefix + "kernel"
        w = state_dict.get(key)
        if w is not None and self.kernel.dim() == 2 and tuple(w.shape) == (1,) + tuple(self.kernel.shape):
            state_dict[key] = w.reshape(self.kernel.shape)        # a 1x1 kernel saved as [1, Cin, Cout]
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)


class _Norm(nn.Module):
    """A MinkowskiBatchNorm: `bn` is the torch BatchNorm1d it wraps (keys normX.bn.*)."""

    def __init__(self, c: int, momentum: float):
        super().__init__()
        self.bn = nn.BatchNorm1d(c, momentum=momentum)


class _Block(nn.Module):
    """BasicBlockBN (misc/fcgf.py:107-158): conv1, norm1, conv2, norm2, no downsample."""

    def __init__(self, c: int, momentum: float):
        super().__init__()
        self.conv1, self.norm1 = _Conv(c, c, 3), _Norm(c, momentum)
        self.conv2, self.norm2 = _Conv(c, c, 3), _Norm(c, momentum)


class ResUNetBN2C(nn.Module):
    """The weights of misc/fcgf.py's ResUNetBN2C with MinkowskiEngine 0.5's names and shapes.  Only the configuration every
    reference caller uses is supported (one input channel, 32 output channels, normalised features); conv1_kernel_size is 7
    for the 3DMatch weights and 5 for the KITTI weights.  Calling the module describes a group of clouds
    (`fcgf_descriptors_many`)."""

    def __init__(self, in_channels: int = 1, out_channels: int = 32, bn_momentum: float = 0.05, conv1_kernel_size: int = 7,
                 normalize_feature: bool = True, D: int = 3):
        super().__init__()
        if in_channels != 1 or out_channels != 32 or not normalize_feature or D != 3:
            raise ValueError("ResUNetBN2C supports in_channels=1, out_channels=32, normalize_feature=True, D=3 only "
                             f"(got {in_channels}, {out_channels}, {normalize_feature}, {D})")
        if conv1_kernel_size not in (5, 7):
            raise ValueError(f"conv1_kernel_size must be 5 or 7 (got {conv1_kernel_size})")
        self.conv1_kernel_size = conv1_kernel_size
        ch, tr, m = CHANNELS, TR_CHANNELS, bn_momentum
        self.conv1, self.norm1, self.block1 = _Conv(1, ch[1], conv1_kernel_size), _Norm(ch[1], m), _Block(ch[1], m)
        self.conv2, self.norm2, self.block2 = _Conv(ch[1], ch[2], 3), _Norm(ch[2], m), _Block(ch[2], m)
        self.conv3, self.norm3, self.block3 = _Conv(ch[2], ch[3], 3), _Norm(ch[3], m), _Block(ch[3], m)
        self.conv4, self.norm4, self.block4 = _Conv(ch[3], ch[4], 3), _Norm(ch[4], m), _Block(ch[4], m)
        self.conv4_tr, self.norm4_tr, self.block4_tr = _Conv(ch[4], tr[4], 3), _Norm(tr[4], m), _Block(tr[4], m)
        self.conv3_tr, self.norm3_tr, self.block3_tr = _Conv(ch[3] + tr[4], tr[3], 3), _Norm(tr[3], m), _Block(tr[3], m)
        self.conv2_tr, self.norm2_tr, self.block2_tr = _Conv(ch[2] + tr[3], tr[2], 3), _Norm(tr[2], m), _Block(tr[2], m)
        self.conv1_tr = _Conv(ch[1] + tr[2], tr[1], 1)
        self.final = _Conv(tr[1], out_channels, 1, bias=True)
        self._handles: Dict[tuple, tuple] = {}     # key -> (handle, its finaliser)
        self.eval()

    def forward(self, clouds: Sequence[torch.Tensor], voxel_size: float):
        return fcgf_descriptors_many(self, clouds, voxel_size)

    def device_weights(self, device: torch.device) -> C.c_void_p:
        """The committed pdsc_fcgf handle of the current weights on `device` (made again when a weight has changed)."""
        index = device.index if device.index is not None else torch.cuda.current_device()
        sd = {k: v for k, v in self.state_dict().items() if not k.endswith("num_batches_tracked")}
        key = (index,) + tuple((k, v.data_ptr(), v._version) for k, v in sd.items())
        if key not in self._handles:
            lib = _capi.load()
            for _, free in self._handles.values():
                free()
            self._handles.clear()
            h = C.c_void_p()
            _capi.check(lib.pdsc_fcgf_create(self.conv1_kernel_size, C.byref(h)))
            free = weakref.finalize(self, lib.pdsc_fcgf_destroy, h)
            for name, v in sd.items():
                a = np.ascontiguousarray(v.detach().cpu().numpy(), dtype=np.float32)
                _capi.check(lib.pdsc_fcgf_set_param(h, name.encode(), a.ctypes.data_as(C.c_void_p), a.size))
            with torch.cuda.device(index):
                _capi.check(lib.pdsc_fcgf_commit(h))
            self._handles[key] = (h, free)
        return self._handles[key][0]


def load_checkpoint(path: str) -> Dict[str, torch.Tensor]:
    """The `state_dict` of a released FCGF checkpoint (`torch.load(path)['state_dict']`, cal_fcgf.py:354)."""
    return torch.load(path, map_location="cpu", weights_only=True)["state_dict"]


def conv1_kernel_size(state_dict: Dict[str, torch.Tensor]) -> int:
    """The conv1 kernel size a checkpoint was trained with, from its `conv1.kernel` shape (343 offsets: 7, 125: 5)."""
    k = state_dict["conv1.kernel"]
    size = {343: 7, 125: 5}.get(int(k.shape[0]))
    if size is None:
        raise ValueError(f"conv1.kernel has shape {tuple(k.shape)}: expected [343, 1, 32] (kernel 7) or [125, 1, 32] (kernel 5)")
    return size


def model_from_checkpoint(path: str) -> ResUNetBN2C:
    """ResUNetBN2C(1, 32, bn_momentum=0.05, conv1_kernel_size=<from the file>, normalize_feature=True) with the file's weights."""
    sd = load_checkpoint(path)
    model = ResUNetBN2C(1, 32, bn_momentum=0.05, conv1_kernel_size=conv1_kernel_size(sd), normalize_feature=True)
    model.load_state_dict(sd)
    return model


@torch.no_grad()
def fcgf_descriptors_many(model: ResUNetBN2C, clouds: Sequence[torch.Tensor],
                          voxel_size: float) -> Tuple[torch.Tensor, torch.Tensor, List[int], torch.Tensor]:
    """FCGF of P device clouds [n_p,3] in one call.  Returns (key points [M,3] float32, descriptors [M,32] float32, offsets (host
    list of P + 1 ints), d_offsets (the same offsets on the device)); cloud p's rows are offsets[p]:offsets[p+1], one per occupied
    voxel in order of its first point, and bit for bit what the cloud gives alone.  One host read, at the end."""
    if not clouds:
        raise ValueError("fcgf_descriptors_many needs at least one cloud")
    dev = clouds[0].device
    if dev.type != "cuda":
        raise _capi.PdscError("pointdsc_b200.fcgf runs on an H100 only: pass CUDA tensors (there is no CPU fallback)")
    for i, c in enumerate(clouds):
        if c.device != dev or c.dim() != 2 or c.shape[1] != 3 or c.shape[0] < 1:
            raise ValueError(f"cloud {i}: expected a [n,3] tensor on {dev} with n >= 1, got {tuple(c.shape)} on {c.device}")
    in_off = [0]
    for c in clouds:
        in_off.append(in_off[-1] + int(c.shape[0]))
    pts = (torch.cat([c.to(torch.float32) for c in clouds]) if len(clouds) > 1 else clouds[0].to(torch.float32)).contiguous()
    keypts, desc, meta = packed_call(model, pts, in_off, voxel_size)
    P = len(clouds)
    h_meta = meta.tolist()                                          # the one host read
    offsets = h_meta[:P + 1]
    for p, s in enumerate(h_meta[P + 1:]):
        if s:
            raise _capi.PdscError(f"cloud {p}: " + "; ".join(m for bit, m in _STATUS.items() if s & bit))
    m = offsets[-1]
    return keypts[:m], desc[:m], offsets, meta[:P + 1]


def packed_call(model: ResUNetBN2C, pts: torch.Tensor, in_off: Sequence[int], voxel_size: float, scratch=None, keypts=None,
                desc=None):
    """One pdsc_fcgf_packed call over packed device points [n,3] float32 with host offsets `in_off`: (key points [n,3], descriptors
    [n,32], meta [2P + 1] int32 = key-point offsets then status), nothing read back.  `scratch`, `keypts`, `desc`: caller-owned
    buffers (tests read the scratch through pdsc_fcgf_scratch_layout); allocated here when None."""
    dev = pts.device
    lib, engine, stream = _capi.device_context(dev)
    h = model.device_weights(dev)
    P, n = len(in_off) - 1, int(in_off[-1])
    h_in, d_in = _capi.offsets(list(in_off), None, dev)
    keypts = torch.empty(n, 3, dtype=torch.float32, device=dev) if keypts is None else keypts
    desc = torch.empty(n, 32, dtype=torch.float32, device=dev) if desc is None else desc
    meta = torch.empty(2 * P + 1, dtype=torch.int32, device=dev)
    if scratch is None:
        nbytes = lib.pdsc_fcgf_packed_scratch_bytes(h, P, h_in)
        if nbytes == 0:
            raise ValueError(f"pdsc_fcgf_packed: unsupported group ({P} clouds, {n} points; at most 2^26 points in all)")
        scratch = _capi.scratch(nbytes, dev, align=256)
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_fcgf_packed(engine, h, P, h_in, C.c_void_p(d_in.data_ptr()), C.c_void_p(pts.data_ptr()),
                                         float(voxel_size), C.c_void_p(keypts.data_ptr()), C.c_void_p(desc.data_ptr()),
                                         C.c_void_p(meta.data_ptr()), C.c_void_p(meta.data_ptr() + 4 * (P + 1)),
                                         C.c_void_p(scratch.data_ptr()), scratch.numel(), stream))
    return keypts, desc, meta


def scratch_layout(model: ResUNetBN2C, in_off: Sequence[int]) -> Tuple[int, List[int]]:
    """(scratch bytes, byte offsets of the regions pdsc_fcgf_scratch_layout reports) of a call over `in_off` (a test aid)."""
    lib = _capi.load()
    h = model.device_weights(torch.device("cuda", torch.cuda.current_device()))
    h_in = (C.c_int32 * len(in_off))(*in_off)
    out = (C.c_int64 * 64)()
    k = lib.pdsc_fcgf_scratch_layout(h, len(in_off) - 1, h_in, out, 64)
    return int(lib.pdsc_fcgf_packed_scratch_bytes(h, len(in_off) - 1, h_in)), [int(v) for v in out[:k]]


def extract_features(model: ResUNetBN2C, xyz, rgb=None, normal=None, voxel_size: float = 0.05, device=None, skip_check=False,
                     is_eval=True):
    """misc/cal_fcgf.py's extract_features: (return_coords = xyz[inds] [m,3] numpy, features [m,32] float32 on the device).
    The point coordinates are taken as float32 (what PLY files and pdsc_read_ply hold); rgb and normal inputs are not supported."""
    if rgb is not None or normal is not None:
        raise ValueError("FCGF with rgb or normal input features is not supported (no reference caller uses it)")
    xyz_np = xyz.detach().cpu().numpy() if torch.is_tensor(xyz) else np.asarray(xyz)
    if xyz_np.ndim != 2 or xyz_np.shape[1] != 3:
        raise ValueError(f"xyz must be [N,3], got {xyz_np.shape}")
    dev = torch.device(device) if device is not None else torch.device("cuda")
    pts = torch.from_numpy(np.ascontiguousarray(xyz_np, dtype=np.float32)).to(dev)
    keypts, feat, _, _ = fcgf_descriptors_many(model, [pts], voxel_size)
    return keypts.cpu().numpy().astype(xyz_np.dtype), feat
