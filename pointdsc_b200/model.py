"""Drop-in `PointDSC` module backed by the H100 engine.

Boundary mirrored (reference models/PointDSC.py):
  * constructor signature and defaults                                   :81-91
  * parameter / buffer names, so `load_state_dict(torch.load('snapshot/<X>/models/model_best.pkl'),
    strict=False)` reports missing=[] and unexpected=['gamma'] exactly as the reference does   :93-113
  * `forward(data: dict) -> dict` with keys corr_pos / src_keypts / tgt_keypts and the presence of
    'testing' selecting test mode; returns final_trans [bs,4,4], final_labels [bs,N], M=None   :128-197

Differences, all deliberate:
  * testing mode accepts bs > 1 and defines it as the loop of bs == 1 reference calls (the reference
    asserts bs == 1, :210/:414);
  * there is NO CPU / PyTorch fallback: the module's sub-modules are parameter containers only, the
    arithmetic lives in libpointdsc_b200.so and every call fails loudly without it;
  * without the 'testing' key the module computes the reference's validation forward (:158-165, :176,
    :190-191: top-S seeds, batch-wide early exit, no refinement, logits as final_labels, M) in eval
    mode only; the training-mode forward (batch statistics in BatchNorm) and the backward pass are
    outside this engine and raise.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Iterable, List, Optional, Sequence

import torch
import torch.nn as nn

from . import _capi

DEFAULT_PRECISION = os.environ.get("POINTDSC_PRECISION", "fp16x3")

_TAP_SPECS = {
    # name: (dtype, shape as a function of (B, N, S, k, C))
    "sc": (torch.float32, lambda B, N, S, k, c: (B, N, N)),
    "features": (torch.float32, lambda B, N, S, k, c: (B, N, c)),
    "normed": (torch.float32, lambda B, N, S, k, c: (B, N, c)),
    "confidence": (torch.float32, lambda B, N, S, k, c: (B, N)),
    "seeds": (torch.int32, lambda B, N, S, k, c: (B, S)),
    "knn_idx": (torch.int32, lambda B, N, S, k, c: (B, S, k)),
    "compat": (torch.float32, lambda B, N, S, k, c: (B, S, k, k)),
    "eig": (torch.float32, lambda B, N, S, k, c: (B, S, k)),
    "power_iters": (torch.int32, lambda B, N, S, k, c: (B,)),
    "seed_trans": (torch.float32, lambda B, N, S, k, c: (B, S, 4, 4)),
    "inlier_counts": (torch.int32, lambda B, N, S, k, c: (B, S)),
    "best": (torch.int32, lambda B, N, S, k, c: (B,)),
    "init_trans": (torch.float32, lambda B, N, S, k, c: (B, 4, 4)),
    "refine_solves": (torch.int32, lambda B, N, S, k, c: (B,)),
    "layer_features": (torch.float32, lambda B, N, S, k, c: (B, N, c)),
    "layer_debug": (torch.float32, lambda B, N, S, k, c: (5, B, N, c)),
    "timeline": (torch.int64, lambda B, N, S, k, c: (2, 16, 4, 8)),
}
_INJECT_DTYPES = {"features": torch.float32, "confidence": torch.float32, "seeds": torch.int32,
                  "knn_idx": torch.int32, "seed_trans": torch.float32}


def _conv(cin, cout):
    return nn.Conv1d(cin, cout, kernel_size=1, bias=True)


class _NonLocalParams(nn.Module):
    """Parameters of one SCNonlocal block, named as in the reference (PointDSC.py:9-25)."""

    def __init__(self, c: int):
        super().__init__()
        h = c // 2
        self.fc_message = nn.Sequential(_conv(c, h), nn.BatchNorm1d(h), nn.ReLU(inplace=True),
                                        _conv(h, h), nn.BatchNorm1d(h), nn.ReLU(inplace=True), _conv(h, c))
        self.projection_q = _conv(c, c)
        self.projection_k = _conv(c, c)
        self.projection_v = _conv(c, c)


class _EncoderParams(nn.Module):
    """Parameters of the NonLocalNet encoder, named as in the reference (PointDSC.py:48-63)."""

    def __init__(self, in_dim: int, num_layers: int, c: int):
        super().__init__()
        self.num_layers = num_layers
        self.blocks = nn.ModuleDict()
        self.layer0 = _conv(in_dim, c)
        for i in range(num_layers):
            self.blocks[f"PointCN_layer_{i}"] = nn.Sequential(_conv(c, c), nn.BatchNorm1d(c), nn.ReLU(inplace=True))
            self.blocks[f"NonLocal_layer_{i}"] = _NonLocalParams(c)


class PointDSC(nn.Module):
    def __init__(self, in_dim=6, num_layers=6, num_channels=128, num_iterations=10, ratio=0.1,
                 inlier_threshold=0.10, sigma_d=0.10, k=40, nms_radius=0.10, *, precision: Optional[str] = None,
                 batch_invariant: bool = False):
        super().__init__()
        self.in_dim = in_dim
        self.num_layers = num_layers
        self.num_iterations = num_iterations
        self.ratio = ratio
        self.num_channels = num_channels
        self.inlier_threshold = inlier_threshold
        self.k = k
        self.nms_radius = nms_radius
        self.precision = precision or DEFAULT_PRECISION
        if self.precision not in _capi.PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(_capi.PRECISIONS)}, got {self.precision!r}")
        # batch-invariant mode (pdsc_set_batch_invariant): every set's result is independent of its call and of the device's
        # SM count, at the cost measured in DESIGN.md §4; a plain attribute, not part of the state dict
        self.batch_invariant = bool(batch_invariant)
        self.sigma = nn.Parameter(torch.tensor([1.0], dtype=torch.float32), requires_grad=True)
        self.sigma_spat = nn.Parameter(torch.tensor([sigma_d], dtype=torch.float32), requires_grad=False)
        self.encoder = _EncoderParams(in_dim, num_layers, num_channels)
        self.classification = nn.Sequential(_conv(num_channels, 32), nn.ReLU(inplace=True), _conv(32, 32),
                                            nn.ReLU(inplace=True), _conv(32, 1))
        for m in self.modules():  # same initialisation scheme as the reference (PointDSC.py:116-121)
            if isinstance(m, nn.Conv1d):
                nn.init.xavier_normal_(m.weight, gain=1)
            elif isinstance(m, nn.BatchNorm1d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        self._engine = None
        self._engine_device = None
        self._engine_hyper = None
        self._pushed_signature = None
        self._pushed_invariant = None
        self._workspaces = {}     # CUDA stream handle -> scratch tensor (two streams never share scratch)
        self._static = {}         # (B, N, stream) -> address-stable buffers of the graph-replay path
        self.graph_rows = 32768   # calls with B * N at most this replay a captured CUDA graph (launch-bound regime)

    # ------------------------------------------------------------------------------------------
    # engine plumbing
    # ------------------------------------------------------------------------------------------
    def _device(self) -> torch.device:
        return self.sigma.device

    def _signature(self):
        return tuple((t._version, t.data_ptr()) for t in self.state_dict(keep_vars=True).values()) + (self.precision,)

    def _hyper(self):
        """Constructor hyper-parameters the engine bakes into its configuration; the reference reads `self.*` on every call,
        so a change after construction (e.g. `model.k = 80`) must reach the engine."""
        return (int(self.in_dim), int(self.num_layers), int(self.num_channels), int(self.num_iterations), float(self.ratio),
                float(self.inlier_threshold), int(self.k), float(self.nms_radius))

    def _ensure_engine(self):
        dev = self._device()
        if dev.type != "cuda":
            raise _capi.PdscError("pointdsc_b200.PointDSC runs on an H100 only: move the module to CUDA "
                                  "(`model.cuda()`); there is no CPU fallback")
        lib = _capi.load()
        index = dev.index if dev.index is not None else torch.cuda.current_device()
        if self._engine is None or self._engine_device != index or self._engine_hyper != self._hyper():
            self._release()
            self._workspaces, self._static = {}, {}
            self._engine_hyper = self._hyper()
            cfg = _capi.Config(self.in_dim, self.num_layers, self.num_channels, self.num_iterations, self.ratio,
                               self.inlier_threshold, float(self.sigma_spat.detach().cpu()[0]), self.k,
                               self.nms_radius, _capi.PRECISIONS[self.precision], index)
            handle = C.c_void_p()
            _capi.check(lib.pdsc_create(C.byref(cfg), C.byref(handle)))
            self._engine, self._engine_device, self._pushed_signature = handle, index, None
            self._pushed_invariant = None
        if self._pushed_invariant != self.batch_invariant:
            _capi.check(lib.pdsc_set_batch_invariant(self._engine, 1 if self.batch_invariant else 0))
            self._pushed_invariant = self.batch_invariant
        sig = self._signature()
        if sig != self._pushed_signature:
            _capi.check(lib.pdsc_set_precision(self._engine, _capi.PRECISIONS[self.precision]))
            for name, t in self.state_dict().items():
                if not t.is_floating_point():
                    continue  # num_batches_tracked
                h = t.detach().to(device="cpu", dtype=torch.float32).contiguous()
                _capi.check(lib.pdsc_set_param(self._engine, name.encode(), C.c_void_p(h.data_ptr()), h.numel()))
            _capi.check(lib.pdsc_commit_params(self._engine))
            self._pushed_signature = sig
        return lib

    def _release(self):
        if self._engine is not None:
            try:
                _capi.load().pdsc_destroy(self._engine)
            except Exception:
                pass
            object.__setattr__(self, "_engine", None)

    def __del__(self):
        try:
            self._release()
        except Exception:  # interpreter shutdown: torch / ctypes may already be torn down
            pass

    def set_precision(self, precision: str):
        if precision not in _capi.PRECISIONS:
            raise ValueError(precision)
        self.precision = precision
        self._workspaces, self._static = {}, {}

    def set_batch_invariant(self, enable: bool):
        """Turn the batch-invariant mode on or off (see the constructor); the next call of any entry point runs in it."""
        self.batch_invariant = bool(enable)
        self._workspaces, self._static = {}, {}

    def launches_per_forward(self, B: int, N: int) -> int:
        lib = self._ensure_engine()
        return int(lib.pdsc_launches_per_forward(self._engine, B, N))

    def profile(self, enable: bool):
        """Turn the engine's CUDA-event stage profiling on/off (pdsc_profile_enable)."""
        lib = self._ensure_engine()
        _capi.check(lib.pdsc_profile_enable(self._engine, 1 if enable else 0))

    def profile_read(self):
        """{span: (milliseconds, launches)} accumulated since the last read (pdsc_profile_read)."""
        lib = self._ensure_engine()
        ms = (C.c_float * len(_capi.SPANS))()
        cnt = (C.c_int32 * len(_capi.SPANS))()
        _capi.check(lib.pdsc_profile_read(self._engine, ms, cnt))
        return {n: (float(ms[i]), int(cnt[i])) for i, n in enumerate(_capi.SPANS)}

    def num_seeds(self, N: int) -> int:
        """Seeds of a set of N correspondences: the length of the reference's slice argsort(...)[:, 0:int(N * ratio)]
        (PointDSC.py:174, :217), as pdsc_num_seeds computes it."""
        m = int(N * self.ratio)
        return min(m, N) if m >= 0 else max(N + m, 0)

    # ------------------------------------------------------------------------------------------
    # the path
    # ------------------------------------------------------------------------------------------
    def forward(self, data: Dict[str, torch.Tensor]) -> Dict[str, Optional[torch.Tensor]]:
        testing = "testing" in data.keys()
        if not testing:
            if self.training:
                raise NotImplementedError(
                    "pointdsc_b200 computes the forward with eval-mode BatchNorm (running statistics) and has no backward "
                    "pass: call model.eval() for validation; training stays with the reference (libs/trainer.py)")
            out = self.run_eval(data["corr_pos"], data["src_keypts"], data["tgt_keypts"])
            return {"final_trans": out["final_trans"], "final_labels": out["final_labels"], "M": out["M"]}
        out = self.run(data["corr_pos"], data["src_keypts"], data["tgt_keypts"])
        return {"final_trans": out["final_trans"], "final_labels": out["final_labels"], "M": None}

    @torch.no_grad()
    def forward_stream(self, batches: Iterable[Dict[str, torch.Tensor]]):
        """Testing-mode forwards over an iterable of HOST batches as a two-deep pipeline: yields, in order, what `forward`
        returns for each element (host tensors).  This is the evaluation drivers' loop (`for data in loader: res = model(data)`,
        evaluation/test_3DMatch.py:64-101) with the copies taken off the critical path: while the device runs the forward of
        batch t, the inputs of batch t + 1 are already crossing to the device and the results of batch t - 1 are crossing back
        (pdsc_forward_host_submit / _wait).  Results are bit-identical to `forward`'s.  Page-locked input tensors
        (`tensor.pin_memory()`, or a DataLoader with pin_memory=True) are needed for the overlap, not for correctness.
        Batches already on the device are simply run in order."""
        lib = self._ensure_engine()
        dev = self._device()
        # results go straight into fresh caller-owned (pageable) tensors, written by the library's device->host copies inside
        # _wait: on the GPU boxes a CPU read of page-locked memory is slow (a 1 MB torch-side clone out of a pinned result buffer
        # took ~5 ms and made the host the bottleneck of the loop), and allocating page-locked memory synchronises the device
        pending = None             # (slot, trans, labels, inputs kept alive)
        count = 0

        def collect(p):
            _capi.check(lib.pdsc_forward_host_wait(self._engine, p[0]))
            return {"final_trans": p[1], "final_labels": p[2], "M": None}

        try:
            for data in batches:
                if "testing" not in data.keys():
                    raise ValueError("forward_stream is the testing-mode loop: every batch needs the 'testing' key")
                cp, s, t = data["corr_pos"], data["src_keypts"], data["tgt_keypts"]
                if cp.device.type != "cpu":
                    if pending is not None:
                        p, pending = pending, None
                        yield collect(p)
                    yield self.forward(data)
                    continue
                if cp.dim() != 3 or s.shape[:2] != cp.shape[:2] or t.shape != s.shape or s.shape[-1] != 3 \
                        or cp.shape[-1] != self.in_dim:
                    raise ValueError(f"expected corr_pos [bs,N,{self.in_dim}] and src/tgt_keypts [bs,N,3], got "
                                     f"{tuple(cp.shape)}, {tuple(s.shape)}, {tuple(t.shape)}")
                cp, s, t = (x.to(torch.float32).contiguous() for x in (cp, s, t))
                B, N = int(cp.shape[0]), int(cp.shape[1])
                b = (torch.empty(B, 4, 4, dtype=torch.float32), torch.empty(B, N, dtype=torch.float32))
                slot = C.c_int32(-1)
                with torch.cuda.device(dev):
                    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
                    _capi.check(lib.pdsc_forward_host_submit(
                        self._engine, B, N, C.c_void_p(cp.data_ptr()), C.c_void_p(s.data_ptr()), C.c_void_p(t.data_ptr()),
                        C.c_void_p(b[0].data_ptr()), C.c_void_p(b[1].data_ptr()), stream, C.byref(slot)))
                cur = (int(slot.value), b[0], b[1], (cp, s, t))
                count += 1
                if pending is not None:
                    p, pending = pending, cur
                    yield collect(p)
                else:
                    pending = cur
            if pending is not None:
                p, pending = pending, None
                yield collect(p)
        finally:
            if pending is not None:      # the consumer stopped early: do not leave a call in flight
                try:
                    lib.pdsc_forward_host_wait(self._engine, pending[0])
                except Exception:
                    pass

    @torch.no_grad()
    def forward_many(self, batches: List[Dict[str, torch.Tensor]]) -> List[Dict[str, Optional[torch.Tensor]]]:
        """Testing-mode forwards of several batches of DIFFERENT sizes in one engine call (pdsc_forward_packed).  Each element
        is what `forward` accepts in testing mode (device tensors [bs_i, N_i, ...] and the 'testing' key); the result is, per
        element, what `forward` returns for it.  All their sets are packed back to back into one mixed-size call, so a loop
        over data of varying N pays one call's latency instead of one per pair.  Within one attention regime (DESIGN.md §3)
        every set's result is bit-identical to that of a `forward` call holding it; with `batch_invariant` on, to that of every
        call holding it."""
        dev = self._device()
        sizes = []
        for i, data in enumerate(batches):
            if "testing" not in data.keys():
                raise ValueError(f"forward_many runs the testing-mode forward: batch {i} has no 'testing' key")
            cp, s, t = data["corr_pos"], data["src_keypts"], data["tgt_keypts"]
            if cp.dim() != 3 or s.shape[:2] != cp.shape[:2] or t.shape != s.shape or s.shape[-1] != 3 \
                    or cp.shape[-1] != self.in_dim:
                raise ValueError(f"batch {i}: expected corr_pos [bs,N,{self.in_dim}] and src/tgt_keypts [bs,N,3], got "
                                 f"{tuple(cp.shape)}, {tuple(s.shape)}, {tuple(t.shape)}")
            if any(x.device.type != "cuda" or x.device != dev for x in (cp, s, t)):
                raise ValueError(f"batch {i}: inputs must be device tensors on {dev} (got {cp.device}, {s.device}, {t.device})")
            sizes.append((int(cp.shape[0]), int(cp.shape[1])))
        if not batches:
            return []
        counts = [n for bs, n in sizes for _ in range(bs)]
        offsets = [0]
        for n in counts:
            offsets.append(offsets[-1] + n)
        cp, s, t = (torch.cat([d[key].to(torch.float32).reshape(-1, d[key].shape[-1]) for d in batches]).contiguous()
                    for key in ("corr_pos", "src_keypts", "tgt_keypts"))
        res = self.forward_packed(cp, s, t, offsets)
        trans, labels = res["final_trans"], res["final_labels"]
        out, set0, row0 = [], 0, 0
        for bs, n in sizes:
            out.append({"final_trans": trans[set0:set0 + bs], "final_labels": labels[row0:row0 + bs * n].view(bs, n), "M": None})
            set0 += bs
            row0 += bs * n
        return out

    @torch.no_grad()
    def forward_packed(self, corr_pos: torch.Tensor, src_keypts: torch.Tensor, tgt_keypts: torch.Tensor, offsets: Sequence[int],
                       d_offsets: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """The testing-mode forward of B sets already packed back to back (pdsc_forward_packed): set b owns rows
        offsets[b]:offsets[b+1] of corr_pos [R,in_dim], src_keypts [R,3] and tgt_keypts [R,3] (device tensors), as
        `frontend.match_many` returns them.  `offsets`: B + 1 host ints; `d_offsets`: the same values as a device int32 tensor
        (uploaded without a stream synchronisation when omitted).  -> {'final_trans' [B,4,4], 'final_labels' [R]}; set b's
        results are what `forward_many` returns for it."""
        dev = self._device()
        offsets = [int(x) for x in offsets]
        R = int(corr_pos.shape[0]) if corr_pos.dim() == 2 else -1
        if corr_pos.dim() != 2 or corr_pos.shape[1] != self.in_dim or tuple(src_keypts.shape) != (R, 3) \
                or tuple(tgt_keypts.shape) != (R, 3):
            raise ValueError(f"expected corr_pos [R,{self.in_dim}] and src/tgt_keypts [R,3], got {tuple(corr_pos.shape)}, "
                             f"{tuple(src_keypts.shape)}, {tuple(tgt_keypts.shape)}")
        if any(x.device.type != "cuda" or x.device != dev for x in (corr_pos, src_keypts, tgt_keypts)):
            raise ValueError(f"inputs must be device tensors on {dev} (got {corr_pos.device}, {src_keypts.device}, {tgt_keypts.device})")
        if len(offsets) < 2 or offsets[-1] != R:
            raise ValueError(f"expected B + 1 >= 2 offsets ending at R = {R}, got {len(offsets)} ending at {offsets[-1:]}")
        lib = self._ensure_engine()
        B = len(offsets) - 1
        h_off, d_off = _capi.offsets(offsets, d_offsets, dev)
        cp, s, t = (x.to(torch.float32).contiguous() for x in (corr_pos, src_keypts, tgt_keypts))
        need = int(lib.pdsc_workspace_bytes_packed(self._engine, B, h_off))
        if need == 0:
            _capi.check(_capi.PDSC_ERR_SHAPE)
        stream_handle = torch.cuda.current_stream(dev).cuda_stream
        workspace = self._workspace_for(dev, need, stream_handle)
        trans = torch.empty(B, 4, 4, dtype=torch.float32, device=dev)
        labels = torch.empty(R, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _capi.check(lib.pdsc_forward_packed(self._engine, B, h_off, C.c_void_p(d_off.data_ptr()), C.c_void_p(cp.data_ptr()),
                                                C.c_void_p(s.data_ptr()), C.c_void_p(t.data_ptr()),
                                                C.c_void_p(trans.data_ptr()), C.c_void_p(labels.data_ptr()),
                                                C.c_void_p(workspace.data_ptr()), workspace.numel(),
                                                C.c_void_p(stream_handle)))
        return {"final_trans": trans, "final_labels": labels}

    def _workspace_for(self, dev, need: int, stream_handle: int) -> torch.Tensor:
        ws = self._workspaces.get(stream_handle)
        if ws is None or ws.numel() < need or ws.device != dev:
            self._workspaces.pop(stream_handle, None)
            if len(self._workspaces) >= 4:          # scratch of streams no longer in use
                self._workspaces.pop(next(iter(self._workspaces)))
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            self._workspaces[stream_handle] = ws
        return ws

    @torch.no_grad()
    def run_eval(self, corr_pos: torch.Tensor, src_keypts: torch.Tensor, tgt_keypts: torch.Tensor, want_M: bool = True,
                 taps: Iterable[str] = ()):
        """The forward WITHOUT the 'testing' key (reference PointDSC.py:158-165, :176, :190-191), eval-mode BatchNorm:
        final_trans [bs,4,4] (best hypothesis, no refinement), final_labels [bs,N] = confidence logits, M [bs,N,N]."""
        lib = self._ensure_engine()
        dev = self._device()
        if corr_pos.device != dev:
            raise ValueError(f"inputs are on {corr_pos.device}, module is on {dev}")
        cp, s, t = (x.to(torch.float32).contiguous() for x in (corr_pos, src_keypts, tgt_keypts))
        B, N = int(cp.shape[0]), int(cp.shape[1])
        S = int(lib.pdsc_num_seeds(self._engine, N))
        k = int(lib.pdsc_num_neighbours(self._engine, N))
        stream = torch.cuda.current_stream(dev).cuda_stream
        ws = self._workspace_for(dev, int(lib.pdsc_workspace_bytes(self._engine, B, N)), stream)
        trans = torch.empty(B, 4, 4, dtype=torch.float32, device=dev)
        conf = torch.empty(B, N, dtype=torch.float32, device=dev)
        M = torch.empty(B, N, N, dtype=torch.float32, device=dev) if want_M else None
        io_ptr, extra = None, {}
        if taps:
            io = _capi.StageIO()
            for name in taps:
                dtype, shape = _TAP_SPECS[name]
                extra[name] = torch.zeros(shape(B, N, S, k, self.num_channels), dtype=dtype, device=dev)
                setattr(io, "out_" + name, extra[name].data_ptr())
            io_ptr = C.byref(io)
        with torch.cuda.device(dev):
            _capi.check(lib.pdsc_forward_eval(self._engine, B, N, C.c_void_p(cp.data_ptr()), C.c_void_p(s.data_ptr()),
                                              C.c_void_p(t.data_ptr()), C.c_void_p(trans.data_ptr()), C.c_void_p(conf.data_ptr()),
                                              C.c_void_p(M.data_ptr()) if want_M else None, io_ptr, C.c_void_p(ws.data_ptr()),
                                              ws.numel(), C.c_void_p(stream)))
        out = {"final_trans": trans, "final_labels": conf, "M": M}
        out.update(extra)
        return out

    @torch.no_grad()
    def run(self, corr_pos: torch.Tensor, src_keypts: torch.Tensor, tgt_keypts: torch.Tensor,
            taps: Iterable[str] = (), inject: Optional[Dict[str, torch.Tensor]] = None, layer_tap: int = 0):
        """Testing-mode forward.  `taps` / `inject` expose the stage boundaries of SURVEY.md §8(a) for the
        parity tests (names: see _TAP_SPECS / _INJECT_DTYPES).  Host tensors take the end-to-end path
        (pdsc_forward_host: H2D + forward + D2H inside the call) and return host tensors."""
        if corr_pos.dim() != 3 or src_keypts.shape[:2] != corr_pos.shape[:2] or tgt_keypts.shape != src_keypts.shape \
                or src_keypts.shape[-1] != 3 or corr_pos.shape[-1] != self.in_dim:
            raise ValueError(f"expected corr_pos [bs,N,{self.in_dim}] and src/tgt_keypts [bs,N,3], got "
                             f"{tuple(corr_pos.shape)}, {tuple(src_keypts.shape)}, {tuple(tgt_keypts.shape)}")
        lib = self._ensure_engine()
        dev = self._device()
        B, N = int(corr_pos.shape[0]), int(corr_pos.shape[1])
        stream_handle = torch.cuda.current_stream(dev).cuda_stream
        stream = C.c_void_p(stream_handle)
        if corr_pos.device.type == "cpu":
            if taps or inject:
                raise ValueError("taps / inject need device tensors")
            cp, s, t = (x.to(torch.float32).contiguous() for x in (corr_pos, src_keypts, tgt_keypts))
            # fresh caller-owned result tensors, written by the library's device->host copies (pageable destination: the
            # 1 MB copy is staged by the driver; a torch-side clone out of a pinned buffer costs more than the copy itself)
            trans = torch.empty(B, 4, 4, dtype=torch.float32)
            labels = torch.empty(B, N, dtype=torch.float32)
            with torch.cuda.device(dev):
                _capi.check(lib.pdsc_forward_host(self._engine, B, N, C.c_void_p(cp.data_ptr()), C.c_void_p(s.data_ptr()),
                                                  C.c_void_p(t.data_ptr()), C.c_void_p(trans.data_ptr()),
                                                  C.c_void_p(labels.data_ptr()), stream))
            return {"final_trans": trans, "final_labels": labels}
        if corr_pos.device != dev:
            raise ValueError(f"inputs are on {corr_pos.device}, module is on {dev}")
        cp, s, t = (x.to(torch.float32).contiguous() for x in (corr_pos, src_keypts, tgt_keypts))
        S = int(lib.pdsc_num_seeds(self._engine, N))
        k = int(lib.pdsc_num_neighbours(self._engine, N))
        need = int(lib.pdsc_workspace_bytes(self._engine, B, N))
        if not taps and not inject and B * N <= self.graph_rows and not torch.cuda.is_current_stream_capturing():
            # launch-bound regime (the evaluation loops' bs = 1): inputs are copied into address-stable buffers and the ~60
            # kernels of the forward are replayed as ONE captured graph (pdsc_forward_graph); results are fresh tensors
            key = (B, N, stream_handle)
            st = self._static.get(key)
            if st is None:
                if len(self._static) >= 8:
                    self._static.pop(next(iter(self._static)))
                st = {"cp": torch.empty_like(cp), "s": torch.empty_like(s), "t": torch.empty_like(t),
                      "trans": torch.empty(B, 4, 4, dtype=torch.float32, device=dev),
                      "labels": torch.empty(B, N, dtype=torch.float32, device=dev),
                      "ws": torch.empty(need, dtype=torch.uint8, device=dev)}
                self._static[key] = st
            st["cp"].copy_(cp); st["s"].copy_(s); st["t"].copy_(t)
            with torch.cuda.device(dev):
                _capi.check(lib.pdsc_forward_graph(self._engine, B, N, C.c_void_p(st["cp"].data_ptr()),
                                                   C.c_void_p(st["s"].data_ptr()), C.c_void_p(st["t"].data_ptr()),
                                                   C.c_void_p(st["trans"].data_ptr()), C.c_void_p(st["labels"].data_ptr()),
                                                   C.c_void_p(st["ws"].data_ptr()), st["ws"].numel(), stream))
            return {"final_trans": st["trans"].clone(), "final_labels": st["labels"].clone()}
        workspace = self._workspace_for(dev, need, stream_handle)
        trans = torch.empty(B, 4, 4, dtype=torch.float32, device=dev)
        labels = torch.empty(B, N, dtype=torch.float32, device=dev)
        io_ptr, extra, keep = None, {}, []
        if taps or inject:
            io = _capi.StageIO()
            for name in taps:
                dtype, shape = _TAP_SPECS[name]
                buf = torch.zeros(shape(B, N, S, k, self.num_channels), dtype=dtype, device=dev)
                extra[name] = buf
                setattr(io, "out_" + name, buf.data_ptr())
            io.layer_tap = int(layer_tap)
            for name, val in (inject or {}).items():
                v = val.to(device=dev, dtype=_INJECT_DTYPES[name]).contiguous()
                keep.append(v)
                setattr(io, "in_" + ("knn_idx" if name == "knn_idx" else name), v.data_ptr())
            io_ptr = C.byref(io)
        _capi.check(lib.pdsc_forward(self._engine, B, N, C.c_void_p(cp.data_ptr()), C.c_void_p(s.data_ptr()),
                                     C.c_void_p(t.data_ptr()), C.c_void_p(trans.data_ptr()),
                                     C.c_void_p(labels.data_ptr()), io_ptr, C.c_void_p(workspace.data_ptr()),
                                     workspace.numel(), stream))
        if keep:
            torch.cuda.current_stream(dev).synchronize()  # injected temporaries must outlive the enqueued work
        out = {"final_trans": trans, "final_labels": labels}
        out.update(extra)
        return out
