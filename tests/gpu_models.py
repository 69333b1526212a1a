"""Set-up the GPU tests share: the snapshot modules and their session cache, the SM count the engine sizes its launches for,
device inputs and byte-level comparisons."""
import os

import numpy as np
import torch

from conftest import load_snapshot
from oracle import pointdsc_oracle as O

_models = {}


def get_model(dataset="3dmatch", precision="fp32", *, k=40, iters=10, invariant=False, fresh=False, num_layers=12, in_dim=6,
              ratio=0.1, inlier_threshold=None, weights=None):
    """A PointDSC module on the device with its engine created: the dataset's constructor arguments (O.default_config;
    inlier_threshold overrides its threshold) and its snapshot, or `weights` = (name, state dict) in its place.

    One module per argument set is kept for the session; a test that changes a module's settings or releases its engine
    asks for a module of its own with fresh=True."""
    from pointdsc_b200 import PointDSC
    key = (dataset, precision, k, iters, invariant, num_layers, in_dim, ratio, inlier_threshold, weights and weights[0])
    if fresh or key not in _models:
        cfg = O.default_config(dataset)
        m = PointDSC(in_dim=in_dim, num_layers=num_layers, num_channels=128, num_iterations=iters, ratio=ratio,
                     inlier_threshold=cfg["inlier_threshold"] if inlier_threshold is None else inlier_threshold,
                     sigma_d=cfg["sigma_d"], k=k, nms_radius=cfg["nms_radius"], precision=precision, batch_invariant=invariant)
        res = m.load_state_dict(load_snapshot(dataset) if weights is None else weights[1], strict=False)
        assert res.missing_keys == [] and res.unexpected_keys == ["gamma"], res
        m = m.cuda().eval()
        m._ensure_engine()
        if fresh:
            return m
        _models[key] = m
    return _models[key]


def release_all():
    """Release every cached module and its engine, and the allocator's cache: for a test that needs the device's memory."""
    for m in _models.values():
        m._release()
    _models.clear()
    torch.cuda.empty_cache()


def sm_count():
    """The SM count the engine sizes its launches for (PDSC_SM_COUNT lowers it, see device_state.cu)."""
    n = torch.cuda.get_device_properties(0).multi_processor_count
    env = os.environ.get("PDSC_SM_COUNT", "")
    return min(n, int(env)) if env.isdigit() and int(env) > 0 else n


def dev(x, dtype=None):
    """An array (or tensor) as a contiguous device tensor, converted to dtype if one is given."""
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype, device="cuda")


def same(a, b):
    """Byte equality (NaN-safe)."""
    a, b = a.contiguous(), b.contiguous()
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def ulps(a, b):
    """|a - b| in float32 units in the last place."""
    def ordered(x):
        i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))


def synth_sets(sizes, preset="3dmatch", seed0=0):
    """Synthetic pairs of N = sizes[i] correspondences (seed seed0 + i, inlier ratio 0.3)."""
    from pointdsc_b200.synth import make_pair
    return [make_pair(seed0 + i, n, preset, 0.3) for i, n in enumerate(sizes)]


def as_batch(pairs):
    """Pairs of one N as a testing-mode batch of device tensors."""
    return {"corr_pos": torch.stack([p["corr_pos"] for p in pairs]).cuda(),
            "src_keypts": torch.stack([p["src_keypts"] for p in pairs]).cuda(),
            "tgt_keypts": torch.stack([p["tgt_keypts"] for p in pairs]).cuda(), "testing": True}
