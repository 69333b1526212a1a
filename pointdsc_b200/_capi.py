"""ctypes binding of the C ABI in include/pointdsc_b200.h.

This is the whole "FFI" a maintainer of the reference would add (the reference is pure Python and
has none of its own): load the shared library, mirror the two structs, declare the entry points,
and pass the arguments every wrapper passes alike (engine and stream, aligned scratch, offsets).
There is deliberately NO fallback: if the library is missing or no H100 is present the import /
engine creation raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("POINTDSC_B200_LIB") or os.path.join(_HERE, "libpointdsc_b200.so")   # env: developer A/B builds

PRECISIONS = {"fp32": 0, "bf16x3": 1, "bf16": 2, "fp16x3": 3}
SPANS = ["sc", "linear", "attention", "head", "seeds", "knn", "nsm", "hypotheses", "refine", "total"]


class PdscError(RuntimeError):
    pass


PDSC_ERR_SHAPE = 3


class Config(C.Structure):
    _fields_ = [
        ("in_dim", C.c_int32), ("num_layers", C.c_int32), ("num_channels", C.c_int32),
        ("num_iterations", C.c_int32), ("ratio", C.c_double), ("inlier_threshold", C.c_double),
        ("sigma_d", C.c_float), ("k", C.c_int32), ("nms_radius", C.c_float),
        ("precision", C.c_int32), ("device", C.c_int32),
    ]


class StageIO(C.Structure):
    _fields_ = [
        ("in_features", C.c_void_p), ("in_confidence", C.c_void_p), ("in_seeds", C.c_void_p),
        ("in_knn_idx", C.c_void_p), ("in_seed_trans", C.c_void_p),
        ("out_sc", C.c_void_p), ("out_features", C.c_void_p), ("out_normed", C.c_void_p),
        ("out_confidence", C.c_void_p), ("out_seeds", C.c_void_p), ("out_knn_idx", C.c_void_p),
        ("out_compat", C.c_void_p), ("out_eig", C.c_void_p), ("out_power_iters", C.c_void_p),
        ("out_seed_trans", C.c_void_p), ("out_inlier_counts", C.c_void_p), ("out_best", C.c_void_p),
        ("out_init_trans", C.c_void_p), ("out_refine_solves", C.c_void_p),
        ("layer_tap", C.c_int32), ("out_layer_features", C.c_void_p), ("out_layer_debug", C.c_void_p), ("out_timeline", C.c_void_p),
    ]


# every symbol include/pointdsc_b200.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "pdsc_create": (C.c_int, [C.POINTER(Config), C.POINTER(C.c_void_p)]),
    "pdsc_destroy": (C.c_int, [C.c_void_p]),
    "pdsc_last_error": (C.c_char_p, []),
    "pdsc_version": (C.c_char_p, []),
    "pdsc_set_param": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64]),
    "pdsc_commit_params": (C.c_int, [C.c_void_p]),
    "pdsc_set_precision": (C.c_int, [C.c_void_p, C.c_int32]),
    "pdsc_set_batch_invariant": (C.c_int, [C.c_void_p, C.c_int32]),
    "pdsc_num_seeds": (C.c_int32, [C.c_void_p, C.c_int32]),
    "pdsc_num_neighbours": (C.c_int32, [C.c_void_p, C.c_int32]),
    "pdsc_workspace_bytes": (C.c_size_t, [C.c_void_p, C.c_int32, C.c_int32]),
    "pdsc_forward": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.POINTER(StageIO), C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_workspace_bytes_packed": (C.c_size_t, [C.c_void_p, C.c_int32, C.c_void_p]),
    "pdsc_forward_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_forward_graph": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_forward_host": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p]),
    "pdsc_forward_host_submit": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]),
    "pdsc_forward_host_wait": (C.c_int, [C.c_void_p, C.c_int32]),
    "pdsc_forward_eval": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.POINTER(StageIO), C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_eval_stats": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "pdsc_eval_stats_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "pdsc_leading_eigenvector_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "pdsc_leading_eigenvector": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_match_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "pdsc_match": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                             C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                             C.c_size_t, C.c_void_p]),
    "pdsc_match_packed_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_void_p, C.c_void_p]),
    "pdsc_match_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_voxel_down_sample_scratch_bytes": (C.c_size_t, [C.c_int64]),
    "pdsc_voxel_down_sample": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_fpfh_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "pdsc_estimate_normals": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_double, C.c_int32, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_compute_fpfh": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_double, C.c_int32, C.c_int32, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_voxel_down_sample_packed_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_void_p]),
    "pdsc_voxel_down_sample_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p,
                                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_fpfh_packed_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_void_p, C.c_int32]),
    "pdsc_estimate_normals_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int32,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_compute_fpfh_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double,
                                           C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_icp_packed_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_void_p]),
    "pdsc_icp_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double,
                                  C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                  C.c_void_p]),
    "pdsc_icp_clouds_packed_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_void_p, C.c_void_p]),
    "pdsc_icp_clouds_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_double, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_information_matrix_packed_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_void_p, C.c_void_p]),
    "pdsc_information_matrix_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                 C.c_void_p]),
    "pdsc_ransac_packed_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_void_p, C.c_int32]),
    "pdsc_ransac_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double,
                                     C.c_int32, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_ransac_packed_hypotheses": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_double, C.c_int32, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                C.c_void_p]),
    "pdsc_spectral_matching_packed_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_void_p]),
    "pdsc_spectral_matching_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_spectral_matching_packed_iterates": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                         C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                         C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_fcgf_create": (C.c_int, [C.c_int32, C.POINTER(C.c_void_p)]),
    "pdsc_fcgf_destroy": (C.c_int, [C.c_void_p]),
    "pdsc_fcgf_set_param": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64]),
    "pdsc_fcgf_commit": (C.c_int, [C.c_void_p]),
    "pdsc_fcgf_packed_scratch_bytes": (C.c_size_t, [C.c_void_p, C.c_int32, C.c_void_p]),
    "pdsc_fcgf_packed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_fcgf_scratch_layout": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32]),
    "pdsc_tsdf_table_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "pdsc_tsdf_touch_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int32, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_tsdf_integrate_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_void_p]),
    "pdsc_tsdf_integrate_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                             C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_double,
                                             C.c_double, C.c_double, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pdsc_extract_vertices_count_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                                     C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                     C.c_void_p]),
    "pdsc_extract_vertices_packed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_size_t,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p]),
    "pdsc_read_ply": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]),
    "pdsc_launches_per_forward": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32]),
    "pdsc_profile_enable": (C.c_int, [C.c_void_p, C.c_int32]),
    "pdsc_profile_read": (C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_int32)]),
}

_lib = None


def load():
    """Load libpointdsc_b200.so (built in-tree by __graft_entry__.build()).  Raises if absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PdscError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(pointdsc_b200 has no CPU or PyTorch fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


_util_engines = {}


def utility_engine(device_index: int):
    """An engine handle for the stateless entry points (pdsc_match*, pdsc_eval_stats*): they only need the device."""
    if device_index not in _util_engines:
        lib = load()
        cfg = Config(6, 12, 128, 10, 0.1, 0.1, 0.1, 40, 0.1, PRECISIONS["fp16x3"], device_index)
        handle = C.c_void_p()
        check(lib.pdsc_create(C.byref(cfg), C.byref(handle)))
        _util_engines[device_index] = handle
    return _util_engines[device_index]


def check(rc: int):
    if rc != 0:
        raise PdscError(f"pointdsc_b200 error {rc}: {load().pdsc_last_error().decode()}")


def device_context(device: torch.device):
    """(library, utility engine, current stream handle) for a call of the stateless entry points on `device`."""
    index = device.index if device.index is not None else torch.cuda.current_device()
    return load(), utility_engine(index), C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def scratch(nbytes: int, device: torch.device, align: int = 8) -> torch.Tensor:
    """A uint8 device buffer of `nbytes` bytes that starts on an `align`-byte boundary: its data_ptr() and numel() are the
    scratch pointer and size an entry point takes.  The allocation is `align` bytes larger, so any start can be aligned."""
    buf = torch.empty(int(nbytes) + align, dtype=torch.uint8, device=device)
    skip = (buf.data_ptr() + align - 1) // align * align - buf.data_ptr()
    return buf[skip:skip + int(nbytes)]


def host_to_device(values, dtype, device) -> torch.Tensor:
    """A small host list as a device tensor without waiting for the stream: staged in page-locked memory, copied
    asynchronously (a copy from pageable memory would synchronise the stream first)."""
    return torch.tensor(values, dtype=dtype).pin_memory().to(device, non_blocking=True)


def offsets(values: Sequence[int], d_offsets: Optional[torch.Tensor], device: torch.device):
    """The B + 1 offsets of a packed call as the packed entry points take them: (host int32 array, device int32 tensor).
    `d_offsets` is the caller's device copy of the same values; when None, `values` is uploaded."""
    h = (C.c_int32 * len(values))(*values)
    if d_offsets is None:
        return h, host_to_device(values, torch.int32, device)
    if d_offsets.dtype != torch.int32 or d_offsets.device != device or d_offsets.numel() != len(values):
        raise ValueError("d_offsets must be a device int32 tensor of B + 1 entries")
    return h, d_offsets.contiguous()
