"""A forward call's plan (pointdsc_b200/csrc/sets.cuh) against its restatement in engine_rules.py, without a GPU.

The host sizes a call's workspace from plan_call and set_table_kernel writes every set's offsets into it from the same
set_sizes and attn_key_split.  tests/call_plan_harness.cu exposes those functions, compiled here with the engine's nvcc flags,
and this module compares them with engine_rules (num_seeds, set_sizes, attn_set_split*, call_splits / call_split,
partial_items): every set size from 2 to 16384 rows at k = 1, 40, 80 and 128, the key split and the call decision at 1, 8, 66,
114 and 132 SMs in both modes, and the totals of a few mixed-size calls."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from engine_rules import (RATIO, attn_set_split, attn_set_split_invariant, call_split, call_splits, num_seeds, partial_items,
                          set_sizes)

HERE = os.path.dirname(os.path.abspath(__file__))
NS = np.arange(2, 16385, dtype=np.int32)
K_CFGS = (1, 40, 80, 128)
SMS = (1, 8, 66, 114, 132)
SIZE_KEYS = ("S", "k", "QT", "KT", "NS", "sc_rowmajor", "sc_tiled", "dist", "knn")
PLAN_KEYS = ("B", "N", "S", "k", "k_min", "R", "sc_rowmajor", "sc_tiled", "seeds", "dist", "knn", "qtiles", "ktiles",
             "attn_items", "attn_split", "attn_invariant", "num_sms", "partial_items")
MIXED = ([41, 257, 1003, 1003, 5000], [2, 3, 16384], [130] * 7, [1000] * 3 + [64, 65], [5000, 2], [16384] * 2)


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    import __graft_entry__ as G
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    lib_path = str(tmp_path_factory.mktemp("call_plan_harness") / "call_plan_harness.so")
    subprocess.run([nvcc] + G.NVCC_FLAGS + ["-I", G.CSRC, "-o", lib_path, os.path.join(HERE, "call_plan_harness.cu")], check=True)
    lib = C.CDLL(lib_path)
    lib.plan_set_sizes.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_int, C.c_void_p]
    lib.plan_key_split.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.plan_call_splits.argtypes = [C.c_longlong, C.c_longlong, C.c_int, C.c_int]
    lib.plan_call.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    for fn in (lib.plan_set_sizes, lib.plan_key_split, lib.plan_call):
        fn.restype = None
    return lib


def _call(lib, Ns, k_cfg, tc, invariant, sms, uniform=False):
    out = np.zeros(len(PLAN_KEYS), np.int64)
    if uniform:
        lib.plan_call(len(Ns), Ns[0], None, RATIO, k_cfg, tc, invariant, sms, out.ctypes.data)
    else:
        offsets = np.concatenate([[0], np.cumsum(Ns)]).astype(np.int32)
        lib.plan_call(len(Ns), 0, offsets.ctypes.data, RATIO, k_cfg, tc, invariant, sms, out.ctypes.data)
    return dict(zip(PLAN_KEYS, out.tolist()))


def _expected(Ns, k_cfg, tc, invariant, sms):
    sizes = [set_sizes(n, k_cfg) for n in Ns]
    total = {key: sum(z[key] for z in sizes) for key in SIZE_KEYS}
    split, items, _ = call_split(Ns, sms, invariant) if tc else (False, 0, None)
    return {"B": len(Ns), "N": max(Ns), "S": max(z["S"] for z in sizes), "k": max(z["k"] for z in sizes),
            "k_min": min([z["k"] for z in sizes if z["S"] > 0], default=k_cfg), "R": sum(Ns),
            "sc_rowmajor": total["sc_rowmajor"], "sc_tiled": total["sc_tiled"], "seeds": total["S"], "dist": total["dist"],
            "knn": total["knn"], "qtiles": total["QT"], "ktiles": total["KT"], "attn_items": items, "attn_split": int(split),
            "attn_invariant": invariant, "num_sms": sms, "partial_items": partial_items(split, items, invariant)}


@pytest.mark.parametrize("k_cfg", K_CFGS)
def test_set_sizes_at_every_n(plan, k_cfg):
    out = np.zeros((len(NS), len(SIZE_KEYS)), np.int64)
    plan.plan_set_sizes(NS.ctypes.data, len(NS), RATIO, k_cfg, out.ctypes.data)
    want = np.array([[set_sizes(int(n), k_cfg)[key] for key in SIZE_KEYS] for n in NS], np.int64)
    bad = np.flatnonzero((out != want).any(axis=1))
    assert bad.size == 0, [(int(NS[i]), out[i].tolist(), want[i].tolist()) for i in bad[:5]]
    assert (out[:, 0] == [num_seeds(int(n)) for n in NS]).all()


@pytest.mark.parametrize("invariant", (0, 1))
@pytest.mark.parametrize("sms", SMS)
def test_key_split_at_every_n(plan, sms, invariant):
    out = np.zeros((len(NS), 2), np.int32)
    plan.plan_key_split(NS.ctypes.data, len(NS), invariant, sms, out.ctypes.data)
    want = np.array([attn_set_split_invariant(int(n)) if invariant else attn_set_split(int(n), sms) for n in NS], np.int32)
    bad = np.flatnonzero((out != want).any(axis=1))
    assert bad.size == 0, [(int(NS[i]), out[i].tolist(), want[i].tolist()) for i in bad[:5]]


@pytest.mark.parametrize("invariant", (0, 1))
@pytest.mark.parametrize("sms", SMS)
def test_call_decision_at_its_edges(plan, sms, invariant):
    """attn_call_splits around every threshold: half the SMs, no set split, the item cap."""
    for qtiles in sorted({1, 2, 3, max(sms // 2 - 1, 1), sms // 2 + 1, sms // 2 + 2, 160, 161}):
        for items in sorted({qtiles - 1, qtiles, qtiles + 1, 2 * qtiles, 319, 320, 321, 1000}):
            got = plan.plan_call_splits(qtiles, items, sms, invariant)
            assert got == int(call_splits(qtiles, items, sms, invariant)), (qtiles, items)


@pytest.mark.parametrize("invariant", (0, 1))
@pytest.mark.parametrize("sms", SMS)
def test_one_set_calls_at_every_n(plan, sms, invariant):
    """The split decision, work items and partial buffers of a call of one set, for every N: the evaluation loops' bs = 1."""
    for n in NS.tolist():
        got = _call(plan, [n], 40, 1, invariant, sms)
        split, items, _ = call_split([n], sms, invariant)
        assert (got["attn_split"], got["attn_items"], got["partial_items"]) == \
            (int(split), items, partial_items(split, items, invariant)), n


@pytest.mark.parametrize("k_cfg", K_CFGS)
def test_mixed_calls(plan, k_cfg):
    """Every total of a few mixed-size calls, tensor-core and SIMT, and a uniform call planned from N alone or from offsets."""
    for Ns in MIXED:
        for sms in SMS:
            for invariant in (0, 1):
                for tc in (0, 1):
                    assert _call(plan, Ns, k_cfg, tc, invariant, sms) == _expected(Ns, k_cfg, tc, invariant, sms), \
                        (Ns, sms, invariant, tc)
    for Ns in ([1000] * 4, [5000], [41] * 33):
        for invariant in (0, 1):
            assert _call(plan, Ns, k_cfg, 1, invariant, 132, uniform=True) == _call(plan, Ns, k_cfg, 1, invariant, 132)
