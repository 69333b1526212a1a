"""Fragment volumes on the H100 (row f9) against oracle/fragments_oracle.py.

The integration is held to the float32 restatement bit for bit: the touched units as a set, then every voxel's tsdf, weight and
colour.  The frames are small (80 x 60, intrinsics scaled by 1/8) views of the synthetic room along a moving camera, so units are
touched by different subsets of a fragment's frames.  The vertices are held to the float64 restatement on the device's own volume:
the same edges in the same order, and positions and colours bit for bit (both round the same operations in the same order).
A fragment's outputs are bit-identical alone, in a group, in either order and at a reduced SM count.  Through the C ABI on
guarded buffers, no output depends on what the table, scratch or outputs held, nothing is written outside them, and unit offsets
above the touch's counts only add empty rows.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from buffer_guards import FLOAT_WORD, PATTERNS, Guarded, fill_words, guarded_input, guarded_output

from oracle import fragments_oracle as O

pytestmark = pytest.mark.gpu

W, H = 80, 60
INTR = (525.0 / 8, 525.0 / 8, 319.5 / 8, 239.5 / 8)
VOXEL, TRUNC = 3.0 / 512, 0.04


def _fragment(n, seed):
    from pointdsc_b200.synth_scene import camera_path, render_rgbd
    poses = camera_path(n, seed)
    fr = [render_rgbd(p, W, H, *INTR) for p in poses]
    return np.stack([f[0] for f in fr]), np.stack([f[1] for f in fr]), np.linalg.inv(poses)


FRAGS = [_fragment(4, 0), _fragment(3, 5)]


def _run(frags):
    from pointdsc_b200.fragments import extract_vertices_packed, integrate_packed
    dep = torch.from_numpy(np.concatenate([f[0] for f in frags])).cuda()
    col = torch.from_numpy(np.concatenate([f[1] for f in frags])).cuda()
    ext = np.concatenate([f[2] for f in frags])
    off = np.concatenate([[0], np.cumsum([len(f[0]) for f in frags])]).tolist()
    vol = integrate_packed(dep, col, ext, off, INTR, VOXEL, TRUNC)
    verts, cols, voff = extract_vertices_packed(vol)
    torch.cuda.synchronize()
    out = []
    for f in range(len(frags)):
        u0, u1 = vol.unit_offsets[f], vol.unit_offsets[f + 1]
        out.append({"keys": vol.unit_keys[u0:u1].cpu().numpy(), "tsdf": vol.tsdf[u0:u1].cpu().numpy(),
                    "weight": vol.weight[u0:u1].cpu().numpy(), "color": vol.color[u0:u1].cpu().numpy(),
                    "verts": verts[voff[f]:voff[f + 1]].cpu().numpy(), "cols": cols[voff[f]:voff[f + 1]].cpu().numpy()})
    return out


@pytest.fixture(scope="module")
def group():
    return _run(FRAGS)


@pytest.mark.parametrize("f", [0, 1])
def test_integration_bit_for_bit(group, f):
    dep, col, ext = FRAGS[f]
    ref = O.integrate(dep, col, ext, INTR, VOXEL, TRUNC)
    got = group[f]
    keys = [tuple(k) for k in got["keys"].tolist()]
    assert keys == sorted(ref), "touched units differ"
    assert len({len(r[0]) for r in ref.values()}) > 1, "every unit saw the same frames: the case does not test the masks"
    for i, k in enumerate(keys):
        _, t, w, c = ref[k]
        t, w, c = t.reshape(16, 16, 16), w.reshape(16, 16, 16), c.reshape(16, 16, 16, 3)
        for name, a, b in (("tsdf", got["tsdf"][i], t), ("weight", got["weight"][i], w), ("color", got["color"][i], c)):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (name, k, int((a != b).sum()))
    assert (got["weight"] > 0).any()


@pytest.mark.parametrize("f", [0, 1])
def test_vertices_against_float64(group, f):
    got = group[f]
    units = {tuple(k): (got["tsdf"][i], got["weight"][i], got["color"][i]) for i, k in enumerate(got["keys"].tolist())}
    rv, rc = O.extract_vertices(units, VOXEL)
    assert got["verts"].shape == rv.shape and len(rv) > 1000
    # the device and the restatement round the same float64 operations in the same order: the same bits
    assert np.array_equal(got["verts"], rv) and np.array_equal(got["cols"], rc)


def test_group_and_order_invariance(group):
    alone = [_run([fr])[0] for fr in FRAGS]
    rev = _run(FRAGS[::-1])[::-1]
    for f in range(len(FRAGS)):
        for name in group[f]:
            a = group[f][name]
            assert np.array_equal(a.view(np.uint8), alone[f][name].view(np.uint8)), ("alone", f, name)
            assert np.array_equal(a.view(np.uint8), rev[f][name].view(np.uint8)), ("reversed", f, name)


def test_unit_capacity_is_reported():
    from pointdsc_b200 import _capi
    from pointdsc_b200.fragments import integrate_packed
    dep, col, ext = FRAGS[0]
    with pytest.raises(_capi.PdscError, match="max_units"):
        integrate_packed(torch.from_numpy(dep).cuda(), torch.from_numpy(col).cuda(), ext, [0, len(dep)], INTR, VOXEL, TRUNC,
                         max_units=8)


def test_blank_frames_give_an_empty_volume():
    from pointdsc_b200.fragments import extract_vertices_packed, integrate_packed
    dep, col, ext = FRAGS[0]
    blank = np.zeros_like(dep[:2])
    both = np.concatenate([blank, dep])
    vol = integrate_packed(torch.from_numpy(both).cuda(), torch.from_numpy(np.concatenate([col[:2], col])).cuda(),
                           np.concatenate([ext[:2], ext]), [0, 2, 2 + len(dep)], INTR, VOXEL, TRUNC)
    verts, _, voff = extract_vertices_packed(vol)
    assert vol.unit_offsets[1] == 0 and voff[1] == 0 and voff[2] == len(verts) > 0


def test_sm_count_does_not_change_a_bit(tmp_path, group):
    here = os.path.dirname(os.path.abspath(__file__))
    code = f"""
import sys, numpy as np
sys.path.insert(0, {here!r})
sys.path.insert(0, {os.path.dirname(here)!r})
import test_gpu_fragments as t
out = t._run(t.FRAGS)
np.savez(sys.argv[1], **{{f"{{f}}_{{k}}": v for f, d in enumerate(out) for k, v in d.items()}})
"""
    path = str(tmp_path / "sm8.npz")
    subprocess.run([sys.executable, "-c", code, path], env=dict(os.environ, PDSC_SM_COUNT="8"), check=True)
    z = np.load(path)
    for f, d in enumerate(group):
        for k, v in d.items():
            assert np.array_equal(v.view(np.uint8), z[f"{f}_{k}"].view(np.uint8)), (f, k)


def _raw(pattern, extra=0):
    """The whole pipeline through the C ABI on guarded buffers prefilled with `pattern`, with `extra` more unit rows for fragment 0
    than the touch counted.  Returns ({output name: host bytes}, unit offsets); every guard is checked."""
    from pointdsc_b200 import _capi
    lib, e, dev = _capi.load(), _capi.utility_engine(0), torch.device("cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = C.c_void_p
    ext = np.concatenate([f[2] for f in FRAGS])
    poses = np.concatenate([ext.reshape(-1, 1, 16), np.linalg.inv(ext).reshape(-1, 1, 16)], 1)
    foff = np.concatenate([[0], np.cumsum([len(f[0]) for f in FRAGS])]).astype(np.int32)
    F = len(FRAGS)
    ins = {"depth": guarded_input(np.concatenate([f[0] for f in FRAGS]), dev),
           "color": guarded_input(np.concatenate([f[1] for f in FRAGS]), dev), "poses": guarded_input(poses, dev),
           "frames": guarded_input(foff, dev)}
    h_f = (C.c_int32 * (F + 1))(*foff.tolist())
    intr = (C.c_double * 4)(*INTR)
    max_units = 4096
    table = Guarded(lib.pdsc_tsdf_table_bytes(F, max_units), 8, dev)
    fill_words(table.inner, FLOAT_WORD[pattern])
    meta = guarded_output(8 * F, 4, dev, pattern)
    _capi.check(lib.pdsc_tsdf_touch_packed(e, F, h_f, P(ins["frames"].ptr), H, W, intr, P(ins["depth"].ptr), P(ins["poses"].ptr), 1000.0,
                                           3.0, VOXEL, TRUNC, max_units, P(meta.ptr), P(meta.ptr + 4 * F), P(table.ptr), table.nbytes,
                                           stream))
    torch.cuda.synchronize()
    counts = meta.typed(torch.int32, (2, F)).cpu().numpy()
    assert not counts[1].any()
    counts = counts[0].copy()
    counts[0] += extra
    uoff = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    U = int(uoff[-1])
    ins["units"] = guarded_input(uoff, dev)
    h_u = (C.c_int32 * (F + 1))(*uoff.tolist())
    outs = {"keys": guarded_output(12 * U, 4, dev, pattern), "tsdf": guarded_output(4 * 4096 * U, 4, dev, pattern),
            "weight": guarded_output(4 * 4096 * U, 4, dev, pattern), "color": guarded_output(12 * 4096 * U, 4, dev, pattern),
            "ends": guarded_output(8 * U, 8, dev, pattern), "voff": guarded_output(8 * (F + 1), 8, dev, pattern)}
    scratch = Guarded(lib.pdsc_tsdf_integrate_scratch_bytes(F, h_u), 8, dev)
    fill_words(scratch.inner, FLOAT_WORD[pattern])
    o = {k: P(g.ptr) for k, g in outs.items()}
    _capi.check(lib.pdsc_tsdf_integrate_packed(e, F, h_f, P(ins["frames"].ptr), h_u, P(ins["units"].ptr), H, W, intr, P(ins["depth"].ptr),
                                               P(ins["color"].ptr), P(ins["poses"].ptr), 1000.0, 3.0, VOXEL, TRUNC, max_units,
                                               P(table.ptr), table.nbytes, o["keys"], o["tsdf"], o["weight"], o["color"],
                                               P(scratch.ptr), scratch.nbytes, stream))
    common = (e, F, h_u, P(ins["units"].ptr), max_units, P(table.ptr), table.nbytes, o["keys"], o["tsdf"], o["weight"])
    _capi.check(lib.pdsc_extract_vertices_count_packed(*common, o["ends"], o["voff"], stream))
    torch.cuda.synchronize()
    V = int(outs["voff"].typed(torch.int64, (F + 1,))[-1])
    outs["verts"] = guarded_output(24 * V, 8, dev, pattern)
    outs["vcols"] = guarded_output(24 * V, 8, dev, pattern)
    _capi.check(lib.pdsc_extract_vertices_packed(*common, o["color"], VOXEL, o["ends"], P(outs["verts"].ptr), P(outs["vcols"].ptr),
                                                 stream))
    torch.cuda.synchronize()
    for name, g in [("table", table), ("meta", meta), ("scratch", scratch)] + list(ins.items()) + list(outs.items()):
        g.check((name, pattern, extra))
    res = {k: g.inner.cpu().numpy() for k, g in outs.items()}
    res["counts"] = meta.inner.cpu().numpy()
    return res, uoff


def test_no_result_depends_on_buffer_contents_and_nothing_is_written_outside():
    ref, _ = _raw("zero")
    for p in PATTERNS[1:]:
        got, _ = _raw(p)
        for k in ref:
            assert np.array_equal(ref[k], got[k]), (p, k)


def test_unit_offsets_above_the_counts_add_empty_rows():
    ref, ro = _raw("zero")
    n0 = int(ro[1])
    for p in ("zero", "ones"):
        got, go = _raw(p, extra=3)
        assert go[1] == n0 + 3
        for k, dt, w in (("keys", np.int32, 3), ("tsdf", np.float32, 4096), ("weight", np.float32, 4096), ("color", np.float32, 12288)):
            a, b = ref[k].view(dt).reshape(-1, w), got[k].view(dt).reshape(-1, w)
            assert np.array_equal(a[:n0].view(np.uint8), b[:n0].view(np.uint8)), (p, k, "fragment 0")
            assert np.array_equal(a[n0:].view(np.uint8), b[n0 + 3:].view(np.uint8)), (p, k, "fragment 1")
            extra = b[n0:n0 + 3]
            assert (extra == np.iinfo(np.int32).min).all() if k == "keys" else not extra.view(np.uint32).any(), (p, k, "extra rows")
        for k in ("verts", "vcols"):
            assert np.array_equal(ref[k], got[k]), (p, k)
