"""The descriptor front end over a group of clouds of different sizes (pdsc_voxel_down_sample_packed,
pdsc_estimate_normals_packed, pdsc_compute_fpfh_packed, descriptors.fpfh_descriptors_many): every cloud's rows bit for bit
those of the single-cloud calls on that cloud, permutation of the clouds, per-cloud status words, poisoned scratch and outputs,
rows past the end, bad offsets, and the packed descriptors through match_many + forward_packed."""
import ctypes as C

import numpy as np
import pytest
import torch

from buffer_guards import FLOAT_WORD, PATTERNS, assert_same, guarded_input, guarded_output, run_guarded, scratch_buffer, tiled
from gpu_models import dev
from pointdsc_b200.synth_scene import rigid, scene

pytestmark = pytest.mark.gpu

VOXEL = 0.08


def group_clouds():
    """A 1-point cloud, a cloud inside one voxel, two identical clouds, a cloud 10^4 m away from the others (a shared min bound
    would put it on another voxel grid) and a larger one."""
    rng = np.random.default_rng(0)
    a = scene(6000, seed=1)
    return [np.array([[0.3, -0.2, 1.5]], np.float32),
            (rng.uniform(0, 0.03, (400, 3)) + 0.5).astype(np.float32),
            a, a.copy(),
            scene(5000, seed=2) + np.float32(1e4),
            scene(20000, seed=3)]


def _lib():
    from pointdsc_b200 import _capi
    return _capi, _capi.load(), _capi.utility_engine(0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def search_packed(kind, pts, offsets, radius, max_nn, normals=None, normalise=0):
    """pdsc_estimate_normals_packed / pdsc_compute_fpfh_packed on device key points -> (out, status [P])."""
    capi, lib, e = _lib()
    P = len(offsets) - 1
    h = (C.c_int32 * (P + 1))(*offsets)
    d_off = dev(offsets, torch.int32)
    m = offsets[-1]
    out = torch.empty(m, 3 if kind == "normals" else 33, dtype=torch.float64, device="cuda")
    status = torch.empty(P, dtype=torch.int32, device="cuda")
    sc = torch.empty(int(lib.pdsc_fpfh_packed_scratch_bytes(P, h, max_nn)), dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())                 # noqa: E731
    if kind == "normals":
        rc = lib.pdsc_estimate_normals_packed(e, P, h, p(d_off), p(pts), radius, max_nn, p(out), p(status), p(sc), sc.numel(), _stream())
    else:
        rc = lib.pdsc_compute_fpfh_packed(e, P, h, p(d_off), p(pts), p(normals), radius, max_nn, normalise, p(out), p(status), p(sc),
                                          sc.numel(), _stream())
    capi.check(rc)
    return out, status.cpu().tolist()


def single_chain(cloud, normalise):
    from pointdsc_b200.descriptors import compute_fpfh, estimate_normals, voxel_down_sample
    kp = voxel_down_sample(dev(cloud, torch.float32), VOXEL)
    nrm = estimate_normals(kp, 2 * VOXEL, 30)
    return kp, nrm, compute_fpfh(kp, nrm, 5 * VOXEL, 100, normalise=normalise)


@pytest.mark.parametrize("normalise", [True, False], ids=["normalised", "raw"])
def test_every_cloud_is_bit_identical_to_the_single_cloud_calls(normalise):
    from pointdsc_b200.descriptors import fpfh_descriptors, fpfh_descriptors_many
    clouds = group_clouds()
    kp, feat, off, d_off = fpfh_descriptors_many([dev(c, torch.float32) for c in clouds], VOXEL, normalise=normalise)
    assert d_off.dtype == torch.int32 and d_off.cpu().tolist() == off and len(off) == len(clouds) + 1
    assert kp.dtype == torch.float32 and feat.dtype == torch.float64 and tuple(feat.shape) == (off[-1], 33)
    nrm, st = search_packed("normals", kp, off, 2 * VOXEL, 30)
    assert st == [0] * len(clouds)
    counts = []
    for p, c in enumerate(clouds):
        s_kp, s_nrm, s_feat = single_chain(c, normalise)
        rows = slice(off[p], off[p + 1])
        assert torch.equal(kp[rows], s_kp), p
        assert torch.equal(nrm[rows], s_nrm), p
        assert torch.equal(feat[rows], s_feat), p
        if normalise:
            assert torch.equal(feat[rows], fpfh_descriptors(dev(c, torch.float32), VOXEL)[1]), p
        counts.append(off[p + 1] - off[p])
    assert counts[0] == 1 and counts[1] == 1                                   # the 1-point cloud, the one-voxel cloud
    assert counts[2] == counts[3] and torch.equal(feat[off[2]:off[3]], feat[off[3]:off[4]])
    assert torch.equal(nrm[off[0]], torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64, device="cuda"))    # below three neighbours
    assert (kp[off[4]:off[5]] > 9000).all()


def test_permuting_the_clouds_permutes_the_outputs():
    from pointdsc_b200.descriptors import fpfh_descriptors_many
    clouds = group_clouds()
    kp, feat, off, _ = fpfh_descriptors_many([dev(c, torch.float32) for c in clouds], VOXEL)
    perm = [5, 2, 0, 4, 1, 3]
    kp2, feat2, off2, _ = fpfh_descriptors_many([dev(clouds[q], torch.float32) for q in perm], VOXEL)
    for i, q in enumerate(perm):
        assert torch.equal(kp2[off2[i]:off2[i + 1]], kp[off[q]:off[q + 1]]), (i, q)
        assert torch.equal(feat2[off2[i]:off2[i + 1]], feat[off[q]:off[q + 1]]), (i, q)


def test_status_lands_on_the_offending_cloud_only():
    from pointdsc_b200 import PdscError
    from pointdsc_b200.descriptors import estimate_normals, fpfh_descriptors_many
    bad = scene(1000, seed=4)
    bad[17, 1] = np.nan
    with pytest.raises(PdscError, match="cloud 1:"):
        fpfh_descriptors_many([dev(scene(1000, seed=5), torch.float32), dev(bad, torch.float32),
                               dev(scene(900, seed=6), torch.float32)], VOXEL)
    # the 4096-candidate overflow on the search of one cloud, next to clean ones
    rng = np.random.default_rng(1)
    sparse = [rng.uniform(0, 100, (n, 3)).astype(np.float32) for n in (300, 70)]
    dense = rng.uniform(0, 0.1, (6000, 3)).astype(np.float32)
    group = [sparse[0], dense, sparse[1]]
    off = np.cumsum([0] + [len(c) for c in group]).tolist()
    pts = dev(np.concatenate(group), torch.float32)
    nrm, st = search_packed("normals", pts, off, 1.0, 30)
    assert st == [0, 2, 0]
    _, st2 = search_packed("fpfh", pts, off, 1.0, 30, normals=nrm)
    assert st2 == [0, 2, 0]
    for p in (0, 2):
        assert torch.equal(nrm[off[p]:off[p + 1]], estimate_normals(dev(group[p], torch.float32), 1.0, 30)), p
    with pytest.raises(PdscError):
        estimate_normals(dev(dense, torch.float32), 1.0, 30)


def _voxel_packed_guarded(clouds, pat):
    capi, lib, e = _lib()
    dev = torch.device("cuda")
    P = len(clouds)
    off = np.cumsum([0] + [len(c) for c in clouds]).astype(np.int32)
    n = int(off[-1])
    h = (C.c_int32 * (P + 1))(*off.tolist())
    ins = {"pts": guarded_input(np.concatenate(clouds), dev), "off": guarded_input(off, dev)}
    need = int(lib.pdsc_voxel_down_sample_packed_scratch_bytes(P, h))
    outs = {"points": guarded_output(n * 12, 4, dev, pat), "offsets": guarded_output((P + 1) * 4, 4, dev, pat),
            "status": guarded_output(P * 4, 4, dev, pat)}
    sc = scratch_buffer(need, 8, pat)
    g = lambda b: C.c_void_p(b.ptr)                        # noqa: E731
    return run_guarded(("voxel_packed", pat), outs, sc, ins, lambda: lib.pdsc_voxel_down_sample_packed(
        e, P, h, g(ins["off"]), g(ins["pts"]), VOXEL, g(outs["points"]), g(outs["offsets"]), g(outs["status"]), g(sc), need,
        _stream()))


def test_poisoned_buffers_and_rows_past_the_end():
    """Scratch and outputs prefilled with every pattern (NaN-like and all-ones words among them), inputs and buffers guarded: the
    results do not change, no guard byte changes, and rows at or beyond out_offsets[P] keep the prefill byte for byte."""
    capi, lib, e = _lib()
    dev = torch.device("cuda")
    clouds = group_clouds()
    ref = None
    for pat in PATTERNS:
        got = _voxel_packed_guarded(clouds, pat)
        off = got["offsets"].view(torch.int32).cpu().tolist()
        assert off[0] == 0 and all(a < b for a, b in zip(off, off[1:])), off
        assert got["status"].view(torch.int32).cpu().tolist() == [0] * len(clouds)
        tail = got["points"][off[-1] * 12:]
        assert torch.equal(tail, tiled(FLOAT_WORD[pat], tail.numel(), dev)), ("row >= out_offsets[P] written", pat)
        got["points"] = got["points"][:off[-1] * 12]
        if ref is None:
            ref = got
        else:
            assert_same(ref, got, ("voxel_packed", pat))
    off = ref["offsets"].view(torch.int32).cpu().tolist()
    kp = ref["points"].view(torch.float32).view(-1, 3).cpu().numpy()
    P, m = len(clouds), off[-1]
    h = (C.c_int32 * (P + 1))(*off)
    ref2 = None
    for pat in PATTERNS:
        g = lambda b: C.c_void_p(b.ptr)                    # noqa: E731
        ins = {"pts": guarded_input(kp, dev), "off": guarded_input(np.array(off, np.int32), dev)}
        res = {}
        for kind, max_nn, radius in (("normals", 30, 2 * VOXEL), ("fpfh", 100, 5 * VOXEL)):
            need = int(lib.pdsc_fpfh_packed_scratch_bytes(P, h, max_nn))
            assert need == int(lib.pdsc_fpfh_scratch_bytes(m, max_nn))
            sc = scratch_buffer(need, 8, pat)
            if kind == "normals":
                outs = {"out": guarded_output(m * 24, 8, dev, pat), "status": guarded_output(P * 4, 4, dev, pat)}
                got = run_guarded((kind, pat), outs, sc, ins, lambda: lib.pdsc_estimate_normals_packed(
                    e, P, h, g(ins["off"]), g(ins["pts"]), radius, max_nn, g(outs["out"]), g(outs["status"]), g(sc), need, _stream()))
                nrm = guarded_input(got["out"].view(torch.float64).view(-1, 3).cpu().numpy(), dev)
            else:
                outs = {"out": guarded_output(m * 33 * 8, 8, dev, pat), "status": guarded_output(P * 4, 4, dev, pat)}
                got = run_guarded((kind, pat), outs, sc, {**ins, "nrm": nrm}, lambda: lib.pdsc_compute_fpfh_packed(
                    e, P, h, g(ins["off"]), g(ins["pts"]), g(nrm), radius, max_nn, 0, g(outs["out"]), g(outs["status"]), g(sc), need,
                    _stream()))
            assert got["status"].view(torch.int32).cpu().tolist() == [0] * P, (kind, pat)
            res[kind] = got["out"]
        if ref2 is None:
            ref2 = res
        else:
            assert_same(ref2, res, ("search_packed", pat))


def test_packed_descriptors_register_a_pair_as_the_per_cloud_chain():
    from conftest import load_snapshot
    from pointdsc_b200 import PointDSC
    from pointdsc_b200.descriptors import fpfh_descriptors, fpfh_descriptors_many
    from pointdsc_b200.frontend import match_many
    R, t = rigid(5)
    src = scene(60000, seed=1)
    tgt = (scene(60000, seed=2).astype(np.float64) @ R.T + t).astype(np.float32)
    model = PointDSC(in_dim=6, num_layers=12, num_channels=128, num_iterations=10, ratio=0.1, inlier_threshold=0.10, sigma_d=0.10,
                     k=40, nms_radius=0.10).cuda().eval()
    model.load_state_dict(load_snapshot("3dmatch"), strict=False)
    kp, feat, off, _ = fpfh_descriptors_many([dev(src, torch.float32), dev(tgt, torch.float32)], VOXEL)
    packed = (feat[off[0]:off[1]], feat[off[1]:off[2]], kp[off[0]:off[1]], kp[off[1]:off[2]])
    (skp, sf), (tkp, tf) = fpfh_descriptors(dev(src, torch.float32), VOXEL), fpfh_descriptors(dev(tgt, torch.float32), VOXEL)
    res = []
    for pair in (packed, (sf, tf, skp, tkp)):
        m = match_many([pair])
        res.append(model.forward_packed(m["corr_pos"], m["src_keypts"], m["tgt_keypts"], m["offsets"], m["d_offsets"]))
    assert torch.equal(res[0]["final_trans"], res[1]["final_trans"])
    assert torch.equal(res[0]["final_labels"], res[1]["final_labels"])
    T = res[0]["final_trans"][0].double().cpu().numpy()
    re = np.degrees(np.arccos(np.clip((np.trace(T[:3, :3].T @ R) - 1) / 2, -1, 1)))
    assert re < 2.0 and np.linalg.norm(T[:3, 3] - t) < 0.05


def test_bad_offsets_are_refused():
    capi, lib, e = _lib()
    pts = torch.zeros(100, 3, dtype=torch.float32, device="cuda")
    nrm = torch.zeros(100, 3, dtype=torch.float64, device="cuda")
    out = torch.empty(100, 33, dtype=torch.float64, device="cuda")
    d_out = torch.empty(8, dtype=torch.int32, device="cuda")
    status = torch.empty(8, dtype=torch.int32, device="cuda")
    sc = torch.empty(1 << 22, dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())                 # noqa: E731
    for offsets in ([0], [1, 50, 100], [0, 50, 50, 100], [0, 60, 50, 100]):
        P = len(offsets) - 1
        h = (C.c_int32 * len(offsets))(*offsets)
        d = dev(offsets, torch.int32)
        assert lib.pdsc_voxel_down_sample_packed_scratch_bytes(P, h) == 0, offsets
        assert lib.pdsc_fpfh_packed_scratch_bytes(P, h, 30) == 0, offsets
        rcs = (lib.pdsc_voxel_down_sample_packed(e, P, h, p(d), p(pts), VOXEL, p(pts), p(d_out), p(status), p(sc), sc.numel(), None),
               lib.pdsc_estimate_normals_packed(e, P, h, p(d), p(pts), 0.1, 30, p(nrm), p(status), p(sc), sc.numel(), None),
               lib.pdsc_compute_fpfh_packed(e, P, h, p(d), p(pts), p(nrm), 0.1, 100, 1, p(out), p(status), p(sc), sc.numel(), None))
        assert rcs == (capi.PDSC_ERR_SHAPE,) * 3, (offsets, rcs)
    from pointdsc_b200.descriptors import fpfh_descriptors_many
    with pytest.raises(ValueError):
        fpfh_descriptors_many([pts, pts[:0]], VOXEL)
    with pytest.raises(ValueError):
        fpfh_descriptors_many([], VOXEL)
