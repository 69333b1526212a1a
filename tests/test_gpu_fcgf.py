"""FCGF on the device (pdsc_fcgf_packed, pointdsc_b200.fcgf) against the float64 restatement in oracle/fcgf_oracle.py.

- Quantisation, the coordinate pyramid and every neighbour table equal the oracle's exactly, cloud by cloud, with negative
  coordinates, a 1-point cloud and a cloud whose bad points (non-finite, beyond 2^20 voxels) are left out with status bit 1.
- Every convolution is checked against float64 of that convolution computed from the device's own input buffers and tables,
  within gamma_(K Cin + 3) (|scale| sum|w||x| + |shift| + |residual|), u = 2^-24 (a fp32 FMA chain of K Cin products, the
  folded BN's FMA with its two fp32-rounded constants, the residual add; ReLU is 1-Lipschitz, so the bound carries through it).
  Absent neighbours contribute nothing on both sides, so a table column the convolution reads in the wrong order or with the
  wrong sign leaves the bound.  The head (conv1_tr, ReLU, final, normalisation) is checked the same way from cat0.
- End to end, the descriptors are within 1e-4 of the float64 network on the oracle's own coordinates (the worst deviation is
  printed); seeded random weights and BN statistics, conv1 kernel 7 and 5.
- A cloud's rows are bit for bit the same alone, in a group and in reversed order, and on repeated calls; results do not depend
  on what the scratch or outputs held, and nothing is written past a cloud's rows or outside the buffers.
"""
import numpy as np
import pytest
import torch

from buffer_guards import FLOAT_WORD, PATTERNS, Guarded, fill_words
from oracle import fcgf_oracle as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
VOXEL = 0.05


def gamma(n):
    return n * U / (1 - n * U)


def random_state_dict(k1, seed):
    """Seeded weights and BN statistics in MinkowskiEngine layout, scaled so activations stay of order one."""
    from pointdsc_b200.fcgf import ResUNetBN2C
    rng = np.random.default_rng(seed)
    sd = {}
    for name, v in ResUNetBN2C(conv1_kernel_size=k1).state_dict().items():
        shape = tuple(v.shape)
        if name.endswith("kernel"):
            fan = int(np.prod(shape[:-1]))
            a = rng.normal(0.0, np.sqrt(2.0 / fan), shape)
        elif name.endswith("running_var"):
            a = rng.uniform(0.5, 2.0, shape)
        elif name.endswith("bn.weight"):
            a = rng.uniform(0.5, 1.5, shape)
        elif name.endswith("num_batches_tracked"):
            sd[name] = torch.zeros((), dtype=torch.int64)
            continue
        else:
            a = rng.normal(0.0, 0.1, shape)
        sd[name] = torch.from_numpy(a.astype(np.float32))
    return sd


_models = {}


def model(k1, seed=0):
    from pointdsc_b200.fcgf import ResUNetBN2C
    if (k1, seed) not in _models:
        m = ResUNetBN2C(conv1_kernel_size=k1)
        res = m.load_state_dict(random_state_dict(k1, seed))
        assert res.missing_keys == [] and res.unexpected_keys == []
        _models[(k1, seed)] = m
    return _models[(k1, seed)]


def sd64(m):
    return {k: v.numpy().astype(np.float64) for k, v in m.state_dict().items()}


def group():
    """Negative coordinates across every stride, a 1-point cloud, a small dense cloud, duplicates, and a larger one."""
    from pointdsc_b200.synth_scene import scene
    a = scene(3000, seed=1) - np.float32(1.5)
    dup = np.concatenate([a[:500], a[:500]])             # every voxel's first point is in the first half
    return [a, np.array([[-0.01, 0.02, -0.51]], np.float32), (np.random.default_rng(5).uniform(-0.2, 0.1, (700, 3))).astype(np.float32),
            dup, scene(6000, seed=2) * np.float32([1, -1, 1])]


def run(m, clouds, scratch_fill=None, out_fill=None, cpu=True, voxel=VOXEL):
    """One packed call; returns (keypts, desc, meta, regions {name: tensor}) with the scratch kept."""
    from pointdsc_b200.fcgf import packed_call, scratch_layout
    in_off = [0]
    for c in clouds:
        in_off.append(in_off[-1] + len(c))
    n = in_off[-1]
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    nbytes, lay = scratch_layout(m, in_off)
    scratch = Guarded(nbytes, 256, pts.device)
    fill_words(scratch.inner, FLOAT_WORD[scratch_fill or "zero"])
    kp = Guarded(n * 12, 16, pts.device)
    ds = Guarded(n * 128, 16, pts.device)
    fill_words(kp.inner, FLOAT_WORD[out_fill or "zero"])
    fill_words(ds.inner, FLOAT_WORD[out_fill or "zero"])
    keypts, desc, meta = packed_call(m, pts, in_off, voxel, scratch=scratch.inner, keypts=kp.typed(torch.float32, (n, 3)),
                                     desc=ds.typed(torch.float32, (n, 32)))
    torch.cuda.synchronize()
    for g, what in ((scratch, "scratch"), (kp, "keypts"), (ds, "desc")):
        g.check(what)
    P = len(clouds)
    k1 = m.conv1_kernel_size
    names = [f"off{l}" for l in range(4)] + [f"coords{l}" for l in range(4)] + ["c1"] + [f"same{l}" for l in range(4)] + \
        [f"down{l}" for l in range(1, 4)] + [f"up{l}" for l in range(3)] + O.FEATS
    assert len(lay) == len(names) == 37
    raw = scratch.inner
    reg = {}
    for i, name in enumerate(names):
        if name.startswith("off"):
            cols, dt = P + 1, torch.int32
            reg[name] = raw[lay[i]:lay[i] + 4 * cols].view(dt)
            continue
        cols = 3 if name.startswith("coords") else (k1 ** 3 if name == "c1" else (O.FEAT_WIDTH.get(name, 27)))
        dt = torch.float32 if name in O.FEAT_WIDTH else torch.int32
        reg[name] = raw[lay[i]:lay[i] + 4 * n * cols].view(dt).view(n, cols)
    return keypts, desc, meta, ({k: v.cpu() for k, v in reg.items()} if cpu else reg), (kp, ds)


@pytest.mark.parametrize("k1", [7, 5])
def test_quantisation_pyramid_and_tables_match_the_oracle(k1):
    m = model(k1)
    clouds = group()
    keypts, desc, meta, reg, _ = run(m, clouds)
    P = len(clouds)
    meta = meta.cpu().tolist()
    assert meta[P + 1:] == [0] * P
    assert meta[:P + 1] == reg["off0"].tolist()
    for p, xyz in enumerate(clouds):
        c0, inds, bad = O.quantize(xyz, VOXEL)
        assert not bad
        levels = O.pyramid(c0)
        mp = O.maps(levels, k1)
        r0 = [int(reg[f"off{l}"][p]) for l in range(4)]
        r1 = [int(reg[f"off{l}"][p + 1]) for l in range(4)]
        for l in range(4):
            assert r1[l] - r0[l] == len(levels[l]), (p, l)
            np.testing.assert_array_equal(reg[f"coords{l}"][r0[l]:r1[l]].numpy(), levels[l], err_msg=f"cloud {p} level {l}")
        np.testing.assert_array_equal(keypts[r0[0]:r1[0]].cpu().numpy(), xyz[inds])
        target = {"c1": 0, **{f"same{l}": l for l in range(4)}, **{f"down{l}": l - 1 for l in range(1, 4)},
                  **{f"up{l}": l + 1 for l in range(3)}}
        for name, want in mp.items():
            lvl = 0 if name == "c1" else int(name[-1])
            got = reg[name][r0[lvl]:r1[lvl]].numpy().astype(np.int64)
            got = np.where(got >= 0, got - r0[target[name]], -1)
            np.testing.assert_array_equal(got, want, err_msg=f"cloud {p} table {name}")


def test_bad_points_are_left_out_with_status_bit_1():
    m = model(7)
    from pointdsc_b200.synth_scene import scene
    good = scene(1500, seed=4) - np.float32(1.5)
    bad = good.copy()
    bad[7] = np.nan
    bad[11, 1] = np.inf
    bad[13, 2] = np.float32(VOXEL * 2 ** 20 * 1.01)
    bad[17, 0] = np.float32(-VOXEL * 2 ** 20 * 1.01)
    keypts, desc, meta, reg, _ = run(m, [good, bad])
    meta = meta.cpu().tolist()
    assert meta[3:] == [0, 1]
    c0, inds, was_bad = O.quantize(bad, VOXEL)
    assert was_bad
    off = meta[:3]
    np.testing.assert_array_equal(reg["coords0"][off[1]:off[2]].numpy(), c0)
    np.testing.assert_array_equal(keypts[off[1]:off[2]].cpu().numpy(), bad[inds])


def _conv_bound_check(step, reg, sd, k1):
    name, kind, level, inp, res, out, cout, norm, relu = step
    tables = {"c1": "c1", "same": f"same{level}", "down": f"down{level}", "up": f"up{level}"}
    nmap = reg[tables[kind]].numpy().astype(np.int64)
    rows = int(reg[f"off{level}"][-1])
    nmap = nmap[:rows]
    W = sd[f"{name}.kernel"]
    K = W.shape[0]
    x = np.ones((rows, 1)) if inp is None else reg[inp[0]].numpy().astype(np.float64)[:, inp[1]:]
    resid = None if res is None else reg[res[0]].numpy().astype(np.float64)[:rows, res[1]:res[1] + cout]
    want = O.apply_step(step, sd, nmap, x, resid)
    got = reg[out[0]].numpy().astype(np.float64)[:rows, out[1]:out[1] + cout]
    g, b = sd[f"{norm}.bn.weight"], sd[f"{norm}.bn.bias"]
    mu, var = sd[f"{norm}.bn.running_mean"], sd[f"{norm}.bn.running_var"]
    scale = g / np.sqrt(var + O.BN_EPS)
    shift = b - mu * scale
    absacc = O.sparse_conv(np.abs(x), nmap, np.abs(W))
    mag = np.abs(scale) * absacc + np.abs(shift) + (0 if resid is None else np.abs(resid))
    bound = gamma(K * x.shape[1] + 3) * mag
    err = np.abs(got - want)
    worst = float((err / np.maximum(bound, 1e-300)).max(initial=0))
    assert np.all(err <= bound), f"{name}: worst error {worst:.3g} of its bound"
    return worst


@pytest.mark.parametrize("k1", [7, 5])
def test_every_layer_within_its_float64_bound(k1):
    m = model(k1, seed=1)
    sd = sd64(m)
    keypts, desc, meta, reg, _ = run(m, group())
    worst = {s[0]: _conv_bound_check(s, reg, sd, k1) for s in O.STEPS}
    # the head, from the device's own cat0
    rows = int(reg["off0"][-1])
    cat0 = reg["cat0"].numpy().astype(np.float64)[:rows]
    w_tr, w_f = sd["conv1_tr.kernel"].reshape(96, 64), sd["final.kernel"].reshape(64, 32)
    h = np.maximum(cat0 @ w_tr, 0.0)
    f = h @ w_f + sd["final.bias"].reshape(32)
    eh = gamma(96) * (np.abs(cat0) @ np.abs(w_tr))
    ef = gamma(65) * (np.abs(h) @ np.abs(w_f) + np.abs(sd["final.bias"].reshape(32))) + eh @ np.abs(w_f)
    nf = np.linalg.norm(f, axis=1, keepdims=True)
    want = f / (nf + 1e-8)
    bound = (np.abs(ef) + np.linalg.norm(ef, axis=1, keepdims=True) * np.abs(want)) / nf + 40 * U
    err = np.abs(desc[:rows].cpu().numpy().astype(np.float64) - want)
    assert np.all(err <= bound), float((err / bound).max())
    print(f"k1={k1}: worst layer error / bound", {k: round(v, 4) for k, v in worst.items()}, "head", float((err / bound).max()))


@pytest.mark.parametrize("k1", [7, 5])
def test_descriptors_match_the_float64_network(k1):
    m = model(k1, seed=2)
    sd = sd64(m)
    clouds = group()
    from pointdsc_b200.fcgf import fcgf_descriptors_many
    keypts, desc, off, _ = fcgf_descriptors_many(m, [torch.from_numpy(c).cuda() for c in clouds], VOXEL)
    worst = 0.0
    for p, xyz in enumerate(clouds):
        kp, want = O.extract_features(sd, xyz, VOXEL, k1)
        np.testing.assert_array_equal(keypts[off[p]:off[p + 1]].cpu().numpy(), kp)
        worst = max(worst, float(np.abs(desc[off[p]:off[p + 1]].cpu().numpy() - want).max()))
    print(f"k1={k1}: worst |descriptor - float64| = {worst:.3g} (asserted <= 1e-4)")
    assert worst <= 1e-4


def test_group_order_repeat_and_buffers_do_not_change_a_cloud():
    m = model(7)
    clouds = group()
    from pointdsc_b200.fcgf import fcgf_descriptors_many
    dev = [torch.from_numpy(c).cuda() for c in clouds]
    kp, ds, off, _ = fcgf_descriptors_many(m, dev, VOXEL)
    rows = [(kp[off[p]:off[p + 1]], ds[off[p]:off[p + 1]]) for p in range(len(clouds))]
    for p, c in enumerate(dev):
        a_kp, a_ds, _, _ = fcgf_descriptors_many(m, [c], VOXEL)
        assert torch.equal(a_kp, rows[p][0]) and torch.equal(a_ds, rows[p][1]), f"cloud {p} alone"
    r_kp, r_ds, r_off, _ = fcgf_descriptors_many(m, dev[::-1], VOXEL)
    P = len(clouds)
    for q in range(P):
        p = P - 1 - q
        assert torch.equal(r_kp[r_off[q]:r_off[q + 1]], rows[p][0]) and torch.equal(r_ds[r_off[q]:r_off[q + 1]], rows[p][1])
    again = fcgf_descriptors_many(m, dev, VOXEL)
    assert torch.equal(again[0], kp) and torch.equal(again[1], ds)
    ref = None
    for pat in PATTERNS:
        keypts, desc, meta, _, (g_kp, g_ds) = run(m, clouds, scratch_fill=pat, out_fill=pat)
        M = int(meta[P])
        got = (keypts[:M].clone(), desc[:M].clone())
        if ref is None:
            ref = got
            assert torch.equal(got[0], kp) and torch.equal(got[1], ds)
        assert torch.equal(got[0].view(torch.int32), ref[0].view(torch.int32)), pat
        assert torch.equal(got[1].view(torch.int32), ref[1].view(torch.int32)), pat
        word = FLOAT_WORD[pat]
        tail_kp = g_kp.inner.view(torch.int32)[M * 3:]
        tail_ds = g_ds.inner.view(torch.int32)[M * 32:]
        as_i32 = word - (1 << 32) if word >= 1 << 31 else word
        assert bool((tail_kp == as_i32).all()) and bool((tail_ds == as_i32).all()), f"{pat}: rows past the end written"


def test_errors():
    from pointdsc_b200 import _capi
    from pointdsc_b200.fcgf import ResUNetBN2C, fcgf_descriptors_many
    import ctypes as C
    lib = _capi.load()
    h = C.c_void_p()
    assert lib.pdsc_fcgf_create(3, C.byref(h)) == 7
    assert lib.pdsc_fcgf_create(7, C.byref(h)) == 0
    a = np.zeros(10, np.float32)
    assert lib.pdsc_fcgf_set_param(h, b"conv1.bias", a.ctypes.data_as(C.c_void_p), 10) == 2
    assert lib.pdsc_fcgf_set_param(h, b"final.bias", a.ctypes.data_as(C.c_void_p), 10) == 3
    assert lib.pdsc_fcgf_commit(h) == 2 and b"missing" in lib.pdsc_last_error()
    lib.pdsc_fcgf_destroy(h)
    with pytest.raises(ValueError):
        fcgf_descriptors_many(model(7), [torch.zeros(0, 3, device="cuda")], VOXEL)
    with pytest.raises(_capi.PdscError):
        fcgf_descriptors_many(model(7), [torch.zeros(4, 3, device="cuda")], -1.0)
    with pytest.raises(ValueError):
        ResUNetBN2C(in_channels=3)


def test_demo_runs_with_fcgf_weights(tmp_path):
    import os
    import demo
    from conftest import GOLDEN
    path = str(tmp_path / "fcgf.pth")
    torch.save({"state_dict": random_state_dict(7, 3)}, path)
    ply = os.path.join(GOLDEN, "ply_cloud_bin_0_first2000.ply")
    out = demo.register(ply, ply, descriptor="fcgf", fcgf_weights=path, verbose=False)
    assert out["key_points"][0] == out["key_points"][1] > 0
    assert out["correspondences"] == out["key_points"][0]
    np.testing.assert_allclose(out["final_trans"], np.eye(4), atol=1e-4)    # a cloud against itself
