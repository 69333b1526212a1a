"""FCGF on the host: the float64 restatement (oracle/fcgf_oracle.py) on hand-worked clouds, the MinkowskiEngine-layout loader
(pointdsc_b200.fcgf.ResUNetBN2C, load_checkpoint, conv1_kernel_size) and cal_fcgf.py with the device call faked."""
import os

import numpy as np
import pytest
import torch

from oracle import fcgf_oracle as O


# ---- the restatement --------------------------------------------------------------------------------------------------
def test_one_voxel():
    xyz = np.array([[0.01, 0.02, 0.03], [0.04, 0.01, 0.0]], np.float32)
    c, inds, bad = O.quantize(xyz, 0.05)
    np.testing.assert_array_equal(c, [[0, 0, 0]])
    np.testing.assert_array_equal(inds, [0])
    assert not bad
    levels = O.pyramid(c)
    assert [l.tolist() for l in levels] == [[[0, 0, 0]]] * 4
    m = O.maps(levels, 7)
    centre = {7: 171, 3: 13}                              # (r, r, r): r + 7 r + 49 r and 1 + 3 + 9
    assert m["c1"].tolist()[0] == [0 if o == centre[7] else -1 for o in range(343)]
    for name in ("same0", "same3", "down1", "up0", "up2"):
        assert m[name].tolist()[0] == [0 if o == centre[3] else -1 for o in range(27)], name


def test_duplicates_choose_the_first_index_and_first_occurrence_order():
    xyz = np.array([[0.35, 0, 0], [0.01, 0, 0], [0.37, 0, 0], [0.0, 0, 0], [0.12, 0, 0]], np.float64)
    c, inds, _ = O.quantize(xyz, 0.1)
    np.testing.assert_array_equal(inds, [0, 1, 4])
    np.testing.assert_array_equal(c[:, 0], [3, 0, 1])


def test_negative_coordinates_floor_toward_minus_infinity():
    xyz = np.array([[-0.01, -0.11, 0.0], [-0.21, 0.19, -0.31]], np.float64)
    c, _, _ = O.quantize(xyz, 0.1)
    np.testing.assert_array_equal(c, [[-1, -2, 0], [-3, 1, -4]])
    lv = O.pyramid(c)
    np.testing.assert_array_equal(lv[1], [[-2, -2, 0], [-4, 0, -4]])
    np.testing.assert_array_equal(lv[2], [[-4, -4, 0], [-4, 0, -4]])
    np.testing.assert_array_equal(lv[3], [[-8, -8, 0], [-8, 0, -8]])


def test_out_of_range_and_non_finite_points_are_left_out():
    xyz = np.array([[0.0, 0, 0], [np.nan, 0, 0], [0.1 * 2 ** 20, 0, 0], [-0.1 * 2 ** 20, 0, 0], [np.inf, 0, 0]])
    c, inds, bad = O.quantize(xyz, 0.1)
    assert bad
    np.testing.assert_array_equal(inds, [0, 3])
    np.testing.assert_array_equal(c[:, 0], [0, -(2 ** 20)])


def _one_hot_state(k1, offset_index, conv, cin, cout):
    """Every parameter zero except the BN (identity) and W[offset_index][i][i] = 1 of `conv`."""
    from pointdsc_b200.fcgf import ResUNetBN2C
    sd = {k: np.zeros(tuple(v.shape)) for k, v in ResUNetBN2C(conv1_kernel_size=k1).state_dict().items()}
    for k in sd:
        if k.endswith("running_var") or k.endswith("bn.weight"):
            sd[k][:] = 1.0 - (O.BN_EPS if k.endswith("running_var") else 0.0)
    W = sd[f"{conv}.kernel"]
    for i in range(min(cin, cout)):
        W[offset_index, i, i] = 1.0
    return sd


@pytest.mark.parametrize("kind", ["same", "down", "up"])
def test_two_voxels_with_one_hot_kernels_pin_offsets_order_and_sign(kind):
    """Two voxels one unit apart along x.  A one-hot kernel at offset index o copies the neighbour at q + o s (q - o s for the
    transposed convolution) and nothing else; o = 14 is (+1, 0, 0) at r = 1, the x-fastest index of convention 4."""
    levels = O.pyramid(np.array([[0, 0, 0], [1, 0, 0]]))
    mp = O.maps(levels, 7)
    plus_x = 1 + 1 * 3 + 1 * 9 + 1                       # (ox, oy, oz) = (1, 0, 0) -> (2) + 3 (1) + 9 (1)
    assert plus_x == 14
    if kind == "same":
        assert mp["same0"][0].tolist() == [0 if o == 13 else (1 if o == 14 else -1) for o in range(27)]
        assert mp["same0"][1, 12] == 0 and mp["same0"][1, 14] == -1
        x = np.array([[1.0] + [0] * 31, [2.0] + [0] * 31])
        step = O.STEPS[1]
        sd = _one_hot_state(7, 14, step[0], 32, 32)
        y = O.apply_step(step, sd, mp["same0"], x, None)
        np.testing.assert_allclose(y[:, 0], [2.0, 0.0])   # row 0 reads row 1 (at +x); row 1 has nothing at +x
    elif kind == "down":
        # both fine voxels fall into coarse (0, 0, 0); coarse q gathers fine q + o * 1
        assert len(levels[1]) == 1
        assert mp["down1"][0].tolist() == [0 if o == 13 else (1 if o == 14 else -1) for o in range(27)]
    else:
        # fine (1, 0, 0) gathers coarse (0, 0, 0) = q - o * 1 at o = (+1, 0, 0); fine (0, 0, 0) at o = (0, 0, 0)
        assert mp["up0"][0].tolist() == [0 if o == 13 else -1 for o in range(27)]
        assert mp["up0"][1].tolist() == [0 if o == 14 else -1 for o in range(27)]


def test_kernel_index_is_x_fastest():
    o = O.offsets(3)
    assert o[0].tolist() == [-1, -1, -1] and o[1].tolist() == [0, -1, -1] and o[3].tolist() == [-1, 0, -1]
    assert o[9].tolist() == [-1, -1, 0] and o[26].tolist() == [1, 1, 1]
    o5 = O.offsets(5)
    assert o5[1].tolist() == [-1, -2, -2] and o5[5].tolist() == [-2, -1, -2] and o5[25].tolist() == [-2, -2, -1]


def test_normalisation_and_forward_shapes():
    from pointdsc_b200.fcgf import ResUNetBN2C
    rng = np.random.default_rng(0)
    sd = {k: rng.normal(0, 0.2, tuple(v.shape)) for k, v in ResUNetBN2C(conv1_kernel_size=5).state_dict().items()}
    for k in sd:
        if k.endswith("running_var"):
            sd[k] = np.abs(sd[k]) + 0.5
    xyz = rng.uniform(-0.5, 0.5, (400, 3))
    kp, desc = O.extract_features(sd, xyz, 0.1, 5)
    assert desc.shape == (len(kp), 32)
    np.testing.assert_allclose(np.linalg.norm(desc, axis=1), 1.0, atol=1e-6)


# ---- the loader ---------------------------------------------------------------------------------------------------
def _me_state_dict(k1, seed=0, one_by_one_3d=False):
    """A seeded state_dict with MinkowskiEngine 0.5's keys and shapes (1x1 kernels as [Cin, Cout] or [1, Cin, Cout])."""
    from pointdsc_b200.fcgf import ResUNetBN2C
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, v in ResUNetBN2C(conv1_kernel_size=k1).state_dict().items():
        t = torch.randn(v.shape, generator=g) if v.dtype == torch.float32 else torch.tensor(7)
        if one_by_one_3d and k in ("conv1_tr.kernel", "final.kernel"):
            t = t[None]
        out[k] = t
    return out


@pytest.mark.parametrize("k1", [7, 5])
@pytest.mark.parametrize("three_d", [False, True])
def test_loader_accepts_minkowski_layout(tmp_path, k1, three_d):
    from pointdsc_b200.fcgf import ResUNetBN2C, conv1_kernel_size, load_checkpoint, model_from_checkpoint
    sd = _me_state_dict(k1, one_by_one_3d=three_d)
    path = str(tmp_path / "w.pth")
    torch.save({"state_dict": sd, "epoch": 3}, path)
    loaded = load_checkpoint(path)
    assert conv1_kernel_size(loaded) == k1
    m = ResUNetBN2C(1, 32, bn_momentum=0.05, conv1_kernel_size=k1, normalize_feature=True)
    res = m.load_state_dict(loaded)
    assert res.missing_keys == [] and res.unexpected_keys == []
    assert tuple(m.conv1.kernel.shape) == (k1 ** 3, 1, 32) and tuple(m.final.kernel.shape) == (64, 32)
    assert tuple(m.final.bias.shape) == (1, 32) and tuple(m.block4.conv1.kernel.shape) == (27, 256, 256)
    assert torch.equal(m.conv1_tr.kernel, sd["conv1_tr.kernel"].reshape(96, 64))
    assert model_from_checkpoint(path).conv1_kernel_size == k1


def test_loader_reports_wrong_keys_and_shapes():
    from pointdsc_b200.fcgf import ResUNetBN2C, conv1_kernel_size
    sd = _me_state_dict(7)
    m = ResUNetBN2C(conv1_kernel_size=5)
    with pytest.raises(RuntimeError, match=r"size mismatch for conv1.kernel: copying a param with shape torch.Size\(\[343, 1, 32\]\)"):
        m.load_state_dict(sd)
    bad = dict(sd)
    del bad["block2.norm1.bn.running_var"]
    bad["block2.norm1.bn.running_varx"] = torch.zeros(64)
    with pytest.raises(RuntimeError, match=r'Missing key\(s\) in state_dict: "block2.norm1.bn.running_var"'):
        ResUNetBN2C(conv1_kernel_size=7).load_state_dict(bad)
    with pytest.raises(ValueError, match=r"conv1.kernel has shape \(27, 1, 32\)"):
        conv1_kernel_size({"conv1.kernel": torch.zeros(27, 1, 32)})
    for kw in ({"in_channels": 3}, {"out_channels": 16}, {"normalize_feature": False}, {"conv1_kernel_size": 3}):
        with pytest.raises(ValueError):
            ResUNetBN2C(**kw)


# ---- cal_fcgf.py ------------------------------------------------------------------------------------------------------
def _fake_describe(calls):
    """cal_fcgf's device call, recorded: the first half of each cloud as key points and unit descriptors."""
    def describe(clouds, voxel_size, weights):
        calls.append([len(c) for c in clouds])
        out = []
        for c in clouds:
            f = np.ones((len(c) // 2, 32), np.float32) / np.sqrt(32.0)
            out.append((c[:len(c) // 2], f))
        return out
    return describe


def test_cal_fcgf_writes_what_evaluate_reads(tmp_path):
    import cal_fcgf
    import evaluate
    src = tmp_path / "data" / "fragments" / "scene"
    src.mkdir(parents=True)
    rng = np.random.default_rng(0)
    clouds = {"cloud_bin_0": rng.normal(size=(50, 3)).astype(np.float32), "cloud_bin_1": rng.normal(size=(30, 3)).astype(np.float32)}
    for k, v in clouds.items():
        np.savez(src / f"{k}.npz", pcd=v)
    np.savez(src / "other.npz", other=np.zeros(3))              # no `pcd`: not an input
    calls = []
    out = tmp_path / "out"
    written = cal_fcgf.run([str(tmp_path / "data")], "weights.pth", 0.05, out_dir=str(out), max_points=60,
                           describe=_fake_describe(calls), log=lambda *a: None)
    assert [os.path.relpath(w, out) for w in written] == ["fragments/scene/cloud_bin_0_fcgf.npz", "fragments/scene/cloud_bin_1_fcgf.npz"]
    assert calls == [[50], [30]]                                # 80 points do not fit one group of 60
    z = np.load(written[0])
    assert sorted(z.files) == ["feature", "points", "xyz"]
    assert z["feature"].dtype == z["xyz"].dtype == z["points"].dtype == np.float32 and z["feature"].shape == (25, 32)
    np.testing.assert_array_equal(z["points"], clouds["cloud_bin_0"])
    xyz, feat = evaluate.load_fragment(str(out), "scene", 0, "fcgf", "cpu")
    np.testing.assert_array_equal(feat.numpy(), z["feature"])
    np.testing.assert_array_equal(xyz.numpy(), z["xyz"])
    assert feat.dtype == torch.float32
