"""cal_fpfh.py on the host: input discovery, output names, keys, dtypes and shapes, the --out mirror and the groups, with the
device stage replaced by the CPU restatement in oracle/fpfh_oracle.py.  The files must load through evaluate.load_fragment."""
import os

import numpy as np
import pytest

import cal_fpfh
import evaluate
from oracle import fpfh_oracle as F

VOXEL = 0.05


def oracle_stage(clouds, voxel):
    """misc/cal_fpfh.py:21-27 per cloud on the CPU: (xyz float32, raw FPFH float32)."""
    out = []
    for c in clouds:
        kp = F.voxel_down_sample(c, voxel)[0].astype(np.float32)
        nrm = F.estimate_normals(kp, 2 * voxel, 30)
        out.append((kp, F.fpfh(kp, nrm, 5 * voxel, 100).astype(np.float32)))
    return out


def write_ply(path, pts):
    with open(path, "wb") as f:
        f.write(f"ply\nformat binary_little_endian 1.0\nelement vertex {len(pts)}\nproperty float x\nproperty float y\n"
                f"property float z\nproperty uchar red\nend_header\n".encode())
        rows = np.zeros(len(pts), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("r", "u1")])
        rows["x"], rows["y"], rows["z"] = pts[:, 0], pts[:, 1], pts[:, 2]
        f.write(rows.tobytes())


def clouds():
    rng = np.random.default_rng(3)
    return {"ply": rng.uniform(0, 0.6, (300, 3)).astype(np.float32),
            "npz": (rng.uniform(0, 0.5, (250, 3)) + [4.0, -2.0, 1.0]).astype(np.float32)}


@pytest.fixture
def tree(tmp_path):
    """fragments/scene-a/cloud_bin_0.ply, fragments/scene-a/cloud_bin_1.npz (pcd) and two files that are not inputs."""
    c = clouds()
    scene = tmp_path / "fragments" / "scene-a"
    scene.mkdir(parents=True)
    write_ply(scene / "cloud_bin_0.ply", c["ply"])
    np.savez(scene / "cloud_bin_1.npz", pcd=c["npz"], color=np.zeros_like(c["npz"]))
    np.savez(scene / "other.npz", xyz=c["npz"])                  # no pcd array: not an input
    (scene / "notes.txt").write_text("not an input")
    return tmp_path


def check_file(path, pts):
    want_xyz, want_feat = oracle_stage([pts], VOXEL)[0]
    with np.load(path) as z:
        assert sorted(z.files) == ["feature", "points", "xyz"]
        assert z["points"].dtype == z["xyz"].dtype == z["feature"].dtype == np.float32
        assert np.array_equal(z["points"], pts)
        assert z["xyz"].shape == want_xyz.shape and z["feature"].shape == (len(want_xyz), 33)
        assert np.array_equal(z["xyz"], want_xyz) and np.array_equal(z["feature"], want_feat)


def test_writes_next_to_the_inputs(tree):
    logged = []
    written = cal_fpfh.run([str(tree / "fragments")], VOXEL, describe=oracle_stage, log=lambda *a: logged.append(a))
    scene = tree / "fragments" / "scene-a"
    assert written == [str(scene / "cloud_bin_0_fpfh.npz"), str(scene / "cloud_bin_1_fpfh.npz")]
    c = clouds()
    check_file(written[0], c["ply"])
    check_file(written[1], c["npz"])
    assert len(logged) == 2
    # a second run does not take its own outputs (no pcd array) as inputs
    assert cal_fpfh.run([str(tree / "fragments")], VOXEL, describe=oracle_stage, log=lambda *a: None) == written


def test_out_mirrors_the_tree_and_load_fragment_reads_it(tree, tmp_path_factory):
    out = tmp_path_factory.mktemp("out")
    before = sorted(os.listdir(tree / "fragments" / "scene-a"))
    written = cal_fpfh.run([str(tree / "fragments")], VOXEL, out_dir=str(out / "fragments"), describe=oracle_stage,
                           log=lambda *a: None)
    assert written == [str(out / "fragments" / "scene-a" / f"cloud_bin_{i}_fpfh.npz") for i in (0, 1)]
    assert sorted(os.listdir(tree / "fragments" / "scene-a")) == before       # nothing written beside the inputs
    c = clouds()
    for i, key in enumerate(("ply", "npz")):
        xyz, feat = evaluate.load_fragment(str(out), "scene-a", i, "fpfh", "cpu")
        want_xyz, want_feat = oracle_stage([c[key]], VOXEL)[0]
        assert np.array_equal(xyz.numpy(), want_xyz)
        f64 = want_feat.astype(np.float64)
        assert np.allclose(feat.numpy(), f64 / (np.linalg.norm(f64, axis=1, keepdims=True) + 1e-6), rtol=0, atol=1e-12)


def test_groups_respect_the_point_budget(tree):
    calls = []

    def stage(cl, voxel):
        calls.append([len(c) for c in cl])
        return oracle_stage(cl, voxel)

    cal_fpfh.run([str(tree / "fragments")], VOXEL, max_points=400, describe=stage, log=lambda *a: None)
    assert calls == [[300], [250]]
    calls.clear()
    cal_fpfh.run([str(tree / "fragments")], VOXEL, max_points=550, describe=stage, log=lambda *a: None)
    assert calls == [[300, 250]]
    assert cal_fpfh.make_groups([5, 1, 9, 2, 2], 4) == [[0], [1], [2], [3, 4]]


def test_empty_cloud_is_skipped(tmp_path):
    np.savez(tmp_path / "empty.npz", pcd=np.zeros((0, 3), np.float32))
    np.savez(tmp_path / "one.npz", pcd=np.array([[1.0, 2.0, 3.0]], np.float32))
    logged = []
    written = cal_fpfh.run([str(tmp_path)], VOXEL, describe=oracle_stage, log=lambda *a: logged.append(a))
    assert written == [str(tmp_path / "one_fpfh.npz")]
    assert any("do not have any points" in str(a[0]) for a in logged)
    assert cal_fpfh.cloud_size(str(tmp_path / "one.npz")) == 1
