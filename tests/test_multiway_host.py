"""Host side of the multiway registration (row f7): the information-matrix restatement against its definition, the pose graph's
JSON, global_optimization, the trajectory error, and multiway.py's scene loop on fakes (which pairs go where, the prune rule at
its exact edges, the pair order, the files written)."""
import os

import numpy as np
import pytest
import torch

import multiway as driver
from multiway_oracle import icp_clouds_packed, information_matrix
from oracle import icp_oracle as O
from pointdsc_b200 import multiway as mw


def _rot(rng, deg):
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    a = np.deg2rad(deg)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def _rigid(rng, deg, shift):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = _rot(rng, deg), rng.normal(size=3) * shift
    return T


# ---------------------------------------------------------------------------------------------------------------- information
@pytest.mark.parametrize("ns,nt,seed", [(1, 1, 0), (50, 300, 1), (2000, 700, 2)])
def test_information_oracle_against_its_definition(ns, nt, seed):
    rng = np.random.default_rng(seed)
    tgt = rng.uniform(-1, 1, (nt, 3)).astype(np.float32)
    src = (tgt[rng.integers(0, nt, ns)] + rng.normal(scale=0.02, size=(ns, 3))).astype(np.float32)
    T = np.eye(4, dtype=np.float32)
    res = information_matrix(src, tgt, T, 0.05)
    info, n = res["info"], res["count"]
    assert res["status"] == 0 and n == len(res["rows"])
    assert np.array_equal(info, info.T)
    assert np.linalg.eigvalsh(info).min() >= -1e-9 * max(1.0, np.abs(info).max())
    assert info[5, 5] == n
    assert np.array_equal(info[3:, 3:], n * np.eye(3))
    # the kept rows are exactly the nearest targets within float32(r^2), found by brute force
    d2 = ((src.astype(np.float64)[:, None] - tgt.astype(np.float64)[None]) ** 2).sum(-1)
    kept = np.nonzero(d2.min(1) < O.radius_sq(0.05))[0]
    assert np.array_equal(res["rows"][:, 0], kept)
    q = tgt[d2.argmin(1)[kept]].astype(np.float64)
    assert np.allclose(info[0, 4], -q[:, 2].sum()) and np.allclose(info[0, 5], q[:, 1].sum())
    assert np.allclose(info[0, 0], (q[:, 1] ** 2 + q[:, 2] ** 2).sum())


def test_information_oracle_moves_the_source_and_reports_status():
    rng = np.random.default_rng(3)
    tgt = rng.uniform(-1, 1, (400, 3)).astype(np.float32)
    T = _rigid(rng, 20, 0.3).astype(np.float32)
    src = ((tgt.astype(np.float64) - T[:3, 3]) @ T[:3, :3].astype(np.float64)).astype(np.float32)   # T^-1 tgt
    assert information_matrix(src, tgt, T, 0.01)["count"] == 400
    assert information_matrix(src, tgt, np.eye(4, dtype=np.float32), 0.01)["count"] < 400
    bad = src.copy()
    bad[7, 1] = np.nan
    res = information_matrix(bad, tgt, T, 0.01)
    assert res["status"] == 1 and not res["info"].any()


def test_icp_packed_two_clouds_matches_icp_per_pair():
    rng = np.random.default_rng(4)
    clouds = [rng.uniform(0, 1, (n, 3)).astype(np.float32) for n in (30, 80, 55)]
    src = np.concatenate([clouds[0], clouds[1]])
    tgt = np.concatenate([clouds[2], clouds[0] + np.float32(0.01)])
    init = np.stack([np.eye(4, dtype=np.float32)] * 2)
    res = icp_clouds_packed(src, tgt, init, [0, 30, 110], [0, 55, 85], 0.1)
    for got, (s, t) in zip(res, [(clouds[0], clouds[2]), (clouds[1], clouds[0] + np.float32(0.01))]):
        ref = O.icp(s, t, np.eye(4, dtype=np.float32), 0.1)
        assert got["iterations"] == ref["iterations"] and np.array_equal(got["trans64"], ref["trans64"])


# ---------------------------------------------------------------------------------------------------------------- pose graph
def _graph(K=8, seed=0, noise=0.0):
    rng = np.random.default_rng(seed)
    poses = [np.eye(4)] + [_rigid(rng, 30, 1.0) for _ in range(K - 1)]
    info = np.diag([400.0, 400.0, 400.0, 1000.0, 1000.0, 1000.0])
    g = mw.PoseGraph([p.copy() for p in poses], [])
    for i in range(K):
        for j in range(i + 1, K):
            g.edges.append(mw.PoseGraphEdge(i, j, np.linalg.inv(poses[j]) @ poses[i], info.copy(), uncertain=j != i + 1))
    for k in range(1, K):
        g.nodes[k] = _rigid(rng, 2.0 * noise, 0.02 * noise) @ g.nodes[k]
    return g, poses


def test_pose_graph_json_round_trip(tmp_path):
    g, _ = _graph(5, 1)
    g.edges[3].confidence = 0.375
    path = str(tmp_path / "g.json")
    mw.write_pose_graph(path, g)
    back = mw.read_pose_graph(path)
    assert len(back.nodes) == 5 and len(back.edges) == len(g.edges)
    assert all(np.array_equal(a, b) for a, b in zip(g.nodes, back.nodes))
    for a, b in zip(g.edges, back.edges):
        assert (a.source, a.target, a.uncertain, a.confidence) == (b.source, b.target, b.uncertain, b.confidence)
        assert np.array_equal(a.transformation, b.transformation) and np.array_equal(a.information, b.information)
    # open3d's layout: column-major matrices
    import json
    doc = json.load(open(path))
    assert doc["class_name"] == "PoseGraph"
    assert doc["nodes"][1]["pose"][12:15] == [float(x) for x in g.nodes[1][:3, 3]]


# From a perturbed start the optimisation stops once the residual is below the criteria's 1e-6 (sum of e^T Info e, Info ~ 1e3 over
# tens of edges): the poses are then within ~1e-5 of the truth.  From the truth itself it takes no step.
@pytest.mark.parametrize("noise,tol", [(0.0, 1e-9), (1.0, 1e-5)])
def test_consistent_graph_returns_the_ground_truth(noise, tol):
    g, poses = _graph(8, 2, noise=noise)
    out = mw.global_optimization(g)
    assert len(out.edges) == len(g.edges)
    assert max(np.abs(a - b).max() for a, b in zip(out.nodes, poses)) < tol


def test_reference_node_keeps_its_pose():
    g, poses = _graph(6, 3, noise=1.0)
    g.nodes = [_rigid(np.random.default_rng(9), 10, 0.5) @ p for p in g.nodes]     # a graph in another world frame
    for ref in (0, 4):
        out = mw.global_optimization(g, reference_node=ref)
        assert np.abs(out.nodes[ref] - g.nodes[ref]).max() < 1e-12


def test_false_loop_closures_are_pruned():
    g, poses = _graph(10, 4, noise=1.0)
    rng = np.random.default_rng(5)
    planted = {(0, 5), (2, 8), (3, 9)}
    for e in g.edges:
        if (e.source, e.target) in planted:
            e.transformation = _rigid(rng, 40, 0.5) @ e.transformation
    first = mw.optimize_pose_graph(g)
    low = {(e.source, e.target) for e in first.edges if e.confidence < 0.25}
    assert low == planted
    out = mw.global_optimization(g)
    kept = {(e.source, e.target) for e in out.edges}
    assert not kept & planted and len(kept) == len(g.edges) - len(planted)
    assert max(np.abs(a - b).max() for a, b in zip(out.nodes, poses)) < 1e-5


def test_residual_does_not_increase_across_accepted_steps():
    g, _ = _graph(9, 6, noise=3.0)
    g.edges[10].transformation = _rigid(np.random.default_rng(1), 30, 0.3) @ g.edges[10].transformation
    hist = []
    mw.optimize_pose_graph(g, history=hist)
    assert len(hist) >= 2
    assert all(b <= a for a, b in zip(hist[:-1], hist[1:])), hist


def test_trajectory_ate():
    rng = np.random.default_rng(7)
    gt = [_rigid(rng, 90, 2.0) for _ in range(12)]
    M = _rigid(rng, 50, 3.0)
    assert mw.trajectory_ate(gt, [M @ p for p in gt]) < 1e-9
    moved = [p.copy() for p in gt]
    moved[3][0, 3] += 0.1
    assert 0.5 < mw.trajectory_ate(gt, moved) < 10.0 / np.sqrt(12) + 1e-9


# ---------------------------------------------------------------------------------------------------------------- the driver
class _Model:
    def __init__(self, log, trans):
        self.log, self.trans = log, trans

    def forward_packed(self, corr_pos, src_keypts, tgt_keypts, offsets, d_offsets=None):
        self.log.append(("forward_packed", len(offsets) - 1))
        return {"final_trans": torch.stack([self.trans.pop(0) for _ in range(len(offsets) - 1)]),
                "final_labels": torch.ones(offsets[-1])}


def _fake_scene(K, n=12):
    g = np.random.default_rng(0)
    gt = [np.eye(4)] + [_rigid(g, 10, 0.2) for _ in range(K - 1)]
    return {"xyz": [torch.from_numpy(g.uniform(size=(n + k, 3)).astype(np.float32)) for k in range(K)],
            "feat": [torch.from_numpy(g.uniform(size=(n + k, 33))) for k in range(K)],
            "gt": gt, "odometry_init": [np.linalg.inv(gt[i + 1]) @ gt[i] for i in range(K - 1)]}


def _install(monkeypatch, log, loop_info):
    """Fakes for the device calls: the odometry ICP returns the initialisation, each loop closure the information matrix
    loop_info[(i, j)] (N correspondences = the source fragment's rows)."""
    def msi(clouds, pairs, inits, **kw):
        log.append(("multi_scale_icp_packed", list(pairs)))
        return inits.clone(), torch.from_numpy(np.stack([np.eye(6) * 100.0] * len(pairs)))

    def match_many(items, use_mutual=False):
        off = np.cumsum([0] + [int(it[2].shape[0]) for it in items]).tolist()
        log.append(("match_many", len(items)))
        return {"corr_pos": torch.zeros(off[-1], 6), "src_keypts": torch.zeros(off[-1], 3), "tgt_keypts": torch.zeros(off[-1], 3),
                "offsets": off, "d_offsets": None}

    def info(src, tgt, trans, so, to, d_src_offsets=None, d_tgt_offsets=None, max_correspondence_distance=None, status=False):
        assert so == to and max_correspondence_distance == pytest.approx(0.07)
        log.append(("information_matrix_packed", len(so) - 1))
        return torch.from_numpy(np.stack([loop_info.pop(0) for _ in range(len(so) - 1)]))

    monkeypatch.setattr(mw, "multi_scale_icp_packed", msi)
    monkeypatch.setattr(driver.frontend, "match_many", match_many)
    monkeypatch.setattr(mw, "information_matrix_packed", info)


def test_driver_routes_pairs_prunes_and_writes(monkeypatch, tmp_path):
    K = 5
    data = _fake_scene(K)
    odo, loops, pairs = driver.scene_pairs(K)
    assert pairs == [(i, j) for i in range(K) for j in range(i + 1, K)]
    assert odo == [(0, 1), (1, 2), (2, 3), (3, 4)]
    assert loops == [(0, 2), (0, 3), (0, 4), (1, 3), (1, 4), (2, 4)]
    # the prune rule at its edges: info[5,5] / N against 0.30 (N = the source fragment's rows, 12 + i), trace(T) == 4
    infos, trans, expect = [], [], []
    rng = np.random.default_rng(1)
    for k, (i, j) in enumerate(loops):
        n = 12 + i
        I6 = np.eye(6)
        T = _rigid(rng, 5, 0.1)
        if k == 0:
            I6[5, 5] = 0.30 * n            # exactly 0.30: kept
        elif k == 1:
            I6[5, 5] = np.nextafter(0.30 * n, 0)    # just below: dropped
        elif k == 2:
            I6[5, 5] = n
            T = np.eye(4)                  # trace 4: dropped
        elif k == 3:
            I6[5, 5] = n
            T = np.diag([1.0, 1.0, 1.0, 1.0]) + np.array([[0, 0, 0, 0.5]] + [[0] * 4] * 3)   # trace 4, not the identity: dropped
        else:
            I6[5, 5] = n
        infos.append(I6)
        trans.append(torch.from_numpy(T.astype(np.float32)))
        expect.append(k in (0, 4, 5))
    assert driver.keep_loop_closure(np.eye(4) * 2, np.diag([1, 1, 1, 1, 1, 3.0]), 10)
    log = []
    _install(monkeypatch, log, infos)
    monkeypatch.setattr(mw, "global_optimization", lambda g, **kw: g.copy())
    prefix = str(tmp_path / "scene_fpfh")
    g, ate = driver.run_scene(_Model(log, trans), data, prefix, use_icp=True, batch_size=4, log=lambda *_: None)
    assert log[0] == ("multi_scale_icp_packed", odo)
    assert log[1:7] == [("match_many", 4), ("forward_packed", 4), ("information_matrix_packed", 4),
                        ("match_many", 2), ("forward_packed", 2), ("information_matrix_packed", 2)]
    kept = [p for p, e in zip(loops, expect) if e]
    g0 = mw.read_pose_graph(prefix + "_0.json")
    assert [(e.source, e.target) for e in g0.edges] == [p for p in pairs if p in odo or p in kept]
    assert [e.uncertain for e in g0.edges] == [p not in odo for p in pairs if p in odo or p in kept]
    assert len(g0.nodes) == K
    # the surviving edges are refined in one call, in the graph's edge order
    assert log[7] == ("multi_scale_icp_packed", [(e.source, e.target) for e in g0.edges]) and len(log) == 8
    for suffix in ("_0.json", "_1.json", "_2.json"):
        assert os.path.exists(prefix + suffix)
    # the odometry nodes: pose = inverse of the accumulated odometry, which the fake ICP left at the ground-truth steps
    assert max(np.abs(a - b).max() for a, b in zip(g0.nodes, data["gt"])) < 1e-5
    assert ate < 1e-3


def test_driver_without_icp_writes_two_graphs(monkeypatch, tmp_path):
    K = 3
    log = []
    _install(monkeypatch, log, [np.eye(6) * 100.0])
    prefix = str(tmp_path / "s")
    driver.run_scene(_Model(log, [torch.eye(4) * 2]), _fake_scene(K), prefix, use_icp=False, log=lambda *_: None)
    assert [x[0] for x in log] == ["multi_scale_icp_packed", "match_many", "forward_packed", "information_matrix_packed"]
    assert os.path.exists(prefix + "_1.json") and not os.path.exists(prefix + "_2.json")


def test_num_node_limit_and_seeded_subsampling():
    assert driver.parse_args([]).num_node == 16384 and driver.parse_args([]).use_icp is True
    assert driver.parse_args(["--use_icp", "false"]).use_icp is False
    with pytest.raises(SystemExit):
        driver.parse_args(["--num_node", "20000"])
    assert driver.subsample(100, 200, 0, 1, 2, 0) is None
    a = driver.subsample(30000, 16384, 0, 1, 5, 0)
    assert len(a) == 16384 and len(np.unique(a)) == 16384
    assert np.array_equal(a, driver.subsample(30000, 16384, 0, 1, 5, 0))
    assert not np.array_equal(a, driver.subsample(30000, 16384, 0, 1, 5, 1))
