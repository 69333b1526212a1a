"""The CPU restatement of the drivers' --use_icp (oracle/icp_oracle.py) on its own: the k-d tree search against brute force,
recovery of an exact rigid motion, the empty and capped runs, and the reference's demo pair."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import icp_oracle as O


def _rigid(seed, deg, cm):
    g = np.random.default_rng(seed)
    ax = g.normal(size=3)
    ax /= np.linalg.norm(ax)
    a = np.deg2rad(deg)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
    T[:3, 3] = g.normal(size=3) * cm / 100
    return T


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_kdtree_equals_brute_force(seed):
    from pointdsc_b200.synth import make_pair
    p = make_pair(seed, 200, "3dmatch")
    src, tgt = p["src_keypts"].numpy(), p["tgt_keypts"].numpy()
    tgt[50:60] = tgt[40:50]                                  # duplicate target positions: the lowest row wins either way
    init = (_rigid(seed, 2.0, 2.0) @ p["gt_trans"].numpy()).astype(np.float32)
    a = O.icp(src, tgt, init, search="kdtree")
    b = O.icp(src, tgt, init, search="brute")
    assert a["iterations"] == b["iterations"] and a["fitness"] == b["fitness"] and a["inlier_rmse"] == b["inlier_rmse"]
    assert np.array_equal(a["trans64"], b["trans64"])
    assert a["margins"] == b["margins"]


def test_recovers_an_exact_rigid_motion():
    # dyadic points and a quarter turn: the target is the exact image of the source in float32, and a start whose rotation is
    # exactly orthogonal keeps every update rigid, so the answer is the motion itself up to float64 rounding
    g = np.random.default_rng(3)
    src = (np.round(g.random((400, 3)) * 3.0 * 1024) / 1024).astype(np.float32)
    truth = np.array([[0.0, -1.0, 0.0, 0.5], [1.0, 0.0, 0.0, -0.25], [0.0, 0.0, 1.0, 0.125], [0.0, 0.0, 0.0, 1.0]])
    tgt = (src.astype(np.float64) @ truth[:3, :3].T + truth[:3, 3]).astype(np.float32)
    assert np.array_equal(tgt.astype(np.float64), src.astype(np.float64) @ truth[:3, :3].T + truth[:3, 3])
    init = truth.astype(np.float32)
    init[:3, 3] += np.float32([0.03, -0.02, 0.025])
    r = O.icp(src, tgt, init)
    assert r["fitness"] == 1.0 and r["status"] == 0 and r["iterations"] >= 2
    assert np.abs(r["trans64"] - truth).max() < 1e-9


def test_no_correspondence_returns_init_after_one_iteration():
    g = np.random.default_rng(6)
    src = g.random((50, 3)).astype(np.float32)
    tgt = (src + 10.0).astype(np.float32)
    init = np.eye(4, dtype=np.float32)
    r = O.icp(src, tgt, init)
    assert r["iterations"] == 1 and r["fitness"] == 0.0 and r["inlier_rmse"] == 0.0 and r["status"] == 0
    assert np.array_equal(r["trans"], init)


def test_status_sets_keep_init():
    g = np.random.default_rng(7)
    src = g.random((20, 3)).astype(np.float32)
    tgt = src.copy()
    tgt[3, 0] = np.inf
    init = np.eye(4, dtype=np.float32)
    r = O.icp(src, tgt, init)
    assert r["status"] == 1 and r["iterations"] == 0 and np.array_equal(r["trans"], init)
    far = src.copy()
    far[0] = [1e6, 0, 0]                                     # 1e7 cells of 0.1 along x: beyond the 2^21-cell grid
    r = O.icp(src, far, init)
    assert r["status"] == 1 and r["iterations"] == 0


@pytest.mark.parametrize("cap", [1, 2, 3])
def test_iteration_cap(cap):
    z = np.load(os.path.join(GOLDEN, "demo_pair_3dmatch.npz"))
    r = O.icp(z["src_keypts"], z["tgt_keypts"], z["final_trans"], max_iteration=cap)
    assert r["iterations"] == cap
    full = O.icp(z["src_keypts"], z["tgt_keypts"], z["final_trans"])
    assert not np.array_equal(r["trans64"], full["trans64"])


def test_demo_pair():
    z = np.load(os.path.join(GOLDEN, "demo_pair_3dmatch.npz"))
    r = O.icp(z["src_keypts"], z["tgt_keypts"], z["final_trans"])
    assert r["iterations"] == 9 and r["status"] == 0
    assert abs(r["fitness"] - 0.8016) < 1e-4 and abs(r["inlier_rmse"] - 0.0421) < 1e-4
    assert 6e-3 < np.abs(r["trans"] - z["final_trans"]).max() < 7e-3
    assert O.margin(r) > 1e-9
    assert len(np.unique(z["tgt_keypts"], axis=0)) == 2024
