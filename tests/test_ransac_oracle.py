"""The CPU restatement of the drivers' --solver RANSAC (oracle/ransac_oracle.py) on its own: its draws against a plain integer
SplitMix64, its selection against a literal transcription of open3d's replace loop, the status-1 and status-2 sets, its labels, and
recovery of the ground truth on synthetic 3DMatch-like and KITTI-like sets."""
import math

import numpy as np
import pytest

from oracle import ransac_oracle as O

M64 = (1 << 64) - 1


def splitmix_int(seed, k):
    z = (seed + k * 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


@pytest.mark.parametrize("seed", [0, 51, (1 << 64) - 3])
def test_generator_equals_integer_splitmix(seed):
    got = O.splitmix64(seed, np.arange(1, 10001, dtype=np.uint64))
    want = [splitmix_int(seed, k) for k in range(1, 10001)]
    assert [int(x) for x in got] == want
    for M in (3, 7, 1000, 16384):
        d = O.draws(seed, 3334, M).reshape(-1)[:10000]
        assert d.tolist() == [(w >> 33) % M for w in want]


def open3d_loop(good, rmse, M):
    """Registration.cpp's loop, transcribed: best starts at fitness 0, rmse 0; replace iff fitness > best or (== and rmse <)."""
    best_fit, best_rmse, best = 0.0, 0.0, -1
    for i, (g, r) in enumerate(zip(good, rmse)):
        fit = g / M
        if fit > best_fit or (fit == best_fit and r < best_rmse):
            best_fit, best_rmse, best = fit, r, i
    return best


@pytest.mark.parametrize("seed", range(8))
def test_selection_equals_the_replace_loop(seed):
    g = np.random.default_rng(seed)
    I, M = 2000, 37
    good = g.integers(0, 6, I)                                   # many ties in good, and zeros
    rmse = np.round(g.random(I), 2)                              # many exact ties in rmse
    rmse[good == 0] = 0.0
    if seed % 2:
        good[:] = np.where(good > 0, 5, 0)                           # every non-empty key ties in good
    want = open3d_loop(good, rmse, M)
    assert O.select(good, rmse) == want
    assert O.select(np.zeros(I, int), np.zeros(I)) == -1 == open3d_loop(np.zeros(I, int), np.zeros(I), M)


def _spread_targets(m, seed=0):
    """One source point repeated m times against m targets scattered over a 1 km cube: every hypothesis maps the source onto the
    mean of its drawn targets, which is no target unless all three draws are the same index."""
    g = np.random.default_rng(seed)
    src = np.tile(np.float32([[1.0, 2.0, 3.0]]), (m, 1))
    tgt = (g.random((m, 3)) * 1000.0).astype(np.float32)
    return src, tgt


def status2_case(m=1000, seed=7, max_iteration=5000):
    src, tgt = _spread_targets(m)
    d = O.draws(seed, max_iteration, m)
    assert not ((d[:, 0] == d[:, 1]) & (d[:, 1] == d[:, 2])).any()
    return src, tgt, np.ones(m, np.float32)


@pytest.mark.parametrize("m", [0, 1, 2])
def test_fewer_than_three_candidates(m):
    g = np.random.default_rng(m)
    src, tgt = g.random((5, 3)).astype(np.float32), g.random((5, 3)).astype(np.float32)
    labels = np.zeros(5, np.float32)
    labels[[1, 3][:m]] = 1.0
    labels[4] = -1.0
    r = O.ransac(src, tgt, labels)
    assert r["status"] == 1 and r["M"] == m and r["best_iteration"] == -1
    assert np.array_equal(r["trans"], np.eye(4, dtype=np.float32)) and not r["labels"].any()
    assert r["fitness"] == 0.0 and r["inlier_rmse"] == 0.0


def test_no_hypothesis_with_an_inlier():
    src, tgt, labels = status2_case()
    r = O.ransac(src, tgt, labels)
    assert r["status"] == 2 and r["best_iteration"] == -1 and not r["good"].any()
    assert np.array_equal(r["trans"], np.eye(4, dtype=np.float32)) and not r["labels"].any()


def _case(preset, n, seed):
    from pointdsc_b200.synth import make_pair
    p = make_pair(seed, n, preset)
    return p["src_keypts"].numpy(), p["tgt_keypts"].numpy(), p["gt_labels"].numpy(), p["gt_trans"].numpy().astype(np.float64)


def test_labels_are_exactly_the_winners_inliers():
    src, tgt, labels, _ = _case("3dmatch", 600, 4)
    labels = labels.copy()
    labels[::7] = 1.0                                            # some outliers among the candidates
    r = O.ransac(src, tgt, labels, max_iteration=500)
    T = r["T"][r["best_iteration"]]
    want = np.zeros(len(src), np.float32)
    for row in range(len(src)):
        if labels[row] > 0:
            x = [sum(T[i, j] * float(src[row, j]) for j in range(3)) + T[i, 3] - float(tgt[row, i]) for i in range(3)]
            want[row] = 1.0 if sum(v * v for v in x) < 0.1 * 0.1 else 0.0
    assert np.array_equal(r["labels"], want)
    assert int(want.sum()) == r["good"][r["best_iteration"]] and r["fitness"] == want.sum() / r["M"]
    assert not (r["labels"] > 0)[labels <= 0].any()


def _re_te(T, gt):
    c = np.clip((np.trace(T[:3, :3].T @ gt[:3, :3]) - 1) / 2, -1, 1)
    return math.degrees(math.acos(c)), float(np.linalg.norm(T[:3, 3] - gt[:3, 3])) * 100


@pytest.mark.parametrize("preset,r,re_thre,te_thre,seed", [("3dmatch", 0.10, 15.0, 30.0, 0), ("3dmatch", 0.10, 15.0, 30.0, 3),
                                                           ("kitti", 0.6, 5.0, 60.0, 1), ("kitti", 0.6, 5.0, 60.0, 2)])
def test_recovers_the_ground_truth(preset, r, re_thre, te_thre, seed):
    src, tgt, labels, gt = _case(preset, 2000, seed)
    labels = labels.copy()
    labels[1500:1800] = 1.0                                      # the network keeps some outliers too
    res = O.ransac(src, tgt, labels, r)
    assert res["status"] == 0
    re, te = _re_te(res["trans"].astype(np.float64), gt)
    assert re < re_thre and te < te_thre, (re, te)
    assert res["labels"][:600].mean() > 0.9 and res["labels"][1500:1800].mean() < 0.05
