"""CPU restatement of the drivers' --solver RANSAC (evaluation/test_3DMatch.py:59-77, evaluation/test_KITTI.py:59-77): open3d 0.9's
`registration_ransac_based_on_correspondence(src, tgt, corres, r, TransformationEstimationPointToPoint(False), 3,
RANSACConvergenceCriteria(5000, 5000))` over the rows the network labelled as inliers, whose inliers then replace pred_labels and
whose transform replaces pred_trans.

TEST INFRASTRUCTURE ONLY.  **Parity unpinned**: open3d is not part of the reference tree or of this image, so this file restates
open3d 0.9's Registration.cpp from memory, in float64 throughout, and the CUDA kernel (pointdsc_b200/csrc/ransac.cu) is tested
against THIS restatement.  Conventions, each recalled from open3d 0.9 and not checkable here unless said otherwise:

  * candidates: the rows with pred_labels > 0 in ascending order (`np.where` in the driver: checkable, test_3DMatch.py:64), M of
    them; source point = src_keypts row, target point = tgt_keypts row, float32 widened to float64;
  * M < ransac_n = 3: open3d's default result (identity, fitness 0, rmse 0, no correspondence).  The driver would then fail at
    `inliers[:, 0]`; here: identity, all-zero labels, status 1;
  * iterations: itr < max_iteration && itr < max_validation, no early exit in 0.9;
  * draws: open3d takes corres[rand() % M] three times, repeats allowed, after srand(time(0)), which no one can replay.  This
    project's draws instead: index = (z >> 33) % M with z = SplitMix64(seed + (3 i + j + 1) * 0x9E3779B97F4A7C15 mod 2^64) for
    draw j = 0, 1, 2 of iteration i (31 bits like glibc's rand(), modulo bias included).  They depend on (seed, i, j) only;
  * solve: the unscaled Umeyama over the 3 drawn pairs (icp_oracle.umeyama: means, demeaned covariance, SVD, reflection fix on
    the smallest singular direction, t = b - R a).  A sample with a non-finite coordinate scores good = 0;
  * score: d^2 = |R p + t - q|^2 in double over every candidate, an inlier iff d^2 < r * r with r * r a DOUBLE product (ICP
    differs: it hands float32(r^2) to FLANN); good = inliers, fitness = good / M, rmse = sqrt(sum d^2 / good), 0 when good = 0;
  * select: best starts at (identity, fitness 0, rmse 0) and hypothesis i replaces it iff fitness > best.fitness or (fitness ==
    best.fitness and rmse < best.rmse): the largest good, then the smallest rmse, then the earliest i among good > 0.  None with
    good > 0: identity, all-zero labels, status 2;
  * outputs: pred_trans = the winner's 3-point solve as float32 (no refit on its inliers), pred_labels = 1 exactly on its inliers.

Every run records the margins that decide whether a float64 computation in another order (the device's) must take the same
discrete decisions: per hypothesis the smallest |d^2 - r * r| over the candidates ('d2_radius') and sigma_2 / sigma_1 of its sample
('sigma_ratio': below rank 2 the rotation is not unique, which two drawn indices that are equal, or three collinear points, cause),
and for the whole run the relative rmse gap from the winner's key to the best key of a hypothesis with the same good and a
different ordered triple ('selection'; inf when no such hypothesis exists).  Hypotheses that drew the same ordered triple compute
the same key bit for bit in any one implementation, so their tie always goes to the earliest.
"""
import numpy as np

from oracle.icp_oracle import umeyama

GOLDEN_GAMMA = 0x9E3779B97F4A7C15
DEFAULT_SEED = 51
_M64 = (1 << 64) - 1


def splitmix64(seed: int, k: np.ndarray) -> np.ndarray:
    """SplitMix64 output for stream positions k (uint64 array): z = seed + k * golden, then the two xor-shift-multiply rounds."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed & _M64) + np.asarray(k, np.uint64) * np.uint64(GOLDEN_GAMMA)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def draws(seed: int, max_iteration: int, M: int) -> np.ndarray:
    """[max_iteration, 3] int64 candidate indices: draw j of iteration i is (z >> 33) % M, z at stream position 3 i + j + 1."""
    k = np.arange(1, 3 * max_iteration + 1, dtype=np.uint64)
    return ((splitmix64(seed, k) >> np.uint64(33)) % np.uint64(M)).astype(np.int64).reshape(max_iteration, 3)


def select(good: np.ndarray, rmse: np.ndarray) -> int:
    """The winning iteration of keys (good [I], rmse [I]): the largest good, then the smallest rmse, then the earliest, among
    good > 0; -1 when no hypothesis has an inlier."""
    good, rmse = np.asarray(good), np.asarray(rmse, np.float64)
    ok = np.nonzero(good > 0)[0]
    if len(ok) == 0:
        return -1
    order = np.lexsort((ok, rmse[ok], -good[ok]))     # last key is primary
    return int(ok[order[0]])


def candidates(labels) -> np.ndarray:
    return np.nonzero(np.asarray(labels, np.float32) > 0)[0]


def ransac(src, tgt, labels, max_correspondence_distance: float = 0.10, max_iteration: int = 5000, seed: int = DEFAULT_SEED,
           chunk: int = 256) -> dict:
    """RANSAC of one set.  src, tgt [N,3] float32, labels [N] (> 0: a candidate).  Returns {'trans' [4,4] float32, 'labels' [N]
    float32, 'fitness', 'inlier_rmse', 'best_iteration' (-1: none), 'status', 'M', 'draws' [I,3], 'good' [I], 'rmse' [I],
    'T' [I,4,4] float64, 'sigma_ratio' [I], 'd2_radius' [I], 'selection'}.  The per-hypothesis arrays are empty when M < 3."""
    src = np.asarray(src, np.float32).astype(np.float64)
    tgt = np.asarray(tgt, np.float32).astype(np.float64)
    rows = candidates(labels)
    N, M, r = len(src), len(rows), float(max_correspondence_distance)
    r2 = r * r
    out = {"trans": np.eye(4, dtype=np.float32), "labels": np.zeros(N, np.float32), "fitness": 0.0, "inlier_rmse": 0.0,
           "best_iteration": -1, "status": 1, "M": M, "draws": np.zeros((0, 3), np.int64), "good": np.zeros(0, np.int64),
           "rmse": np.zeros(0), "T": np.zeros((0, 4, 4)), "sigma_ratio": np.zeros(0), "d2_radius": np.zeros(0), "selection": np.inf}
    if M < 3:
        return out
    p, q = src[rows], tgt[rows]
    idx = draws(seed, max_iteration, M)
    I = max_iteration
    T = np.tile(np.eye(4), (I, 1, 1))
    ratio = np.full(I, np.inf)
    ok = np.ones(I, bool)
    for i in range(I):
        a, b = p[idx[i]], q[idx[i]]
        if not (np.isfinite(a).all() and np.isfinite(b).all()):
            ok[i] = False
            continue
        R, t, ratio[i] = umeyama(a, b)
        T[i, :3, :3], T[i, :3, 3] = R, t
    good = np.zeros(I, np.int64)
    rmse = np.zeros(I)
    margin = np.full(I, np.inf)
    for i0 in range(0, I, chunk):
        i1 = min(I, i0 + chunk)
        e = np.einsum("hij,mj->hmi", T[i0:i1, :3, :3], p) + T[i0:i1, None, :3, 3] - q[None]
        d2 = (e * e).sum(-1)                                           # [h, M]
        with np.errstate(invalid="ignore"):
            inl = d2 < r2
            gap = np.abs(d2 - r2)
        gap = np.where(np.isfinite(gap), gap, np.inf)
        inl &= ok[i0:i1, None]
        good[i0:i1] = inl.sum(1)
        s = np.where(inl, d2, 0.0).sum(1)
        with np.errstate(invalid="ignore", divide="ignore"):
            rmse[i0:i1] = np.where(good[i0:i1] > 0, np.sqrt(s / np.maximum(good[i0:i1], 1)), 0.0)
        margin[i0:i1] = np.where(ok[i0:i1], gap.min(1), np.inf)
    best = select(good, rmse)
    out.update(draws=idx, good=good, rmse=rmse, T=T, sigma_ratio=ratio, d2_radius=margin, best_iteration=best)
    if best < 0:
        out["status"] = 2
        return out
    e = p @ T[best, :3, :3].T + T[best, :3, 3] - q
    inl = (e * e).sum(-1) < r2
    labels_out = np.zeros(N, np.float32)
    labels_out[rows[inl]] = 1.0
    same = (good == good[best]) & np.any(idx != idx[best], axis=1)
    sel = np.inf
    if same.any():
        gap = float(np.min(np.abs(rmse[same] - rmse[best])))
        sel = gap / rmse[best] if rmse[best] > 0 else (np.inf if gap > 0 else 0.0)
    out.update(trans=T[best].astype(np.float32), labels=labels_out, fitness=good[best] / M, inlier_rmse=float(rmse[best]),
               status=0, selection=sel)
    return out


def ransac_packed(src, tgt, labels, offsets, max_correspondence_distance: float = 0.10, max_iteration: int = 5000,
                  seed: int = DEFAULT_SEED) -> list:
    """`ransac` of every set b of a packed group: rows offsets[b]:offsets[b+1] of src / tgt [R,3] and labels [R]."""
    return [ransac(src[a:b], tgt[a:b], labels[a:b], max_correspondence_distance, max_iteration, seed)
            for a, b in zip(offsets[:-1], offsets[1:])]


def qualifies(result, margin: float = 1e-9) -> np.ndarray:
    """[I] bool: hypotheses whose every recorded margin exceeds `margin` (their good and rmse must match any float64 order)."""
    return (result["d2_radius"] > margin) & (result["sigma_ratio"] > margin)
