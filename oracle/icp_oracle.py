"""CPU restatement of the drivers' --use_icp refinement (evaluation/benchmark_utils.py:40-55, called from
evaluation/test_3DMatch.py:79-80, evaluation/test_KITTI.py:79-80, multiway/test_multi.py:53-54): open3d 0.9's
`registration_icp(src, tgt, 0.10, init, TransformationEstimationPointToPoint(False), ICPConvergenceCriteria())` over the pair's
correspondence key points (source = src_keypts, target = tgt_keypts, the rows the forward consumes).

TEST INFRASTRUCTURE ONLY.  **Parity unpinned**: open3d is not part of the reference tree or of this image, so this file restates
open3d 0.9's RegistrationICP from its published source, in float64 throughout, and the CUDA kernel (pointdsc_b200/csrc/icp.cu) is
tested against THIS restatement.  Conventions, named because open3d leaves them to FLANN or because they are recalled rather than
checked:

  * correspondence: the nearest target row of every source row, kept iff d^2 < float32(r * r) (open3d's SearchHybrid hands
    `float(radius * radius)` to FLANN; recalled from open3d's source, not checkable here);
  * ties in d^2 go to the lowest target row (FLANN's pick depends on its tree order; duplicate target positions, common because
    matching maps many sources onto one target, give the same coordinates whichever row wins);
  * fitness = |C| / N, inlier_rmse = sqrt(sum d^2 / |C|), 0 when C is empty;
  * update: Umeyama without scaling over C (means, demeaned covariance, SVD, reflection fix on the smallest singular direction),
    the identity when C is empty; T <- U T and the moved cloud P <- U P incrementally, as open3d transforms its copy of the cloud;
  * stop after `max_iteration` updates, or as soon as |d fitness| < 1e-6 and |d rmse| < 1e-6 (ICPConvergenceCriteria defaults);
  * a set with a non-finite coordinate, or whose target spans 2^21 or more grid cells of side max(r, sqrt(float32(r * r))) along
    an axis, is not refined: status 1, T = init, 0 iterations, fitness = rmse = 0 (the device kernel's cell index limit).

Every run records the margins that decide whether a float64 computation in another order (the device's) must take the same
discrete decisions: the smallest |d^2 - r^2_f| of a nearest neighbour, the smallest gap in d^2 between the nearest and the next
distinct target position, the smallest distance of |d rmse| from the 1e-6 criterion, and the smallest sigma_2 / sigma_1 of an
update over two or more correspondences (below rank 2 the rotation is not unique and any two SVDs may pick different ones).
`late_margins` are the same margins without the first correspondence search, for runs built so that the first search decides
at an exact edge on purpose.  `decide`, a hook on every search, can override its outcome: that is how a test shows that a
decision it placed on an edge matters.
"""
import numpy as np
from scipy.spatial import cKDTree

RELATIVE_FITNESS = 1e-6
RELATIVE_RMSE = 1e-6
MAX_CELLS = 1 << 21


def radius_sq(r: float) -> float:
    """float32(r * r) as float64: the squared radius open3d hands to FLANN."""
    return float(np.float32(r * r))


def cell_side(r: float) -> float:
    return max(r, float(np.sqrt(radius_sq(r))))


def umeyama(a: np.ndarray, b: np.ndarray):
    """(R, t, sigma_2 / sigma_1) of the rigid transform that maps a [n,3] onto b [n,3] in the least-squares sense."""
    if len(a) == 0:
        return np.eye(3), np.zeros(3), np.inf
    am, bm = a.mean(0), b.mean(0)
    H = (a - am).T @ (b - bm)                       # H[i, j] = sum_n a_i b_j
    if not np.any(H):
        return np.eye(3), bm - am, np.inf
    U, S, Vt = np.linalg.svd(H)
    d = 1.0 if np.linalg.det(Vt.T @ U.T) >= 0 else -1.0
    R = Vt.T @ np.diag([1.0, 1.0, d]) @ U.T
    ratio = S[1] / S[0] if len(a) >= 2 else np.inf
    return R, bm - R @ am, ratio


class _Targets:
    """Nearest target row of query points: exact float64 (d^2, row) minimum, lowest row on ties."""

    def __init__(self, tgt: np.ndarray, r: float, search: str):
        self.tgt, self.r2f, self.search = tgt, radius_sq(r), search
        # distinct positions, each represented by its lowest row (np.unique keeps the first occurrence)
        self.pos, self.first = np.unique(tgt, axis=0, return_index=True)
        self.bound = 2.0 * cell_side(r)                 # candidates further than this never decide anything
        if search == "kdtree":
            self.tree = cKDTree(self.pos)

    def nearest(self, P: np.ndarray):
        """(row [N] int64 or -1, d2 [N], gap [N] = d^2 of the next distinct position - d^2 of the nearest)."""
        if self.search == "kdtree":
            k = min(2, len(self.pos))
            _, idx = self.tree.query(P, k=k, distance_upper_bound=self.bound)
            idx = idx.reshape(len(P), k)
            ok = idx < len(self.pos)
            safe = np.where(ok, idx, 0)
            d2 = np.where(ok, ((P[:, None, :] - self.pos[safe]) ** 2).sum(-1), np.inf)
        else:                                          # brute force over every distinct position
            d2all = ((P[:, None, :] - self.pos[None, :, :]) ** 2).sum(-1)
            k = min(2, len(self.pos))
            safe = np.argsort(d2all, axis=1, kind="stable")[:, :k]
            d2 = np.take_along_axis(d2all, safe, 1)
            d2 = np.where(d2 < self.bound * self.bound, d2, np.inf)
        # exact order of the candidates by (d^2, row)
        rows = self.first[safe]
        swap = (d2[:, 1] < d2[:, 0]) | ((d2[:, 1] == d2[:, 0]) & (rows[:, 1] < rows[:, 0])) if k == 2 else np.zeros(len(P), bool)
        d1 = np.where(swap, d2[:, 1], d2[:, 0]) if k == 2 else d2[:, 0]
        r1 = np.where(swap, rows[:, 1], rows[:, 0]) if k == 2 else rows[:, 0]
        with np.errstate(invalid="ignore"):                # inf - inf where neither candidate exists
            gap = np.abs(d2[:, 1] - d2[:, 0]) if k == 2 else np.full(len(P), np.inf)
        r1 = np.where(np.isfinite(d1), r1, -1)
        return r1, d1, gap


def _status(src: np.ndarray, tgt: np.ndarray, r: float) -> int:
    if not (np.isfinite(src).all() and np.isfinite(tgt).all()):
        return 1
    lo = tgt.min(0)
    cells = np.floor((tgt - lo) / cell_side(r))
    return 1 if (cells >= MAX_CELLS).any() else 0


def icp(src, tgt, init, max_correspondence_distance: float = 0.10, max_iteration: int = 30, search: str = "kdtree",
        decide=None, record: bool = False) -> dict:
    """Point-to-point ICP of one set.  src, tgt [N,3] float32 (row j of src corresponds to nothing in particular: the target is
    searched), init [4,4] float32.  Returns {'trans' [4,4] float32, 'trans64', 'fitness', 'inlier_rmse', 'iterations', 'status',
    'margins' and 'late_margins': {'d2_radius', 'nn_gap', 'rmse_criterion', 'sigma_ratio'}}.

    decide(search, row, d2, keep) -> (row, keep), when given, sees every correspondence search (0 = the one before the first
    update): the nearest target row of every source row (-1: none), its d^2 and whether it is kept, and returns the rows and
    the kept mask to use.  record=True adds 'updates': the (moved source, target) point pairs of every update."""
    src = np.asarray(src, np.float32).astype(np.float64)
    tgt = np.asarray(tgt, np.float32).astype(np.float64)
    T = np.asarray(init, np.float32).astype(np.float64)
    r = float(max_correspondence_distance)
    margins = {"d2_radius": np.inf, "nn_gap": np.inf, "rmse_criterion": np.inf, "sigma_ratio": np.inf}
    late = dict(margins)
    if _status(src, tgt, r):
        return {"trans": T.astype(np.float32), "trans64": T, "fitness": 0.0, "inlier_rmse": 0.0, "iterations": 0, "status": 1,
                "margins": margins, "late_margins": late, "updates": []}
    N = len(src)
    targets = _Targets(tgt, r, search)
    r2f = targets.r2f

    searches = 0
    updates = []

    def correspondences(P):
        nonlocal searches
        row, d2, gap = targets.nearest(P)
        found = row >= 0
        if found.any():
            for m in (margins, late) if searches else (margins,):
                m["d2_radius"] = min(m["d2_radius"], float(np.abs(d2[found] - r2f).min()))
                m["nn_gap"] = min(m["nn_gap"], float(gap[found].min()))
        keep = found & (d2 < r2f)
        if decide is not None:
            row, keep = decide(searches, row.copy(), d2, keep.copy())
        searches += 1
        n = int(keep.sum())
        rmse = float(np.sqrt(d2[keep].sum() / n)) if n else 0.0
        return np.nonzero(keep)[0], row[keep], n / N, rmse

    P = src @ T[:3, :3].T + T[:3, 3]
    cs, ct, fitness, rmse = correspondences(P)
    iterations = 0
    for _ in range(max_iteration):
        R, t, ratio = umeyama(P[cs], tgt[ct])
        if record:
            updates.append((P[cs].copy(), tgt[ct].copy()))
        for m in (margins, late):
            m["sigma_ratio"] = min(m["sigma_ratio"], ratio)
        U = np.eye(4)
        U[:3, :3], U[:3, 3] = R, t
        T = U @ T
        P = P @ R.T + t
        iterations += 1
        cs, ct, f2, r2 = correspondences(P)
        for m in (margins, late):
            m["rmse_criterion"] = min(m["rmse_criterion"], abs(abs(rmse - r2) - RELATIVE_RMSE))
        done = abs(fitness - f2) < RELATIVE_FITNESS and abs(rmse - r2) < RELATIVE_RMSE
        fitness, rmse = f2, r2
        if done:
            break
    return {"trans": T.astype(np.float32), "trans64": T, "fitness": fitness, "inlier_rmse": rmse, "iterations": iterations,
            "status": 0, "margins": margins, "late_margins": late, "updates": updates}


def icp_packed(src, tgt, init, offsets, max_correspondence_distance: float = 0.10, max_iteration: int = 30) -> list:
    """`icp` of every set b of a packed group: rows offsets[b]:offsets[b+1] of src / tgt [R,3], init [B,4,4]."""
    return [icp(src[a:b], tgt[a:b], init[i], max_correspondence_distance, max_iteration)
            for i, (a, b) in enumerate(zip(offsets[:-1], offsets[1:]))]


def margin(result) -> float:
    """The smallest recorded margin of a run (inf when no decision was close to anything)."""
    return min(result["margins"].values())
