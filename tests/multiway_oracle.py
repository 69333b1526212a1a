"""Float64 restatements of the multiway registration's device calls (row f7), for the tests that check them: ICP between two
clouds per pair (pdsc_icp_clouds_packed) and open3d's information matrix (pdsc_information_matrix_packed).  Both reuse
oracle/icp_oracle.py's conventions as they stand: its single-set `icp` (which already takes a source and a target of different
sizes, fitness = |C| / Ns), its nearest-target search (exact (d^2, row) minimum, ties to the lowest row) and its status rule."""
import numpy as np

from oracle import icp_oracle as O


def icp_clouds_packed(src, tgt, init, src_offsets, tgt_offsets, max_correspondence_distance: float = 0.07,
                      max_iteration: int = 30) -> list:
    """`O.icp` of every pair b of a two-cloud group: source rows src_offsets[b]:src_offsets[b+1] of src, target rows
    tgt_offsets[b]:tgt_offsets[b+1] of tgt, init [B,4,4]."""
    return [O.icp(src[src_offsets[b]:src_offsets[b + 1]], tgt[tgt_offsets[b]:tgt_offsets[b + 1]], init[b], max_correspondence_distance,
                  max_iteration) for b in range(len(src_offsets) - 1)]


def information_matrix(src, tgt, trans, max_correspondence_distance: float) -> dict:
    """open3d 0.9's get_information_matrix_from_point_clouds(src, tgt, r, trans), restated in float64 (recalled from its source,
    not checkable here; the device call is pdsc_information_matrix_packed).  Conventions:

      * the source [Ns,3] float32 is moved by trans [4,4] float32, in float64;
      * correspondences as `O.icp`'s: the nearest target row of every moved source row, kept iff d^2 < float32(r * r), ties to
        the lowest row;
      * every kept correspondence with target point (x, y, z) adds G G^T for the rows (0, z, -y, 1, 0, 0), (-z, 0, x, 0, 1, 0),
        (y, -x, 0, 0, 0, 1) of G, so info[5,5] = |C| and info[3:,3:] = |C| I;
      * status 1 (a non-finite coordinate, or a target spanning 2^21 or more cells): the zero matrix.

    Returns {'info' [6,6] float64, 'count', 'status', 'rows' (the kept (source, target) rows), 'margins': {'d2_radius',
    'nn_gap'}}: the smallest |d^2 - r^2_f| of a nearest neighbour and the smallest gap between the nearest and the next distinct
    target, the margins a float64 computation in another order must clear to keep the same correspondences."""
    src = np.asarray(src, np.float32).astype(np.float64)
    tgt = np.asarray(tgt, np.float32).astype(np.float64)
    T = np.asarray(trans, np.float32).astype(np.float64)
    r = float(max_correspondence_distance)
    margins = {"d2_radius": np.inf, "nn_gap": np.inf}
    if O._status(src, tgt, r):
        return {"info": np.zeros((6, 6)), "count": 0, "status": 1, "rows": np.zeros((0, 2), np.int64), "margins": margins}
    targets = O._Targets(tgt, r, "kdtree")
    P = src @ T[:3, :3].T + T[:3, 3]
    row, d2, gap = targets.nearest(P)
    found = row >= 0
    if found.any():
        margins["d2_radius"] = float(np.abs(d2[found] - targets.r2f).min())
        margins["nn_gap"] = float(gap[found].min())
    keep = found & (d2 < targets.r2f)
    q = tgt[row[keep]]
    x, y, z = q[:, 0], q[:, 1], q[:, 2]
    zero, one = np.zeros_like(x), np.ones_like(x)
    G = np.stack([np.stack([zero, z, -y, one, zero, zero], 1),
                  np.stack([-z, zero, x, zero, one, zero], 1),
                  np.stack([y, -x, zero, zero, zero, one], 1)], 1)          # [|C|, 3, 6]
    info = np.einsum("cki,ckj->ij", G, G)
    return {"info": info, "count": int(keep.sum()), "status": 0,
            "rows": np.stack([np.nonzero(keep)[0], row[keep]], 1), "margins": margins}
