"""The spectral-matching baseline SM (baseline_scripts/baseline_3DMatch.py:19-53) restated in float64, with the margins the GPU
tests need.  Torch float64 on whatever device the inputs live on: CPU for the host tests, the GPU for the large sets.

Per set of N rows (corr [N,6] the centred corr_pos, src / tgt [N,3], tau the inlier threshold):
  1. M_ij = ||c_j[0:3] - c_i[0:3]|| - ||c_j[3:6] - c_i[3:6]||;  M_ij = max(0, 4.5 - M_ij^2 / 2 / sigma^2), sigma = tau / 3;
     M_ii = 0  (:20-37).
  2. v = 1, then exactly ten v <- M v / (||M v|| + 1e-6)  (:40-44).
  3. S = int(N * 0.1); labels = 1 on the first S rows of v sorted descending, lowest row first on ties  (:47-49; the
     reference's argsort is unstable, so any order of tied entries is a valid reference output).
  4. T = rigid_transform_3d(src, tgt, v * labels) (models/common.py:7-45): centroids over sum w + 1e-6, H = Am^T diag(w) Bm,
     R = V diag(1, 1, det(V U^T)) U^T, t = cb - R ca.  H = 0 (S = 0, or every weight 0) is defined as the identity.
Margins: `gap` = v_(S) - v_(S+1) of the sorted float64 v (inf when S is 0 or N), `clamp` = the smallest |4.5 - m^2 / (2
sigma^2)| over the off-diagonal pairs, the distance of an entry from the clamp at 0.
"""
import math

import torch

ITERATIONS = 10
TOP_RATIO = 0.1


def num_selected(N, top_ratio=TOP_RATIO):
    return int(N * top_ratio)


def unclamped(corr, inlier_threshold, rows=slice(None)):
    """4.5 - m^2 / (2 sigma^2) of the rows `rows` against every row, float64 [rows, N]."""
    c = corr.to(torch.float64)
    ci = c[rows]
    ds = torch.cdist(ci[:, :3], c[:, :3], compute_mode="donot_use_mm_for_euclid_dist")
    dt = torch.cdist(ci[:, 3:], c[:, 3:], compute_mode="donot_use_mm_for_euclid_dist")
    sigma = inlier_threshold / 3.0
    return 4.5 - (ds - dt) ** 2 / 2.0 / sigma ** 2


def compat(corr, inlier_threshold, chunk=2048):
    """M [N,N] float64 of step 1."""
    N = corr.shape[0]
    M = torch.empty(N, N, dtype=torch.float64, device=corr.device)
    for r0 in range(0, N, chunk):
        M[r0:r0 + chunk] = unclamped(corr, inlier_threshold, slice(r0, r0 + chunk)).clamp_min(0.0)
    M.fill_diagonal_(0.0)
    return M


def power(M, iterations=ITERATIONS):
    """Every iterate of step 2: [iterations + 1, N], row 0 the start vector of ones."""
    v = torch.ones(M.shape[0], dtype=M.dtype, device=M.device)
    its = [v]
    for _ in range(iterations):
        u = M @ v
        v = u / (torch.linalg.norm(u) + 1e-6)
        its.append(v)
    return torch.stack(its)


def select(v, S):
    """Labels [N] of step 3 and the sorted order (descending value, ascending row)."""
    order = torch.sort(-v, stable=True).indices
    labels = torch.zeros_like(v)
    labels[order[:S]] = 1.0
    return labels, order


def weighted_kabsch(src, tgt, w):
    """Step 4 in float64: T [4,4] of rigid_transform_3d(src, tgt, w), and H."""
    a, b, w = (x.to(torch.float64) for x in (src, tgt, w))
    w = torch.where(w < 0, torch.zeros_like(w), w)
    den = w.sum() + 1e-6
    ca = (a * w[:, None]).sum(0) / den
    cb = (b * w[:, None]).sum(0) / den
    H = (a - ca).T @ ((b - cb) * w[:, None])
    T = torch.eye(4, dtype=torch.float64, device=a.device)
    if bool((H != 0).any()):
        U, _, Vh = torch.linalg.svd(H)
        V = Vh.T
        D = torch.eye(3, dtype=torch.float64, device=a.device)
        D[2, 2] = torch.sign(torch.linalg.det(V @ U.T))
        R = V @ D @ U.T
        T[:3, :3] = R
        T[:3, 3] = cb - R @ ca
    return T, H


def sm(corr, src, tgt, inlier_threshold, iterations=ITERATIONS, top_ratio=TOP_RATIO, M=None):
    """The four steps on one set.  Returns a dict: M, its (float64) iterates, v, labels, order, S, trans, H, gap, clamp."""
    N = corr.shape[0]
    M = compat(corr, inlier_threshold) if M is None else M
    its = power(M, iterations)
    v = its[-1]
    S = num_selected(N, top_ratio)
    labels, order = select(v, S)
    trans, H = weighted_kabsch(src, tgt, v * labels)
    vs = v[order]
    gap = float(vs[S - 1] - vs[S]) if 0 < S < N else math.inf
    clamp = math.inf
    for r0 in range(0, N, 2048):
        x = unclamped(corr, inlier_threshold, slice(r0, r0 + 2048)).abs()
        idx = torch.arange(r0, min(r0 + 2048, N), device=x.device)
        x[idx - r0, idx] = math.inf
        clamp = min(clamp, float(x.min()))
    return dict(M=M, iterates=its, v=v, labels=labels, order=order, S=S, trans=trans, H=H, gap=gap, clamp=clamp)
