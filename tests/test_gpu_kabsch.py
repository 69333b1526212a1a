"""The geometric back end against float64: the 3x3 Kabsch solver (csrc/svd3.cuh), the per-seed hypotheses, hypothesis
scoring and selection, and the post-refinement (csrc/select_refine.cu), on degenerate geometry and at every k.  Needs an
H100: `-m gpu`.

Part 1 runs `pdsc::kabsch_rotation` alone through a test-only harness (tests/kabsch_harness.cu, compiled here with the
engine's nvcc flags) on ~10^5 matrices, in float (the forward's solves, against LAPACK) and in double (ICP's updates, with
the families built in float64 and eps64 = 2^-52 in the bound, against a long-double Jacobi: `kabsch_ld`).  Parts 2 and 3 go
through the engine with injected stage inputs.

Error model used by every tolerance below (eps = 2^-23, the fp32 unit roundoff):
  * the solver: |R - R64|max <= C_SVD * eps * s1 / (s2 + d s3), where s are the singular values of the float32 H and
    d = det(V U^T): the signed polar factor of H is governed by s2 + d s3 (its smallest singular-value pair sum);
  * fp32 arithmetic before the solver perturbs H by at most E_H per entry (see `_h_error`), which moves the polar factor
    by at most 2 |dH|_F / (s2 + d s3) <= 6 E_H / (s2 + d s3) (the perturbation bound of the polar factor, |dH|_F <= 3 E_H).
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import load_snapshot
from float64_bounds import (C_PRE, C_SVD, EPS, EPS64, _gap, assert_rotations, check_transforms, kabsch64, kabsch_ld,
                            weighted_kabsch64)
from gpu_models import get_model
from oracle import pointdsc_oracle as O

pytestmark = pytest.mark.gpu

PRECISIONS = os.environ.get("PDSC_TEST_PRECISIONS", "fp32,fp16x3").split(",")
HERE = os.path.dirname(os.path.abspath(__file__))


def residual_band(T, src, tgt, thr):
    """Width of the band around thr inside which an fp32 residual ||R p + t - q|| may land on either side.  The kernels form
    R p + t with a 3-term fma chain and one add (<= 3 eps (|p|_1 + |t|) per coordinate), subtract q (eps |q|), square and
    sum (3 eps relative) and compare with a threshold rounded to fp32: |d32 - d64| <= 6 eps (|p|_1 + |t|max + |q|max) +
    2 eps d.  The band is 8 eps (that magnitude + thr).  In part 3's sets, built with 100 points on the threshold, 305
    (3DMatch) and 310 (KITTI) (hypothesis, point) pairs fall inside it."""
    mag = np.abs(src).sum(1) + np.abs(T[:3, 3]).max() + np.abs(tgt).max(1)
    return 8.0 * EPS * (mag + thr)


def residuals64(T, src, tgt):
    return np.linalg.norm(src @ T[:3, :3].T + T[:3, 3] - tgt, axis=1)


# ---------------------------------------------------------------------------------------------------
# part 1: the solver alone
# ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def kabsch_gpu(tmp_path_factory):
    """kabsch_rotation from pointdsc_b200/csrc/svd3.cuh, built as the engine builds it (same nvcc flags: sm_90a, -O3, the
    default -fmad=true) into a session temp directory.  run(H) solves in H's scalar: float32 or float64."""
    import __graft_entry__ as G
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    lib_path = str(tmp_path_factory.mktemp("kabsch_harness") / "kabsch_harness.so")
    subprocess.run([nvcc] + G.NVCC_FLAGS + ["-I", G.CSRC, "-o", lib_path, os.path.join(HERE, "kabsch_harness.cu")], check=True)
    lib = C.CDLL(lib_path)
    for fn in (lib.kabsch_harness_run, lib.kabsch_harness_run_f64):
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        fn.restype = C.c_int

    def run(H):
        dtype = np.float64 if H.dtype == np.float64 else np.float32
        h = torch.from_numpy(np.ascontiguousarray(H, dtype).reshape(-1, 9)).cuda()
        r = torch.empty_like(h)
        torch.cuda.synchronize()
        fn = lib.kabsch_harness_run_f64 if dtype == np.float64 else lib.kabsch_harness_run
        rc = fn(h.data_ptr(), r.data_ptr(), h.shape[0])
        assert rc == 0, f"harness launch failed: CUDA error {rc}"
        return r.cpu().numpy().reshape(-1, 3, 3)
    return run


def _orthogonal(rng, n, proper=None):
    q, r = np.linalg.qr(rng.standard_normal((n, 3, 3)))
    q = q * np.sign(np.diagonal(r, axis1=1, axis2=2))[:, None, :]
    if proper is not None:
        flip = (np.linalg.det(q) > 0) != proper
        q[flip, :, 0] *= -1
    return q


def _compose(rng, s, proper_u=None, proper_v=None, dtype=np.float32):
    """H = U diag(s) V^T with random orthogonal U, V (float64), rounded to `dtype`."""
    s = np.asarray(s, np.float64)
    U, V = _orthogonal(rng, len(s), proper_u), _orthogonal(rng, len(s), proper_v)
    return ((U * s[:, None, :]) @ np.swapaxes(V, 1, 2)).astype(dtype)


SMALL_S2_RATIOS = np.concatenate([np.logspace(-6, -16, 21), [0.0]])


def solver_families(seed=0, dtype=np.float32):
    """The part-1 inputs, built in float64 and rounded once to `dtype` (float64: not rounded at all)."""
    rng = np.random.default_rng(seed)
    f = {}
    n = 100000
    s = np.sort(np.exp(rng.uniform(-4.0, 0.0, (n, 3))), axis=1)[:, ::-1] * np.exp(rng.uniform(-3, 3, (n, 1)))
    f["random"] = _compose(rng, s, dtype=dtype)
    ratios = np.concatenate([np.logspace(0, -8, 17), [0.0]])
    cond = np.stack([np.ones_like(ratios), np.full_like(ratios, 0.5), ratios], 1)
    f["condition"] = _compose(rng, np.repeat(cond, 300, axis=0), dtype=dtype)
    f["rank1"] = _compose(rng, np.tile([[1.0, 0.0, 0.0]], (500, 1)) * np.exp(rng.uniform(-3, 3, (500, 1))), dtype=dtype)
    rep = [[1.0, 1.0, 0.3], [1.0, 0.3, 0.3], [1.0, 1.0, 1.0], [1.0, 1.0, 0.0]]
    f["repeated"] = _compose(rng, np.repeat(np.array(rep), 500, axis=0), dtype=dtype)
    # det(H) < 0: U V^T a reflection, with s3 = 0 and with s3 tiny and negative (H = U diag(s1, s2, -tiny) V^T, U V^T proper)
    f["reflection"] = _compose(rng, np.tile([[1.0, 0.6, 0.2]], (1000, 1)), True, False, dtype)
    f["reflection_rank2"] = _compose(rng, np.tile([[1.0, 0.6, 0.0]], (1000, 1)), True, False, dtype)
    tiny = np.stack([np.ones(1000), np.full(1000, 0.7), -np.logspace(-2, -9, 1000)], 1)
    f["reflection_tiny"] = _compose(rng, tiny, True, True, dtype)
    base = f["random"][:2000]
    perm = np.array([rng.permutation(3) for _ in range(2000)])
    signs = rng.choice([-1.0, 1.0], (2000, 1, 3)).astype(dtype)
    f["layout"] = np.take_along_axis(base, perm[:, None, :], axis=2) * signs
    diag = np.zeros((1000, 3, 3), dtype)
    diag[:, [0, 1, 2], [0, 1, 2]] = (rng.uniform(0.1, 2.0, (1000, 3)) * rng.choice([-1, 1], (1000, 3))).astype(dtype)
    f["diagonal"] = diag
    # few significant bits: 2^e H stays exact down to the subnormal range (entries are multiples of 2^-149 / 2^-1074 there)
    f["integer"] = rng.integers(-64, 65, (2000, 3, 3)).astype(dtype)
    small = f["random"][2000:3000].copy()
    tiny_factor = dtype(1e-20) if dtype == np.float32 else dtype(1e-150)
    small[:500, 1, :] *= tiny_factor      # one row many orders smaller
    small[500:, :, 2] *= tiny_factor      # one column
    f["small_row_col"] = small
    f["zero"] = np.zeros((4, 3, 3), dtype)
    bad = f["random"][:6].copy()
    bad[0, 0, 0], bad[1, 2, 1], bad[2, 1, 1] = np.nan, np.inf, -np.inf
    bad[3] = np.nan
    bad[4, 0, :] = np.inf
    bad[5, 1, 2], bad[5, 0, 0] = np.nan, np.inf
    f["nonfinite"] = bad
    # a small SECOND singular value (`condition` shrinks only s3): s2 / s1 from 1e-6 down to 1e-16, and 0, with s3 = 0, with
    # s3 = s2 / 2 and U V^T proper (d = +1), and with s3 = s2 / 2 and U V^T a reflection (d = -1, gap s2 / 2).  Around
    # s2 / s1 ~ 1e-13 the double solver's rank-1 branch decides whether u2 comes from H or is made up.
    r2 = np.repeat(SMALL_S2_RATIOS, 150)
    one = np.ones_like(r2)
    f["small_s2"] = np.concatenate([_compose(rng, np.stack([one, r2, 0.0 * r2], 1), dtype=dtype),
                                    _compose(rng, np.stack([one, r2, 0.5 * r2], 1), True, True, dtype),
                                    _compose(rng, np.stack([one, r2, 0.5 * r2], 1), True, False, dtype)])
    return f


SCALE_EXPONENTS = [-149, -140, -130, -126, -60, 0, 60, 120]
# float64: 2^e H is exact for the integer family from the smallest subnormal (2^-1074) up to 2^1000 (|H| <= 64)
SCALE_EXPONENTS_64 = [-1074, -1060, -1040, -1022, -600, -60, 0, 60, 600, 1000]
# |R R^T - I| and |det R - 1| in float64: R sums three products of unit vectors, each normalised by a reciprocal square root
# and built by cross products (~8 roundings, as in float), and the float64 check itself rounds R R^T and the LU determinant
# (~4 more): 16 eps64 = 3.6e-15.  Measured on an H100 (80 GB HBM3, 700 W) over every part-1 input: 1.55e-15 and 1.78e-15.
ROT_TOL_64 = 16.0 * EPS64


def _solver_against_float64(kabsch_gpu, dtype):
    """Part 1 in one scalar: every family and its 2^e copies through the device solver, against kabsch64.  Returns the
    worst ratios."""
    eps, exps = (EPS, SCALE_EXPONENTS) if dtype == np.float32 else (EPS64, SCALE_EXPONENTS_64)
    rot_tol = 1e-6 if dtype == np.float32 else ROT_TOL_64
    # R u1 = v1 for rank 1: float measured 2.4 eps (1e-6 = 8.4 eps); float64 gets 16 eps64 (8.4 eps and the reference's own
    # rounding), measured 3.0 eps64
    u1_tol = 1e-6 if dtype == np.float32 else 16.0 * EPS64
    fam = solver_families(dtype=dtype)
    names = list(fam)
    base = np.concatenate([fam[k] for k in names])
    sizes = [len(fam[k]) for k in names]
    # the scaled copies of every finite family: 2^e H rounded to `dtype`
    finite = np.isfinite(base).all(axis=(1, 2))
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        scaled = [(base.astype(np.float64) * 2.0 ** e).astype(dtype) for e in exps]
    R_all = kabsch_gpu(np.concatenate([base] + scaled))
    assert R_all.dtype == dtype
    R_base = R_all[:len(base)]
    R_scaled = [R_all[len(base) * (i + 1):len(base) * (i + 2)] for i in range(len(exps))]

    # always a rotation: every input, subnormal, huge, zero and non-finite H included
    labels = np.concatenate([np.repeat(names, sizes)] + [np.char.add(np.repeat(names, sizes), f" * 2^{e}") for e in exps])
    nonfinite = ~np.isfinite(R_all).all(axis=(1, 2))
    assert not nonfinite.any(), ("non-finite R for", sorted(set(labels[nonfinite])))
    assert_rotations(R_all, "all inputs", rot_tol)
    ident = ~finite | ~(np.abs(base) > 0).any(axis=(1, 2))
    assert ident.sum() == 4 + 6
    assert (R_base[ident] == np.eye(3, dtype=dtype)).all()          # H = 0 and non-finite H: exactly the identity
    for Hs, Rs in zip(scaled, R_scaled):
        z = ~(np.abs(Hs) > 0).any(axis=(1, 2)) | ~np.isfinite(Hs).all(axis=(1, 2))
        assert (Rs[z] == np.eye(3, dtype=dtype)).all()

    # accurate wherever the rotation is defined (s2 + d s3 > 0)
    worst = {}
    off = 0
    for name, nrow in zip(names, sizes):
        H = base[off:off + nrow].astype(np.float64)
        R = R_base[off:off + nrow].astype(np.float64)
        off += nrow
        if name in ("zero", "nonfinite"):
            continue
        R64, s, d, U, V = kabsch64(H) if dtype == np.float32 else kabsch_ld(H)
        gap = _gap(s, d)
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.abs(R - R64).max(axis=(1, 2)) / (eps * s[:, 0] / gap)
        # below the solver's rank-1 threshold (s2 / s1 <= sqrt(KabschTol::rank): 1e-6 in float, 1.8e-15 in double) u2 is made
        # up and only R u1 = v1 is promised.  In double the bound is >= 2 there already; in float it is 1.9 at s2 / s1 = 1e-6
        # (the float constant 1e-12 sits 10% above (8 eps)^2), so rows within 5% of the threshold are held to u1 alone
        rank1 = s[:, 1] <= 1.05 * (1e-6 if dtype == np.float32 else np.sqrt(3.2e-30)) * s[:, 0]
        ok = (gap > 0) & ~rank1
        assert (ratio[ok] <= C_SVD).all(), (name, float(ratio[ok].max()), np.flatnonzero(ok & (ratio > C_SVD))[:8])
        with np.errstate(divide="ignore", invalid="ignore"):
            tol_u1 = np.where(s[:, 0] > s[:, 1], C_SVD * eps * s[:, 0] / (s[:, 0] - s[:, 1]), np.inf)
        err_u1 = np.abs(np.einsum("pij,pj->pi", R, U[:, :, 0]) - V[:, :, 0]).max(1)
        assert (err_u1[rank1] <= tol_u1[rank1]).all(), (name, float(err_u1[rank1].max()))
        # the worst ratio where the bound says something (C_SVD times it below 2, the distance between any two rotations)
        with np.errstate(divide="ignore", invalid="ignore"):
            informative = ok & (C_SVD * eps * s[:, 0] / gap < 2.0)
        worst[name] = float(np.max(ratio[informative], initial=0.0))
        if name == "rank1":
            # only the first singular pair is defined: R maps u1 onto v1; the rotation about that axis is arbitrary
            err = np.abs(np.einsum("pij,pj->pi", R, U[:, :, 0]) - V[:, :, 0]).max()
            assert err <= u1_tol, err
            worst["rank1_u1"] = float(err) / eps
        if name == "reflection":
            assert (d < 0).all()                     # the det(V U^T) = -1 branch is what these exercise
        if name == "reflection_tiny":                # |s3| >= 1.6e-5: float32 rounding of H cannot flip det(H)'s sign
            assert (d[:400] < 0).all()
        if name == "small_s2":
            # the family is not vacuous: rows whose bound is below 0.1 at s2 / s1 <= 1e-12, where the double solver's rank-1
            # branch once made u2 up
            if dtype == np.float64:
                tight = ok & (s[:, 1] <= 1e-12 * s[:, 0]) & (C_SVD * eps * s[:, 0] / np.where(ok, gap, 1.0) < 0.1)
                assert tight.sum() >= 300, int(tight.sum())
                # the reflected third with s2 / s1 >= 1e-12 (float64 rounding of H cannot flip det(H)'s sign there): d = -1
                third = 2 * len(SMALL_S2_RATIOS) * 150
                assert (d[third:third + 13 * 150] < 0).all()
    orth = float(np.abs(R_all.astype(np.float64) @ np.swapaxes(R_all, 1, 2) - np.eye(3)).max())
    det = float(np.abs(np.linalg.det(R_all.astype(np.float64)) - 1).max())

    # scale invariance, bit for bit, wherever the scaled matrix is exactly 2^e times H
    for e, Hs, Rs in zip(exps, scaled, R_scaled):
        with np.errstate(over="ignore", invalid="ignore"):
            exact = finite & (np.ldexp(Hs.astype(np.float64), -e) == base.astype(np.float64)).all(axis=(1, 2))
        exact &= (np.abs(base) > 0).any(axis=(1, 2))
        assert exact.sum() >= 2000, (e, int(exact.sum()))                    # the integer family at least
        bad = exact & ~(Rs == R_base).all(axis=(1, 2))
        assert not bad.any(), (e, int(bad.sum()), np.flatnonzero(bad)[:8], labels[:len(base)][bad][:8])
    return worst, orth, det


def test_kabsch_solver_against_float64(kabsch_gpu):
    worst, orth, det = _solver_against_float64(kabsch_gpu, np.float32)
    print("part 1 float worst |R - R64| / (eps s1 / (s2 + d s3)) (rank1_u1: |R u1 - v1| / eps):",
          {k: round(v, 2) for k, v in worst.items()}, "worst |R R^T - I|, |det R - 1|: %.3g %.3g" % (orth, det))


def test_kabsch_solver_double_against_float64(kabsch_gpu):
    """kabsch_rotation<double>, the ICP update's solver, on part 1's families built in float64, with eps = 2^-52 in the bound
    and the same C_SVD.  Worst ratio measured on an H100 (80 GB HBM3, 700 W) where the bound is below 2: 5.6 (random; repeated
    5.3, condition 3.8, small s2 0.33).  Before KabschTol<double>::rank was scaled to double the small-s2 family reached 1.3e4."""
    worst, orth, det = _solver_against_float64(kabsch_gpu, np.float64)
    print("part 1 double worst |R - R64| / (eps64 s1 / (s2 + d s3)) (rank1_u1: |R u1 - v1| / eps64):",
          {k: round(v, 2) for k, v in worst.items()}, "worst |R R^T - I|, |det R - 1|: %.3g %.3g (tolerance %.3g)" % (
              orth, det, ROT_TOL_64))


# ---------------------------------------------------------------------------------------------------
# part 2: seed hypotheses on the engine's own inputs
# ---------------------------------------------------------------------------------------------------
def _rot(rng):
    return _orthogonal(rng, 1, True)[0]


def seed_geometry_set(seed=0):
    """N = 1000 points (S = 100 seeds, k = 40), neighbourhoods of chosen seeds overwritten with degenerate geometry.
    Returns src, tgt (float32), knn_idx [S,k] (seed i's neighbours) and {family: [seed indices]}."""
    from pointdsc_b200.synth import make_pair
    rng = np.random.default_rng(seed)
    N, S, k = 1000, 100, 40
    p = make_pair(900 + seed, N, "3dmatch", 0.5)
    src = p["src_keypts"].numpy().astype(np.float64)
    tgt = p["tgt_keypts"].numpy().astype(np.float64)
    knn = np.stack([rng.choice(np.delete(np.arange(N), i), k, replace=False) for i in range(S)])
    fam, block = {}, 0

    def put(name, a, b):
        nonlocal block
        rows = np.arange(100 + 40 * block, 140 + 40 * block)
        seed_i = block
        src[rows], tgt[rows] = a, b
        knn[seed_i] = rows
        fam.setdefault(name, []).append(seed_i)
        block += 1

    for rep in range(2):
        R, t = _rot(rng), rng.uniform(-1, 1, 3)
        F = _rot(rng)                                               # the plane's frame
        uv = np.c_[rng.uniform(-1, 1, (k, 2)), np.zeros(k)] @ F.T + rng.uniform(0, 3, 3)
        put("plane", uv, uv @ R.T + t)                              # rank-2 H
        M = F @ np.diag([-1.0, 1.0, 1.0]) @ F.T                     # a mirror that maps the plane onto itself
        put("plane_mirrored", uv, uv @ M.T @ R.T + t)               # rank 2, mirrored in the target
        thick = uv + 0.02 * rng.standard_normal((k, 1)) * F[:, 2]
        M3 = F @ np.diag([1.0, 1.0, -1.0]) @ F.T                    # mirror through the plane: det(V U^T) = -1, s3 > 0
        put("slab_mirrored", thick, thick @ M3.T @ R.T + t)
        line = rng.uniform(-1, 1, (k, 1)) * _rot(rng)[:, 0] + rng.uniform(0, 3, 3)
        put("line", line, line @ R.T + t)                           # rank 1
        put("point_origin", np.zeros((k, 3)), np.tile(rng.uniform(-2, 2, 3), (k, 1)))   # H = 0 exactly: R = I, t = cb - ca
        put("point", np.tile(rng.uniform(0, 3, 3), (k, 1)), np.tile(rng.uniform(0, 3, 3), (k, 1)))
        a = rng.uniform(-80, 80, (k, 3))                            # KITTI scale: +-80 units, 20x the 3DMatch spread
        put("kitti", a, a @ R.T + 20 * t + 0.1 * rng.standard_normal((k, 3)))
        a = 1000.0 + rng.uniform(-1, 1, (k, 3))                     # 10^3 units off the origin: the fp32 centroids cancel
        put("far", a, a @ R.T + 1000.0 * t + 0.01 * rng.standard_normal((k, 3)))
    return src.astype(np.float32), tgt.astype(np.float32), knn.astype(np.int32), fam


@pytest.mark.parametrize("precision", PRECISIONS)
def test_seed_kabsch_on_degenerate_neighbourhoods(precision):
    m = get_model("3dmatch", precision)
    src, tgt, knn, fam = seed_geometry_set()
    N, S, k = src.shape[0], knn.shape[0], knn.shape[1]
    rng = np.random.default_rng(1)
    # identical features: the feature compatibility is 1, the spatial one decides the eigenvector (non-negative weights)
    feat = np.tile(rng.standard_normal(128).astype(np.float32), (N, 1))
    corr = np.concatenate([src, tgt], 1)
    corr -= corr.mean(0)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()[None]  # noqa: E731
    inj = {"features": dev(feat), "confidence": dev(np.zeros(N, np.float32)), "seeds": dev(np.arange(S, dtype=np.int32)),
           "knn_idx": dev(knn)}
    out = m.run(dev(corr), dev(src), dev(tgt), taps=["eig", "seed_trans", "inlier_counts", "knn_idx"], inject=inj)
    assert np.array_equal(out["knn_idx"][0].cpu().numpy(), knn)
    eig = out["eig"][0].cpu().numpy().astype(np.float64)
    T = out["seed_trans"][0].cpu().numpy()
    a, b = src.astype(np.float64)[knn], tgt.astype(np.float64)[knn]
    ref = weighted_kabsch64(a, b, eig / (eig.sum(1, keepdims=True) + 1e-6))
    r = check_transforms(T, ref, "seed_trans")
    print(f"part 2 geometry ({precision}) worst error/tolerance:", {x: round(v, 3) for x, v in r.items() if x != "tol_R"})
    s, d = ref["s"], ref["d"]
    # the families reach the branches they are built for, and the comparison is not vacuous there
    assert (s[fam["plane"], 2] <= 1e-5 * s[fam["plane"], 0]).all()
    assert (s[fam["line"], 1] <= 1e-5 * s[fam["line"], 0]).all()
    assert (d[fam["slab_mirrored"]] < 0).all()
    for name in ("plane", "plane_mirrored", "slab_mirrored", "kitti"):
        assert (r["tol_R"][fam[name]] < 1e-2).all(), (name, r["tol_R"][fam[name]])
    # 10^3 units off the origin with a spread of 1: the centroids' fp32 error is 10^3 times larger relative to the spread
    assert (r["tol_R"][fam["far"]] < 0.5).all(), r["tol_R"][fam["far"]]
    # H = 0 exactly: R = I and t = cb - ca
    for i in fam["point_origin"]:
        assert np.array_equal(T[i, :3, :3], np.eye(3, dtype=np.float32))
        assert np.abs(T[i, :3, 3] - (ref["cb"][i] - ref["ca"][i])).max() <= C_PRE * EPS * ref["Mb"][i]
    check_counts(T, src, tgt, out["inlier_counts"][0].cpu().numpy(), float(m.inlier_threshold))


K_SWEEP = [1, 2, 3, 31, 32, 33, 39, 40, 41, 47, 48, 49, 79, 80, 81, 88, 89, 96, 127, 128]
ORACLE_K = (33, 79, 88, 128)    # one per NSM kernel family: one warp (<= 40), 4-warp tensor core (41-80), SIMT (81-88, > 88)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("k", K_SWEEP)
def test_k_sweep_knn_compat_seed_kabsch(k, precision):
    from pointdsc_b200.synth import make_pair
    m = get_model("3dmatch", precision, k=k)
    n = 300                                                    # S = 30 seeds, k <= n - 1
    p = make_pair(500 + k, n, "3dmatch", 0.6)
    args = [p[x][None].cuda() for x in ("corr_pos", "src_keypts", "tgt_keypts")]
    out = m.run(*args, taps=["normed", "seeds", "knn_idx", "compat", "eig", "seed_trans"])
    normed = out["normed"][0].cpu().numpy().astype(np.float64)
    seeds = out["seeds"][0].cpu().numpy().astype(np.int64)
    got = out["knn_idx"][0].cpu().numpy().astype(np.int64)
    S = seeds.shape[0]
    assert got.shape == (S, k)

    # kNN: k distinct neighbours, the seed left out where it is strictly nearest, the float64 ranking wherever it is
    # separated by more than the fp32 distance noise (the rule of test_gpu_parity.test_knn_given_reference_features)
    assert all(len(set(row)) == k for row in got)
    dist = 2.0 - 2.0 * (normed[seeds] @ normed.T)
    ref = np.argsort(dist, axis=1, kind="stable")[:, 1:k + 1]
    d_got, d_ref = np.take_along_axis(dist, got, 1), np.take_along_axis(dist, ref, 1)
    assert np.abs(d_got - d_ref).max() < 1e-5
    full = np.sort(dist, axis=1)[:, :k + 2]
    gap_lo = full[:, 1:k + 1] - full[:, 0:k]
    gap_hi = full[:, 2:k + 2] - full[:, 1:k + 1] if full.shape[1] == k + 2 else np.full_like(gap_lo, 1.0)
    sep = (gap_lo > 1e-5) & (gap_hi > 1e-5)
    assert np.array_equal(got[sep], ref[sep])
    self_first = full[:, 1] - full[:, 0] > 1e-5
    assert not any(int(sd) in r for sd, r, f in zip(seeds, got, self_first) if f)

    # compatibility (oracle.seed_compatibility's formula in float64) on the engine's neighbourhoods
    src, tgt = p["src_keypts"].numpy().astype(np.float64), p["tgt_keypts"].numpy().astype(np.float64)
    sigma, sigma_d = float(m.sigma.detach().cpu()[0]), float(m.sigma_spat.detach().cpu()[0])
    f = normed[got]
    fm = np.maximum(1.0 - (1.0 - f @ np.swapaxes(f, 1, 2)) / sigma ** 2, 0.0)
    la = np.linalg.norm(src[got][:, :, None] - src[got][:, None], axis=-1)
    lb = np.linalg.norm(tgt[got][:, :, None] - tgt[got][:, None], axis=-1)
    cm = fm * np.maximum(1.0 - (la - lb) ** 2 / sigma_d ** 2, 0.0)
    cm[:, np.arange(k), np.arange(k)] = 0.0
    compat = out["compat"][0].cpu().numpy().reshape(S, k, k)
    # 2e-5, the bound of test_compat_power_kabsch_given_reference_neighbourhoods, in both modes: the tensor-core Gram of
    # fp16x3 (k <= 80: fp16 hi/lo split, only the lo*lo product dropped, <= 2^-22 of |f_i||f_j| = 1) stays at fp32 grade.
    # Measured on an H100 over the sweep: 6.2e-6 in fp32, 1.2e-5 in fp16x3 (k = 40).
    assert np.abs(compat - cm).max() < 2e-5, float(np.abs(compat - cm).max())
    print(f"part 2 k={k} ({precision}): max |compat - compat64| = {np.abs(compat - cm).max():.3g}")

    # seed transforms: float64 Kabsch on the tapped eigenvector
    eig = out["eig"][0].cpu().numpy().astype(np.float64)
    kab = weighted_kabsch64(src[got], tgt[got], eig / (eig.sum(1, keepdims=True) + 1e-6))
    check_transforms(out["seed_trans"][0].cpu().numpy(), kab, f"seed_trans k={k}")
    T = out["final_trans"][0].cpu().numpy()
    assert_rotations(T[None, :3, :3], "final_trans", 1e-5)

    if k in ORACLE_K:
        sd = load_snapshot("3dmatch")
        cfg = dict(O.default_config("3dmatch"), k=k)
        ro = O.forward_testing(sd, cfg, p["corr_pos"], p["src_keypts"], p["tgt_keypts"])
        assert float((ro["final_trans"] - p["gt_trans"]).abs().max()) < 0.05      # the oracle registers this pair
        assert float((out["final_trans"][0].cpu() - ro["final_trans"]).abs().max()) < 1e-4
        assert int((out["final_labels"][0].cpu() != ro["final_labels"]).sum()) <= 2


@pytest.mark.parametrize("precision", PRECISIONS)
def test_large_k_set_in_a_mixed_call(precision):
    """k = 128: N = 41 (k = 40, one-warp NSM), N = 90 (k = 89, SIMT with repeated Gram passes) and N = 300 (k = 128) in one
    forward_many call, bit for bit what single calls give."""
    from pointdsc_b200.synth import make_pair
    m = get_model("3dmatch", precision, k=128)
    pairs = [make_pair(70 + i, n, "3dmatch", 0.5) for i, n in enumerate([41, 300, 90])]
    batch = lambda ps: {"corr_pos": torch.stack([q["corr_pos"] for q in ps]).cuda(),  # noqa: E731
                        "src_keypts": torch.stack([q["src_keypts"] for q in ps]).cuda(),
                        "tgt_keypts": torch.stack([q["tgt_keypts"] for q in ps]).cuda(), "testing": True}
    out = m.forward_many([batch([q]) for q in pairs])
    for q, o in zip(pairs, out):
        b = batch([q])
        one = m.run(b["corr_pos"], b["src_keypts"], b["tgt_keypts"])
        assert torch.equal(o["final_trans"], one["final_trans"])
        assert torch.equal(o["final_labels"], one["final_labels"])


# ---------------------------------------------------------------------------------------------------
# part 3: scoring, selection and refinement given injected hypotheses
# ---------------------------------------------------------------------------------------------------
def check_counts(T, src, tgt, counts, thr):
    """Engine inlier counts against float64 ||R p + t - q|| < thr: exact outside the fp32 band, either side inside it.
    Returns the number of (hypothesis, point) pairs inside the band."""
    src64, tgt64 = src.astype(np.float64), tgt.astype(np.float64)
    in_band = 0
    for i in range(T.shape[0]):
        Ti = T[i].astype(np.float64)
        d = residuals64(Ti, src64, tgt64)
        band = np.abs(d - thr) <= residual_band(Ti, src64, tgt64, thr)
        sure = int((d < thr)[~band].sum())
        assert sure <= int(counts[i]) <= sure + int(band.sum()), (i, int(counts[i]), sure, int(band.sum()))
        in_band += int(band.sum())
    return in_band


def _inputs(src, tgt):
    corr = np.concatenate([src, tgt], 1)
    corr -= corr.mean(0)
    return [torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()[None] for x in (corr, src, tgt)]


def _T(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def scoring_set(dataset, seed=0):
    """N = 1000 (S = 100 hypotheses): half inliers of a ground-truth motion (noise <= 0.3 thr), 100 points placed exactly at
    distance thr from it (they land in the fp32 band), the rest outliers.  Hypotheses: perturbed ground truths, and the
    exact ground truth at rows 7, 23 and 61 (equal counts: the first, 7, must win)."""
    rng = np.random.default_rng(seed)
    thr = O.default_config(dataset)["inlier_threshold"]
    scale = 3.0 if dataset == "3dmatch" else 50.0
    N, S = 1000, 100
    src = rng.uniform(0, scale, (N, 3))
    R, t = _rot(rng), rng.uniform(0, scale / 3, 3)
    warped = src @ R.T + t
    dirs = rng.standard_normal((N, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    tgt = warped + dirs * rng.uniform(0, 0.3 * thr, (N, 1))
    tgt[500:600] = warped[500:600] + dirs[500:600] * thr                      # on the threshold
    tgt[600:] = rng.uniform(0, scale, (400, 3))                               # outliers
    hyps = []
    for i in range(S):
        # every perturbed hypothesis is >= 0.9 thr off in translation: it loses a share of the inliers, so the ground truth
        # keeps the largest count
        shift = rng.standard_normal(3)
        shift *= rng.uniform(0.9, 2.0) * thr / np.linalg.norm(shift)
        hyps.append(_T(_rot_small(rng, rng.uniform(0.0, 1.0) * thr / scale) @ R, t + shift))
    for i in (7, 23, 61):
        hyps[i] = _T(R, t)
    return src.astype(np.float32), tgt.astype(np.float32), np.stack(hyps).astype(np.float32), thr


@pytest.mark.parametrize("dataset", ["3dmatch", "kitti"])
def test_inlier_counts_and_first_maximum_selection(dataset):
    m = get_model(dataset, "fp32")
    src, tgt, hyps, thr = scoring_set(dataset)
    out = m.run(*_inputs(src, tgt), taps=["inlier_counts", "best", "init_trans"],
                inject={"seed_trans": torch.from_numpy(hyps).cuda()[None]})
    counts = out["inlier_counts"][0].cpu().numpy()
    in_band = check_counts(hyps, src, tgt, counts, thr)
    assert in_band >= 100, in_band                       # the band is not vacuous: the points placed on thr fall in it
    print(f"part 3 counts {dataset}: {in_band} (hypothesis, point) pairs in the band")
    assert counts[7] == counts[23] == counts[61] == counts.max()
    best = int(out["best"][0])
    assert best == int(np.argmax(counts)) == 7           # exact ties go to the first maximum
    assert np.array_equal(out["init_trans"][0].cpu().numpy(), hyps[best])
    T = hyps[best].astype(np.float64)
    d = residuals64(T, src.astype(np.float64), tgt.astype(np.float64))
    band = np.abs(d - thr) <= residual_band(T, src.astype(np.float64), tgt.astype(np.float64), thr)
    labels = out["final_labels"][0].cpu().numpy()
    assert np.array_equal((labels > 0.5)[~band], (d < thr)[~band])          # the winner's inlier mask


def test_one_seed_and_no_seeds():
    m = get_model("3dmatch", "fp32")
    thr = 0.10
    src, tgt, hyps, _ = scoring_set("3dmatch", seed=3)
    # N = 15: S = 1, the only hypothesis is selected
    sub = slice(490, 505)
    out = m.run(*_inputs(src[sub], tgt[sub]), taps=["best", "init_trans", "inlier_counts"],
                inject={"seed_trans": torch.from_numpy(hyps[7:8]).cuda()[None]})
    assert out["inlier_counts"].shape == (1, 1) and int(out["best"][0]) == 0
    assert np.array_equal(out["init_trans"][0].cpu().numpy(), hyps[7])
    # N = 7 < 10: no seeds, the identity is the initial transform and the refinement starts from it
    rng = np.random.default_rng(4)
    s7 = rng.uniform(0, 1, (7, 3)).astype(np.float32)
    t7 = (s7 + rng.uniform(-0.02, 0.02, (7, 3))).astype(np.float32)
    t7[5:] += 1.0
    out = m.run(*_inputs(s7, t7), taps=["best", "init_trans", "refine_solves"])
    assert int(out["best"][0]) == 0
    assert np.array_equal(out["init_trans"][0].cpu().numpy(), np.eye(4, dtype=np.float32))
    d = residuals64(np.eye(4), s7.astype(np.float64), t7.astype(np.float64))
    assert np.array_equal(out["final_labels"][0].cpu().numpy() > 0.5, d < thr)
    ref = refine64(np.eye(4), s7, t7, O.refinement_threshold(thr))
    assert int(out["refine_solves"][0]) == ref["solves"] == 1
    check_refined(out["final_trans"][0].cpu().numpy(), ref, "N=7")


def refine64(T0, src, tgt, tau, max_iters=20):
    """oracle.post_refinement in float64, from the engine's own (float32) initial transform.  Besides the result it keeps,
    per solve, what the tolerance needs: the float64 solve (weighted_kabsch64) and a bound on how far the engine's weights
    may be from these, and the smallest distance of any residual from tau over all iterations (`margin`, units of tau)."""
    src64, tgt64 = src.astype(np.float64), tgt.astype(np.float64)
    T = np.asarray(T0, np.float64).copy()
    prev, solves, margin = 0, 0, np.inf
    last, prev_R, prev_t = None, 0.0, 0.0
    mag = np.abs(src64).sum(1).max() + np.abs(tgt64).max()
    dd0 = 8.0 * EPS * (mag + tau)                 # fp32 residual error (residual_band)

    def bounds(sol, dd):
        # the weight 1 / (1 + (d/tau)^2) moves by at most 0.65 |dd| / tau when a residual moves by dd.  A weight change
        # leaves the fit's rotation alone except through the fit's residuals nu = n - R m: it moves H's polar factor like
        # an error of sum |dw| |m| |nu| in H (the R m part of n only adds a symmetric positive term in H R)
        nu = np.abs(sol["n"] - sol["m"] @ sol["R"][0].T).max(1)
        EH = sol["EH"][0] + 0.65 * dd / tau * float((np.abs(sol["m"]).max(1) * nu).sum())
        gap = _gap(sol["s"], sol["d"])[0]
        bR = min(2.0, (C_SVD * EPS * sol["s"][0, 0] + 6.0 * EH) / gap) if gap > 0 else 2.0
        return EH, bR, 3.0 * bR * sol["Ma"][0] + C_PRE * EPS * (sol["Ma"][0] + sol["Mb"][0])

    for _ in range(max_iters):
        d = residuals64(T, src64, tgt64)
        margin = min(margin, float(np.min(np.abs(d - tau))) / tau)
        inl = d < tau
        cnt = int(inl.sum())
        if cnt == prev:
            break
        prev = cnt
        w = 1.0 / (1.0 + (d / tau) ** 2)
        sol = weighted_kabsch64(src64[inl][None], tgt64[inl][None], w[inl][None])
        sol["m"], sol["n"] = src64[inl] - sol["ca"][0], tgt64[inl] - sol["cb"][0]
        # the engine's residuals also carry the previous solve's transform error.  With the inlier set fixed by the margin
        # every solve is a weighted fit of consistent points, which does not amplify an error of the transform it starts
        # from, so the previous solve's own bound (fp32 residuals only) stands for it.  (Chaining worst cases instead
        # grows by ~10^2 per solve and makes the 20-solve comparison vacuous.)
        EH, _, _ = bounds(sol, dd0 + 3.0 * prev_R * np.abs(src64).max() + prev_t)
        _, prev_R, prev_t = bounds(sol, dd0)
        sol["EH"] = np.array([EH])
        T = _T(sol["R"][0], sol["t"][0])
        last = sol
        solves += 1
    return dict(T=T, solves=solves, margin=margin, sol=last)


def check_refined(T, ref, what):
    if ref["sol"] is None:
        return None
    T = np.asarray(T, np.float64)
    assert np.abs(T - ref["T"]).max() <= 2.0    # shape / sanity before the bounded comparison
    return check_transforms(T[None], ref["sol"], what)


def refinement_case(case, dataset, seed=0):
    """(src, tgt, initial transform, required margin in units of tau').  Margins: every residual at every iteration is
    below 0.5 tau' or above 2 tau' (|d - tau'| >= 0.5 tau'), except for the 20-iteration chain (see below)."""
    rng = np.random.default_rng(seed)
    tau = O.refinement_threshold(O.default_config(dataset)["inlier_threshold"])
    L = 30.0 * tau                                                 # extent of the inlier cloud
    R, t = _rot(rng), rng.uniform(-L, L, 3)
    if case == "chain":
        # 60 clusters of 4 + j points, all with the same centred source cloud shape and centroid, cluster j displaced by
        # x_j = sum_{i<j} 0.3 tau' 0.96^i along one axis: the fit (R stays exact, H is symmetric positive definite in the
        # source frame) moves the translation towards the denser clusters ahead, taking in new clusters at every solve,
        # for more than 20 solves.  Its margin is smaller: every residual stays >= 5e-3 tau' from tau' (float64 check
        # below; 6.6e-3 tau' as built), about 40 times the fp32 residual band (`residual_band`) at these magnitudes.
        x = np.concatenate([[0.0], np.cumsum(0.3 * tau * 0.96 ** np.arange(59))])
        srcs, tgts = [], []
        for j, xj in enumerate(x):
            c = rng.uniform(-L, L, (4 + j, 3))
            c -= c.mean(0)
            srcs.append(c)
            tgts.append(c @ R.T + t + R[:, 0] * xj)
        return np.concatenate(srcs), np.concatenate(tgts), _T(R, t), 5e-3
    n_in, n_out = 300, 200
    src = rng.uniform(-L, L, (n_in + n_out, 3))
    if case == "planar":
        F = _rot(rng)
        src[:n_in] = np.c_[rng.uniform(-L, L, (n_in, 2)), np.zeros(n_in)] @ F.T   # the inliers' H is rank 2
    dirs = rng.standard_normal((n_in + n_out, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    warped = src @ R.T + t
    tgt = warped + dirs * rng.uniform(0, 0.2 * tau, (n_in + n_out, 1))
    tgt[n_in:] = warped[n_in:] + dirs[n_in:] * rng.uniform(4 * tau, 8 * tau, (n_out, 1))
    ang = 0.05 * tau / L                                          # initial error: <= 0.15 tau' at the cloud's edge
    T0 = _T(_rot_small(rng, ang) @ R, t + rng.uniform(-0.05, 0.05, 3) * tau)
    if case == "zero_inliers":
        T0 = _T(R, t + 100.0 * tau)
    return src, tgt, T0, 0.5


def _rot_small(rng, ang):
    ax = rng.standard_normal(3)
    ax /= np.linalg.norm(ax)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


@pytest.mark.parametrize("case", ["generic", "planar", "zero_inliers", "chain"])
@pytest.mark.parametrize("dataset", ["3dmatch", "kitti"])           # tau' = 0.10 and 1.2
def test_refinement_given_injected_hypothesis(dataset, case):
    m = get_model(dataset, "fp32")
    src, tgt, T0, need_margin = refinement_case(case, dataset)
    src, tgt, T0 = src.astype(np.float32), tgt.astype(np.float32), T0.astype(np.float32)
    S = m.num_seeds(src.shape[0])
    hyps = torch.from_numpy(np.tile(T0, (S, 1, 1))).cuda()[None]
    out = m.run(*_inputs(src, tgt), taps=["init_trans", "refine_solves"], inject={"seed_trans": hyps})
    assert np.array_equal(out["init_trans"][0].cpu().numpy(), T0)
    tau = O.refinement_threshold(float(m.inlier_threshold))
    ref = refine64(T0, src, tgt, tau)
    assert ref["margin"] >= need_margin, ref["margin"]           # the construction keeps every residual clear of tau'
    solves = int(out["refine_solves"][0])
    assert solves == ref["solves"], (solves, ref["solves"])
    T = out["final_trans"][0].cpu().numpy()
    if case == "zero_inliers":
        assert solves == 0 and np.array_equal(T, T0)              # no inliers: no solve, the initial transform back
        return
    if case == "chain":
        assert solves == 20                                      # stops at the iteration cap
    if case == "planar":
        s = ref["sol"]["s"][0]
        assert s[2] <= 1e-5 * s[0], s
    # the last solve's bound (refine64); measured on an H100, the worst error over every case is 0.003 of it
    r = check_refined(T, ref, f"refine {dataset} {case}")
    print(f"part 3 refinement {dataset}/{case}: solves={solves} margin={ref['margin']:.3g} worst error/tolerance:",
          {x: round(v, 3) for x, v in r.items() if x != "tol_R"})
