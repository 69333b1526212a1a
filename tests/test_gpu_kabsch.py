"""The geometric back end against float64: the 3x3 Kabsch solver (csrc/svd3.cuh), the per-seed hypotheses, hypothesis
scoring and selection, and the post-refinement (csrc/select_refine.cu), on degenerate geometry and at every k.  Needs an
H100: `-m gpu`.

Part 1 runs `pdsc::kabsch_rotation` alone through a test-only harness (tests/kabsch_harness.cu, compiled here with the
engine's nvcc flags) on ~10^5 matrices.  Parts 2 and 3 go through the engine with injected stage inputs.

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
from oracle import pointdsc_oracle as O

pytestmark = pytest.mark.gpu

PRECISIONS = os.environ.get("PDSC_TEST_PRECISIONS", "fp32,fp16x3").split(",")
HERE = os.path.dirname(os.path.abspath(__file__))
EPS = 2.0 ** -23
# Solver constant: |R - R64|max <= C_SVD * eps * s1 / (s2 + d s3).  Worst measured on an H100 over the ~1.1e5 matrices of
# part 1: 5.2 (repeated singular values; random 4.7, ill-conditioned 3.8, reflected 1.8, rank 2 1.8), so 16 leaves 3x.
C_SVD = 16.0
# Pre-solver fp32 term (`_h_error`): per-entry bound on |H32 - H64| in units of eps * (its magnitude terms).  Derivation: a
# weighted centroid is a 4-term fma chain per lane, a 5-level warp tree and a division by a sum with the same error, so it
# is off by <= 20 eps * max|a|; a centred coordinate then by <= 21 eps * max|a|; each H entry sums k products of such terms
# (4 fma per lane + the tree: 10 eps relative).  32 covers all three with margin.  Measured on an H100 (part 2's degenerate
# neighbourhoods): the worst error is 0.002 of the rotation tolerance, 0.018 of the translation one and 0.008 of the centroid
# one; the bounds are worst cases, the typical rounding errors cancel.
C_PRE = 32.0

_models = {}


def get_model(dataset, precision="fp32", k=40):
    from pointdsc_b200 import PointDSC
    key = (dataset, precision, k)
    if key not in _models:
        cfg = O.default_config(dataset)
        m = PointDSC(in_dim=6, num_layers=12, num_channels=128, num_iterations=10, ratio=0.1,
                     inlier_threshold=cfg["inlier_threshold"], sigma_d=cfg["sigma_d"], k=k,
                     nms_radius=cfg["nms_radius"], precision=precision)
        res = m.load_state_dict(load_snapshot(dataset), strict=False)
        assert res.missing_keys == [] and res.unexpected_keys == ["gamma"]
        _models[key] = m.cuda().eval()
    return _models[key]


# ---------------------------------------------------------------------------------------------------
# float64 references
# ---------------------------------------------------------------------------------------------------
def kabsch64(H):
    """R = V diag(1, 1, det(V U^T)) U^T of H [..., 3, 3] (float64, H = U S V^T, H = sum w a b^T so that b ~= R a).
    Returns R, singular values s [..., 3] (descending), d = det(V U^T), U, V."""
    U, s, Vt = np.linalg.svd(H)
    V = np.swapaxes(Vt, -1, -2)
    d = np.sign(np.linalg.det(V @ np.swapaxes(U, -1, -2)))
    D = np.broadcast_to(np.eye(3), H.shape).copy()
    D[..., 2, 2] = d
    return V @ D @ np.swapaxes(U, -1, -2), s, d, U, V


def _gap(s, d):
    return s[..., 1] + d * s[..., 2]


def _h_error(w, a, b, m, n):
    """Per-entry bound on |H32 - H64| from fp32 centroids, centring and sums.  w [P,k], a/b the points [P,k,3], m/n the
    centred points [P,k,3] (all float64).  Ma, Mb: the coordinates' magnitude, which the centroid errors scale with."""
    Ma, Mb = np.abs(a).max(axis=(1, 2)), np.abs(b).max(axis=(1, 2))
    mi, ni = np.abs(m).max(axis=2), np.abs(n).max(axis=2)
    return C_PRE * EPS * (Ma * (w * ni).sum(1) + Mb * (w * mi).sum(1) + (w * mi * ni).sum(1)), Ma, Mb


def weighted_kabsch64(a, b, w):
    """oracle.pointdsc_oracle.weighted_kabsch in float64 (the oracle builds its identity in float32): negative weights -> 0,
    centroids over sum(w) + 1e-6, H = Am^T diag(w) Bm, t = cb - R ca.  a, b [P,k,3], w [P,k].
    Returns R [P,3,3], t [P,3], ca, cb, H, and the H error bound with its magnitudes."""
    w = np.where(w < 0, 0.0, w)
    den = w.sum(1) + 1e-6
    ca = (a * w[..., None]).sum(1) / den[:, None]
    cb = (b * w[..., None]).sum(1) / den[:, None]
    m, n = a - ca[:, None], b - cb[:, None]
    H = np.einsum("pki,pkj,pk->pij", m, n, w)
    R, s, d, U, V = kabsch64(H)
    t = cb - np.einsum("pij,pj->pi", R, ca)
    EH, Ma, Mb = _h_error(w, a, b, m, n)
    return dict(R=R, t=t, ca=ca, cb=cb, H=H, s=s, d=d, U=U, V=V, EH=EH, Ma=Ma, Mb=Mb)


def assert_rotations(R, what, tol=1e-6):
    """Finite, orthonormal and det = +1 to `tol`.  1e-6 is ~8 fp32 roundings of a product of unit vectors; the worst measured
    on an H100 over every part-1 input is 8.6e-7 (|R R^T - I|) and 8.9e-7 (|det R - 1|)."""
    R = np.asarray(R, np.float64)
    assert np.isfinite(R).all(), what
    orth = np.abs(R @ np.swapaxes(R, -1, -2) - np.eye(3)).max(axis=(-1, -2))
    det = np.abs(np.linalg.det(R) - 1.0)
    assert orth.max() <= tol and det.max() <= tol, (what, float(orth.max()), float(det.max()))


def check_transforms(T, ref, what):
    """Engine transforms T [P,4,4] against a weighted_kabsch64 result.  Returns the worst ratios (error / tolerance)."""
    T = np.asarray(T, np.float64)
    R, t = T[:, :3, :3], T[:, :3, 3]
    assert_rotations(R, what)
    s, d, EH, Ma, Mb = ref["s"], ref["d"], ref["EH"], ref["Ma"], ref["Mb"]
    gap = _gap(s, d)
    with np.errstate(divide="ignore", invalid="ignore"):
        # rotation: solver term + pre-solver term over the signed gap; >= 2 is vacuous (entries of two rotations)
        tol_R = np.where(gap > 0, (C_SVD * EPS * s[:, 0] + 6.0 * EH) / gap, np.inf)
        # the first singular pair is defined whenever s1 > s2, the gap of singular vectors: R u1 = v1 (rank 1 included)
        tol_u1 = np.where(s[:, 0] > s[:, 1], (C_SVD * EPS * s[:, 0] + 6.0 * EH) / (s[:, 0] - s[:, 1]), np.inf)
    err_R = np.abs(R - ref["R"]).max(axis=(1, 2))
    assert (err_R <= tol_R).all(), (what, np.flatnonzero(err_R > tol_R)[:8], err_R[err_R > tol_R][:8], tol_R[err_R > tol_R][:8])
    err_u1 = np.abs(np.einsum("pij,pj->pi", R, ref["U"][:, :, 0]) - ref["V"][:, :, 0]).max(1)
    assert (err_u1 <= tol_u1).all(), (what, err_u1[err_u1 > tol_u1][:8], tol_u1[err_u1 > tol_u1][:8])
    # t = cb - R ca: its error is the rotation's error at the centroid plus the centroids' own (<= 20 eps Ma, see C_PRE)
    tol_t = 3.0 * np.minimum(tol_R, 2.0) * Ma + C_PRE * EPS * (Ma + Mb)
    err_t = np.abs(t - ref["t"]).max(1)
    assert (err_t <= tol_t).all(), (what, err_t[err_t > tol_t][:8], tol_t[err_t > tol_t][:8])
    # whatever R is, it maps the weighted centroid onto the target centroid (no division by a gap): the centroids' errors
    # (<= 20 eps each), R times the source one (3 terms) and the rounding of t = cb - R ca: 96 eps (Ma + Mb)
    err_c = np.abs(np.einsum("pij,pj->pi", R, ref["ca"]) + t - ref["cb"]).max(1)
    tol_c = 96.0 * EPS * (Ma + Mb)
    assert (err_c <= tol_c).all(), (what, err_c[err_c > tol_c][:8], tol_c[err_c > tol_c][:8])
    ratio = lambda e, tl: float(np.max(np.where(np.isfinite(tl) & (tl < 2), e / tl, 0.0), initial=0.0))  # noqa: E731
    return dict(R=ratio(err_R, tol_R), u1=ratio(err_u1, tol_u1), t=ratio(err_t, tol_t), c=ratio(err_c, tol_c), tol_R=tol_R)


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
    default -fmad=true) into a session temp directory."""
    import __graft_entry__ as G
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    lib_path = str(tmp_path_factory.mktemp("kabsch_harness") / "kabsch_harness.so")
    subprocess.run([nvcc] + G.NVCC_FLAGS + ["-I", G.CSRC, "-o", lib_path, os.path.join(HERE, "kabsch_harness.cu")], check=True)
    lib = C.CDLL(lib_path)
    lib.kabsch_harness_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    lib.kabsch_harness_run.restype = C.c_int

    def run(H32):
        h = torch.from_numpy(np.ascontiguousarray(H32, np.float32).reshape(-1, 9)).cuda()
        r = torch.empty_like(h)
        torch.cuda.synchronize()
        rc = lib.kabsch_harness_run(h.data_ptr(), r.data_ptr(), h.shape[0])
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


def _compose(rng, s, proper_u=None, proper_v=None):
    """H = U diag(s) V^T with random orthogonal U, V (float64), rounded to float32."""
    s = np.asarray(s, np.float64)
    U, V = _orthogonal(rng, len(s), proper_u), _orthogonal(rng, len(s), proper_v)
    return ((U * s[:, None, :]) @ np.swapaxes(V, 1, 2)).astype(np.float32)


def solver_families(seed=0):
    rng = np.random.default_rng(seed)
    f = {}
    n = 100000
    s = np.sort(np.exp(rng.uniform(-4.0, 0.0, (n, 3))), axis=1)[:, ::-1] * np.exp(rng.uniform(-3, 3, (n, 1)))
    f["random"] = _compose(rng, s)
    ratios = np.concatenate([np.logspace(0, -8, 17), [0.0]])
    cond = np.stack([np.ones_like(ratios), np.full_like(ratios, 0.5), ratios], 1)
    f["condition"] = _compose(rng, np.repeat(cond, 300, axis=0))
    f["rank1"] = _compose(rng, np.tile([[1.0, 0.0, 0.0]], (500, 1)) * np.exp(rng.uniform(-3, 3, (500, 1))))
    rep = [[1.0, 1.0, 0.3], [1.0, 0.3, 0.3], [1.0, 1.0, 1.0], [1.0, 1.0, 0.0]]
    f["repeated"] = _compose(rng, np.repeat(np.array(rep), 500, axis=0))
    # det(H) < 0: U V^T a reflection, with s3 = 0 and with s3 tiny and negative (H = U diag(s1, s2, -tiny) V^T, U V^T proper)
    f["reflection"] = _compose(rng, np.tile([[1.0, 0.6, 0.2]], (1000, 1)), True, False)
    f["reflection_rank2"] = _compose(rng, np.tile([[1.0, 0.6, 0.0]], (1000, 1)), True, False)
    tiny = np.stack([np.ones(1000), np.full(1000, 0.7), -np.logspace(-2, -9, 1000)], 1)
    f["reflection_tiny"] = _compose(rng, tiny, True, True)
    base = f["random"][:2000]
    perm = np.array([rng.permutation(3) for _ in range(2000)])
    signs = rng.choice([-1.0, 1.0], (2000, 1, 3)).astype(np.float32)
    f["layout"] = np.take_along_axis(base, perm[:, None, :], axis=2) * signs
    diag = np.zeros((1000, 3, 3), np.float32)
    diag[:, [0, 1, 2], [0, 1, 2]] = (rng.uniform(0.1, 2.0, (1000, 3)) * rng.choice([-1, 1], (1000, 3))).astype(np.float32)
    f["diagonal"] = diag
    # few significant bits: 2^e H stays exact down to the subnormal range (entries are multiples of 2^-149 there)
    f["integer"] = rng.integers(-64, 65, (2000, 3, 3)).astype(np.float32)
    small = f["random"][2000:3000].copy()
    small[:500, 1, :] *= np.float32(1e-20)      # one row many orders smaller
    small[500:, :, 2] *= np.float32(1e-20)      # one column
    f["small_row_col"] = small
    f["zero"] = np.zeros((4, 3, 3), np.float32)
    bad = f["random"][:6].copy()
    bad[0, 0, 0], bad[1, 2, 1], bad[2, 1, 1] = np.nan, np.inf, -np.inf
    bad[3] = np.nan
    bad[4, 0, :] = np.inf
    bad[5, 1, 2], bad[5, 0, 0] = np.nan, np.inf
    f["nonfinite"] = bad
    return f


SCALE_EXPONENTS = [-149, -140, -130, -126, -60, 0, 60, 120]


def test_kabsch_solver_against_float64(kabsch_gpu):
    fam = solver_families()
    names = list(fam)
    base = np.concatenate([fam[k] for k in names])
    sizes = [len(fam[k]) for k in names]
    # the scaled copies of every finite family: 2^e H rounded to float32
    finite = np.isfinite(base).all(axis=(1, 2))
    scaled = [(base.astype(np.float64) * 2.0 ** e).astype(np.float32) for e in SCALE_EXPONENTS]
    R_all = kabsch_gpu(np.concatenate([base] + scaled))
    R_base = R_all[:len(base)]
    R_scaled = [R_all[len(base) * (i + 1):len(base) * (i + 2)] for i in range(len(SCALE_EXPONENTS))]

    # always a rotation: every input, subnormal, huge, zero and non-finite H included
    labels = np.concatenate([np.repeat(names, sizes)] + [np.char.add(np.repeat(names, sizes), f" * 2^{e}")
                                                         for e in SCALE_EXPONENTS])
    nonfinite = ~np.isfinite(R_all).all(axis=(1, 2))
    assert not nonfinite.any(), ("non-finite R for", sorted(set(labels[nonfinite])))
    assert_rotations(R_all, "all inputs")
    ident = ~finite | ~(np.abs(base) > 0).any(axis=(1, 2))
    assert ident.sum() == 4 + 6
    assert (R_base[ident] == np.eye(3, dtype=np.float32)).all()          # H = 0 and non-finite H: exactly the identity
    for Hs, Rs in zip(scaled, R_scaled):
        z = ~(np.abs(Hs) > 0).any(axis=(1, 2)) | ~np.isfinite(Hs).all(axis=(1, 2))
        assert (Rs[z] == np.eye(3, dtype=np.float32)).all()

    # accurate wherever the rotation is defined (s2 + d s3 > 0)
    worst = {}
    off = 0
    for name, nrow in zip(names, sizes):
        H = base[off:off + nrow].astype(np.float64)
        R = R_base[off:off + nrow].astype(np.float64)
        off += nrow
        if name in ("zero", "nonfinite"):
            continue
        R64, s, d, U, V = kabsch64(H)
        gap = _gap(s, d)
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.abs(R - R64).max(axis=(1, 2)) / (EPS * s[:, 0] / gap)
        ok = gap > 0
        worst[name] = float(np.max(ratio[ok], initial=0.0))
        assert (ratio[ok] <= C_SVD).all(), (name, worst[name], np.flatnonzero(ratio > C_SVD)[:8])
        if name == "rank1":
            # only the first singular pair is defined: R maps u1 onto v1; the rotation about that axis is arbitrary
            err = np.abs(np.einsum("pij,pj->pi", R, U[:, :, 0]) - V[:, :, 0]).max()
            assert err <= 1e-6, err              # measured on an H100: 2.8e-7 (2.4 eps)
            worst["rank1_u1"] = float(err) / EPS
        if name == "reflection":
            assert (d < 0).all()                     # the det(V U^T) = -1 branch is what these exercise
        if name == "reflection_tiny":                # |s3| >= 1.6e-5: float32 rounding of H cannot flip det(H)'s sign
            assert (d[:400] < 0).all()
    print("part 1 worst |R - R64| / (eps s1 / (s2 + d s3)) (rank1_u1: |R u1 - v1| / eps):",
          {k: round(v, 2) for k, v in worst.items()}, "worst |R R^T - I|, |det R - 1|: %.3g %.3g" % (
              np.abs(R_all.astype(np.float64) @ np.swapaxes(R_all, 1, 2) - np.eye(3)).max(),
              np.abs(np.linalg.det(R_all.astype(np.float64)) - 1).max()))

    # scale invariance, bit for bit, wherever the float32 scaled matrix is exactly 2^e times the float32 H
    for e, Hs, Rs in zip(SCALE_EXPONENTS, scaled, R_scaled):
        exact = finite & (Hs.astype(np.float64) == base.astype(np.float64) * 2.0 ** e).all(axis=(1, 2))
        exact &= (np.abs(base) > 0).any(axis=(1, 2))
        assert exact.sum() >= 2000, (e, int(exact.sum()))                    # the integer family at least
        bad = exact & ~(Rs == R_base).all(axis=(1, 2))
        assert not bad.any(), (e, int(bad.sum()), np.flatnonzero(bad)[:8])


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
    m = get_model("3dmatch", precision, 40)
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
    m = get_model("3dmatch", precision, k)
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
    m = get_model("3dmatch", precision, 128)
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
    m = get_model(dataset, "fp32", 40)
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
    m = get_model("3dmatch", "fp32", 40)
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
    m = get_model(dataset, "fp32", 40)
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
