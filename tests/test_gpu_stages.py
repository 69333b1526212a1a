"""The stages between the encoder and Kabsch against float64, on every launch path they take: the SC matrix (csrc/sc_matrix.cu),
the normalisation and confidence head (csrc/head.cu), seed selection (csrc/seeds.cu), the seed-row distances and kNN selection
(csrc/knn_tc.cu, csrc/nsm.cu), the power iteration (csrc/nsm.cu) and the validation forward's M.  Needs an H100: `-m gpu`.

Several kernels choose a second launch path from the batch, N or the SM count (the NMS tile kernel, the head's grid-stride
loop, several seed CTAs and key chunks in the seed-row distances, the kNN select's scalar loads).  Every test sizes its
batch from the device's SM count and asserts that it reached the path it targets.  The stages are driven through
`PointDSC.run` taps and injections (features, confidence, seeds) and `run_eval` taps.

Error model (u = 2^-24, the fp32 unit roundoff; gamma(n) = n u / (1 - n u)):
  * inputs are fp32 and exact in float64; every reference below is float64 on the engine's own fp32 inputs or taps;
  * an fp32 sum of n terms in any order, fma or not, is within gamma(n) * sum |terms| of the exact sum; for non-negative
    terms that is a relative error;
  * sqrt, division and a single add / multiply add one rounding (u relative) each.
Each tolerance is derived beside its assertion from these rules, and the worst measured error / tolerance ratio on an
H100 is recorded next to its constant.
"""
import os

import numpy as np
import pytest
import torch

from conftest import load_snapshot
from float64_bounds import E_KNN, U, check_power, gamma
from gpu_models import dev, get_model, sm_count
from oracle import pointdsc_oracle as O

pytestmark = pytest.mark.gpu

PRECISIONS = os.environ.get("PDSC_TEST_PRECISIONS", "fp32,fp16x3").split(",")


def release(m):
    """Drop a model's cached workspaces after a call whose workspace (it holds the SC matrix) runs to gigabytes."""
    m._workspaces.clear()
    torch.cuda.empty_cache()


def run_injected(m, feat, src, tgt, taps, **inject):
    """A testing-mode call that starts at the head: features [B,N,128] injected (the encoder does not run), plus any of
    confidence / seeds / knn_idx."""
    B, N = feat.shape[:2]
    inj = {"features": dev(feat.astype(np.float32))}
    inj.update({name: dev(v) for name, v in inject.items()})
    out = m.run(torch.zeros(B, N, 6, device="cuda"), dev(src.astype(np.float32)), dev(tgt.astype(np.float32)),
                taps=taps, inject=inj)
    return {name: out[name].cpu().numpy() for name in taps}


def points(rng, B, N, side):
    return rng.uniform(0, side, (B, N, 3)).astype(np.float32), rng.uniform(0, side, (B, N, 3)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------
# 1. the SC matrix: row-major (fp32) and tiled (tensor-core modes) layouts
# ---------------------------------------------------------------------------------------------------
# Bound (`sc64`): a length of fp32 points is within 3.5 u of the exact one (the differences are exact to u, the fma chain of
# the squares adds gamma(3), the square root halves that and adds u): 4 u ds.  The rounded difference ds - dt is then within
# E = 4 u (ds + dt) + u |d|; its square within 2 |d| E + E^2 + u d^2; the division by the fp32 sigma_d^2 (itself rounded:
# u) and 1 - q add 2 u q + u; max(0, .) is 1-Lipschitz.  Measured on an H100 (80GB HBM3) over every case: worst error / bound
# = 0.64 (3DMatch, N = 5000; KITTI 0.61).
SC_N = [2, 10, 63, 64, 65, 127, 128, 129, 257, 1003, 2000, 5000]


def sc64(src, tgt, s32):
    """float64 SC [N,N] and the bound of |SC32 - SC64| for fp32 points src/tgt [N,3] and the fp32 sigma_d s32."""
    p, q = src.astype(np.float64), tgt.astype(np.float64)
    s2 = float(s32) ** 2
    sc, tol = np.empty((len(p), len(p))), np.empty((len(p), len(p)))
    for r0 in range(0, len(p), 512):
        ds = np.sqrt(((p[r0:r0 + 512, None] - p[None]) ** 2).sum(-1))
        dt = np.sqrt(((q[r0:r0 + 512, None] - q[None]) ** 2).sum(-1))
        d = ds - dt
        E = 4 * U * (ds + dt) + U * np.abs(d)
        sc[r0:r0 + 512] = np.maximum(1.0 - d * d / s2, 0.0)
        tol[r0:r0 + 512] = (2 * np.abs(d) * E + E * E + U * d * d) / s2 + 2 * U * d * d / s2 + U
    return sc, tol


@pytest.mark.parametrize("dataset", ["3dmatch", "kitti"])
@pytest.mark.parametrize("n", SC_N)
def test_sc_matrix_both_layouts_against_float64(n, dataset):
    from pointdsc_b200.synth import make_pair
    pairs = [make_pair(7000 + 10 * n + i, n, dataset, 0.5) for i in range(3)]
    args = [torch.stack([p[x] for p in pairs]).cuda() for x in ("corr_pos", "src_keypts", "tgt_keypts")]
    sigma_d = np.float32(O.default_config(dataset)["sigma_d"])
    got = {}
    for precision in PRECISIONS:
        m = get_model(dataset, precision)
        sc3 = m.run(*args, taps=["sc"])["sc"].cpu().numpy()
        sc1 = m.run(*[a[:1] for a in args], taps=["sc"])["sc"].cpu().numpy()
        assert np.array_equal(sc1[0], sc3[0]), precision              # a set's SC does not depend on its call
        got[precision] = sc3
    # the two layouts replay the same rounded sequence (div_by_const is the correctly rounded quotient): bit for bit
    first = got[PRECISIONS[0]]
    for precision in PRECISIONS[1:]:
        assert np.array_equal(got[precision], first), precision
    worst = 0.0
    for b, p in enumerate(pairs):
        sc = first[b]
        assert np.array_equal(sc, sc.T)                              # (x_i - x_j)^2 == (x_j - x_i)^2 in fp32
        assert (np.diagonal(sc) == 1.0).all()
        # the fixtures' bar against the oracle (test_gpu_parity.test_sc_matrix)
        _, ref = O.sc_matrix(p["src_keypts"], p["tgt_keypts"], float(sigma_d))
        ref = ref.numpy()
        assert np.abs(sc - ref).max() <= 1e-6
        assert (sc == ref).mean() >= 0.999
        ref64, tol = sc64(p["src_keypts"].numpy(), p["tgt_keypts"].numpy(), sigma_d)
        err = np.abs(sc - ref64)
        assert (err <= tol).all(), (b, float(err.max()), np.argwhere(err > tol)[:4])
        worst = max(worst, float((err / tol).max()))
        if n >= 64:
            assert (sc > 0).sum() > n, "SC is not vacuous: some off-diagonal pairs are consistent"
    print(f"SC {dataset} N={n}: worst |SC - SC64| / bound = {worst:.3g}")


# ---------------------------------------------------------------------------------------------------
# 2. the head: normalisation and the confidence MLP on injected features
# ---------------------------------------------------------------------------------------------------
# normed: the squared norm sums 128 non-negative products (gamma(128) relative), the square root halves that and adds u,
# the division adds u: |n32 - n64| <= C_NORMED u |n64| per entry, C_NORMED = 64 + 3.  Measured on an H100 (80GB HBM3):
# worst error 6.9 u |n64| (0.10 of the bound); the confidence's worst error is 1.2e-3 of its running-error bound.
C_NORMED = 67.0


def mlp64(feat, sd):
    """float64 confidence [R] and its running-error bound: per layer gamma(n + 1) (|b| + sum |W| |h|) for the n-term fma
    chain that starts at the bias (the last layer: 32 fmas from 0 and the bias add), plus |W| times the input's bound
    (ReLU is 1-Lipschitz)."""
    w = {i: sd[f"classification.{i}.weight"].double().numpy()[:, :, 0] for i in (0, 2, 4)}
    bb = {i: sd[f"classification.{i}.bias"].double().numpy() for i in (0, 2, 4)}
    x = feat.astype(np.float64)
    h1 = x @ w[0].T + bb[0]
    e1 = gamma(129) * (np.abs(x) @ np.abs(w[0]).T + np.abs(bb[0]))
    a1 = np.maximum(h1, 0.0)
    h2 = a1 @ w[2].T + bb[2]
    e2 = gamma(33) * ((a1 + e1) @ np.abs(w[2]).T + np.abs(bb[2])) + e1 @ np.abs(w[2]).T
    a2 = np.maximum(h2, 0.0)
    o = (a2 @ w[4].T + bb[4])[:, 0]
    e3 = (gamma(33) * ((a2 + e2) @ np.abs(w[4]).T + np.abs(bb[4])) + e2 @ np.abs(w[4]).T)[:, 0]
    return o, e3


def head_features(rng, B, N):
    f = (rng.standard_normal((B, N, 128)) * rng.uniform(0.1, 3.0, (B, N, 1))).astype(np.float32)
    flat = f.reshape(-1, 128)
    R = flat.shape[0]
    if R >= 3:
        flat[0] = 0.0                                          # a zero row: F.normalize gives 0
        flat[R // 2] = flat[R - 1]                             # an exact duplicate
    if R >= 8:
        flat[2] = (rng.standard_normal(128) * 1e-15).astype(np.float32)    # norm below the 1e-12 clamp
        flat[5::7] = flat[3]                                   # many copies of one row, in different warps and passes
    return f


def check_head(m, sd, feat, rng, what):
    B, N = feat.shape[:2]
    src, tgt = points(rng, B, N, 3.0)
    # first a call with other features of the same shape: rows the kernel fails to write keep that call's values
    run_injected(m, -head_features(rng, B, N), src, tgt, ["normed"])
    out = run_injected(m, feat, src, tgt, ["normed", "confidence"])
    x = feat.reshape(-1, 128).astype(np.float64)
    normed, conf = out["normed"].reshape(-1, 128), out["confidence"].reshape(-1)
    den = np.maximum(np.sqrt((x * x).sum(1)), float(np.float32(1e-12)))
    n64 = x / den[:, None]
    err = np.abs(normed - n64)
    tol = C_NORMED * U * np.abs(n64)
    assert (err <= tol).all(), (what, np.argwhere(err > tol)[:4])
    zero = ~(x != 0).any(1)
    assert (normed[zero] == 0.0).all()
    # identical rows give identical outputs, bit for bit, wherever they land
    _, first, inv = np.unique(feat.reshape(-1, 128), axis=0, return_index=True, return_inverse=True)
    inv = inv.reshape(-1)
    assert np.array_equal(normed, normed[first[inv]]) and np.array_equal(conf, conf[first[inv]])
    o64, e64 = mlp64(x, sd)
    cerr = np.abs(conf - o64)
    assert (cerr <= e64).all(), (what, float(cerr.max()), np.argwhere(cerr > e64)[:4])
    return float(np.max(np.where(n64 != 0, err / (U * np.abs(n64) + 1e-300), 0.0))), float((cerr / e64).max())


@pytest.mark.parametrize("precision", PRECISIONS)
def test_head_against_float64(precision):
    m = get_model("3dmatch", precision)
    sd = load_snapshot("3dmatch")
    rng = np.random.default_rng(11)
    sms = sm_count()
    worst_n, worst_c = 0.0, 0.0
    # R = 2 .. 31: one partial warp tile
    for n in range(2, 32):
        a, b = check_head(m, sd, head_features(rng, 1, n), rng, f"R={n}")
        worst_n, worst_c = max(worst_n, a), max(worst_c, b)
    a, b = check_head(m, sd, head_features(rng, 1, 1000), rng, "R=1000")
    worst_n, worst_c = max(worst_n, a), max(worst_c, b)
    # more rows than one pass of the capped grid (sms CTAs x 8 warps x 32 rows): the grid-stride loop runs again
    B = max(40, -(-(8 * 32 * sms + 1) // 1000))
    assert B * 1000 > 8 * 32 * sms
    a, b = check_head(m, sd, head_features(rng, B, 1000), rng, f"R={B * 1000}")
    worst_n, worst_c = max(worst_n, a), max(worst_c, b)
    release(m)
    print(f"head ({precision}): worst |normed - n64| = {worst_n:.3g} u |n64|; worst |conf - c64| / bound = {worst_c:.3g}")


# ---------------------------------------------------------------------------------------------------
# 3. seeds: testing-mode NMS (warp and tile kernels) and the validation forward's top-S
# ---------------------------------------------------------------------------------------------------
# The engine decides ||x_i - x_j|| >= R without a square root (d2_min, seeds.cu); the oracle computes the fp32 length as the
# reference does and compares it with the fp32 R.  They must agree index for index.  Against float64 a decision can differ
# only through a pair (i, j), s_j > s_i, whose float64 distance is within the fp32 length error of R: 4 u max(d, R) (see
# the SC bound above).
def nms_sets(rng, family, B, N, R):
    """B sets of N points: `ties` quantised confidences in [-0.5, 1.25] (many ties and exact zeros), `negative` 90 %
    negative confidences (the seed list's tail is the suppressed points, keys +0 and -0, in index order).  The cloud's
    density gives each point about three others within R.  From N >= 160 the last rows are pairs placed at fp32
    distance R and a few ulps either side of it, far from everything else, the second point of a pair scoring higher."""
    side = R * (N * 4.19 / 3.0) ** (1.0 / 3.0)
    src = rng.uniform(0, side, (B, N, 3)).astype(np.float32)
    if family == "ties":
        conf = (rng.integers(-2, 6, (B, N)) / 4.0).astype(np.float32)
    else:
        conf = np.where(rng.uniform(size=(B, N)) < 0.9, -rng.uniform(0.01, 1.0, (B, N)),
                        rng.uniform(0.0, 1.0, (B, N))).astype(np.float32)
        conf[:, ::13] = 0.0
    pairs = []
    if N >= 160:
        r32 = np.float32(R)
        deltas = [r32]
        lo = hi = r32
        for _ in range(3):
            lo, hi = np.nextafter(lo, np.float32(0)), np.nextafter(hi, np.float32(1e9))
            deltas += [lo, hi]
        for p, delta in enumerate(deltas):
            i, j = N - 2 - 2 * p, N - 1 - 2 * p                # the last rows: never early in the zero-key tail
            y = np.float32(-(10 + 20 * p) * R)
            src[:, i] = (0.0, y, 0.0)
            src[:, j] = (delta, y, 0.0)
            conf[:, i], conf[:, j] = 10.0 + 2 * p, 11.0 + 2 * p
            d32 = np.sqrt(np.float32(delta) * np.float32(delta))        # = length3(-delta, 0, 0) in fp32
            pairs.append((i, j, d32))
    return src, conf, pairs


def nms_reference(src, conf, R):
    """oracle.pick_seeds's local-max mask on fp32 distances (O.pairwise_length's expression, a block of rows at a time),
    the float64 mask and the points whose float64 decision hinges on a pair inside the fp32 band of R."""
    p32 = torch.from_numpy(src)
    s = torch.from_numpy(conf)
    r32 = torch.tensor(R, dtype=torch.float32)
    p64 = p32.double()
    R64 = float(r32)
    N = len(src)
    mask32, mask64, amb = (torch.empty(N, dtype=torch.bool) for _ in range(3))
    for r0 in range(0, N, 1024):
        rows = slice(r0, r0 + 1024)
        dist = torch.norm(p32[rows, None, :] - p32[None, :, :], dim=-1)
        mask32[rows] = ((s[rows, None] >= s[None, :]) | (dist >= r32)).all(-1)
        d64 = ((p64[rows, None, :] - p64[None, :, :]) ** 2).sum(-1).sqrt()
        higher = s[rows, None] < s[None, :]
        mask64[rows] = (~higher | (d64 >= R64)).all(-1)
        amb[rows] = (higher & ((d64 - R64).abs() <= 4 * U * torch.clamp(d64, min=R64))).any(-1)
    return mask32.numpy(), mask64.numpy(), amb.numpy()


def seeds_oracle(conf, mask32, S):
    key = torch.from_numpy(conf) * torch.from_numpy(mask32).float()
    return torch.sort(key, descending=True, stable=True)[1][:S].numpy()


_nms_refs = {}


def check_nms_set(key, src, conf, R, S, got, pairs):
    if key not in _nms_refs:
        mask32, mask64, amb = nms_reference(src, conf, R)
        want = seeds_oracle(conf, mask32, S)
        if len(src) <= 2048:                                   # the blocked oracle is oracle.pick_seeds itself
            p = torch.from_numpy(src)
            assert np.array_equal(want, O.pick_seeds(O.pairwise_length(p), torch.from_numpy(conf), R, S).numpy())
        assert np.array_equal(mask32[~amb], mask64[~amb])      # fp32 decisions = float64 outside the band
        _nms_refs[key] = (want, int(amb.sum()))
    want, n_amb = _nms_refs[key]
    assert np.array_equal(got, want), (key, np.flatnonzero(got != want)[:8], got[:8], want[:8])
    # the pairs at distance R and one ulp either side: the lower-scoring point keeps its score (and follows its partner in the
    # list) iff its fp32 distance is >= R
    for i, j, d32 in pairs:
        pos = np.flatnonzero(got == j)
        assert len(pos) == 1 and pos[0] + 1 < len(got), (i, j)
        assert (got[pos[0] + 1] == i) == (d32 >= np.float32(R)), (i, j, d32)
    return n_amb


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("n", [9, 10, 257, 16384])
@pytest.mark.parametrize("family,dataset", [("ties", "3dmatch"), ("negative", "kitti")])
def test_nms_seeds_both_kernels(family, dataset, n, precision):
    m = get_model(dataset, precision)
    R = float(np.float32(O.default_config(dataset)["nms_radius"]))
    S = m.num_seeds(n)
    sms = sm_count()
    tiles = -(-n // 256)
    B = -(-2 * sms // tiles)                     # nms_key_kernel<256> runs when B * ceil(N / 256) >= 2 * SMs
    assert B * tiles >= 2 * sms and tiles < 2 * sms
    rng = np.random.default_rng(100 + n)
    src, conf, pairs = nms_sets(rng, family, B, n, R)
    feat = np.random.default_rng(1).standard_normal((1, n, 128)).astype(np.float32)
    tgt = src + np.float32(0.01)
    batch = run_injected(m, np.broadcast_to(feat, (B, n, 128)), src, tgt, ["seeds"], confidence=conf)["seeds"]
    assert batch.shape == (B, S)
    if S == 0:
        return
    if n == 16384:
        assert len(pairs) == 7
        assert {np.float32(R), np.nextafter(np.float32(R), np.float32(0)), np.nextafter(np.float32(R), np.float32(1))} \
            <= {d for _, _, d in pairs}, "the pairs reach R and one ulp either side"
    check_sets = range(B) if n <= 2048 else [0]
    single = [0, 1, B - 1] if n <= 2048 else [0, B - 1]
    n_amb = 0
    for b in single:                             # bs = 1: nms_key_warp_kernel, the same seeds
        one = run_injected(m, feat, src[b:b + 1], tgt[b:b + 1], ["seeds"], confidence=conf[b:b + 1])["seeds"][0]
        assert np.array_equal(one, batch[b]), b
    for b in check_sets:
        n_amb += check_nms_set((family, n, b), src[b], conf[b], R, S, batch[b], pairs)
    if n >= 160:
        assert n_amb >= 1, "some decisions hinge on a pair inside the fp32 band"
    release(m)
    print(f"NMS {family} N={n} B={B}: {n_amb} points decided inside the fp32 band")


# ---------------------------------------------------------------------------------------------------
# 4. kNN on injected features and seeds
# ---------------------------------------------------------------------------------------------------
# Two ranks may swap only where their float64 distances lie within 2 E_KNN (float64_bounds.py derives E_KNN).
def knn_features(rng, N):
    """Clustered unit-scale rows (N / 20 centres) with 2 % exact duplicates of other rows."""
    centres = rng.standard_normal((N // 20 + 1, 128))
    f = centres[rng.integers(0, len(centres), N)] + 0.35 * rng.standard_normal((N, 128))
    dup = rng.choice(N, N // 50, replace=False)
    f[dup] = f[rng.integers(0, N, len(dup))]
    return f.astype(np.float32), dup


def check_knn(got, normed, seeds, k):
    """The float64 ranking wherever separated, the same distance at every rank, no duplicates, ignore_self, and exact
    duplicate rows in ascending index order.  Returns (separated fraction, worst ratio)."""
    got = got.astype(np.int64)
    nm = normed.astype(np.float64)
    dist = 2.0 - 2.0 * (nm[seeds] @ nm.T)
    order = np.argsort(dist, axis=1, kind="stable")
    ref = order[:, 1:k + 1]
    assert all(len(set(r)) == k for r in got)
    d_got, d_ref = np.take_along_axis(dist, got, 1), np.take_along_axis(dist, ref, 1)
    assert np.abs(d_got - d_ref).max() <= 2 * E_KNN, float(np.abs(d_got - d_ref).max())
    full = np.take_along_axis(dist, order[:, :k + 2], 1)
    gap_lo = full[:, 1:k + 1] - full[:, 0:k]
    gap_hi = full[:, 2:k + 2] - full[:, 1:k + 1] if full.shape[1] == k + 2 else np.ones_like(gap_lo)
    sep = (gap_lo > 2 * E_KNN) & (gap_hi > 2 * E_KNN)
    assert np.array_equal(got[sep], ref[sep]), np.argwhere((got != ref) & sep)[:8]
    self_first = full[:, 1] - full[:, 0] > 2 * E_KNN
    assert not any(int(sd) in r for sd, r, f in zip(seeds, got, self_first) if f)
    # exact duplicate rows have bitwise identical distances in both modes (identical operands, identical per-element
    # accumulation): they are selected lowest index first, and a higher copy never without the lower ones
    _, inv, cnt = np.unique(normed, axis=0, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    gid = np.where(cnt[inv] > 1, inv, -1)
    n_dup = 0
    for row, sd in zip(got, seeds):
        gr = gid[row]
        for g in np.unique(gr[gr >= 0]):
            members = np.flatnonzero(inv == g)
            pos = np.flatnonzero(gr == g)
            n_dup += 1
            present = row[pos]
            assert np.array_equal(present, np.sort(present)), (sd, present)
            # the lowest copy is missing only when it was the dropped rank 0 (the seed's own copy group)
            ok = np.array_equal(present, members[:len(present)]) or (
                sd in members and pos[0] == 0 and np.array_equal(present, members[1:len(present) + 1]))
            assert ok, (sd, present, members)
    assert n_dup > 0
    return float(sep.mean()), float(np.abs(d_got - d_ref).max() / (2 * E_KNN))


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("k", [40, 128])
@pytest.mark.parametrize("n", [1001, 1290, 2003, 5000, 16384])
def test_knn_against_float64(n, k, precision):
    m = get_model("3dmatch", precision, k=k)
    S = m.num_seeds(n)
    sms = sm_count()
    seed_ctas = -(-S // 128)
    if n == 1290:
        assert S > 128                                        # two seed CTAs per set
    if n % 4:
        assert n in (1001, 1290, 2003)                        # knn_select_kernel's scalar-load branch
    assert seed_ctas < sms                                    # bs = 1: the keys are split into several chunks
    B = -(-sms // seed_ctas)                                  # the batch: seed CTAs x sets >= SMs, one chunk
    assert B * seed_ctas >= sms
    rng = np.random.default_rng(n + k)
    feats = [knn_features(rng, n) for _ in range(2)]
    seeds = []
    for f, dup in feats:
        s = rng.choice(n, S, replace=False)
        s[:5] = dup[:5]                                       # some seeds have an exact copy elsewhere
        seeds.append(s.astype(np.int32))
    src, tgt = points(rng, 1, n, 3.0)
    # first a call with other features: distance entries the kernels fail to write keep that call's values
    run_injected(m, knn_features(rng, n)[0][None], src, tgt, ["knn_idx"], seeds=seeds[0][None])
    one = run_injected(m, feats[0][0][None], src, tgt, ["knn_idx", "normed"], seeds=seeds[0][None])
    sep, ratio = check_knn(one["knn_idx"][0], one["normed"][0], seeds[0], k)
    assert sep >= 0.2, sep                                    # a non-trivial share of ranks is separated
    # the batch: the same set first, another last, the rest filler
    fill = np.random.default_rng(5).standard_normal((B, n, 128)).astype(np.float32)
    fill[0], fill[-1] = feats[0][0], feats[1][0]
    bseeds = np.tile(seeds[0], (B, 1))
    bseeds[-1] = seeds[1]
    bsrc, btgt = np.broadcast_to(src, (B, n, 3)), np.broadcast_to(tgt, (B, n, 3))
    batch = run_injected(m, fill, bsrc, btgt, ["knn_idx", "normed"], seeds=bseeds)
    assert np.array_equal(batch["knn_idx"][0], one["knn_idx"][0])     # chunking does not change a distance
    if n <= 5000:
        sep2, ratio2 = check_knn(batch["knn_idx"][-1], batch["normed"][-1], seeds[1], k)
        ratio = max(ratio, ratio2)
    release(m)
    print(f"kNN N={n} k={k} ({precision}) B={B}: separated {sep:.2f}, worst |d64(got) - d64(ref)| / (2 E) = {ratio:.3g}")


# ---------------------------------------------------------------------------------------------------
# 5. the power iteration on the tapped compatibility
# ---------------------------------------------------------------------------------------------------
# float64_bounds.check_power: eig within its worst-case bound and statistical band, power_iters equal to the float64 exit
# wherever that exit is sure.
POWER_K = [1, 2, 3, 31, 32, 33, 39, 40, 41, 47, 48, 49, 79, 80, 81, 88, 89, 96, 127, 128]


def power_batch(N, B):
    from pointdsc_b200.synth import make_pair
    pairs = [make_pair(3000 + i, N, "3dmatch", 0.1 + 0.7 * i / max(B - 1, 1)) for i in range(B)]
    return [torch.stack([p[x] for p in pairs]).cuda() for x in ("corr_pos", "src_keypts", "tgt_keypts")]


def run_power_case(precision, k, iters, B=8, N=400):
    m = get_model("3dmatch", precision, k=k, iters=iters)
    out = m.run(*power_batch(N, B), taps=["compat", "eig", "power_iters"])
    S = m.num_seeds(N)
    compat = out["compat"].cpu().numpy().reshape(B, S, k, k)
    eig = out["eig"].cpu().numpy()
    pit = out["power_iters"].cpu().numpy()
    worst, worst_band, compared = 0.0, 0.0, 0
    for b in range(B):
        r, rb, sure = check_power(compat[b], eig[b], pit[b], k, iters)
        worst, worst_band, compared = max(worst, r), max(worst_band, rb), compared + int(sure)
    return worst, worst_band, compared, pit


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("k", POWER_K)
def test_power_iteration_against_float64(k, precision):
    worst, worst_band, compared, pit = run_power_case(precision, k, 10)
    assert compared >= 1, ("no set's exit could be compared", pit)
    print(f"power k={k} ({precision}): iterations {pit.tolist()}, exits compared {compared}/8, worst eig error / bound "
          f"{worst:.3g}, / band {worst_band:.3g}")


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("k", [40, 80, 128])
@pytest.mark.parametrize("iters", [1, 16])                 # 16 is kMaxIters, the largest cap the engine accepts
def test_power_iteration_caps(iters, k, precision):
    worst, worst_band, compared, pit = run_power_case(precision, k, iters)
    if iters == 1:
        assert (pit == 1).all()
    assert compared >= 1, ("no set's exit could be compared", pit)
    print(f"power cap={iters} k={k} ({precision}): iterations {pit.tolist()}, worst eig error / bound {worst:.3g}")


# ---------------------------------------------------------------------------------------------------
# 6. the validation forward: top-S seeds and M
# ---------------------------------------------------------------------------------------------------
# M = clamp(1 - (1 - f_i . f_j) / sigma^2, 0, 1): the fp32 dot is within gamma(128) sum |f_i| |f_j|, 1 - dot adds
# u |1 - dot|, the division by the fp32 sigma^2 (itself rounded: u) 2 u q, and 1 - q u; the clamp is 1-Lipschitz.
# Measured on an H100 (80GB HBM3): worst error / bound = 0.097 (N = 2000).
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("n", [257, 1003, 2000])
def test_validation_seeds_and_M(n, B, precision):
    from pointdsc_b200.synth import make_pair
    m = get_model("3dmatch", precision)
    pairs = [make_pair(8100 + n + i, n, "3dmatch", 0.4) for i in range(B)]
    args = [torch.stack([p[x] for p in pairs]).cuda() for x in ("corr_pos", "src_keypts", "tgt_keypts")]
    out = m.run_eval(*args, taps=["normed", "confidence", "seeds"])
    M = out["M"].cpu().numpy()
    normed, conf, seeds = (out[x].cpu().numpy() for x in ("normed", "confidence", "seeds"))
    assert np.array_equal(out["final_labels"].cpu().numpy(), conf)
    S = m.num_seeds(n)
    s2 = float(m.sigma.detach().cpu()[0]) ** 2
    worst = 0.0
    for b in range(B):
        want = O.top_confidence_seeds(torch.from_numpy(conf[b]), S).numpy()
        assert np.array_equal(seeds[b], want), b
        f = normed[b].astype(np.float64)
        dot = f @ f.T
        q = (1.0 - dot) / s2
        m64 = np.clip(1.0 - q, 0.0, 1.0)
        np.fill_diagonal(m64, 0.0)
        tol = (gamma(128) * (np.abs(f) @ np.abs(f).T) + U * np.abs(1.0 - dot)) / s2 + 2 * U * np.abs(q) + U
        assert (np.diagonal(M[b]) == 0.0).all()
        assert (M[b] >= 0.0).all() and (M[b] <= 1.0).all()
        err = np.abs(M[b] - m64)
        assert (err <= tol).all(), (b, float(err.max()), np.argwhere(err > tol)[:4])
        worst = max(worst, float((err / tol).max()))
        assert (M[b] > 0).mean() > 0.01                     # not vacuous: similar features exist
    print(f"validation N={n} B={B} ({precision}): worst |M - M64| / bound = {worst:.3g}")
