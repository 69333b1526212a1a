"""The spectral-matching baseline on the device (csrc/spectral_matching.cu, `spectral.spectral_matching_packed`) against the
float64 restatement of oracle/sm_oracle.py, its contracts, and `evaluate.py --method SM`.

Error model (u = 2^-24, gamma(n) = n u / (1 - n u), as in float64_bounds.py).  The reference is the float64 SM on the device's
own fp32 rows.  Write m = ds - dt for a pair (ds, dt the exact source / target lengths), c = 4.5 / tau^2.
  M entries.  Each squared difference carries 3 roundings and the two additions 2 more: ds^2 within gamma(5) relative, so
    |ds' - ds| <= gamma(4) ds after the square root and its rounding (dt alike), and |m' - m| <= e_m = gamma(5) (ds + dt).
    y' = fl(fl(m'^2) fl32(c)) is within (2 |m| e_m + e_m^2) c (1 + gamma(3)) + gamma(3) c m^2 of m^2 c, and 4.5 - y' rounds once
    more (at most 4.5 u where it is not clamped).  With e = that sum and Mu = 4.5 - m^2 c, the clamp max(0, .) is 1-Lipschitz
    and flat below 0, so |M'_ij - M_ij| <= W_ij = max(0, Mu + e) - max(0, Mu - e) (0 on the diagonal, both exact).  W is
    symmetric (fl(x_j - x_i) = -fl(x_i - x_j)), so |E|_2 <= max_i sum_j W_ij = E_N; |M|_2 <= max_i sum_j M_ij = M_N.
  One step.  u_t' = M' v_t-1' with fp32 sums: each lane's fma chain holds ceil(N / 32) terms and warp_sum adds 5 levels, so
    |u' - M' v'| <= g M' |v'| entrywise, g = gamma(ceil(N / 32) + 6).  With x_t = M v_t-1 (float64) and delta_t-1 the norm
    distance of the iterates,
        |u_t' - x_t| <= a_t = E_N (|v_t-1| + delta_t-1) + M_N delta_t-1 + g (M_N + E_N) (|v_t-1| + delta_t-1).
    f(x) = x / (|x| + 1e-6) has Jacobian norm 1 / (|x| + 1e-6) and every point of the segment has |z| >= |x_t| - a_t, so
    |f(u') - f(x_t)| <= a_t / (|x_t| - a_t + 1e-6); the fp32 norm (a thread-strided fma sum, warp tree and eight warps:
    gamma(ceil(N / 256) + 13) relative on the square, half that on the root, plus the root's, the + 1e-6's and the division's
    roundings) moves v_t' by at most e_n = gamma(ceil(N / 256) + 16) relative, and |f| <= 1:
        delta_t <= min(2, a_t / (|x_t| - a_t + 1e-6) + e_n)     (2 when |x_t| <= a_t: two vectors of norm <= 1).
  v is checked entrywise against delta_10 (a norm bound covers every entry); that end-to-end bound is loose, and
  test_gpu_spectral_steps.py checks every iterate on its own against a per-entry bound of one step.
  pdsc_leading_eigenvector on the materialised fp32 M has the same one-step model with its own orders: ceil(N / 32) fmas per
  lane and the tree again, and a norm summed over ceil(N / 8) per-CTA partials of at most 32 squares each:
  e_n = gamma(ceil(N / 8) + 40).
Labels.  Always: the top S = int(N * 0.1) of the device's own v, descending, lowest row first on ties, exactly.  Against float64:
  a row whose float64 entry is above the (S+1)-th largest by more than 2 delta_10 is selected, one below the S-th by more than
  2 delta_10 is not; where the selection gap v_(S) - v_(S+1) exceeds 2 delta_10 the labels equal the oracle's.
T.  float64_bounds.check_transforms on a float64 Kabsch of the device's own weights (v' * labels') over all N rows.  The fp32
  centroids and H of weighted_kabsch.cuh are sums in double of fp32 products, inside _h_error's C_PRE model.  Rank-deficient
  selections (S <= 2, collinear rows: no unique rotation) are checked on their own terms: R orthonormal with det 1, and the
  value gap sigma_1 + sigma_2 + d sigma_3 - tr(R H) within C_VALUE eps (|H|_1 + sum EH) + 3 sum EH (tests/ransac_samples.py's
  form with the fp32 eps and H error).  H = 0 gives T = I bit for bit.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from float64_bounds import EPS, _h_error, assert_rotations, check_transforms, entry_width, gamma, weighted_kabsch64
from oracle import sm_oracle as O
from ransac_samples import C_VALUE

pytestmark = pytest.mark.gpu

THR = {"3dmatch": 0.10, "kitti": 0.6}
WORST = {}


def _note(what, r):
    WORST[what] = max(WORST.get(what, 0.0), float(r))


def make_set(seed, n, preset, ratio=0.3):
    from pointdsc_b200.synth import make_pair
    p = make_pair(seed, n, preset, ratio)
    return p["corr_pos"].numpy(), p["src_keypts"].numpy(), p["tgt_keypts"].numpy()


def run(sets, thr, d_offsets=False):
    """One packed call over sets [(corr, src, tgt)] -> (trans [B,4,4], labels [R], v [R]) as numpy."""
    from pointdsc_b200.spectral import spectral_matching_packed
    off = np.cumsum([0] + [len(s[0]) for s in sets]).tolist()
    cat = lambda i: torch.from_numpy(np.ascontiguousarray(np.concatenate([s[i] for s in sets]))).cuda()   # noqa: E731
    d_off = torch.tensor(off, dtype=torch.int32, device="cuda") if d_offsets else None
    T, lab, v = spectral_matching_packed(cat(0), cat(1), cat(2), off, d_offsets=d_off, inlier_threshold=thr, eigenvector=True)
    torch.cuda.synchronize()
    return T.cpu().numpy(), lab.cpu().numpy(), v.cpu().numpy(), off


def power_bound(M, W, iterates, e_n):
    """delta_10 of the header, from the float64 M, W and iterates (row 0 the start vector)."""
    N = M.shape[0]
    M_N = float(M.sum(1).max())
    E_N = float(W.sum(1).max())
    g = gamma(math.ceil(N / 32) + 6)
    delta = 0.0
    for t in range(1, iterates.shape[0]):
        nv = float(torch.linalg.norm(iterates[t - 1]))
        x = float(torch.linalg.norm(M @ iterates[t - 1]))
        a = E_N * (nv + delta) + M_N * delta + g * (M_N + E_N) * (nv + delta)
        den = x - a + 1e-6
        delta = 2.0 if den <= 0 else min(2.0, a / den + e_n)
        delta *= 1 + 1e-9                              # the float64 evaluation of the bound itself
    return delta


def sm_norm_error(N):
    return gamma(math.ceil(N / 256) + 16)


def check_set(corr, src, tgt, thr, T, labels, v, where):
    """One set's device outputs against the oracle (header).  Returns delta_10."""
    N = len(corr)
    c = torch.from_numpy(corr).cuda()
    o = O.sm(c, torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda(), thr)
    S = o["S"]
    W = entry_width(c, thr)
    delta = power_bound(o["M"], W, o["iterates"], sm_norm_error(N))
    del W
    v64 = o["v"].cpu().numpy()
    err = np.abs(v.astype(np.float64) - v64)
    assert (err <= delta).all(), (where, float(err.max()), delta)
    _note("v / delta", err.max() / delta if delta > 0 else 0.0)
    # labels: the device's own top S, exactly
    own = np.zeros(N, np.float32)
    own[np.argsort(-v, kind="stable")[:S]] = 1.0
    assert np.array_equal(labels, own), (where, "labels are not the top S of the device's v")
    # against float64 where the margin decides
    if 0 < S < N:
        vs = np.sort(v64)[::-1]
        assert (labels[v64 > vs[S] + 2 * delta] == 1).all(), where
        assert (labels[v64 < vs[S - 1] - 2 * delta] == 0).all(), where
        if o["gap"] > 2 * delta:
            assert np.array_equal(labels, o["labels"].cpu().numpy().astype(np.float32)), where
    # T on the device's own weights
    w = (v * labels).astype(np.float64)
    if not w.any():
        assert np.array_equal(T, np.eye(4, dtype=np.float32)), (where, "H = 0 must give the identity")
        return delta
    a, b = src.astype(np.float64)[None], tgt.astype(np.float64)[None]
    ref = weighted_kabsch64(a, b, w[None])
    assert np.array_equal(T[3], np.array([0, 0, 0, 1], np.float32)), where
    R = T[:3, :3].astype(np.float64)
    assert_rotations(R[None], where)
    s, d, H = ref["s"][0], ref["d"][0], ref["H"][0]
    if s[1] > 1e-4 * s[0]:
        r = check_transforms(T[None], ref, where)
        _note("T rotation / tol", r["R"])
    # the value gap, on every set (the only rotation check of a rank-deficient one)
    m = a - ref["ca"][:, None]
    n = b - ref["cb"][:, None]
    EH, _, _ = _h_error(w[None], a, b, m, n)
    sumE = 9.0 * float(EH[0])
    gap = s[0] + s[1] + d * s[2] - float(np.trace(R @ H))
    bound = C_VALUE * EPS * (np.abs(H).sum() + sumE) + 3.0 * sumE
    assert gap <= bound, (where, gap, bound)
    _note("value gap / bound", max(gap, 0.0) / bound)
    return delta


SIZES = [2, 9, 10, 11, 31, 32, 33, 255, 256, 257, 511, 512, 513, 1000, 1024, 5000, 16384]


@pytest.mark.parametrize("preset", ["3dmatch", "kitti"])
def test_parity_alone(preset):
    """Every size from 2 to 16,384 rows, tile and warp-row edges included, one set per call."""
    thr = THR[preset]
    for i, n in enumerate(SIZES):
        if preset == "kitti" and n > 5000:
            continue
        s = make_set(1000 + i, n, preset, (0.1, 0.3, 0.6)[i % 3])
        T, lab, v, _ = run([s], thr)
        check_set(*s, thr, T[0], lab, v, (preset, n))
    print(f"{preset}: worst {WORST}")


def test_mixed_group_parity_and_invariance():
    """64 sets of the 3DMatch-like mix (tools/mixed_batch_bench.py) in one call: each against the oracle, and bit for bit the
    same as alone and in reverse order."""
    rng = np.random.default_rng(100)
    u = rng.random(64)
    lo = np.where(u < 0.1, 200, np.where(u < 0.7, 1000, 3000))
    hi = np.where(u < 0.1, 1000, np.where(u < 0.7, 3000, 6001))
    sizes = [int(rng.integers(a, b)) for a, b in zip(lo, hi)]
    sets = [make_set(2000 + b, n, "3dmatch", 0.05 + 0.5 * (b % 5) / 4) for b, n in enumerate(sizes)]
    T, lab, v, off = run(sets, 0.10, d_offsets=True)
    Tr, labr, vr, offr = run(sets[::-1], 0.10)
    for b, s in enumerate(sets):
        a, e = off[b], off[b + 1]
        rb = len(sets) - 1 - b
        ar, er = offr[rb], offr[rb + 1]
        assert np.array_equal(T[b], Tr[rb]) and np.array_equal(lab[a:e], labr[ar:er]) and np.array_equal(v[a:e], vr[ar:er]), b
        if b % 8 == 0:
            T1, lab1, v1, _ = run([s], 0.10)
            assert np.array_equal(T[b], T1[0]) and np.array_equal(lab[a:e], lab1) and np.array_equal(v[a:e], v1), b
        check_set(*s, 0.10, T[b], lab[a:e], v[a:e], ("mixed", b, len(s[0])))
    print(f"mixed: worst {WORST}")


def test_edge_families():
    """S = 0 (N < 10), all rows outliers (M = 0: v = 0 after one step, T = I), duplicate rows, all inliers, collinear rows."""
    sets = []
    for n in range(2, 10):
        sets.append(make_set(3000 + n, n, "3dmatch", 0.5))
    n = 40
    i = np.arange(n, dtype=np.float32)
    z = np.zeros(n, np.float32)
    src = np.stack([i, z, z], 1)
    tgt = np.stack([3 * i, z, z], 1)
    corr = np.concatenate([src, tgt], 1)
    sets.append(((corr - corr.mean(0)).astype(np.float32), src, tgt))
    c, s, t = make_set(3100, 300, "3dmatch", 0.4)
    c[150:], s[150:], t[150:] = c[:150], s[:150], t[:150]
    sets.append((c, s, t))
    sets.append(make_set(3101, 600, "3dmatch", 1.0))
    sets.append(make_set(3102, 600, "kitti", 1.0))
    # collinear: every source row on one line, targets the same line moved rigidly (H of rank 1 whatever is selected)
    x = np.linspace(-1, 1, 200, dtype=np.float32)
    src = np.stack([x, 0.5 * x, -x], 1).astype(np.float32)
    tgt = (src @ np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]], np.float32).T + np.float32(0.3)).astype(np.float32)
    corr = np.concatenate([src, tgt], 1)
    sets.append(((corr - corr.mean(0)).astype(np.float32), src, tgt))
    # S <= 2 with inliers: N = 10 .. 29
    for n in (10, 19, 20, 29):
        sets.append(make_set(3200 + n, n, "3dmatch", 1.0))
    T, lab, v, off = run(sets, 0.10)
    for b, st in enumerate(sets):
        a, e = off[b], off[b + 1]
        check_set(*st, 0.10, T[b], lab[a:e], v[a:e], ("edge", b, len(st[0])))
    for b in range(8):                                       # S = 0
        assert lab[off[b]:off[b + 1]].sum() == 0 and np.array_equal(T[b], np.eye(4, dtype=np.float32))
    b = 8                                                    # all outliers
    assert not v[off[b]:off[b + 1]].any() and np.array_equal(lab[off[b]:off[b + 1]], (np.arange(40) < 4).astype(np.float32))
    assert np.array_equal(T[b], np.eye(4, dtype=np.float32))
    print(f"edges: worst {WORST}")


def test_cross_check_with_materialised_power_iteration():
    """The fused eigenvector and pdsc_leading_eigenvector(early_exit=0) on the fp32 M, materialised with the kernel's own
    operations, both within the float64 bound."""
    from pointdsc_b200.spectral import leading_eigenvector
    for n, preset, seed in ((1000, "3dmatch", 4000), (5000, "3dmatch", 4001), (2000, "kitti", 4002)):
        thr = THR[preset]
        s = make_set(seed, n, preset, 0.3)
        T, lab, v, _ = run([s], thr)
        c = torch.from_numpy(s[0]).cuda()
        d = c[None, :, :] - c[:, None, :]
        ds = torch.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])
        dt = torch.sqrt((d[..., 3] * d[..., 3] + d[..., 4] * d[..., 4]) + d[..., 5] * d[..., 5])
        del d
        m = ds - dt
        M32 = torch.clamp_min(4.5 - (m * m) * torch.tensor(4.5 / thr ** 2, dtype=torch.float32), 0.0)
        M32.fill_diagonal_(0.0)
        del ds, dt, m
        ve, it = leading_eigenvector(M32[None].contiguous(), 10, early_exit=False)
        assert int(it[0]) == 10
        o = O.sm(c, torch.from_numpy(s[1]).cuda(), torch.from_numpy(s[2]).cuda(), thr)
        W = entry_width(c, thr)
        d_sm = power_bound(o["M"], W, o["iterates"], sm_norm_error(n))
        d_eig = power_bound(o["M"], W, o["iterates"], gamma(math.ceil(n / 8) + 40))
        v64 = o["v"].cpu().numpy()
        assert np.abs(v - v64).max() <= d_sm, (n, preset)
        assert np.abs(ve[0].cpu().numpy() - v64).max() <= d_eig, (n, preset)
        print(f"N={n} {preset}: fused {np.abs(v - v64).max() / d_sm:.3g}, materialised "
              f"{np.abs(ve[0].cpu().numpy() - v64).max() / d_eig:.3g} of the bound")


# ---------------------------------------------------------------------------------------------------
# the C ABI: guarded buffers, graph replay, errors
# ---------------------------------------------------------------------------------------------------
def _abi(sets):
    from pointdsc_b200 import _capi
    lib, eng = _capi.load(), _capi.utility_engine(0)
    off = np.cumsum([0] + [len(s[0]) for s in sets]).tolist()
    cat = lambda i: torch.from_numpy(np.ascontiguousarray(np.concatenate([x[i] for x in sets]))).cuda()   # noqa: E731
    corr, src, tgt = cat(0), cat(1), cat(2)
    d_off = torch.tensor(off, dtype=torch.int32, device="cuda")
    h_off = (C.c_int32 * len(off))(*off)
    need = int(lib.pdsc_spectral_matching_packed_scratch_bytes(len(sets), h_off))
    P = lambda x: None if x is None else C.c_void_p(x if isinstance(x, int) else x.data_ptr())           # noqa: E731

    def call(trans, labels, eig, scratch, nbytes, stream=None, h=h_off, B=len(sets), thr=0.10, its=False):
        """pdsc_spectral_matching_packed, or pdsc_spectral_matching_packed_iterates when `its` (the iterates buffer) is given."""
        st = (stream or torch.cuda.current_stream()).cuda_stream
        args = (eng, B, h, P(d_off), P(corr), P(src), P(tgt), thr, P(trans), P(labels), P(eig))
        if its is not False:
            return lib.pdsc_spectral_matching_packed_iterates(*args, P(its), P(scratch), nbytes, C.c_void_p(st))
        return lib.pdsc_spectral_matching_packed(*args, P(scratch), nbytes, C.c_void_p(st))
    torch.cuda.synchronize()
    return call, need, off


def _abi_group():
    return [make_set(5000 + b, n, "3dmatch", 0.3) for b, n in enumerate((5, 700, 33, 2048, 513))]


def test_memory_contract():
    """Every output is written within its bounds and the same whatever the output and scratch buffers held, with and without
    the iterates output (pdsc_spectral_matching_packed_iterates); the other outputs do not depend on it."""
    from buffer_guards import PATTERNS, guarded_output, scratch_buffer
    from pointdsc_b200.spectral import spectral_matching_packed
    sets = _abi_group()
    T, lab, v, _ = run(sets, 0.10)
    call, need, off = _abi(sets)
    B, R = len(sets), off[-1]
    cat = lambda i: torch.from_numpy(np.ascontiguousarray(np.concatenate([x[i] for x in sets]))).cuda()   # noqa: E731
    its = spectral_matching_packed(cat(0), cat(1), cat(2), off, iterates=True)[2].cpu().numpy()
    assert np.array_equal(its[-1], v)
    want = {"trans": T, "labels": lab, "eig": v}
    for pattern in PATTERNS:
        outs = {"trans": guarded_output(64 * B, 16, torch.device("cuda"), pattern),
                "labels": guarded_output(4 * R, 4, torch.device("cuda"), pattern),
                "eig": guarded_output(4 * R, 4, torch.device("cuda"), pattern)}
        scratch = scratch_buffer(need, 16, pattern)
        assert call(outs["trans"].ptr, outs["labels"].ptr, outs["eig"].ptr, scratch.ptr, need) == 0
        torch.cuda.synchronize()
        scratch.check(("scratch", pattern))
        for name, g in outs.items():
            g.check((name, pattern))
            assert np.array_equal(g.inner.cpu().numpy(), np.ascontiguousarray(want[name]).view(np.uint8).reshape(-1)), (name, pattern)
        # without the optional eigenvector output
        lab_only = guarded_output(4 * R, 4, torch.device("cuda"), pattern)
        assert call(outs["trans"].ptr, lab_only.ptr, None, scratch.ptr, need) == 0
        torch.cuda.synchronize()
        lab_only.check(("labels without eig", pattern))
        assert np.array_equal(lab_only.inner.cpu().numpy(), lab.view(np.uint8))
        # with the iterates output: all ten rows written, and the same bytes in every other output
        outs["its"] = guarded_output(4 * 10 * R, 4, torch.device("cuda"), pattern)
        for name in ("trans", "labels", "eig"):
            outs[name] = guarded_output(outs[name].nbytes, outs[name].align, torch.device("cuda"), pattern)
        want["its"] = its
        assert call(outs["trans"].ptr, outs["labels"].ptr, outs["eig"].ptr, scratch.ptr, need, its=outs["its"].ptr) == 0
        torch.cuda.synchronize()
        scratch.check(("scratch with iterates", pattern))
        for name, g in outs.items():
            g.check((name, "with iterates", pattern))
            assert np.array_equal(g.inner.cpu().numpy(), np.ascontiguousarray(want[name]).view(np.uint8).reshape(-1)), \
                (name, "with iterates", pattern)


def test_graph_replay_and_errors():
    from pointdsc_b200 import _capi
    sets = _abi_group()
    call, need, off = _abi(sets)
    B, R = len(sets), off[-1]
    scratch = _capi.scratch(need, torch.device("cuda"), 16)

    def outs():
        return (torch.empty(B, 4, 4, device="cuda"), torch.empty(R, device="cuda"), torch.empty(R, device="cuda"),
                torch.empty(10, R, device="cuda"))
    eager = outs()
    assert call(*eager[:3], scratch, need, its=eager[3]) == 0
    graphed = outs()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            assert call(*graphed[:3], scratch, need, stream=s, its=graphed[3]) == 0
    torch.cuda.current_stream().wait_stream(s)
    for x in graphed:
        x.fill_(7.0)
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, graphed):
        assert torch.equal(a, b)
    assert torch.equal(eager[3][-1], eager[2])
    lib = _capi.load()
    fn = "pdsc_spectral_matching_packed"
    # short scratch, null outputs, a bad threshold
    eager = eager[:3]
    assert call(*eager, scratch, need - 1) != 0 and fn in lib.pdsc_last_error().decode()
    assert call(None, eager[1], None, scratch, need) != 0 and fn in lib.pdsc_last_error().decode()
    assert call(*eager, scratch, need, thr=0.0) != 0 and fn in lib.pdsc_last_error().decode()
    assert call(*eager, scratch, need, thr=0.0, its=None) != 0 and fn + "_iterates" in lib.pdsc_last_error().decode()
    # bad offsets: not starting at 0, an empty set, a set above 16,384 rows
    for bad in ([1, 5, 700], [0, 5, 5], [0, 16385]):
        h = (C.c_int32 * len(bad))(*bad)
        assert call(*eager, scratch, need, h=h, B=len(bad) - 1) != 0 and fn in lib.pdsc_last_error().decode(), bad
        assert lib.pdsc_spectral_matching_packed_scratch_bytes(len(bad) - 1, h) == 0
    torch.cuda.synchronize()
    from pointdsc_b200.spectral import spectral_matching_packed
    with pytest.raises(_capi.PdscError):
        z = torch.zeros(16385, 6, device="cuda")
        spectral_matching_packed(z, z[:, :3].contiguous(), z[:, :3].contiguous(), [0, 16385])


def test_spectral_matching_batched_matches_packed():
    """spectral_matching [bs,N,...] is the packed call with offsets b * N."""
    from pointdsc_b200.spectral import spectral_matching
    sets = [make_set(6000 + b, 800, "3dmatch", 0.3) for b in range(3)]
    T, lab, _, _ = run(sets, 0.10)
    st = lambda i: torch.from_numpy(np.stack([s[i] for s in sets])).cuda()   # noqa: E731
    T2, lab2 = spectral_matching(st(0), st(1), st(2), 0.10)
    assert np.array_equal(T, T2.cpu().numpy()) and np.array_equal(lab.reshape(3, 800), lab2.cpu().numpy())


def test_evaluate_method_sm():
    """evaluate.py --synthetic 4 --method SM: the same statistics at --batch_size 1 and 4; RANSAC and ICP are refused."""
    import evaluate
    cols = [c for c in range(len(evaluate.COLUMNS)) if c not in (9, 10)]
    s1, _ = evaluate.main(["--synthetic", "4", "--method", "SM", "--batch_size", "1"])
    s4, _ = evaluate.main(["--synthetic", "4", "--method", "SM", "--batch_size", "4"])
    assert len(s1) == 4 and np.array_equal(s1[:, cols], s4[:, cols])
    for extra in (["--solver", "RANSAC"], ["--use_icp"]):
        with pytest.raises(SystemExit):
            evaluate.main(["--synthetic", "1", "--method", "SM"] + extra)
