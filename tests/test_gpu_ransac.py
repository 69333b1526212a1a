"""Device RANSAC (pointdsc_b200.ransac, csrc/ransac.cu) against the float64 CPU restatement oracle/ransac_oracle.py, hypothesis by
hypothesis, on the packed interface the evaluation loop uses; its decision edges; a set's independence from its call; its memory,
graph and error contracts; and the evaluate.py --solver RANSAC loop.

Every hypothesis the device scores is replayed by the oracle from the same draws.  Its good is exact and its rmse agrees to 1e-12
relative (plus what the rounding of a thin sample's rotation moves it by: `rmse_tolerance`) whenever its margins (the smallest
|d^2 - r * r| and sigma_2 / sigma_1 of its sample) exceed 1e-9.  The device's winner
is the oracle's whenever the selection margin exceeds 1e-9, and otherwise ties the oracle's best key to 1e-12; its T is within 2
float32 ulps of the oracle's T for that iteration and its labels are exactly the oracle's.  The open3d rule applied to the device's
own keys gives the device's winner in every case, ties included.  Every hypothesis, rank-deficient samples included, also passes
the checks of tests/ransac_samples.py, which need no unique rotation: its rotation, the optimal value of its sample, its
translation, and its key recounted from its own transform; the winner's T and labels are its own transform's even when its
sample is degenerate."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from gpu_models import get_model, ulps
from oracle import ransac_oracle as O
from ransac_samples import check_set

pytestmark = pytest.mark.gpu

MARGIN = 1e-9
RADIUS = {"3dmatch": 0.10, "kitti": 0.6}
SIZES = [3, 4, 41, 1000, 5000, 12000, 16384]


def _pair(preset, n, seed=0):
    from pointdsc_b200.synth import make_pair
    p = make_pair(seed, n, preset)
    return p["src_keypts"].numpy(), p["tgt_keypts"].numpy(), p["gt_labels"].numpy(), p


def _forward_labels(preset, p):
    m = get_model(preset, "fp32")
    out = m({"corr_pos": p["corr_pos"][None].cuda(), "src_keypts": p["src_keypts"][None].cuda(),
             "tgt_keypts": p["tgt_keypts"][None].cuda(), "testing": True})
    return out["final_labels"][0].float().cpu().numpy()


def _device(src, tgt, labels, offsets=None, **kw):
    """ransac_packed with info and hypotheses on numpy inputs; returns a dict of numpy arrays."""
    from pointdsc_b200.ransac import ransac_packed
    if offsets is None:
        offsets = [0, len(src)]
    d = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()      # noqa: E731
    trans, lab, info = ransac_packed(d(src), d(tgt), d(labels), offsets, info=True, hypotheses=True, **kw)
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in info.items()}
    out.update(trans=trans.cpu().numpy(), labels=lab.cpu().numpy())
    return out


def rmse_tolerance(ref):
    """[I] the rmse difference two float64 solves of the same sample may show: 1e-12 relative, plus what the rotation's own
    rounding moves a residual by.  A 3-point sample's rotation is determined to about 16 eps / (sigma_2 / sigma_1) (svd3.cuh), and a
    rotation error dR moves R p + t - q by up to 2 |dR| max|p|, so a thin triangle far from the origin can move the rmse by more
    than 1e-12 of itself in either implementation.  0 for a sample with H = 0 (ratio inf: R = I in both)."""
    pts = np.abs(ref["_src"][O.candidates(ref["_labels_in"])])
    ext = float(pts[np.isfinite(pts)].max())
    with np.errstate(divide="ignore"):
        return 1e-12 * ref["rmse"] + 2 * 16 * 2.0 ** -52 * ext / ref["sigma_ratio"]


def _check(dev, b, ref, rows=slice(None)):
    """Device set b against the oracle's run `ref`: every qualifying hypothesis, the selection, T and the labels; and every
    hypothesis against the checks of ransac_samples.check_set."""
    check_set(dev, b, ref["_src"], ref["_tgt"], ref["_labels_in"], ref["_r"], max_iteration=dev["hyp_good"].shape[1],
              seed=ref["_seed"], rows=rows)
    assert int(dev["status"][b]) == ref["status"]
    if ref["status"] == 1:
        assert not dev["hyp_good"][b].any() and not dev["hyp_rmse"][b].any()
    else:
        good, rmse = dev["hyp_good"][b], dev["hyp_rmse"][b]
        q = O.qualifies(ref, MARGIN)
        assert q.mean() > (0.5 if ref["M"] >= 12 else 0.25), q.mean()      # M = 3: 6 + 3 of the 27 triples have full rank or H = 0
        assert np.array_equal(good[q], ref["good"][q])
        assert np.all(np.abs(rmse[q] - ref["rmse"][q]) <= rmse_tolerance(ref)[q])
        # the open3d rule on the device's own keys gives the device's winner
        best = int(dev["best_iteration"][b])
        assert best == O.select(good, rmse)
        wb = ref["best_iteration"]
        if ref["status"] == 0 and not (q[best] and q[wb]):
            return      # a degenerate sample won on either side: check_set has checked the device's winner, T and labels
        if ref["status"] == 0:
            if ref["selection"] > MARGIN:
                assert best == wb
            else:
                assert ref["good"][best] == ref["good"][wb] and abs(ref["rmse"][best] - ref["rmse"][wb]) <= 1e-12 * ref["rmse"][wb]
            assert ulps(dev["trans"][b], ref["T"][best].astype(np.float32)).max() <= 2
            assert float(dev["fitness"][b]) == ref["good"][best] / ref["M"]
            assert float(dev["inlier_rmse"][b]) == float(rmse[best])
            inl = np.zeros_like(ref["labels"])
            T = ref["T"][best]
            cand = O.candidates(ref["_labels_in"])
            e = ref["_src"][cand] @ T[:3, :3].T + T[:3, 3] - ref["_tgt"][cand]
            inl[cand[(e * e).sum(-1) < ref["_r"] ** 2]] = 1.0
            assert np.array_equal(dev["labels"][rows], inl)
            if best == wb:
                assert np.array_equal(dev["labels"][rows], ref["labels"])
            return
        assert best == -1
    assert np.array_equal(dev["trans"][b], np.eye(4, dtype=np.float32)) and not dev["labels"][rows].any()
    assert int(dev["best_iteration"][b]) == -1 and float(dev["fitness"][b]) == 0.0 and float(dev["inlier_rmse"][b]) == 0.0


def _oracle(src, tgt, labels, r, **kw):
    ref = O.ransac(src, tgt, labels, r, **kw)
    ref.update(_src=np.asarray(src, np.float32).astype(np.float64), _tgt=np.asarray(tgt, np.float32).astype(np.float64),
               _labels_in=labels, _r=r, _seed=kw.get("seed", O.DEFAULT_SEED))
    return ref


# ---------------------------------------------------------------------------------------------------
# 1-2. parity per hypothesis, and the selection on the device's own keys
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("source", ["gt", "forward", "all"])
@pytest.mark.parametrize("preset", ["3dmatch", "kitti"])
@pytest.mark.parametrize("n", SIZES)
def test_parity_per_hypothesis(n, preset, source):
    src, tgt, labels, p = _pair(preset, n)
    if source == "forward":
        if n < 4:
            pytest.skip("the forward needs more rows than seeds")
        labels = _forward_labels(preset, p)
    elif source == "all":
        labels = np.ones(n, np.float32)
    r = RADIUS[preset]
    _check(_device(src, tgt, labels, max_correspondence_distance=r), 0, _oracle(src, tgt, labels, r))


def test_parity_demo_pair():
    z = np.load(os.path.join(GOLDEN, "demo_pair_3dmatch.npz"))
    src, tgt, labels = z["src_keypts"], z["tgt_keypts"], z["final_labels"].reshape(-1).astype(np.float32)
    ref = _oracle(src, tgt, labels, 0.10)
    assert ref["status"] == 0
    _check(_device(src, tgt, labels), 0, ref)


# ---------------------------------------------------------------------------------------------------
# 3. decision edges: iteration 0 draws a triple whose solve is exact, R = I and t dyadic-exact
# ---------------------------------------------------------------------------------------------------
def edge_set(r):
    """A set whose rows 0-2 are a triple related by a pure translation t (their x coordinates equal, so the demeaned covariance
    is diag(0, 8 s^2, 6 s^2): no Jacobi rotation, R = I exactly, and t_x = r - float32(r) exactly), then candidates whose residual
    lies along x only, ex = float32(r) + t_x - qx, exact in double: d^2 = r * r exactly (not an inlier); the nearest double below
    r * r that such a residual reaches (an inlier; two or three steps below, as the 2^-53-relative grid of ex allows); and, where
    float32(r^2) != r * r, a d^2 strictly between the two (decided by the double product).  A last row is not a candidate.
    Returns (src, tgt, labels, intended label of each edge candidate)."""
    f32 = np.float32
    T = r * r
    tx = r - float(f32(r))
    hi = float(f32(tx))
    lo = tx - hi
    s, ty, tz, cy, cz = 0.125, 0.25, -0.5, 0.5, 0.75
    yz = ((2, 1), (-2, 1), (0, -2))
    src = [(-lo, cy + s * y, cz + s * z) for y, z in yz]
    tgt = [(hi, cy + s * y + ty, cz + s * z + tz) for y, z in yz]
    step = 2.0 ** -56 if r == 0.125 else float(np.spacing(r))       # the grid of ex just below r
    px = float(f32(r))

    def cand(m):
        qx = m * step
        assert float(f32(qx)) == qx
        return (px, 0.5, 0.25), (qx, 0.5 + ty, 0.25 + tz), (px + tx) - qx

    want = []
    p, q, ex = cand(0)
    assert ex * ex == T
    src.append(p), tgt.append(q), want.append(0.0)
    m = next(m for m in range(1, 64) if cand(m)[2] ** 2 < T)
    p, q, ex = cand(m)
    below = ex * ex
    steps, v = 0, T
    while v > below:
        v, steps = np.nextafter(v, 0.0), steps + 1
    assert 1 <= steps <= 3
    src.append(p), tgt.append(q), want.append(1.0)
    if float(f32(T)) != T:
        p, q, ex = cand(-(1 << 22) if float(f32(T)) > T else (1 << 22))
        a, b = sorted((T, float(f32(T))))
        assert a < ex * ex < b
        src.append(p), tgt.append(q), want.append(1.0 if ex * ex < T else 0.0)
    src.append((0.0, 0.0, 0.0)), tgt.append((5.0, 5.0, 5.0))
    labels = np.ones(len(src), np.float32)
    labels[-1] = 0.0
    return np.array(src, np.float32), np.array(tgt, np.float32), labels, want


def edge_seed(M):
    """The first seed whose iteration 0 draws the triple (rows 0, 1, 2 in any order)."""
    return next(s for s in range(1 << 20) if sorted(O.draws(s, 1, M)[0].tolist()) == [0, 1, 2])


@pytest.mark.parametrize("r", [0.1, 0.6, 0.125])
def test_decision_edges(r):
    src, tgt, labels, want = edge_set(r)
    seed = edge_seed(int((labels > 0).sum()))
    ref = O.ransac(src, tgt, labels, r, max_iteration=1, seed=seed)
    assert np.array_equal(ref["T"][0][:3, :3], np.eye(3)) and ref["T"][0][0, 3] == r - float(np.float32(r))
    assert ref["status"] == 0 and list(ref["labels"][3:-1]) == want and ref["labels"][:3].all()
    dev = _device(src, tgt, labels, max_correspondence_distance=r, max_iteration=1, seed=seed)
    assert int(dev["status"][0]) == 0 and int(dev["best_iteration"][0]) == 0
    assert np.array_equal(dev["labels"], ref["labels"])
    assert int(dev["hyp_good"][0, 0]) == ref["good"][0] == 3 + sum(want)
    assert float(dev["hyp_rmse"][0, 0]) == ref["rmse"][0]
    assert np.array_equal(dev["trans"][0], ref["trans"])


# ---------------------------------------------------------------------------------------------------
# 4. a set's result is its own: one group == reversed == each set alone == another SM count, bit for bit
# ---------------------------------------------------------------------------------------------------
def status2_set(m=1000, seed=51, max_iteration=5000):
    """One source point repeated against targets scattered over a 1 km cube: a hypothesis maps it onto the mean of its drawn
    targets, which is no target unless its three draws are one index (none are, for this seed)."""
    g = np.random.default_rng(0)
    src = np.tile(np.float32([[1.0, 2.0, 3.0]]), (m, 1))
    tgt = (g.random((m, 3)) * 1000.0).astype(np.float32)
    d = O.draws(seed, max_iteration, m)
    assert not ((d[:, 0] == d[:, 1]) & (d[:, 1] == d[:, 2])).any()
    return src, tgt, np.ones(m, np.float32)


def invariance_group():
    sets = []
    for m in (0, 1, 2, 3):                                           # M = 0, 1, 2, 3 among 9 rows
        s, t, _, _ = _pair("3dmatch", 9, 10 + m)
        lab = np.zeros(9, np.float32)
        lab[[1, 4, 6][:m] if m < 3 else [0, 2, 5]] = 1.0
        sets.append((s, t, lab))
    s, t, lab, _ = _pair("3dmatch", 300, 5)
    s = s.copy()
    s[17, 1] = np.nan                                                # a non-finite candidate
    sets.append((s, t, lab))
    sets.append(status2_set())
    for preset, n, seed in (("3dmatch", 1000, 1), ("kitti", 5000, 2), ("3dmatch", 12000, 3)):
        s, t, lab, _ = _pair(preset, n, seed)
        lab = lab.copy()
        lab[n // 2:n // 2 + n // 10] = 1.0
        sets.append((s, t, lab))
    return sets


def _run_group(sets, **kw):
    off = np.cumsum([0] + [len(s) for s, _, _ in sets]).tolist()
    return _device(np.concatenate([s for s, _, _ in sets]), np.concatenate([t for _, t, _ in sets]),
                   np.concatenate([lab for _, _, lab in sets]), off, **kw), off


def _same(a, b):
    return np.array_equal(np.atleast_1d(a).view(np.uint8), np.atleast_1d(b).view(np.uint8))


KEYS = ["trans", "fitness", "inlier_rmse", "best_iteration", "status", "hyp_good", "hyp_rmse", "hyp_trans"]


def test_group_equals_reversed_and_alone():
    sets = invariance_group()
    assert len(sets) == 9
    packed, off = _run_group(sets)
    rev, roff = _run_group(sets[::-1])
    B = len(sets)
    for b, st in enumerate(sets):
        alone, _ = _run_group([st])
        for k in KEYS:
            assert _same(packed[k][b], alone[k][0]) and _same(packed[k][b], rev[k][B - 1 - b]), (b, k)
        rows = packed["labels"][off[b]:off[b + 1]]
        assert _same(rows, alone["labels"]) and _same(rows, rev["labels"][roff[B - 1 - b]:roff[B - b]]), b
    assert list(packed["status"]) == [1, 1, 1, 0, 0, 2, 0, 0, 0]
    for b in (4, 5, 6, 7, 8):
        s, t, lab = sets[b]
        _check(packed, b, _oracle(s, t, lab, 0.10), rows=slice(off[b], off[b + 1]))


def _dump(path):
    sets = invariance_group()
    out, _ = _run_group(sets)
    np.savez(path, **out)


def test_sm_count_does_not_matter(tmp_path):
    runs = {}
    for sms in (None, 16):
        env = dict(os.environ)
        env.pop("PDSC_SM_COUNT", None)
        if sms is not None:
            env["PDSC_SM_COUNT"] = str(sms)
        path = tmp_path / f"sm_{sms}.npz"
        subprocess.run([sys.executable, os.path.abspath(__file__), str(path)], env=env, check=True,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        runs[sms] = np.load(path)
    assert sorted(runs[None].files) == sorted(runs[16].files)
    for k in runs[None].files:
        assert _same(runs[None][k], runs[16][k]), k


def test_seeds_and_iteration_caps():
    s, t, lab, _ = _pair("3dmatch", 1000, 1)
    a = _device(s, t, lab)
    again = _device(s, t, lab)
    other = _device(s, t, lab, seed=52)
    for k in KEYS + ["labels"]:
        assert _same(a[k], again[k]), k
    assert not np.array_equal(a["hyp_good"], other["hyp_good"])
    for cap in (1, 2, 3, 5000):
        d = _device(s, t, lab, max_iteration=cap)
        ref = _oracle(s, t, lab, 0.10, max_iteration=cap)
        assert d["hyp_good"].shape == (1, cap)
        assert np.array_equal(d["hyp_good"][0], a["hyp_good"][0, :cap])        # the draws do not depend on the cap
        _check(d, 0, ref)


# ---------------------------------------------------------------------------------------------------
# 5. memory contract, graph capture, errors
# ---------------------------------------------------------------------------------------------------
def _raw(lib, eng, off, d_off, src, tgt, lab, outs, scratch, nbytes, r=0.10, max_iteration=5000, seed=51):
    h = (C.c_int32 * len(off))(*off)
    P = lambda x: C.c_void_p(x) if isinstance(x, int) else (C.c_void_p(x.data_ptr()) if x is not None else None)   # noqa: E731
    return lib.pdsc_ransac_packed(eng, len(off) - 1, h, P(d_off), P(src), P(tgt), P(lab), float(r), int(max_iteration),
                                  C.c_uint64(seed), *[P(o) for o in outs], P(scratch), nbytes,
                                  C.c_void_p(torch.cuda.current_stream().cuda_stream))


def _group_tensors(sets):
    off = np.cumsum([0] + [len(s) for s, _, _ in sets]).tolist()
    cat = lambda i: torch.from_numpy(np.concatenate([x[i] for x in sets])).cuda()     # noqa: E731
    return off, torch.tensor(off, dtype=torch.int32, device="cuda"), cat(0), cat(1), cat(2)


OUT_SPECS = [("trans", 4, lambda B, R, I: B * 16), ("labels", 4, lambda B, R, I: R), ("fitness", 8, lambda B, R, I: B),
             ("inlier_rmse", 8, lambda B, R, I: B), ("best_iteration", 4, lambda B, R, I: B), ("status", 4, lambda B, R, I: B),
             ("hyp_good", 4, lambda B, R, I: B * I), ("hyp_rmse", 8, lambda B, R, I: B * I)]


def test_memory_contract():
    from buffer_guards import PATTERNS, guarded_output, scratch_buffer
    from pointdsc_b200 import _capi
    lib, eng = _capi.load(), _capi.utility_engine(0)
    sets = invariance_group()
    off, d_off, src, tgt, lab = _group_tensors(sets)
    B, R, I = len(sets), off[-1], 5000
    need = int(lib.pdsc_ransac_packed_scratch_bytes(B, (C.c_int32 * (B + 1))(*off), I))
    assert need > 0
    ref, _ = _run_group(sets)
    for pattern in PATTERNS:
        outs = {name: guarded_output(size * n(B, R, I), size, torch.device("cuda"), pattern) for name, size, n in OUT_SPECS}
        scratch = scratch_buffer(need, 16, pattern)
        assert _raw(lib, eng, off, d_off, src, tgt, lab, [g.ptr for g in outs.values()], scratch.ptr, need) == 0
        torch.cuda.synchronize()
        scratch.check(("scratch", pattern))
        for (name, size, _), g in zip(OUT_SPECS, outs.values()):
            g.check((name, pattern))
            want = np.ascontiguousarray(ref[name]).view(np.uint8).reshape(-1)
            assert np.array_equal(g.inner.cpu().numpy(), want), (name, pattern)


def test_graph_replay_equals_eager():
    from pointdsc_b200 import _capi
    lib, eng = _capi.load(), _capi.utility_engine(0)
    sets = invariance_group()
    off, d_off, src, tgt, lab = _group_tensors(sets)
    B, R, I = len(sets), off[-1], 5000
    need = int(lib.pdsc_ransac_packed_scratch_bytes(B, (C.c_int32 * (B + 1))(*off), I))
    scratch = _capi.scratch(need, torch.device("cuda"), 16)

    def outs():
        return [torch.empty(n(B, R, I) * size, dtype=torch.uint8, device="cuda") for _, size, n in OUT_SPECS]
    eager = outs()
    assert _raw(lib, eng, off, d_off, src, tgt, lab, eager, scratch, need) == 0
    graphed = outs()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            assert _raw(lib, eng, off, d_off, src, tgt, lab, graphed, scratch, need) == 0
    torch.cuda.current_stream().wait_stream(s)
    for x in graphed:
        x.fill_(0xAB)
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, graphed):
        assert torch.equal(a, b)


def test_errors():
    from pointdsc_b200 import _capi
    from pointdsc_b200.ransac import ransac_packed, ransac_refine
    lib, eng = _capi.load(), _capi.utility_engine(0)
    sets = invariance_group()[3:6]
    off, d_off, src, tgt, lab = _group_tensors(sets)
    B, R, I = len(sets), off[-1], 100
    need = int(lib.pdsc_ransac_packed_scratch_bytes(B, (C.c_int32 * (B + 1))(*off), I))
    scratch = torch.empty(need + 32, dtype=torch.uint8, device="cuda")
    base = (scratch.data_ptr() + 15) // 16 * 16
    trans, labels = torch.empty(B, 4, 4, device="cuda"), torch.empty(R, device="cuda")
    outs = [trans, labels] + [None] * 6
    call = lambda **kw: _raw(lib, eng, kw.pop("off", off), d_off, kw.pop("src", src), tgt, lab, kw.pop("outs", outs),   # noqa: E731
                             kw.pop("scratch", base), kw.pop("nbytes", need), **{"max_iteration": I, **kw})
    assert call() == 0
    # offsets
    assert call(off=[0, 5, 5, off[-1]]) == 3
    assert call(off=[1, 5, 9, off[-1]]) == 3
    assert lib.pdsc_ransac_packed_scratch_bytes(3, (C.c_int32 * 4)(0, 5, 5, 9), I) == 0
    assert lib.pdsc_ransac_packed_scratch_bytes(0, (C.c_int32 * 1)(0), I) == 0
    assert lib.pdsc_ransac_packed_scratch_bytes(B, (C.c_int32 * (B + 1))(*off), 0) == 0
    # arguments
    for r in (0.0, -0.1, float("nan"), float("inf")):
        assert call(r=r) == 1, r
    assert call(max_iteration=0) == 1
    assert call(src=None) == 1
    assert call(outs=[trans, None] + [None] * 6) == 1
    assert call(outs=[None, labels] + [None] * 6) == 1
    # scratch
    assert call(nbytes=need - 1) == 5
    assert call(scratch=base + 8) == 5
    assert call(scratch=None) == 5
    assert "pdsc_ransac_packed" in lib.pdsc_last_error().decode()
    # Python
    with pytest.raises(_capi.PdscError):
        ransac_packed(src, tgt, lab, off, max_correspondence_distance=0.0)
    with pytest.raises(_capi.PdscError):
        ransac_packed(src, tgt, lab, off, max_iteration=0)
    with pytest.raises(ValueError):
        ransac_packed(src, tgt, lab, [0, 5, 5, off[-1]])
    with pytest.raises(ValueError):
        ransac_packed(src[1:], tgt[1:], lab[1:], off)
    with pytest.raises(ValueError):
        ransac_refine(src[None], tgt[None], lab[None, :-1])
    with pytest.raises(_capi.PdscError):
        ransac_packed(src.cpu(), tgt.cpu(), lab.cpu(), off)


def test_ransac_refine_equals_packed():
    from pointdsc_b200.ransac import ransac_packed, ransac_refine
    pairs = [_pair("3dmatch", 500, s) for s in (0, 1, 2)]
    src = torch.from_numpy(np.stack([p[0] for p in pairs])).cuda()
    tgt = torch.from_numpy(np.stack([p[1] for p in pairs])).cuda()
    lab = torch.from_numpy(np.stack([p[2] for p in pairs])).cuda()
    a, la = ransac_refine(src, tgt, lab)
    b, lb = ransac_packed(src.reshape(-1, 3), tgt.reshape(-1, 3), lab.reshape(-1), [0, 500, 1000, 1500])
    assert a.shape == (3, 4, 4) and la.shape == (3, 500) and torch.equal(a, b) and torch.equal(la.reshape(-1), lb)


# ---------------------------------------------------------------------------------------------------
# 6. evaluate.py --solver RANSAC
# ---------------------------------------------------------------------------------------------------
def test_evaluate_solver_ransac():
    import evaluate
    flags = ["--synthetic", "8", "--batch_invariant", "--solver", "RANSAC"]
    cols = [c for c in range(len(evaluate.COLUMNS)) if c not in (9, 10)]
    plain, _ = evaluate.main(["--synthetic", "8", "--batch_invariant", "--batch_size", "1"])
    for icp in ([], ["--use_icp"]):
        s1, _ = evaluate.main(flags + ["--batch_size", "1"] + icp)
        s4, _ = evaluate.main(flags + ["--batch_size", "4"] + icp)
        assert np.array_equal(s1[:, cols], s4[:, cols]), icp
        assert (s1[:, 5:9] != plain[:, 5:9]).any()                  # RANSAC's labels, not the network's


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    _dump(sys.argv[1])
