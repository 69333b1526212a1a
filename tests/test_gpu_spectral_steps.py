"""The spectral-matching baseline's power iteration (csrc/spectral_matching.cu) one step at a time: every iterate the device
writes (`spectral_matching_packed(..., iterates=True)`, pdsc_spectral_matching_packed_iterates) against one float64 step from
the device's own previous iterate, on every launch path the power kernel takes.

Error model (u = 2^-24, gamma(n) = n u / (1 - n u); W the entry width of test_gpu_spectral_matching.py's header, |M' - M| <= W
entrywise for the fp32 entries M' the kernel forms).  Step t takes the device's iterate v' = v'_t-1 (v'_0 = 1 exactly) and
writes v'_t.  The reference is y_t = x / (|x| + 1e-6), x = M v', with M the float64 matrix on the device's fp32 rows.
  The sum.  u_i' = sum_j M'_ij v'_j: lane l runs one fma per column j = l mod 32 in ascending order, ceil(N / 32) of them, and
    warp_sum's xor tree adds 5 levels, so |u_i' - (M' v')_i| <= gamma(ceil(N / 32) + 6) (|M'| |v'|)_i (one level spare).  With
    |M'| <= M + W:
        |u_i' - x_i| <= a_i = (W |v'|)_i + g ((M + W) |v'|)_i,    g = gamma(ceil(N / 32) + 6).
  The norm.  sum u'^2 is a thread-strided fma chain (ceil(N / 256) terms per thread), a warp tree (5) and the eight warps'
    partials added in order (8): within gamma(ceil(N / 256) + 13) relative (every term >= 0).  Half of that after the square
    root, plus the root's, the + 1e-6's and the division's roundings: the fp32 division moves v_t' from u' / (|u'| + 1e-6) by
    at most e_n = gamma(ceil(N / 256) + 16) relative (generous: half the sum's terms would do), plus |1e-6f - 1e-6| / D on the
    denominator, D = |u'| + 1e-6.
  The normalisation.  |u' - x|_2 <= |a|_2, so D >= D_lo = max(|x| - |a|, 0) + 1e-6, and with D0 = |x| + 1e-6
        |u_i' / D - y_i| <= a_i / D_lo + |x_i| |a|_2 / (D_lo D0).
  So per entry
        |v_t,i' - y_t,i| <= tol_i = a_i / D_lo + |x_i| |a|_2 / (D_lo D0) + (e_n + |1e-6f - 1e-6| / D_lo) (|x_i| + a_i) / D_lo,
  plus gamma64(N + 8) (M |v'| + |x|) / D_lo for the float64 evaluation itself.  Worst measured on an H100 (80GB HBM3, 700 W
  power limit) over this module's sets: 0.096 of tol (the CPU rehearsal's emulated kernel: 0.12).
The check can tell.  The same float64 step with a bug built in, on the same device iterate: M_ii = 4.5 (diagonal not zeroed),
  the last column dropped, the last (partial) 512-column tile dropped, sigma = tau in place of tau / 3, and a start vector
  other than 1 (1 on even rows, 0 on odd ones; step 1 only).  Every set of at least three rows must move by at least
  TELL = 10 tolerances under every bug at some step, else the case is too weak to check the kernel and fails.  (At N = 2 M is
  one symmetric entry: a shifted diagonal leaves the direction of M v alone when that entry is positive, and a dropped column
  changes nothing when it is 0, so no two-row set can tell both.)  Smallest margins over this module's sets on an H100:
  diagonal 13.8, last column 32.6, last tile 234, sigma = tau 4.7e4, start vector 1.0e3 tolerances.
Labels.  Exactly the top S = int(N * 0.1) of iterate 10, lowest row first on ties, and iterate 10 is bit for bit the
  eigenvector output.  Against float64 where it decides, from the final step's own bound: with y = y_10 and tol from v'_9, if
  every row of float64's top S has y - tol above every other row's y + tol, the device's selection is float64's.  The
  constructed sets below (S tight inliers among N = 10 S rows) must reach that decision.
Launch paths.  RW (rows per warp) in {4, 2, 1} is chosen from the call's CTA count and the SM count (engine_rules
  .sm_rows_per_warp); each value is reached, read back from the launched kernel's name, and a set's iterates are bit for bit
  the same in every composition and alone.
The CPU rehearsal (unmarked) emulates the kernel's fp32 step in numpy (its entries bit for bit, its lane order and xor tree,
  its norm order; each fma rounded through float64, so up to one extra rounding per fma, inside the spare tree level) and
  shows that it stays within tol while a kernel with each bug planted does not.
"""
import math
import re

import numpy as np
import pytest
import torch

from engine_rules import SM_TILE, num_seeds, sm_rows_per_warp
from float64_bounds import entry_width, gamma, gamma64
from oracle import sm_oracle as O

ITERS = 10
TELL = 10.0             # a bug must move some step by this many tolerances; smallest seen on an H100: 13.8 (diagonal)
THR = {"3dmatch": 0.10, "kitti": 0.6}
D6 = abs(float(np.float32(1e-6)) - 1e-6)
BUGS = ("diagonal", "last column", "last tile", "sigma = tau", "start vector")
WORST = {}


def _note(what, r):
    WORST[what] = max(WORST.get(what, 0.0), float(r))


def _low(what, r):
    WORST[what] = min(WORST.get(what, math.inf), float(r))


# ---------------------------------------------------------------------------------------------------
# the float64 step, its tolerance and the bugs
# ---------------------------------------------------------------------------------------------------
def step_bound(M, W, v):
    """(y, tol) of the header for one step from the iterate v (float64, M's device)."""
    N = M.shape[0]
    av = v.abs()
    x = M @ v
    mv = M @ av
    wv = W @ av
    a = wv + gamma(math.ceil(N / 32) + 6) * (mv + wv)
    nx, na = float(torch.linalg.norm(x)), float(torch.linalg.norm(a))
    d0, dlo = nx + 1e-6, max(nx - na, 0.0) + 1e-6
    en = gamma(math.ceil(N / 256) + 16)
    ax = x.abs()
    tol = a / dlo + ax * na / (dlo * d0) + (en + D6 / dlo) * (ax + a) / dlo + gamma64(N + 8) * (mv + ax) / dlo
    return x / d0, tol * (1 + 1e-9)


def normalise(x):
    return x / (float(torch.linalg.norm(x)) + 1e-6)


def bugged_step(bug, M, Msig, v, t):
    """y of one step with `bug` built in, from the iterate v (None where the bug does not act at step t)."""
    N = M.shape[0]
    if bug == "diagonal":
        return normalise(M @ v + 4.5 * v)
    if bug == "last column":
        return normalise(M[:, :N - 1] @ v[:N - 1])
    if bug == "last tile":
        c0 = (N - 1) // SM_TILE * SM_TILE
        return normalise(M[:, :c0] @ v[:c0])
    if bug == "sigma = tau":
        return normalise(Msig @ v)
    if bug == "start vector":
        return normalise(M @ start_vector(N, v)) if t == 1 else None
    raise ValueError(bug)


def start_vector(N, like):
    s = torch.zeros(N, dtype=torch.float64, device=like.device)
    s[::2] = 1.0
    return s


def ratio(err, tol):
    """max err / tol, inf where tol = 0 < err."""
    r = torch.where(tol > 0, err / torch.where(tol > 0, tol, torch.ones_like(tol)), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def check_steps(corr, thr, its, where, device, tell=True):
    """Every step of one set's iterates its [10,N] (fp32 numpy) against the float64 step from the previous one (header).
    Returns (per-step worst error / tol, {bug: largest deviation / tol over the steps}, y_10, tol_10)."""
    N = len(corr)
    c = torch.from_numpy(np.ascontiguousarray(corr)).to(device)
    M = O.compat(c, thr)
    W = entry_width(c, thr)
    Msig = O.compat(c, 3.0 * thr) if tell else None          # sigma = tau: the threshold three times over
    V = torch.from_numpy(its.astype(np.float64)).to(device)
    prev = torch.ones(N, dtype=torch.float64, device=device)
    steps, moved = [], {b: 0.0 for b in BUGS}
    for t in range(1, ITERS + 1):
        y, tol = step_bound(M, W, prev)
        r = ratio((V[t - 1] - y).abs(), tol)
        steps.append(r)
        if tell:
            for bug in BUGS:
                yb = bugged_step(bug, M, Msig, prev, t)
                if yb is not None:
                    moved[bug] = max(moved[bug], ratio((yb - y).abs(), tol))
        prev = V[t - 1]
    del M, W, Msig
    return steps, moved, y, tol


def assert_steps(corr, thr, its, where, device):
    """check_steps, asserted: every step within tol, and every bug told apart (sets of three rows or more)."""
    steps, moved, y, tol = check_steps(corr, thr, its, where, device, tell=len(corr) >= 3)
    bad = [t + 1 for t, r in enumerate(steps) if not r <= 1.0]
    assert not bad, (where, "steps outside the bound", bad, [steps[t - 1] for t in bad])
    _note("step error / tol", max(steps))
    if len(corr) >= 3:
        weak = {b: r for b, r in moved.items() if not r >= TELL}
        assert not weak, (where, "the check cannot tell these bugs (largest deviation / tol)", weak)
        for b, r in moved.items():
            _low(f"{b}: deviation / tol (smallest)", r)
    return y, tol


def decided_labels(y, tol, S):
    """float64's top S of y (descending, lowest row first) when the final step's bound decides it, else None."""
    N = y.shape[0]
    if not 0 < S < N:
        return None
    order = torch.sort(-y, stable=True).indices
    top, rest = order[:S], order[S:]
    if float((y[top] - tol[top]).min()) <= float((y[rest] + tol[rest]).max()):
        return None
    lab = np.zeros(N, np.float32)
    lab[top.cpu().numpy()] = 1.0
    return lab


def top_s(v, S):
    lab = np.zeros(len(v), np.float32)
    lab[np.argsort(-v, kind="stable")[:S]] = 1.0
    return lab


# ---------------------------------------------------------------------------------------------------
# sets
# ---------------------------------------------------------------------------------------------------
def make_set(seed, n, preset="3dmatch", ratio=0.3):
    """A synthetic pair (pointdsc_b200.synth) with its rows reversed, so that the inliers come last and the last column and
    the last tile carry compatible rows."""
    from pointdsc_b200.synth import make_pair
    p = make_pair(seed, n, preset, ratio)
    return tuple(np.ascontiguousarray(p[k].numpy()[::-1]) for k in ("corr_pos", "src_keypts", "tgt_keypts"))


def make_gap_set(seed, n):
    """Exactly S = int(N * 0.1) noise-free inliers of one rigid motion (the last S rows) among uniform outliers in a 3 m cube:
    a wide selection gap."""
    rng = np.random.default_rng(seed)
    S = num_seeds(n)
    src = rng.uniform(0, 3, (n, 3))
    q, r = np.linalg.qr(rng.standard_normal((3, 3)))
    q *= np.sign(np.diag(r))
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    tgt = rng.uniform(0, 3, (n, 3))
    tgt[n - S:] = src[n - S:] @ q.T + rng.uniform(0, 1, 3)
    corr = np.concatenate([src, tgt], 1)
    corr = corr - corr.mean(0)
    return corr.astype(np.float32), src.astype(np.float32), tgt.astype(np.float32)


# ---------------------------------------------------------------------------------------------------
# the CPU rehearsal: the kernel's fp32 step in numpy
# ---------------------------------------------------------------------------------------------------
def emulate_entries(corr, thr, sigma_bug=False, diagonal_bug=False):
    """M' [N,N] fp32 of sm_entry, bit for bit: every operation rounded on its own, no contraction."""
    c = corr.astype(np.float32)
    d = c[None, :, :] - c[:, None, :]
    ds = np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])
    dt = np.sqrt((d[..., 3] * d[..., 3] + d[..., 4] * d[..., 4]) + d[..., 5] * d[..., 5])
    m = ds - dt
    tau = 3.0 * thr if sigma_bug else thr
    M = np.maximum(np.float32(4.5) - (m * m) * np.float32(4.5 / (tau * tau)), np.float32(0.0))
    if not diagonal_bug:
        np.fill_diagonal(M, 0.0)
    return M


def _fma(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def _xor_tree(x):
    """warp_sum over the last axis (32 lanes): lane l adds lane l ^ o for o = 16 .. 1; lane 0's value."""
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        x = (x + x[..., lanes ^ o]).astype(np.float32)
    return x[..., 0]


def emulate_step(M, v, cols=None):
    """One iteration: sm_power_kernel's u = M' v (lane l: columns l, l + 32, ... in order, then the xor tree) over the
    columns `cols` (default all), then sm_norm_kernel's v = u / (sqrt(sum u^2) + 1e-6)."""
    N = M.shape[0]
    n = N if cols is None else cols
    acc = np.zeros((N, 32), np.float32)
    for j0 in range(0, n, 32):
        k = min(32, n - j0)
        acc[:, :k] = _fma(M[:, j0:j0 + k], v[None, j0:j0 + k], acc[:, :k])
    u = _xor_tree(acc)
    K = -(-N // 256)
    up = np.zeros(K * 256, np.float32)
    up[:N] = u
    ss = np.zeros(256, np.float32)
    for r in range(K):
        ss = _fma(up[r * 256:(r + 1) * 256], up[r * 256:(r + 1) * 256], ss)
    part = _xor_tree(ss.reshape(8, 32))
    t = np.float32(0.0)
    for w in range(8):
        t = np.float32(t + part[w])
    den = np.float32(np.sqrt(t) + np.float32(1e-6))
    return (u / den).astype(np.float32)


def emulate(corr, thr, bug=None):
    """The kernel's ten iterates [10,N] fp32, with `bug` (one of BUGS) planted."""
    N = len(corr)
    M = emulate_entries(corr, thr, sigma_bug=bug == "sigma = tau", diagonal_bug=bug == "diagonal")
    v = np.ones(N, np.float32)
    if bug == "start vector":
        v = np.zeros(N, np.float32)
        v[::2] = 1.0
    cols = {"last column": N - 1, "last tile": (N - 1) // SM_TILE * SM_TILE}.get(bug)
    its = []
    for _ in range(ITERS):
        v = emulate_step(M, v, cols)
        its.append(v)
    return np.stack(its)


REHEARSAL = [("3dmatch", 33, 0.5), ("3dmatch", 257, 0.3), ("3dmatch", 700, 0.1), ("kitti", 600, 0.3), ("gap", 1000, None)]


@pytest.mark.parametrize("case", REHEARSAL, ids=lambda c: f"{c[0]}-{c[1]}")
def test_rehearsal_on_the_cpu(case):
    """The emulated fp32 kernel stays within every step's bound, every bug moves the float64 step by >= TELL tolerances, and
    an emulated kernel with each bug planted fails the check."""
    preset, n, r = case
    s = make_gap_set(7000 + n, n) if preset == "gap" else make_set(7000 + n, n, preset, r)
    thr = THR.get(preset, 0.10)
    its = emulate(s[0], thr)
    y, tol = assert_steps(s[0], thr, its, ("rehearsal", preset, n), "cpu")
    if preset == "gap":
        assert decided_labels(y, tol, num_seeds(n)) is not None
    for bug in BUGS:
        steps, _, _, _ = check_steps(s[0], thr, emulate(s[0], thr, bug), (bug,), "cpu", tell=False)
        print(f"rehearsal {preset} N={n}: planted {bug!r}: worst step error / tol {max(steps):.3g}")
        assert max(steps) > TELL, (bug, steps)
    print(f"rehearsal {preset} N={n}: {WORST}")


def test_rehearsal_rows_per_warp_rule():
    """sm_rows_per_warp at the edges of its two thresholds."""
    for sms in (16, 114, 132):
        want = 2 * sms
        assert sm_rows_per_warp([32 * want], sms) == 4 and sm_rows_per_warp([32 * want - 32], sms) == 2
        assert sm_rows_per_warp([16 * want], sms) == 2 and sm_rows_per_warp([16 * want - 16], sms) == 1
        assert sm_rows_per_warp([1] * want, sms) == 4 and sm_rows_per_warp([1] * (want - 1), sms) == 1


# ---------------------------------------------------------------------------------------------------
# the device
# ---------------------------------------------------------------------------------------------------
def run(sets, thr):
    """One packed call -> (labels [R], eigenvector [R], iterates [10,R], offsets, the RW values the power kernel ran)."""
    from torch.profiler import ProfilerActivity, profile

    from pointdsc_b200.spectral import spectral_matching_packed
    off = np.cumsum([0] + [len(s[0]) for s in sets]).tolist()
    cat = lambda i: torch.from_numpy(np.ascontiguousarray(np.concatenate([s[i] for s in sets]))).cuda()   # noqa: E731
    args = (cat(0), cat(1), cat(2))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _, lab, v, its = spectral_matching_packed(*args, off, inlier_threshold=thr, eigenvector=True, iterates=True)
        torch.cuda.synchronize()
    rws = {int(m.group(1)) for e in prof.events() for m in [re.search(r"sm_power_kernel<(\d)>", e.name)] if m}
    return lab.cpu().numpy(), v.cpu().numpy(), its.cpu().numpy(), off, rws


def check_call(sets, thr, where):
    """Every set of one call, step by step; returns the call's outputs (run) for identity checks."""
    from gpu_models import sm_count
    lab, v, its, off, rws = run(sets, thr)
    want = sm_rows_per_warp([len(s[0]) for s in sets], sm_count())
    assert rws == {want}, (where, "the power kernel ran RW", rws, "the rule says", want)
    for b, s in enumerate(sets):
        a, e = off[b], off[b + 1]
        N = e - a
        w = where + (b, N)
        assert np.array_equal(its[ITERS - 1, a:e].view(np.uint32), v[a:e].view(np.uint32)), (w, "iterate 10 is not the eigenvector")
        assert np.array_equal(lab[a:e], top_s(its[ITERS - 1, a:e], num_seeds(N))), (w, "labels are not the top S of iterate 10")
        y, tol = assert_steps(s[0], thr, its[:, a:e], w, "cuda")
        dec = decided_labels(y, tol, num_seeds(N))
        if dec is not None:
            assert np.array_equal(lab[a:e], dec), (w, "labels differ from float64's where the final step decides")
            WORST["labels decided by float64"] = WORST.get("labels decided by float64", 0) + 1
    return lab, v, its, off, want


EDGES = [2, 9, 10, 31, 32, 33, 511, 512, 513, 1023, 1024, 1025, 16384]


@pytest.mark.gpu
def test_tile_and_warp_row_edges():
    """Every tile and warp-row edge, each set alone and all of them in one call, every step against float64; the group's
    iterates bit for bit the sets' own."""
    sets = [make_set(8000 + n, n, "3dmatch", (0.1, 0.3, 0.6)[i % 3]) for i, n in enumerate(EDGES)]
    alone = {}
    for s in sets:
        _, _, its, _, rw = check_call([s], 0.10, ("alone",))
        alone[len(s[0])] = (its, rw)
    _, _, its, off, rw = check_call(sets, 0.10, ("group",))
    for b, s in enumerate(sets):
        n = len(s[0])
        assert np.array_equal(its[:, off[b]:off[b + 1]].view(np.uint32), alone[n][0].view(np.uint32)), (n, rw, alone[n][1])
    print(f"edges: RW alone {sorted({a[1] for a in alone.values()})}, group {rw}; {WORST}")


@pytest.mark.gpu
def test_kitti_steps():
    for i, n in enumerate((33, 700, 2049, 5000)):
        check_call([make_set(8100 + i, n, "kitti", (0.1, 0.3, 0.6)[i % 3])], THR["kitti"], ("kitti",))
    print(f"kitti: {WORST}")


def _compositions(target, sms):
    """For RW = 4, 2, 1: companion set sizes that make a call with `target` take that RW (None if no single companion size
    of up to 16,384 rows, repeated at most four times, does)."""
    out = {}
    for rw in (1, 2, 4):
        for k in range(0, 5):
            hit = [n for n in ([0] if k == 0 else range(2, 16385)) if sm_rows_per_warp([target] + [n] * k, sms) == rw]
            if hit:
                out[rw] = [hit[0]] * k
                break
    return out


@pytest.mark.gpu
def test_every_rows_per_warp():
    """RW = 4, 2 and 1 each reached (the rule restated in engine_rules, the launched kernel read back), the same set's
    iterates bit for bit the same under each, and a group whose largest set sizes the grid while the small sets' CTAs leave
    early."""
    from gpu_models import sm_count
    sms = sm_count()
    target = make_set(8200, 1025, "3dmatch", 0.3)
    comp = _compositions(1025, sms)
    assert sorted(comp) == [1, 2, 4], ("a composition for every RW at this SM count", sms, comp)
    ref = None
    seen = set()
    for rw, companions in sorted(comp.items()):
        sets = [target] + [make_set(8300 + i, n, "3dmatch", 0.3) for i, n in enumerate(companions)]
        _, _, its, off, got = check_call(sets, 0.10, ("RW", rw))
        assert got == rw
        seen.add(got)
        mine = its[:, :off[1]]
        if ref is None:
            ref = mine
        assert np.array_equal(mine.view(np.uint32), ref.view(np.uint32)), ("iterates depend on RW", rw)
    assert seen == {1, 2, 4}
    # the grid sized by a 16,384-row set; every other set's CTAs past its last row return at once
    sets = [make_set(8400, 16384, "3dmatch", 0.2), make_set(8401, 2, "3dmatch", 1.0), make_set(8402, 33, "3dmatch", 0.3),
            target, make_set(8403, 513, "3dmatch", 0.6)]
    _, _, its, off, rw = check_call(sets, 0.10, ("early exit",))
    assert np.array_equal(its[:, off[3]:off[4]].view(np.uint32), ref.view(np.uint32))
    for b in (1, 2, 4):
        _, _, its1, _, _ = run([sets[b]], 0.10)
        assert np.array_equal(its[:, off[b]:off[b + 1]].view(np.uint32), its1.view(np.uint32)), b
    print(f"RW reached {sorted(seen)} at {sms} SMs (companions {comp}); {WORST}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [100, 1000, 5000, 16384])
def test_labels_where_float64_decides(n):
    """S tight inliers among N = 10 S rows: the final step's bound decides the selection, and the device's is float64's."""
    key = "labels decided by float64"
    before = WORST.get(key, 0)
    check_call([make_gap_set(8500 + n, n)], 0.10, ("gap",))
    assert WORST.get(key, 0) == before + 1, ("the float64 label comparison did not run", n)
    print(f"gap N={n}: {WORST}")


@pytest.mark.gpu
def test_every_iterate_slot_is_written():
    """Through the C ABI on guarded buffers prefilled with each of buffer_guards.PATTERNS: all ten rows of every set written,
    nothing outside them, and the same bytes whatever the buffers held."""
    import ctypes as C

    from buffer_guards import PATTERNS, guarded_output, scratch_buffer
    from pointdsc_b200 import _capi
    sets = [make_set(8600 + i, n, "3dmatch", 0.3) for i, n in enumerate((5, 700, 33, 2048, 513))]
    _, _, its, off, _ = run(sets, 0.10)
    lib, eng = _capi.load(), _capi.utility_engine(0)
    B, R = len(sets), off[-1]
    cat = lambda i: torch.from_numpy(np.ascontiguousarray(np.concatenate([x[i] for x in sets]))).cuda()   # noqa: E731
    corr, src, tgt = cat(0), cat(1), cat(2)
    d_off = torch.tensor(off, dtype=torch.int32, device="cuda")
    h_off = (C.c_int32 * len(off))(*off)
    need = int(lib.pdsc_spectral_matching_packed_scratch_bytes(B, h_off))
    P = C.c_void_p
    dev = torch.device("cuda")
    for pattern in PATTERNS:
        trans, labels = guarded_output(64 * B, 16, dev, pattern), guarded_output(4 * R, 4, dev, pattern)
        it = guarded_output(4 * ITERS * R, 4, dev, pattern)
        scratch = scratch_buffer(need, 16, pattern)
        rc = lib.pdsc_spectral_matching_packed_iterates(eng, B, h_off, P(d_off.data_ptr()), P(corr.data_ptr()), P(src.data_ptr()),
                                                        P(tgt.data_ptr()), 0.10, P(trans.ptr), P(labels.ptr), None, P(it.ptr),
                                                        P(scratch.ptr), need, P(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, lib.pdsc_last_error().decode()
        torch.cuda.synchronize()
        for name, g in (("trans", trans), ("labels", labels), ("iterates", it), ("scratch", scratch)):
            g.check((name, pattern))
        got = it.inner.cpu().numpy().view(np.float32).reshape(ITERS, R)
        assert np.array_equal(got.view(np.uint32), its.view(np.uint32)), (pattern, "an iterate slot kept the buffer's fill")
