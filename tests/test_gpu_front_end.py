"""The front-end rows against float64, on every launch path they take: descriptor matching (csrc/frontend.cu through
`frontend.match`), the N x N power iteration (csrc/eig_power.cu through `spectral.leading_eigenvector`), the evaluation
statistics (csrc/eval_stats.cu through `metrics.eval_stats`) and the FPFH neighbour search, normals and voxel grid
(csrc/fpfh.cu through `descriptors.*`).  The GPU tests are marked one by one (`-m gpu`, an H100); the tests of section 5
check this file's own float64 helpers and bounds on the CPU.

Several kernels choose a launch path from the shapes, the pointer or the SM count: the matcher's column-chunk count and
its fp64 shared-memory opt-in, the compaction's passes, the power iteration's rows per CTA R, its bulk-copy path and its
tile ring, the search's bitonic size P.  Every test recomputes the kernel's choice (engine_rules.py: `match_plan`,
`eig_plan`, `search_plan`) and asserts that it reached the path it targets.

Error model (float64_bounds.py's, u = 2^-24 for fp32 and 2^-53 for fp64, gamma(n) = n u / (1 - n u)):
  * inputs are exact in float64; every reference below is float64 on the kernel's own fp32 / fp64 inputs;
  * a sum of n terms in any order, fma or not, is within gamma(n) sum |terms| of the exact sum;
  * sqrt, division and a single add / multiply add one rounding (u relative) each; CUDA's acosf adds 2 ulp.
Each tolerance is derived beside its assertion from these rules, and the worst measured error / tolerance ratio on an
H100 is recorded next to its constant.
"""
import math

import numpy as np
import pytest
import torch

from buffer_guards import (RE_THRE, TE_THRE, check_network_input, keypoints, match_descriptors, mean_candidates, run_match,
                           stats_case, surface)
from engine_rules import CAND_CAP, EIG_COLS, EIG_ROWS, MATCH_MAX_CHUNKS, eig_plan, match_plan, search_plan
from float64_bounds import U, U64, check_power, gamma, gamma64
from gpu_models import sm_count
from oracle import fpfh_oracle as F
from oracle import frontend_oracle as FO
from oracle import metrics_oracle as MO

GOLDEN_FRONT = ["frontend_fcgf32_n300_m0", "frontend_fcgf32_n300_m1", "frontend_fpfh33_n500_m0", "frontend_fpfh33_n500_m1",
                "frontend_ties_n64_m0"]


def golden(name):
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name + ".npz"))


# ---------------------------------------------------------------------------------------------------
# 1. matching
# ---------------------------------------------------------------------------------------------------
# The kernel forms y = fl(fl(2 - 2 dot) + fl_T(1e-6)) in the descriptors' type T and compares fl(sqrt(y)) with a strict '<'.
# Bound (`match_err`) on |y - x|, x = 2 - 2 a.b + 1e-6 in exact arithmetic: the ascending-channel FMA chain is within
# gamma(D) S, S = sum |a_i b_i|, doubled by 2 dot (exact); the subtraction and the add round once each (2.01 u (x + 2 gamma S));
# fl_T(1e-6) is within u 1e-6 of 1e-6; the float64 reference x carries the same terms at 2^-53.  The square root merges
# values within an ulp: the kernel may return column j only if sqrt(y_j) (1 - u) <= sqrt(y_min) (1 + u), i.e.
#   x_j - e_j <= (x_min + e_min) (1 + 4.01 u)                         (`nearest64`: the allowed columns)
# Columns holding bit-identical descriptors have bit-identical distances (one FMA chain in the same order), so where every
# allowed column is a copy of one descriptor the kernel must return the lowest of them.
# Measured on an H100 (80GB HBM3, 700 W): worst (x_chosen - x_min) / E = 0.022 (fp32, D = 15), 0.013 (fp64, D = 39); the
# index is determined for 97-100 % of the rows.
MATCH_PAIRS = [(1, 1), (1, 5000), (5000, 1), (2, 63), (63, 2), (64, 65), (65, 64), (127, 128), (128, 129), (129, 127),
               (1023, 1025), (1025, 1024), (1024, 1023), (2, 5000), (5000, 64), (5000, 5000), (129, 4091)]
MATCH_D = [("fp32", d) for d in (1, 15, 16, 17, 32, 48, 64)] + [("fp64", d) for d in (1, 17, 33, 38, 39, 64)]


def match_err(x, S, D, fp64):
    u, g = (U64, gamma64(D)) if fp64 else (U, gamma(D))
    return 2 * g * S + 2.01 * u * (x + 2 * g * S) + u * 1e-6 + 2 * gamma64(D) * S + 2.01 * U64 * x


def nearest64(a, b, fp64, probe=None):
    """For every row of a, the columns of b the kernel may return: (want = the lowest allowed column, sure = every allowed
    column holds one descriptor, single = one allowed column, ok [len(probe)] = whether each probe (row, col) is allowed,
    worst (x_col - x_min) / (E of the col) over the probes)."""
    uT = U64 if fp64 else U
    D = a.shape[1]
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    gid = np.unique(b, axis=0, return_inverse=True)[1].reshape(-1)
    want = np.empty(len(a), np.int64)
    sure = np.empty(len(a), bool)
    single = np.empty(len(a), bool)
    pr, pc = probe if probe is not None else (np.zeros(0, np.int64), np.zeros(0, np.int64))
    ok = np.zeros(len(pr), bool)
    worst = 0.0
    for r0 in range(0, len(a), 512):
        blk = slice(r0, r0 + 512)
        x = 2.0 - 2.0 * (a64[blk] @ b64.T) + 1e-6
        e = match_err(x, np.abs(a64[blk]) @ np.abs(b64).T, D, fp64)
        r = np.arange(len(x))
        m = x.argmin(1)
        lim = (x[r, m] + e[r, m]) * (1 + 4.01 * uT)
        allowed = x - e <= lim[:, None]
        want[blk] = allowed.argmax(1)
        gmax = np.where(allowed, gid[None, :], -1).max(1)
        gmin = np.where(allowed, gid[None, :], len(b)).min(1)
        sure[blk] = gmin == gmax
        single[blk] = allowed.sum(1) == 1
        sel = (pr >= r0) & (pr < r0 + len(x))
        if sel.any():
            rr, cc = pr[sel] - r0, pc[sel]
            ok[sel] = allowed[rr, cc]
            E = e[rr, cc] + e[rr, m[rr]] + 4.01 * uT * (x[rr, m[rr]] + e[rr, m[rr]])
            worst = max(worst, float(((x[rr, cc] - x[rr, m[rr]]) / E).max()))
    return want, sure, single, ok, worst


def check_match(sd, td, sk, tk, outs, exact_mean=False):
    """outs: {mutual: kernel output}.  Returns (rows whose index is determined, rows, worst ratio)."""
    fp64 = sd.dtype == np.float64
    ns = len(sd)
    rows_probe = [np.arange(ns), outs[False]["corr"][:, 1]] if False in outs else [np.zeros(0, np.int64)] * 2
    if True in outs:
        kept = outs[True]["corr"]
        rows_probe = [np.concatenate([rows_probe[0], kept[:, 0]]), np.concatenate([rows_probe[1], kept[:, 1]])]
    want_r, sure_r, single_r, ok_r, worst = nearest64(sd, td, fp64, rows_probe)
    assert ok_r.all(), np.flatnonzero(~ok_r)[:8]
    if False in outs:
        corr = outs[False]["corr"]
        assert np.array_equal(corr[:, 0], np.arange(ns))
        assert np.array_equal(corr[sure_r, 1], want_r[sure_r]), np.flatnonzero(corr[:, 1] != want_r)[:8]
    if True in outs:
        kept = outs[True]["corr"]
        assert np.all(np.diff(kept[:, 0]) > 0)                     # ascending source order
        want_c, sure_c, _, ok_c, w2 = nearest64(td, sd, fp64, (kept[:, 1], kept[:, 0]))
        assert ok_c.all()
        worst = max(worst, w2)
        det = sure_r & sure_c[want_r]                               # both argmins determined
        expect = want_c[want_r] == np.arange(ns)
        is_kept = np.zeros(ns, bool)
        is_kept[kept[:, 0]] = True
        assert np.array_equal(is_kept[det], expect[det]), np.flatnonzero(det & (is_kept != expect))[:8]
        ks = sure_r[kept[:, 0]]
        assert np.array_equal(kept[ks, 1], want_r[kept[ks, 0]])
    for out in outs.values():
        check_network_input(out, sk, tk, exact_mean)
    return int(sure_r.sum()), ns, worst


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,D", MATCH_D)
def test_match_sweep_against_float64(dtype, D):
    fp64 = dtype == "fp64"
    sms = sm_count()
    rng = np.random.default_rng(100 * D + fp64)
    kinds, partial, smem_seen, sep, rows, worst = set(), False, set(), 0, 0, 0.0
    for ns, nt in MATCH_PAIRS:
        sd, td = match_descriptors(rng, ns, nt, D, np.float64 if fp64 else np.float32)
        sk, tk = keypoints(rng, ns), keypoints(rng, nt)
        outs = {mutual: run_match(sd, td, sk, tk, mutual) for mutual in (False, True)}
        s, r, w = check_match(sd, td, sk, tk, outs)
        sep, rows, worst = sep + s, rows + r, max(worst, w)
        for rr, cc in ((ns, nt), (nt, ns)):                         # the mutual check's swapped launch has rows = Nt
            chunks, per, smem = match_plan(rr, cc, D, fp64, sms)
            kinds.add("1" if chunks == 1 else ("max" if chunks == MATCH_MAX_CHUNKS else "mid"))
            partial |= chunks > 1 and cc % per != 0 and cc % (32 if fp64 else 64) != 0
            smem_seen.add(smem)
    assert kinds == {"1", "mid", "max"}, kinds                     # one chunk, several, capped at kMatchMaxChunks
    assert partial                                                  # a partial last chunk ending in a partial tile
    assert all((s > 48 * 1024) == (fp64 and D >= 39) for s in smem_seen)    # the dynamic shared-memory opt-in from fp64 D = 39
    assert sep >= 0.8 * rows, (sep, rows)                           # most rows have one admissible descriptor
    print(f"match {dtype} D={D}: determined {sep}/{rows}, worst (x_chosen - x_min) / E = {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["fp32", "fp64"])
def test_match_exact_ties_across_tiles_and_chunks(dtype):
    """Exact duplicate targets in one tile, in two tiles of one chunk and in two chunks (and three copies spread over all
    three), each the clear nearest of ten sources: every source must take the lowest copy.  Exact duplicate sources in
    one tile and in two column chunks of the swapped launch: only the lowest is kept by the mutual check."""
    fp64 = dtype == "fp64"
    dt = np.float64 if fp64 else np.float32
    tt, D = (32, 39) if fp64 else (64, 32)
    ns, nt = 300, 3000
    sms = sm_count()
    chunks, per, _ = match_plan(ns, nt, D, fp64, sms)
    chunks_sw, per_sw, _ = match_plan(nt, ns, D, fp64, sms)
    assert chunks > 1 and chunks_sw > 1 and per >= tt + 8
    groups = [(per + 3, per + 8), (2 * per + 1, 2 * per + tt + 2), (5, 7 * per + 11),
              (3 * per + 2, 3 * per + tt + 4, (chunks - 1) * per + 6)]
    assert all(p < nt for g in groups for p in g)
    assert groups[0][0] // tt == groups[0][1] // tt                              # one tile
    assert groups[1][0] // per == groups[1][1] // per and groups[1][0] // tt != groups[1][1] // tt
    assert groups[2][0] // per != groups[2][1] // per                            # two chunks
    src_copies = [(2, 250), (3, 7)]
    assert 2 // per_sw != 250 // per_sw and 3 // (tt) == 7 // tt
    rng = np.random.default_rng(7 + fp64)
    unit = lambda f: f / np.linalg.norm(f, axis=-1, keepdims=True)      # noqa: E731
    td = unit(rng.standard_normal((nt, D)))
    sd = unit(rng.standard_normal((ns, D)))
    centres = unit(rng.standard_normal((len(groups), D)))
    members = {}
    for k, g in enumerate(groups):
        td[list(g)] = centres[k]
        members[k] = np.arange(20 + 10 * k, 30 + 10 * k)
        sd[members[k]] = unit(centres[k] + 0.05 * rng.standard_normal((10, D)))
    for k, (i, j) in enumerate(src_copies):
        sd[[i, j]] = centres[k]
    td, sd = td.astype(dt), sd.astype(dt)
    sk, tk = keypoints(rng, ns), keypoints(rng, nt)
    outs = {mutual: run_match(sd, td, sk, tk, mutual) for mutual in (False, True)}
    check_match(sd, td, sk, tk, outs)
    want_r, sure_r, _, _, _ = nearest64(sd, td, fp64)
    chosen = outs[False]["corr"][:, 1]
    for k, g in enumerate(groups):
        assert sure_r[members[k]].all() and (want_r[members[k]] == min(g)).all()
        assert (chosen[members[k]] == min(g)).all(), (k, g, chosen[members[k]])
    kept = set(outs[True]["corr"][:, 0].tolist())
    for i, j in src_copies:
        assert i in kept and j not in kept, (i, j)
    print(f"ties {dtype}: {chunks} chunks of {per} columns, swapped launch {chunks_sw} chunks of {per_sw}")


@pytest.mark.gpu
@pytest.mark.parametrize("grid", [False, True], ids=["uniform", "dyadic"])
def test_match_network_input_across_compaction_passes(grid):
    """Ns = 5000: compact_center_kernel's 1024-thread loop runs five passes, the kept rows are spread over them (mutual: a
    sparse subset), and corr_pos is fl32(v - mean) with the fp64 mean rounded to fp32; on a dyadic grid the fp64 sums
    are exact, and so is every corr_pos entry."""
    rng = np.random.default_rng(31 + grid)
    ns, nt, D = 5000, 4000, 32
    sd, td = match_descriptors(rng, ns, nt, D, np.float32)
    if grid:
        sk = (rng.integers(-2 ** 19, 2 ** 19, (ns, 3)) * 2.0 ** -10).astype(np.float32)
        tk = (rng.integers(-2 ** 19, 2 ** 19, (nt, 3)) * 2.0 ** -10).astype(np.float32)
    else:
        sk, tk = keypoints(rng, ns), keypoints(rng, nt)
    outs = {mutual: run_match(sd, td, sk, tk, mutual) for mutual in (False, True)}
    check_match(sd, td, sk, tk, outs, exact_mean=grid)
    for mutual, out in outs.items():
        blocks = np.unique(out["corr"][:, 0] // 1024)
        assert len(out["corr"]) > 1024 and len(blocks) == 5, (mutual, len(out["corr"]), blocks)
    assert 1024 < len(outs[True]["corr"]) < ns


# ---------------------------------------------------------------------------------------------------
# 2. the N x N power iteration
# ---------------------------------------------------------------------------------------------------
# One step on the kernel's own iterate v_t (non-negative M and v): each u_j is an fp32 sum of N products, within
# gamma(N) w_j of w = M64 v_t; the norm sums N rounded squares of those (3 gamma(N + 1) relative), the square root halves
# that and adds u, the add of fl(1e-6) and the division add u each, the float64 reference 4 gamma64(N):
#   |v_t+1 - normalise(w)| <= (1.01 (gamma(N) + 1.5 gamma(N + 1) + 4 u) + 4 gamma64(N)) normalise(w)     per entry.
# The whole run at the cap goes through float64_bounds.check_power with k = N (its Hilbert-metric bound and exit rule).
# Measured on an H100 (80GB HBM3, 700 W): worst one-step error / bound = 0.13 (1.5e-4 at N = 24576); whole run / check_power's
# bound 0.011.


def eig_cases(sms):
    """(B, N, misaligned, matrix) covering every R regime, both copy paths and the ring's parity."""
    k_mid = max(2, 2 * round(sms / 32))             # N = 512 k + 4: R ~ 16, k + 1 tiles (odd)
    k_32 = 2 * ((128 * sms - 64) // 1024)           # N = 512 k + 4 just under 4 SMs x 32 rows: R clamped from ~63
    b_w = -(-4 * sms // (1536 // EIG_ROWS))         # B sets of N = 1536 fill >= 4 CTAs per SM: R = 32, three tiles
    return [(1, 1, False, "rand"), (1, 2, False, "rand"), (1, 3, True, "rand"), (2, 4, False, "rand"), (2, 4, True, "rand"),
            (1, 512, False, "rand"), (3, 516, False, "rand"), (1, 516, True, "spectral"), (2, 1003, False, "spectral"),
            (1, 1024, True, "rand"), (1, 512 * k_mid + 4, False, "spectral"), (1, 3072, True, "rand"),
            (1, 512 * k_32 + 4, False, "rand"), (b_w, 1536, False, "rand"), (b_w, 1536, True, "rand")]


def eig_matrix(kind, B, N, seed):
    if kind == "spectral":                            # test_gpu_next_rows.test_leading_eigenvector_spectral_matching_matrix's
        from pointdsc_b200.synth import make_pair
        ms = []
        for b in range(B):
            p = make_pair(seed + b, N, "3dmatch", 0.3)
            ds = torch.cdist(p["src_keypts"], p["src_keypts"]) - torch.cdist(p["tgt_keypts"], p["tgt_keypts"])
            m = torch.clamp(4.5 - ds ** 2 / 2 / (0.1 / 3) ** 2, min=0)
            m.fill_diagonal_(0)
            ms.append(m)
        return torch.stack(ms).float().cuda()
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(B, N, N, device="cuda", generator=g).add_(0.5).clamp_(0, 1)


def misalign(M):
    """The same matrix 4 bytes past a 16-byte boundary, contiguous."""
    B, N, _ = M.shape
    out = torch.empty(B * N * N + 1, device="cuda")[1:].view(B, N, N)
    out.copy_(M)
    assert out.is_contiguous() and out.data_ptr() % 16 == 4
    return out


def eig_step64(M, v):
    """normalise(M64 v) per set in float64 on the device, 2048 rows at a time."""
    B, N, _ = M.shape
    v64 = v.double()[:, :, None]
    w = torch.empty(B, N, dtype=torch.float64, device=M.device)
    for r0 in range(0, N, 2048):
        w[:, r0:r0 + 2048] = torch.bmm(M[:, r0:r0 + 2048].double(), v64)[:, :, 0]
    return w / (w.norm(dim=1, keepdim=True) + 1e-6)


def eig_step_tol(N, ref):
    return (1.01 * (gamma(N) + 1.5 * gamma(N + 1) + 4 * U) + 4 * gamma64(N)) * ref


def eig_one_step(M, t):
    """v_t+1 of the kernel against normalise(M64 v_t) on its own v_t; returns the worst error / bound."""
    from pointdsc_b200.spectral import leading_eigenvector
    B, N, _ = M.shape
    vt, it = leading_eigenvector(M, t, early_exit=False)
    vt1, it1 = leading_eigenvector(M, t + 1, early_exit=False)
    assert (it == t).all() and (it1 == t + 1).all()
    ref = eig_step64(M, vt)
    err = (vt1.double() - ref).abs()
    tol = eig_step_tol(N, ref)
    assert bool((err <= tol).all()), (N, t, float(err.max()), float((err / (tol + 1e-300)).max()))
    return float((err / tol.clamp_min(1e-300)).max())


@pytest.mark.gpu
def test_leading_eigenvector_every_launch_path():
    from pointdsc_b200.spectral import leading_eigenvector
    sms = sm_count()
    seen, worst, worst_run, exits = set(), 0.0, 0.0, 0
    for i, (B, N, mis, kind) in enumerate(eig_cases(sms)):
        M = eig_matrix(kind, B, N, 500 + i)
        if mis:
            M = misalign(M)
        plan = eig_plan(B, N, M.data_ptr(), sms)
        seen |= {plan["regime"], ("tma" if plan["tma"] else "plain") + ("-misaligned" if mis and N % 4 == 0 else "")}
        if plan["last_rows"] < plan["R"]:
            seen.add("partial-cta")
        seen.add("ntiles=" + ("1" if plan["ntiles"] == 1 else "2" if plan["ntiles"] == 2 else
                              "odd" if plan["ntiles"] % 2 else "even"))
        seen.add("N%512==0" if N % 512 == 0 else ("N%512==4" if N % 512 == 4 else ""))
        for t in (1, 4):
            worst = max(worst, eig_one_step(M, t))
        if N <= 4200:                                # the whole run at the cap on the host (float64 M)
            v, it = leading_eigenvector(M, 10, early_exit=True)
            M64 = M.double().cpu().numpy()
            v, it = v.cpu().numpy(), it.cpu().numpy()
            for b in range(B):
                r, _, sure = check_power(M64[b][None], v[b][None], it[b], N, 10)
                worst_run, exits = max(worst_run, r), exits + int(sure)
        del M
        torch.cuda.empty_cache()
    need = {"clamp8", "mid", "clamp32", "waves", "tma", "plain", "plain-misaligned", "partial-cta", "ntiles=1", "ntiles=2",
            "ntiles=odd", "N%512==0", "N%512==4"}
    assert need <= seen, need - seen
    assert exits >= 5
    print(f"eig paths {sorted(seen - {''})}: worst one-step error / bound {worst:.3g}, whole run / bound {worst_run:.3g}, "
          f"{exits} exits compared")


@pytest.mark.gpu
def test_leading_eigenvector_largest_n():
    """N = 24576, the largest N whose vector fits in shared memory beside the ring (R = 32, many waves): two steps on the
    kernel's own iterates; N = 24577 is rejected before any launch."""
    from pointdsc_b200 import PdscError
    from pointdsc_b200.spectral import leading_eigenvector
    N = 24576
    M = eig_matrix("rand", 1, N, 77)
    plan = eig_plan(1, N, M.data_ptr(), sm_count())
    assert plan["regime"] == "waves" and plan["tma"] and plan["ntiles"] == 48
    assert 2 * 32 * EIG_COLS * 4 + 64 + N * 4 <= 227 * 1024
    worst = max(eig_one_step(M, 1), eig_one_step(M, 2))
    del M
    torch.cuda.empty_cache()
    with pytest.raises(PdscError, match="24577"):
        leading_eigenvector(torch.empty(1, N + 1, N + 1, device="cuda"), 1)
    print(f"eig N={N}: worst one-step error / bound {worst:.3g}")


@pytest.mark.gpu
def test_leading_eigenvector_per_set_exit():
    """One batch: a rank-one M (exits at iteration 2) beside a block matrix with lambda2 / lambda1 = 0.99 (runs to the cap).
    iters_run is per set and equals the exit recomputed from the kernel's own iterates wherever every allclose decision
    up to it is outside the fp32 comparison's rounding band (|d| u + 3 u (1e-8 + 1e-5 |v|)); the converged set is frozen
    bit for bit at its exit while the other keeps iterating, and the other equals the early_exit=False run."""
    from pointdsc_b200.spectral import leading_eigenvector
    N, cap = 1000, 10
    rng = np.random.default_rng(3)
    a = rng.uniform(0.5, 1.0, N)
    rank1 = np.outer(a, a)
    block = np.zeros((N, N))
    n1 = 400
    block[:n1, :n1] = 1.0 / n1
    block[n1:, n1:] = 0.99 / (N - n1)
    block += 1e-7 * rng.uniform(0, 1, (N, N))
    M = torch.from_numpy(np.stack([rank1, block]).astype(np.float32)).cuda()
    its = [np.ones((2, N), np.float32)]
    for t in range(1, cap + 1):
        v, it = leading_eigenvector(M, t, early_exit=False)
        assert (it.cpu().numpy() == t).all()                  # no latch without early_exit
        its.append(v.cpu().numpy())
    exit_own = []
    for b in range(2):
        ex, sure = cap, True
        for t in range(1, cap + 1):
            vn, vo = its[t][b].astype(np.float64), its[t - 1][b].astype(np.float64)
            d = np.abs(vn - vo)
            margin = d - (1e-8 + 1e-5 * np.abs(vo))
            band = U * d + 3 * U * (1e-8 + 1e-5 * np.abs(vo))
            sure &= bool((margin < -band).all() or (margin > band).any())
            if (margin <= 0).all():
                ex = t
                break
        assert sure, b
        exit_own.append(ex)
    v, it = leading_eigenvector(M, cap, early_exit=True)
    v, it = v.cpu().numpy(), it.cpu().numpy()
    assert it.tolist() == exit_own and exit_own[0] == 2 and exit_own[1] == cap, (it, exit_own)
    capped, _ = leading_eigenvector(M, exit_own[0], early_exit=True)     # same B and N: the same R
    assert np.array_equal(v[0], capped.cpu().numpy()[0]) and np.array_equal(v[0], its[exit_own[0]][0])
    assert np.array_equal(v[1], its[cap][1])
    for b in range(2):
        check_power(M.double().cpu().numpy()[b][None], v[b][None], it[b], N, cap)


# ---------------------------------------------------------------------------------------------------
# 3. evaluation statistics
# ---------------------------------------------------------------------------------------------------
# RE: the trace of R^T R_gt is 3 fp32 dots of 3 and two adds, within gamma(5) S (S = sum |T_ij G_ij|); (tr - 1) rounds
# once, / 2 is exact, the clamp is 1-Lipschitz: dc.  acos moves by at most dc / sqrt(1 - m^2), m = |c| + dc, and never by
# more than acos(1 - dc) (its steepest interval ends at +-1); acosf adds 2 ulp (4 u relative), * 180 and / pi_f (which is
# within u of pi) 3 u.  TE: the three differences round once each (u on the length), the sum of squares gamma(3) (halved by
# the root), the root and * 100 once each: 4.6 u TE.  RMSE: per point the warped coordinate is within gamma(4) A_c
# (A_c = sum_k |r_ck x_k| + |t_c|), the difference adds u |d_c|, the length gamma(3) / 2 + u; the fp64 sum gamma64(N + 1) and
# the final fp32 rounding u.  Counts and the ratios of exact fp32 integers are exact.
# Measured on an H100 (80GB HBM3, 700 W): worst RE / TE / RMSE error / bound = 0.49 / 0.62 / 0.22.
STATS_N = [1, 31, 255, 256, 257, 5000, 2 ** 20]


def stats64(pred, gt, src, tgt, pl, gl):
    """float64 columns [B,10] of fp32 inputs, bounds for RE / TE / RMSE, the exact fp32 values of the count / ratio columns
    and flags (clamp active, the three zero denominators)."""
    T, G = pred.astype(np.float64), gt.astype(np.float64)
    B, N = pl.shape
    prod = T[:, :3, :3] * G[:, :3, :3]
    tr, S = prod.sum((1, 2)), np.abs(prod).sum((1, 2))
    dtr = 1.01 * gamma(5) * S
    dc = (dtr + U * (np.abs(tr - 1) + dtr)) / 2
    c_raw = (tr - 1) / 2
    c = np.clip(c_raw, -1, 1)
    th = np.arccos(c)
    m = np.abs(c) + dc
    steep = np.where(m < 1, dc / np.sqrt(np.maximum(1 - m * m, 1e-300)), np.inf)
    rad = np.minimum(steep, np.arccos(1 - np.minimum(dc, 2)))
    deg = 180 / math.pi
    re, re_tol = th * deg, deg * (rad + 4 * U * (th + rad)) + 3.1 * U * deg * (th + rad)
    d = T[:, :3, 3] - G[:, :3, 3]
    te = 100 * np.sqrt((d * d).sum(1))
    te_tol = 4.6 * U * te
    x = src.astype(np.float64)
    w = np.einsum("bck,bnk->bnc", T[:, :3, :3], x) + T[:, None, :3, 3]
    A = np.einsum("bck,bnk->bnc", np.abs(T[:, :3, :3]), np.abs(x)) + np.abs(T[:, None, :3, 3])
    dd = w - tgt.astype(np.float64)
    dist = np.sqrt((dd * dd).sum(2))
    Ec = gamma(4) * A + U * (np.abs(dd) + gamma(4) * A)
    e = Ec.sum(2) + (gamma(3) / 2 + U) * (dist + Ec.sum(2))
    rmse = dist.mean(1)
    rmse_tol = e.mean(1) + U * (rmse + e.mean(1)) + gamma64(N + 1) * (dist + e).mean(1)
    p, g = pl > 0, gl > 0
    tp, fp, fn, gs = ((p & g).sum(1), (p & ~g).sum(1), (~p & g).sum(1), g.sum(1))
    f = np.float32
    exact = np.zeros((B, 10), np.float32)
    exact[:, 3], exact[:, 4], exact[:, 5] = gs, f(gs) / f(N), tp
    with np.errstate(invalid="ignore", divide="ignore"):
        exact[:, 6] = np.where(tp + fp > 0, f(tp) / f(tp + fp), 0)
        exact[:, 7] = np.where(tp + fn > 0, f(tp) / f(tp + fn), 0)
        exact[:, 8] = np.where(2 * tp + fp + fn > 0, f(2) * f(tp) / (f(2) * f(tp) + f(fp) + f(fn)), 0)
    return {"re": re, "re_tol": re_tol, "te": te, "te_tol": te_tol, "rmse": rmse, "rmse_tol": rmse_tol, "exact": exact,
            "clamp": (c_raw + dc < -1) | (c_raw - dc > 1), "den0": np.stack([tp + fp == 0, tp + fn == 0, 2 * tp + fp + fn == 0], 1)}


def check_stats(got, ref):
    """got [B,10] fp32 against stats64; returns the worst (RE, TE, RMSE) error / bound and the success flags compared."""
    assert np.array_equal(got[:, 3:9], ref["exact"][:, 3:9]), np.argwhere(got[:, 3:9] != ref["exact"][:, 3:9])[:8]
    out = []
    for col, key in ((1, "re"), (2, "te"), (9, "rmse")):
        err = np.abs(got[:, col].astype(np.float64) - ref[key])
        tol = ref[key + "_tol"]
        assert (err <= tol).all(), (key, np.flatnonzero(err > tol)[:8], float((err / np.maximum(tol, 1e-300)).max()))
        out.append(float(np.where(tol > 0, err / np.maximum(tol, 1e-300), 0).max()))
    far = (np.abs(ref["te"] - TE_THRE) > ref["te_tol"]) & (np.abs(ref["re"] - RE_THRE) > ref["re_tol"])
    want = ((ref["te"] < TE_THRE) & (ref["re"] < RE_THRE)).astype(np.float32)
    assert np.array_equal(got[far, 0], want[far])
    assert set(np.unique(got[:, 0]).tolist()) <= {0.0, 1.0}
    return out, int(far.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("n", STATS_N)
def test_eval_stats_against_float64(n):
    from pointdsc_b200.metrics import eval_stats
    B = 2000 if n <= 257 else (64 if n <= 5000 else 2)
    rng = np.random.default_rng(n)
    pred, gt, src, tgt, pl, gl = stats_case(rng, B, n)
    got = eval_stats(*(torch.from_numpy(a).cuda() for a in (pred, gt, src, tgt, pl, gl)), re_thre=RE_THRE,
                     te_thre=TE_THRE).cpu().numpy()
    ref = stats64(pred, gt, src, tgt, pl, gl)
    worst, compared = check_stats(got, ref)
    assert compared >= B // 2
    if B >= 8:
        assert got[0, 1] == 0.0 and got[0, 2] == 0.0 and got[0, 0] == 1.0           # pred == gt
        assert ref["clamp"][1] and abs(float(got[1, 1]) - 180.0) <= ref["re_tol"][1] and got[1, 0] == 0.0
        assert abs(float(got[1, 1]) - 180.0) <= 180.0 * 7 * U                        # clamped to -1: acosf(-1) * 180 / pi_f
        assert got[2, 2] == np.float32(TE_THRE) and got[2, 1] == 0.0 and got[2, 0] == 0.0     # TE == te_thre: not a success
        assert ref["den0"][3, 0] and ref["den0"][5, 1] and ref["den0"][6, 2]         # each zero denominator is reached
        assert (got[3, 6] == 0.0 and got[5, 7] == 0.0 and (got[6, 6:9] == 0.0).all())
    print(f"eval_stats N={n} B={B}: worst RE / TE / RMSE error / bound = {worst[0]:.3g} / {worst[1]:.3g} / {worst[2]:.3g}, "
          f"success compared {compared}/{B}")


# ---------------------------------------------------------------------------------------------------
# 4. FPFH search boundaries, normals, voxel grid
# ---------------------------------------------------------------------------------------------------
# Normals: both sides form the fp64 covariance of the same neighbours (sums of at most max_nn + 1 terms around a mean that
# itself carries gamma64(cnt) max |p|), so each entry is within 2 gamma64(cnt + 3) (max |p|^2 + w2); Davis-Kahan turns
# that into a normal within C_NORMAL (cnt + 3) u64 (max |p|^2 + w2) / gap, gap = w1 - w0 (C_NORMAL = 8 covers both
# covariances and both symmetric eigensolvers).  Compared where gap > 1e-3 w2.  FPFH: counts are exact, the oracle adds
# 100 / (cnt - 1) cnt times (the kernel multiplies once) and sums the parts in another order: within
# 4 (max_nn + 24) u64 (|f| + 100).  Measured on an H100 (80GB HBM3, 700 W): worst normal error / bound = 1.3e-5 (sweep),
# 2.7e-6 (lattice), 2.4e-5 (4096 candidates); worst FPFH error / bound = 0.015.
C_NORMAL = 8.0
SEARCH_MAX_NN = [1, 2, 31, 32, 33, 64, 65, 128, 129, 255, 256]


def check_normals(got, pts, radius, max_nn):
    """Normals against the oracle where the eigen-gap is healthy; returns (compared, worst error / bound)."""
    want = F.estimate_normals(pts, radius, max_nn)
    p = pts.astype(np.float64)
    pmax2 = float((p * p).sum(1).max())
    assert np.allclose(np.linalg.norm(got, axis=1), 1.0, atol=1e-12)
    compared, worst = 0, 0.0
    for i, (idx, _) in enumerate(F.hybrid_neighbours(pts, radius, max_nn)):
        if len(idx) < 3:
            assert np.array_equal(got[i], [0.0, 0.0, 1.0])
            continue
        w = np.linalg.eigvalsh(np.cov(p[idx].T, bias=True))
        if w[1] - w[0] <= 1e-3 * w[2]:
            continue
        tol = C_NORMAL * (len(idx) + 3) * U64 * (pmax2 + w[2]) / (w[1] - w[0])
        err = min(np.abs(got[i] - want[i]).max(), np.abs(got[i] + want[i]).max())
        assert err <= tol, (i, err, tol)
        compared, worst = compared + 1, max(worst, err / tol)
    return compared, worst


@pytest.mark.gpu
@pytest.mark.parametrize("max_nn", SEARCH_MAX_NN)
def test_normals_every_bitonic_size(max_nn):
    from pointdsc_b200.descriptors import estimate_normals
    m = 2003
    P, warps = search_plan(max_nn)
    assert m % 8 and m % warps and P >= max_nn and (P == 2 or P // 2 < max_nn)
    pts = surface(np.random.default_rng(max_nn), m)
    radius = math.sqrt(1.5 * max(max_nn, 4) / (math.pi * m))        # ~1.5 max_nn points inside: the cap cuts most
    got = estimate_normals(torch.from_numpy(pts).cuda(), radius, max_nn).cpu().numpy()
    compared, worst = check_normals(got, pts, radius, max_nn)
    if max_nn >= 31:
        assert compared >= m // 2
    print(f"normals max_nn={max_nn} (P={P}, {warps} warps/CTA): compared {compared}/{m}, worst error / bound {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("max_nn,shells", [(30, 5.5), (45, 5.5), (85, 8.5)])
def test_normals_tie_selection_on_a_lattice(max_nn, shells):
    """A dyadic 14^3 lattice in random index order: fp32 squared distances are exact, so max_nn cuts through a shell of
    equal distances (27 | 33, 33 | 57, 81 | 93 points inside) and the kernel must keep the lowest indices of that shell, as
    the oracle does; another subset changes the covariance.  A cluster of 60 exact duplicates (more than max_nn, nothing
    else in range) takes warp_select's all-keys-equal branch."""
    from pointdsc_b200.descriptors import estimate_normals
    rng = np.random.default_rng(max_nn)
    h = 0.25
    g = np.stack(np.meshgrid(*[np.arange(14)] * 3, indexing="ij"), -1).reshape(-1, 3) * h - 1.75
    pts = np.concatenate([g[rng.permutation(len(g))], np.full((60, 3), 10.0)]).astype(np.float32)
    order = rng.permutation(len(pts))
    pts = pts[order]
    cluster = np.flatnonzero(order >= len(g))
    radius = h * math.sqrt(shells)
    assert np.float32(radius * radius) == np.float32(shells * h * h)
    got = estimate_normals(torch.from_numpy(pts).cuda(), radius, max_nn).cpu().numpy()
    compared, worst = check_normals(got, pts, radius, max_nn)
    cut = 0
    p = pts.astype(np.float64)
    for i, (idx, d2) in enumerate(F.hybrid_neighbours(pts, radius, 10 ** 6)):
        if len(idx) > max_nn and d2[max_nn - 1] == d2[max_nn] and len(set(d2.tolist())) > 1:
            w = np.linalg.eigvalsh(np.cov(p[idx[:max_nn]].T, bias=True))
            cut += int(w[1] - w[0] > 1e-3 * w[2])
    assert cut >= 200, cut                                      # healthy points whose neighbourhood cuts a shell
    want = F.estimate_normals(pts, radius, max_nn)
    assert np.array_equal(got[cluster], want[cluster])
    print(f"lattice max_nn={max_nn}: {cut} shell cuts with a healthy gap, compared {compared}, worst error / bound {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("max_nn", [1, 2, 33, 129, 256])
def test_fpfh_every_bitonic_size(max_nn):
    from pointdsc_b200.descriptors import compute_fpfh, estimate_normals
    m = 1003
    P, warps = search_plan(max_nn)
    assert m % 8 and m % warps
    rng = np.random.default_rng(1000 + max_nn)
    pts = np.concatenate([surface(rng, m - 40), np.full((40, 3), 5.0, np.float32)])    # + 40 duplicates > 33
    kp = torch.from_numpy(pts).cuda()
    # independent continuous normals: points that share a neighbourhood get normals equal to within rounding, and the pair
    # feature's frame choice (acos |n1.d| > acos |n2.d|) between two such points is then decided by rounding on either side
    nrm = estimate_normals(kp, 0.08, 30) + 0.05 * torch.from_numpy(rng.standard_normal((m, 3))).cuda()
    nrm = nrm / nrm.norm(dim=1, keepdim=True)
    radius = math.sqrt(1.5 * max(max_nn, 4) / (math.pi * m))
    worst = 0.0
    raw = F.fpfh(pts, nrm.cpu().numpy(), radius, max_nn)
    for normalise in (False, True):
        got = compute_fpfh(kp, nrm, radius, max_nn, normalise=normalise).cpu().numpy()
        want = raw
        if normalise:
            want = want / (np.linalg.norm(want, axis=1, keepdims=True) + 1e-6)
        tol = 4 * (max_nn + 24) * U64 * (np.abs(want) + (1.0 if normalise else 100.0))
        err = np.abs(got - want)
        assert (err <= tol).all(), (normalise, np.argwhere(err > tol)[:4], float((err / tol).max()))
        worst = max(worst, float((err / tol).max()))
    assert (np.count_nonzero(want, axis=1) > 3).mean() > 0.5 or max_nn <= 2
    print(f"fpfh max_nn={max_nn} (P={P}): worst error / bound {worst:.3g}")


@pytest.mark.gpu
def test_search_candidate_cap_boundary():
    """4096 points all within the radius of each other: exactly the 4096 candidates a warp holds, accepted and equal to
    the oracle; one point more raises with status bit 2 (and only bit 2)."""
    from pointdsc_b200 import PdscError
    from pointdsc_b200.descriptors import _STATUS, estimate_normals
    rng = np.random.default_rng(4096)
    pts = rng.uniform(0, 0.01, (CAND_CAP + 1, 3)).astype(np.float32)
    got = estimate_normals(torch.from_numpy(pts[:CAND_CAP]).cuda(), 1.0, 30).cpu().numpy()
    compared, worst = check_normals(got, pts[:CAND_CAP], 1.0, 30)
    assert compared >= CAND_CAP // 2
    with pytest.raises(PdscError) as exc:
        estimate_normals(torch.from_numpy(pts).cuda(), 1.0, 30)
    assert str(exc.value) == _STATUS[2]
    print(f"candidate cap: compared {compared}, worst error / bound {worst:.3g}")


@pytest.mark.gpu
def test_voxel_boundaries_largest_index_and_table_step():
    from pointdsc_b200 import PdscError
    from pointdsc_b200.descriptors import _STATUS, voxel_down_sample
    vals = np.array([-1.0, -0.75, -0.5, -0.0, 0.0, 0.25, 0.5, 1.0], np.float32)
    g = np.stack(np.meshgrid(vals, vals, np.array([-0.0, 0.0, 0.5, 1.0], np.float32), indexing="ij"), -1).reshape(-1, 3)
    rng = np.random.default_rng(5)
    cases = [(g[rng.permutation(len(g))], 0.5), (rng.uniform(-3, 3, (512, 3)).astype(np.float32), 0.4),
             (rng.uniform(-3, 3, (513, 3)).astype(np.float32), 0.4),
             (np.array([[0, 0, 0], [2097151.0, 0, 0]], np.float32), 1.0)]
    for pts, voxel in cases:
        got = voxel_down_sample(torch.from_numpy(pts).cuda(), voxel).cpu().numpy()
        want, _ = F.voxel_down_sample(pts, voxel)
        assert got.shape == want.shape, (len(pts), got.shape, want.shape)
        # the fp64 sum / count of the oracle and the 2^-40-voxel fixed point of the kernel, both rounded to fp32 once
        assert np.abs(got.astype(np.float64) - want).max() <= np.spacing(np.float32(np.abs(want).max()))
    assert np.array_equal(got, [[0, 0, 0], [2097151.0, 0, 0]])                  # voxel index 2^21 - 1 accepted
    with pytest.raises(PdscError) as exc:
        voxel_down_sample(torch.tensor([[0, 0, 0], [2097151.5, 0, 0]], device="cuda"), 1.0)
    assert str(exc.value) == _STATUS[1]


# ---------------------------------------------------------------------------------------------------
# 5. the helpers themselves (CPU)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [1, 17, 64])
def test_match_bound_covers_numpy_fp32(D):
    """numpy's fp32 distance (BLAS order) lies within match_err of the float64 x, its argmin is an allowed column and
    equals `want` wherever nearest64 is sure; the fp64 distance lies within it of a long-double x."""
    rng = np.random.default_rng(D)
    sd, td = match_descriptors(rng, 300, 700, D, np.float32)
    x64 = 2.0 - 2.0 * (sd.astype(np.float64) @ td.astype(np.float64).T) + 1e-6
    S = np.abs(sd.astype(np.float64)) @ np.abs(td.astype(np.float64)).T
    x32 = (np.float32(2) - np.float32(2) * (sd @ td.T)) + np.float32(1e-6)
    assert (np.abs(x32 - x64) <= match_err(x64, S, D, False)).all()
    chosen = np.sqrt(x32).argmin(1)
    want, sure, single, ok, _ = nearest64(sd, td, False, (np.arange(300), chosen))
    assert ok.all() and np.array_equal(chosen[sure], want[sure]) and single.mean() > 0.6
    sd, td = match_descriptors(rng, 60, 80, D, np.float64)
    xl = 2 - 2 * (sd.astype(np.longdouble) @ td.astype(np.longdouble).T) + np.longdouble(1e-6)
    x = 2 - 2 * (sd @ td.T) + 1e-6
    Sl = np.abs(sd) @ np.abs(td).T
    assert (np.abs(x - xl).astype(np.float64) <= match_err(np.asarray(xl, np.float64), Sl, D, True)).all()


def test_match_plan_reaches_every_chunk_regime_on_an_h100():
    """The sweep's pairs reach one chunk, several and the cap in both dtypes on 132 SMs; the fp64 opt-in starts at D = 39."""
    for fp64 in (False, True):
        kinds = {match_plan(r, c, 32, fp64, 132)[0] for ns, nt in MATCH_PAIRS for r, c in ((ns, nt), (nt, ns))}
        assert 1 in kinds and MATCH_MAX_CHUNKS in kinds and any(1 < k < MATCH_MAX_CHUNKS for k in kinds)
    assert match_plan(1, 1, 38, True, 132)[2] <= 48 * 1024 < match_plan(1, 1, 39, True, 132)[2]
    assert match_plan(1, 1, 64, False, 132)[2] <= 48 * 1024
    regimes = {eig_plan(B, N, 4 if mis else 16, 132)["regime"] for B, N, mis, _ in eig_cases(132)}
    assert {"clamp8", "mid", "clamp32", "waves"} <= regimes
    assert [search_plan(n)[0] for n in SEARCH_MAX_NN] == [2, 2, 32, 32, 64, 64, 128, 128, 256, 256, 256]


@pytest.mark.parametrize("name", GOLDEN_FRONT)
def test_match_helpers_agree_with_frontend_oracle(name):
    """On the reference fixtures: the oracle's matches are allowed columns, equal to `want` where sure (the ties fixture:
    everywhere), its mutual subset equals the one determined by the two float64 argmins, and its corr_pos lies within
    one fp32 rounding of v - mean."""
    z = golden(name)
    sd, td, mutual = z["src_desc"], z["tgt_desc"], bool(z["use_mutual"])
    corr = FO.match(sd, td, mutual)
    assert np.array_equal(corr, z["corr"])
    fp64 = sd.dtype == np.float64
    want_r, sure_r, _, ok, _ = nearest64(sd, td, fp64, (corr[:, 0], corr[:, 1]))
    assert ok.all()
    assert np.array_equal(corr[sure_r[corr[:, 0]], 1], want_r[corr[sure_r[corr[:, 0]], 0]])
    if "ties" in name:
        assert sure_r.all()
    if mutual:
        want_c, sure_c, _, _, _ = nearest64(td, sd, fp64)
        det = sure_r & sure_c[want_r]
        kept = np.zeros(len(sd), bool)
        kept[corr[:, 0]] = True
        assert np.array_equal(kept[det], (want_c[want_r] == np.arange(len(sd)))[det])
    v = np.concatenate([z["src_keypts"][corr[:, 0]], z["tgt_keypts"][corr[:, 1]]], 1).astype(np.float64)
    ref = v - v.mean(0)
    # the reference's fp32 mean: gamma(M) mean |v| + u |mean|; its subtraction: u |v - m|
    tol = U * np.abs(ref) + 1.01 * (gamma(len(v)) * np.abs(v).mean(0) + U * np.abs(v.mean(0)))
    assert (np.abs(z["corr_pos"] - ref) <= tol).all()


def test_mean_candidates_reproduce_fp32_centring():
    """On dyadic inputs the single candidate is numpy's own fp32(fp64 mean); on general inputs the candidates bracket it."""
    rng = np.random.default_rng(2)
    v = (rng.integers(-2 ** 19, 2 ** 19, 3000) * 2.0 ** -10).astype(np.float32)
    (m,) = mean_candidates(v, True)
    assert m == np.float32(v.astype(np.float64).sum() / len(v))
    w = rng.uniform(-3, 3, 3000).astype(np.float32)
    assert np.float32(w.astype(np.float64).mean()) in mean_candidates(w, False)


def stats32_numpy(pred, gt, src, tgt):
    """numpy's fp32 RE, TE and the mean distance (fp64 accumulation), in an operation order other than the kernel's."""
    f = np.float32
    tr = np.zeros(len(pred), f)
    for j in range(3):
        tr = tr + ((pred[:, 0, j] * gt[:, 0, j] + pred[:, 1, j] * gt[:, 1, j]) + pred[:, 2, j] * gt[:, 2, j])
    c = np.clip((tr - f(1)) / f(2), f(-1), f(1))
    re = np.arccos(c) * f(180) / f(math.pi)
    d = pred[:, :3, 3] - gt[:, :3, 3]
    te = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]) * f(100)
    R, t = pred[:, :3, :3], pred[:, :3, 3]
    w = [((R[:, None, c, 0] * src[..., 0] + R[:, None, c, 1] * src[..., 1]) + R[:, None, c, 2] * src[..., 2]) + t[:, None, c]
         for c in range(3)]
    dd = [w[c] - tgt[..., c] for c in range(3)]
    dist = np.sqrt((dd[0] * dd[0] + dd[1] * dd[1]) + dd[2] * dd[2])
    return re, te, (dist.astype(np.float64).sum(1) / src.shape[1]).astype(f)


@pytest.mark.parametrize("n", [1, 31, 257])
def test_stats_bounds_cover_numpy_fp32(n):
    rng = np.random.default_rng(n)
    pred, gt, src, tgt, pl, gl = stats_case(rng, 300, n)
    ref = stats64(pred, gt, src, tgt, pl, gl)
    re, te, rmse = stats32_numpy(pred, gt, src, tgt)
    assert (np.abs(re - ref["re"]) <= ref["re_tol"]).all()
    assert (np.abs(te - ref["te"]) <= ref["te_tol"]).all()
    assert (np.abs(rmse - ref["rmse"]) <= ref["rmse_tol"]).all()
    assert ref["clamp"][1] and ref["te"][2] == TE_THRE and ref["re"][0] == 0.0
    assert ref["den0"][3, 0] and ref["den0"][5, 1] and ref["den0"][6, 2]
    far = (np.abs(ref["te"] - TE_THRE) > ref["te_tol"]) & (np.abs(ref["re"] - RE_THRE) > ref["re_tol"])
    assert far.mean() > 0.5


def test_stats_helpers_agree_with_metrics_oracle():
    """The reference's fixtures (its own fp32 module): counts and flags exact, the ratios within one fp32 rounding of the
    exact fp32 ones, RE / TE within stats64's bounds (RMSE: plus the fp32 mean's gamma(N))."""
    z = golden("metrics_cases")
    for i in range(int(z["num_cases"])):
        g = {k: z[f"c{i}_{k}"][None] for k in ("pred", "gt", "src", "tgt", "pred_labels", "gt_labels")}
        ref = stats64(g["pred"], g["gt"], g["src"], g["tgt"], g["pred_labels"], g["gt_labels"])
        thr = (15.0, 30.0) if str(z[f"c{i}_dataset"]) == "3dmatch" else (5.0, 60.0)
        row = np.asarray(MO.stats_row(*(torch.from_numpy(g[k][0]) for k in ("pred", "gt", "src", "tgt", "pred_labels",
                                                                            "gt_labels")), *thr), np.float64)
        assert np.array_equal(z[f"c{i}_row"][[0, 3, 5]], row[[0, 3, 5]])
        assert row[3] == ref["exact"][0, 3] and row[5] == ref["exact"][0, 5]
        assert (np.abs(row[[4, 6, 7, 8]] - ref["exact"][0, [4, 6, 7, 8]]) <= U * np.abs(row[[4, 6, 7, 8]])).all()
        assert abs(row[1] - ref["re"][0]) <= ref["re_tol"][0], i
        assert abs(row[2] - ref["te"][0]) <= ref["te_tol"][0], i
        n = g["src"].shape[1]
        assert abs(row[9] - ref["rmse"][0]) <= ref["rmse_tol"][0] + (gamma(n) + U) * ref["rmse"][0], i


def test_eig_step_bound_covers_numpy_fp32():
    """numpy's fp32 GEMV (BLAS order), sum of squares and normalisation lie within eig_step_tol of the float64 step."""
    rng = np.random.default_rng(0)
    for N in (3, 516, 1003):
        M = np.clip(rng.standard_normal((N, N)) + 0.5, 0, 1).astype(np.float32)
        v = rng.uniform(0, 1, N).astype(np.float32)
        u = M @ v
        nrm = np.sqrt((u * u).sum(dtype=np.float32)) + np.float32(1e-6)
        v32 = u / nrm
        w = M.astype(np.float64) @ v.astype(np.float64)
        ref = w / (np.linalg.norm(w) + 1e-6)
        assert (np.abs(v32 - ref) <= eig_step_tol(N, ref)).all()
