"""Groups of pairs of different sizes in one call each: matching (pdsc_match_packed through `frontend.match_many`), the
evaluation statistics (pdsc_eval_stats_packed through `metrics.eval_stats_packed`), the forward of already-packed rows
(`PointDSC.forward_packed`) and the grouped loop of evaluate.py that chains them.

Contract: a pair's (set's) results in a packed call are bit for bit those of the single-pair (uniform) entry point on that
pair alone, whatever else is in the call and whichever column chunking the call's size selects.  Matching's float64 checks
(test_gpu_front_end.py) therefore carry over from the single-pair path; here a packed call is compared with it.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from test_gpu_front_end import check_network_input, keypoints, match_descriptors, match_plan, run_match, stats_case
from test_gpu_memory_contract import (FLOAT_WORD, PATTERNS, assert_same, guarded_input, guarded_output, run_guarded,
                                      scratch_buffer, tiled)
from test_gpu_mixed_batch import as_batch, get_model, synth_sets
from test_gpu_stages import sm_count

pytestmark = pytest.mark.gpu

MATCH_CASES = [("fp32", 32), ("fp64", 33)]      # FCGF, FPFH
MATCH_MAX_CHUNKS = 32
# (Ns, Nt) per pair: one row / one column, sizes off the 128-row and 64 / 32-column tiles, Ns > Nt and Nt > Ns
GROUP = [(1, 1), (130, 70), (70, 130), (1, 300), (300, 1), (1000, 999), (257, 2000), (63, 65)]


def packed_plan(rows, cols, D, fp64, sms):
    """(row CTAs, chunks, grid.y) of one nearest_columns launch of a packed call (frontend.cu): pair p owns the row tiles
    [tile0(p), tile0(p+1)), tile0(p) = (offset_p + 127 p) // 128; the chunk count comes from the call's row CTAs as
    match_plan computes it for one pair; a pair's columns per chunk are whole tiles, and grid.y is the most chunks any pair
    fills."""
    tt = 32 if fp64 else 64
    tiles = (sum(rows) + 127 * len(rows)) // 128
    chunks = min(max(-(-4 * sms // tiles), 1), MATCH_MAX_CHUNKS)
    grid_y = 1
    for c in cols:
        per = -(-(-(-c // chunks)) // tt) * tt
        grid_y = max(grid_y, -(-c // per))
    return tiles, chunks, grid_y


def make_group(rng, shapes, D, dtype, dyadic=False):
    """Per pair (sd, td, sk, tk): sources near random targets with exact copies (match_descriptors), plus exact duplicate
    targets on either side of a column-tile boundary and duplicate sources on either side of a row-tile boundary."""
    tt = 32 if dtype == np.float64 else 64
    out = []
    for ns, nt in shapes:
        sd, td = match_descriptors(rng, ns, nt, D, dtype)
        if nt > tt:
            td[tt] = td[tt - 1]
            if ns > 5:
                sd[5] = td[tt - 1]                   # the clear nearest of both copies: the first one must win
        if ns > 128:
            sd[128] = sd[127]
        if dyadic:
            sk = (rng.integers(-2 ** 19, 2 ** 19, (ns, 3)) * 2.0 ** -10).astype(np.float32)
            tk = (rng.integers(-2 ** 19, 2 ** 19, (nt, 3)) * 2.0 ** -10).astype(np.float32)
        else:
            sk, tk = keypoints(rng, ns), keypoints(rng, nt)
        out.append((sd, td, sk, tk))
    return out


def run_many(group, mutual):
    from pointdsc_b200.frontend import match_many
    d = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()      # noqa: E731
    out = match_many([tuple(d(x) for x in g) for g in group], use_mutual=mutual)
    assert out["d_offsets"].dtype == torch.int32 and out["d_offsets"].cpu().tolist() == out["offsets"]
    return {"corr": out["corr"].cpu().numpy(), "corr_pos": out["corr_pos"].cpu().numpy(), "src": out["src_keypts"].cpu().numpy(),
            "tgt": out["tgt_keypts"].cpu().numpy(), "offsets": out["offsets"]}


def compare_with_single(group, mutual, exact=False):
    """Packed matching against `match` on each pair alone: every output bit for bit, per-pair counts equal; corr_pos also
    passes the candidate-mean check; a second run is bit-identical.  Returns the packed output."""
    got = run_many(group, mutual)
    off = got["offsets"]
    assert len(off) == len(group) + 1 and off[0] == 0
    if not mutual:
        assert off == list(np.cumsum([0] + [len(g[0]) for g in group]))
    for p, (sd, td, sk, tk) in enumerate(group):
        one = run_match(sd, td, sk, tk, mutual)
        a, b = off[p], off[p + 1]
        assert b - a == len(one["corr"]), (p, b - a, len(one["corr"]))
        sl = {k: got[k][a:b] for k in ("corr", "corr_pos", "src", "tgt")}
        for k in sl:
            assert np.array_equal(sl[k], one[k]), (p, k)
        assert (sl["corr"][:, 1] < len(td)).all() and (sl["corr"][:, 0] < len(sd)).all()
        check_network_input(sl, sk, tk, exact)
    again = run_many(group, mutual)
    for k in ("corr", "corr_pos", "src", "tgt"):
        assert np.array_equal(again[k], got[k]), k
    return got


# ---------------------------------------------------------------------------------------------------
# 1-3. matching
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,D", MATCH_CASES)
@pytest.mark.parametrize("mutual", [False, True], ids=["plain", "mutual"])
def test_packed_match_equals_single_pairs(dtype, D, mutual):
    fp64 = dtype == "fp64"
    rng = np.random.default_rng(11 * D + mutual)
    group = make_group(rng, GROUP, D, np.float64 if fp64 else np.float32)
    got = compare_with_single(group, mutual)
    if mutual:
        assert got["offsets"][-1] < sum(len(g[0]) for g in group)
    # the duplicate targets straddling a column tile: source 5 of the pairs that have them takes the first copy (the
    # first of all exact copies of that descriptor: match_descriptors plants more)
    tt = 32 if fp64 else 64
    for p, (sd, td, _, _) in enumerate(group):
        if len(td) > tt and len(sd) > 5 and not mutual:
            first = int(np.flatnonzero((td == td[tt - 1]).all(1))[0])
            assert got["corr"][got["offsets"][p] + 5, 1] == first, p


@pytest.mark.parametrize("dtype,D", MATCH_CASES)
def test_packed_match_centring_exact_on_a_dyadic_grid(dtype, D):
    rng = np.random.default_rng(5 + D)
    group = make_group(rng, GROUP, D, np.float64 if dtype == "fp64" else np.float32, dyadic=True)
    for mutual in (False, True):
        compare_with_single(group, mutual, exact=True)


@pytest.mark.parametrize("mutual", [False, True], ids=["plain", "mutual"])
def test_pairs_are_isolated(mutual):
    """Exact copies of pair p's sources planted among pair p + 1's targets are never chosen by pair p (its own targets are
    only near its sources, the copies would be exact), and the mutual check keeps no cross-pair match."""
    rng = np.random.default_rng(3 + mutual)
    D = 32
    group = make_group(rng, [(300, 200), (250, 400), (129, 65)], D, np.float32)
    for p in range(len(group) - 1):
        sd, _, _, _ = group[p]
        _, td_next, _, _ = group[p + 1]
        k = min(len(sd), len(td_next)) // 2
        td_next[:k] = sd[:k]                           # pair p + 1's targets hold exact copies of pair p's sources
    got = compare_with_single(group, mutual)
    off = got["offsets"]
    for p, (sd, td, _, _) in enumerate(group):
        corr = got["corr"][off[p]:off[p + 1]]
        assert (corr[:, 1] < len(td)).all()
        if p + 1 < len(group):
            # a cross-pair match would be exact: apart from the sources with an exact copy among the pair's own targets,
            # every distance pair p sees is its own and none is zero
            own = (sd[:, None, :] == td[None, :, :]).all(-1).any(1)
            c = corr[~own[corr[:, 0]]]
            d = 2 - 2 * np.einsum("ij,ij->i", sd[c[:, 0]].astype(np.float64), td[c[:, 1]].astype(np.float64))
            assert len(c) > 0 and (d > 1e-4).all(), p


def plan_groups(sms):
    """Groups whose packed plan reaches one chunk, several and the chunk cap, each with a pair whose own plan differs."""
    many = max(1, -(-4 * sms // 67)) + 1                 # pairs of 8500 rows (67 tiles each): at least 4 x SM row CTAs
    return {"1": [(8500, 700 + 37 * i) for i in range(many)] + [(200, 3000)],
            "mid": [(1000, 999), (1003, 1500), (2000, 700), (130, 4000)],
            "max": [(100, 3000), (1, 5000), (33, 2049)]}


@pytest.mark.parametrize("mutual", [False, True], ids=["plain", "mutual"])
def test_plan_does_not_change_indices(mutual):
    sms = sm_count()
    rng = np.random.default_rng(17 + mutual)
    kinds, differs = set(), 0
    for want, shapes in plan_groups(sms).items():
        rows, cols = [s for s, _ in shapes], [t for _, t in shapes]
        tiles, chunks, grid_y = packed_plan(rows, cols, 32, False, sms)
        kind = "1" if chunks == 1 else ("max" if chunks == MATCH_MAX_CHUNKS else "mid")
        assert kind == want, (want, chunks)
        kinds.add(kind)
        differs += sum(match_plan(s, t, 32, False, sms)[0] != chunks for s, t in shapes)
        group = make_group(rng, shapes, 32, np.float32)
        got = run_many(group, mutual)
        for p, (sd, td, sk, tk) in enumerate(group):
            one = run_match(sd, td, sk, tk, mutual)
            assert np.array_equal(got["corr"][got["offsets"][p]:got["offsets"][p + 1]], one["corr"]), (want, p)
        print(f"plan {want}: {tiles} row CTAs, {chunks} chunks, grid.y {grid_y}")
    assert kinds == {"1", "mid", "max"}, kinds
    assert differs >= 3


# ---------------------------------------------------------------------------------------------------
# 4. statistics
# ---------------------------------------------------------------------------------------------------
def test_packed_stats_equal_per_set_stats():
    from pointdsc_b200.metrics import eval_stats, eval_stats_packed
    rng = np.random.default_rng(21)
    sizes = [1, 255, 256, 257, 1000, 3, 5000, 2]
    sets = [stats_case(rng, 1, n) for n in sizes]
    cat = lambda i, shape: torch.from_numpy(np.concatenate([s[i].reshape(shape) for s in sets])).cuda()   # noqa: E731
    off = [0] + list(np.cumsum(sizes))
    got = eval_stats_packed(cat(0, (-1, 4, 4)), cat(1, (-1, 4, 4)), cat(2, (-1, 3)), cat(3, (-1, 3)), cat(4, (-1,)),
                            cat(5, (-1,)), off, re_thre=15.0, te_thre=30.0)
    assert got.shape == (len(sizes), 10)
    for b, s in enumerate(sets):
        one = eval_stats(*(torch.from_numpy(a).cuda() for a in s), re_thre=15.0, te_thre=30.0)
        assert torch.equal(got[b], one[0]), (sizes[b], got[b], one[0])


# ---------------------------------------------------------------------------------------------------
# 5. forward of packed rows
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp16x3", "fp32"])
def test_forward_packed_equals_forward_many(precision):
    m = get_model("3dmatch", precision)
    sizes = [41, 1000, 2, 257, 130]
    pairs = synth_sets(sizes, seed0=300)
    many = m.forward_many([as_batch([p]) for p in pairs])
    cat = lambda k: torch.cat([p[k] for p in pairs]).cuda()      # noqa: E731
    off = [0] + list(np.cumsum(sizes))
    res = m.forward_packed(cat("corr_pos"), cat("src_keypts"), cat("tgt_keypts"), off)
    assert res["final_trans"].shape == (len(sizes), 4, 4) and res["final_labels"].shape == (off[-1],)
    for b, o in enumerate(many):
        assert torch.equal(res["final_trans"][b], o["final_trans"][0]), b
        assert torch.equal(res["final_labels"][off[b]:off[b + 1]], o["final_labels"][0]), b


# ---------------------------------------------------------------------------------------------------
# 6. memory contract of pdsc_match_packed (the pattern of test_gpu_memory_contract.py)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fp64", [False, True], ids=["fp32", "fp64"])
def test_match_packed_poison_guards_and_rows_past_the_end(fp64):
    """Scratch at exactly 8 B and pdsc_match_packed_scratch_bytes, poisoned; outputs prefilled; identical results under every
    poison; no guard byte changed; rows at or beyond out_offsets[P] keep the prefill byte for byte."""
    from pointdsc_b200 import _capi
    lib = _capi.load()
    dev = torch.device("cuda")
    e = _capi.utility_engine(0)
    D = 33 if fp64 else 32
    dt = np.float64 if fp64 else np.float32
    rng = np.random.default_rng(40 + fp64)
    group = make_group(rng, [(300, 200), (1, 1), (129, 700), (64, 3)], D, dt)
    so = np.cumsum([0] + [len(g[0]) for g in group]).astype(np.int32)
    to = np.cumsum([0] + [len(g[1]) for g in group]).astype(np.int32)
    P, ns = len(group), int(so[-1])
    ins = {"sd": guarded_input(np.concatenate([g[0] for g in group]), dev), "td": guarded_input(np.concatenate([g[1] for g in group]), dev),
           "sk": guarded_input(np.concatenate([g[2] for g in group]), dev), "tk": guarded_input(np.concatenate([g[3] for g in group]), dev),
           "so": guarded_input(so, dev), "to": guarded_input(to, dev)}
    h_so, h_to = (C.c_int32 * (P + 1))(*so.tolist()), (C.c_int32 * (P + 1))(*to.tolist())
    need = int(lib.pdsc_match_packed_scratch_bytes(P, h_so, h_to))
    assert need == int(lib.pdsc_match_scratch_bytes(ns, int(to[-1])))
    for mutual in (0, 1):
        ref = None
        for pat in PATTERNS:
            outs = {"corr": guarded_output(ns * 8, 4, dev, pat), "offsets": guarded_output((P + 1) * 4, 4, dev, pat),
                    "corr_pos": guarded_output(ns * 24, 4, dev, pat), "src": guarded_output(ns * 12, 4, dev, pat),
                    "tgt": guarded_output(ns * 12, 4, dev, pat)}
            sc = scratch_buffer(need, 8, pat)
            Pp = lambda g: C.c_void_p(g.ptr)     # noqa: E731
            got = run_guarded((mutual, pat), outs, sc, ins, lambda: lib.pdsc_match_packed(
                e, P, D, h_so, h_to, Pp(ins["so"]), Pp(ins["to"]), Pp(ins["sd"]), Pp(ins["td"]), int(fp64), Pp(ins["sk"]),
                Pp(ins["tk"]), mutual, Pp(outs["corr"]), Pp(outs["offsets"]), Pp(outs["corr_pos"]), Pp(outs["src"]),
                Pp(outs["tgt"]), Pp(sc), need, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
            off = got["offsets"].view(torch.int32).cpu().tolist()
            assert off[0] == 0 and all(a < b for a, b in zip(off, off[1:])) and off[-1] <= ns, off
            assert mutual or off == so.tolist()
            M = off[-1]
            for name, row in (("corr", 8), ("corr_pos", 24), ("src", 12), ("tgt", 12)):
                tail = got[name][M * row:]
                assert torch.equal(tail, tiled(FLOAT_WORD[pat], tail.numel(), dev)), (name, "row >= out_offsets[P] written", pat)
                got[name] = got[name][:M * row]
            if ref is None:
                ref = got
            else:
                assert_same(ref, got, ("match_packed", mutual, pat))


# ---------------------------------------------------------------------------------------------------
# 7. loud errors
# ---------------------------------------------------------------------------------------------------
def test_errors_are_loud():
    from pointdsc_b200 import _capi
    from pointdsc_b200.frontend import match, match_many
    from pointdsc_b200.metrics import eval_stats_packed
    rng = np.random.default_rng(8)
    d = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()      # noqa: E731
    g32 = [tuple(d(x) for x in g) for g in make_group(rng, [(50, 40), (30, 60)], 32, np.float32)]
    g64 = [tuple(d(x) for x in g) for g in make_group(rng, [(50, 40)], 32, np.float64)]
    with pytest.raises(ValueError):                                    # mixed dtypes: as match raises for one pair
        match_many([g32[0], g64[0]])
    with pytest.raises(ValueError):
        match(g32[0][0], g64[0][1], g32[0][2], g64[0][3])
    wide = [tuple(d(x) for x in g) for g in make_group(rng, [(20, 20)], 65, np.float32)]
    with pytest.raises(_capi.PdscError):                               # D > 64
        match_many(wide)
    with pytest.raises(_capi.PdscError):
        match(*wide[0])
    empty = (g32[1][0][:0], g32[1][1], g32[1][2][:0], g32[1][3])
    with pytest.raises(_capi.PdscError):                               # an empty pair
        match_many([g32[0], empty])
    with pytest.raises(_capi.PdscError):
        match(*empty)
    # non-increasing offsets through the C ABI
    lib = _capi.load()
    e = _capi.utility_engine(0)
    sd, td = torch.cat([g[0] for g in g32]), torch.cat([g[1] for g in g32])
    sk, tk = torch.cat([g[2] for g in g32]), torch.cat([g[3] for g in g32])
    outs = [torch.empty(80, k, dtype=dt, device="cuda") for k, dt in ((2, torch.int32), (6, torch.float32), (3, torch.float32),
                                                                      (3, torch.float32))]
    d_out = torch.empty(3, dtype=torch.int32, device="cuda")
    sc = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    for so, to in (([0, 50, 50], [0, 40, 100]), ([0, 50, 80], [0, 40, 40]), ([1, 50, 80], [0, 40, 100]),
                   ([0, 60, 50], [0, 40, 100])):
        h_so, h_to = (C.c_int32 * 3)(*so), (C.c_int32 * 3)(*to)
        d_so = torch.tensor(so + to, dtype=torch.int32, device="cuda")
        assert lib.pdsc_match_packed_scratch_bytes(2, h_so, h_to) == 0
        rc = lib.pdsc_match_packed(e, 2, 32, h_so, h_to, C.c_void_p(d_so.data_ptr()), C.c_void_p(d_so.data_ptr() + 12),
                                   C.c_void_p(sd.data_ptr()), C.c_void_p(td.data_ptr()), 0, C.c_void_p(sk.data_ptr()),
                                   C.c_void_p(tk.data_ptr()), 0, C.c_void_p(outs[0].data_ptr()), C.c_void_p(d_out.data_ptr()),
                                   C.c_void_p(outs[1].data_ptr()), C.c_void_p(outs[2].data_ptr()), C.c_void_p(outs[3].data_ptr()),
                                   C.c_void_p(sc.data_ptr()), sc.numel(), None)
        assert rc == _capi.PDSC_ERR_SHAPE, (so, to, rc)
    trans = torch.eye(4, device="cuda").expand(2, 4, 4).contiguous()
    with pytest.raises(_capi.PdscError):                               # an empty set of the statistics
        eval_stats_packed(trans, trans, sk[:50], sk[:50], sk[:50, 0], sk[:50, 0], [0, 50, 50])
    # a pair keeping fewer than two correspondences reaches the forward: the error the single-pair path raises
    m = get_model("3dmatch", "fp16x3")
    one = tuple(d(x) for x in make_group(rng, [(1, 30)], 32, np.float32)[0])
    packed = match_many([g32[0], one])
    assert packed["offsets"][-1] - packed["offsets"][-2] == 1
    with pytest.raises(_capi.PdscError):
        m.forward_packed(packed["corr_pos"], packed["src_keypts"], packed["tgt_keypts"], packed["offsets"])
    single = match(*one)
    with pytest.raises(_capi.PdscError):
        m({"corr_pos": single["corr_pos"], "src_keypts": single["src_keypts"], "tgt_keypts": single["tgt_keypts"], "testing": True})


# ---------------------------------------------------------------------------------------------------
# 8. evaluate.py: the packed group loop against the single-pair loop
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mutual", [False, True], ids=["plain", "mutual"])
def test_evaluate_packed_groups_equal_single_pairs(mutual):
    import evaluate
    extra = ["--use_mutual"] if mutual else []
    s1, _ = evaluate.main(["--synthetic", "4", "--batch_size", "1"] + extra)
    s4, _ = evaluate.main(["--synthetic", "4", "--batch_size", "4"] + extra)
    assert s1.shape == s4.shape == (4, len(evaluate.COLUMNS))
    # fixed by matching and labels alone
    assert np.array_equal(s1[:, 3], s4[:, 3]) and np.array_equal(s1[:, 4], s4[:, 4])
    assert np.array_equal(s1[:, 0], s4[:, 0])
    assert np.array_equal(s1[:, 11], s4[:, 11])
    # the rest: test_evaluate_groups_equal_single_pairs' tolerances (the two calls may run different attention regimes)
    ok = s1[:, 0] == 1
    assert np.abs(s1[ok, 1] - s4[ok, 1]).max(initial=0) < 1e-2 and np.abs(s1[ok, 2] - s4[ok, 2]).max(initial=0) < 0.1
    assert np.abs(s1[:, 6] - s4[:, 6]).max() < 1e-2 and np.abs(s1[:, 7] - s4[:, 7]).max() < 1e-2
    assert (s4[:, 9] > 0).all() and (s4[:, 10] >= 0).all()
