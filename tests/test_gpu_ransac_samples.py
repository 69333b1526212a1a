"""Device RANSAC (csrc/ransac.cu) on every hypothesis it scores, against the float64 checks of tests/ransac_samples.py that need no
unique rotation: rank-deficient samples (repeated draws, collinear or coincident points, H = 0) and small candidate sets, where
such samples win most often.  Each family runs as one packed group and every set again alone, bit for bit alike (hyp_trans
included).  The worst error / bound of each check is printed at the end of every test."""
import numpy as np
import pytest
import torch

from oracle import ransac_oracle as O
from ransac_samples import (DEGENERATE, NEAR_RATIOS, check_set, collinear_set, duplicate_sets, exact_motion,
                            near_collinear_triple, point_sets, report, small_m_sets)

pytestmark = pytest.mark.gpu

KEYS = ["trans", "fitness", "inlier_rmse", "best_iteration", "status", "hyp_good", "hyp_rmse", "hyp_trans"]


def run(sets, r, max_iteration, seed=O.DEFAULT_SEED):
    """ransac_packed of the sets as one group; returns (numpy outputs, offsets)."""
    from pointdsc_b200.ransac import ransac_packed
    off = np.cumsum([0] + [len(s) for s, _, _ in sets]).tolist()
    d = lambda i: torch.from_numpy(np.ascontiguousarray(np.concatenate([x[i] for x in sets]))).cuda()   # noqa: E731
    trans, lab, info = ransac_packed(d(0), d(1), d(2), off, max_correspondence_distance=r, max_iteration=max_iteration,
                                     seed=seed, info=True, hypotheses=True)
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in info.items()}
    out.update(trans=trans.cpu().numpy(), labels=lab.cpu().numpy())
    return out, off


def _same(a, b):
    return np.array_equal(np.atleast_1d(a).view(np.uint8), np.atleast_1d(b).view(np.uint8))


def run_family(sets, r, max_iteration=1000, seed=O.DEFAULT_SEED):
    """The group, each set alone (bit for bit), and check_set on every set.  Returns the check_set results."""
    dev, off = run(sets, r, max_iteration, seed)
    res = []
    for b, st in enumerate(sets):
        alone, _ = run([st], r, max_iteration, seed)
        for k in KEYS:
            assert _same(dev[k][b], alone[k][0]), (b, k)
        assert _same(dev["labels"][off[b]:off[b + 1]], alone["labels"]), b
        res.append(check_set(dev, b, *st, r, max_iteration=max_iteration, seed=seed, rows=slice(off[b], off[b + 1])))
    print("worst error / bound:", report())
    return res


def degenerate_winner(res):
    return res["best"] >= 0 and not res["ratio"][res["best"]] > DEGENERATE


# ---------------------------------------------------------------------------------------------------
# small candidate sets
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [3, 4, 5, 6, 8, 12, 16, 32])
def test_small_m(M):
    degenerate = 0
    for preset, r in (("3dmatch", 0.10), ("kitti", 0.6)):
        sets = small_m_sets(M, preset)
        assert len(sets) >= 12 and all(int((lab > 0).sum()) == M for _, _, lab in sets)
        res = run_family(sets, r)
        degenerate += sum(degenerate_winner(x) for x in res)
    print(f"M = {M}: {degenerate} of 24 winners are degenerate")
    if M <= 8:
        assert degenerate > 0, "the family holds no degenerate winner"


# ---------------------------------------------------------------------------------------------------
# duplicate rows
# ---------------------------------------------------------------------------------------------------
def matched_without_mutual(seed=4):
    """pdsc_match with mutual = False on a synthetic pair whose 60 source descriptors are noisy copies of 15 target descriptors:
    every target row is the match of about four sources."""
    from pointdsc_b200.frontend import match
    g = np.random.default_rng(seed)
    td = g.standard_normal((15, 32))
    sd = td[np.arange(60) % 15] + 0.05 * g.standard_normal((60, 32))
    td /= np.linalg.norm(td, axis=1, keepdims=True)
    sd /= np.linalg.norm(sd, axis=1, keepdims=True)
    sk = (g.random((60, 3)) * 2.0).astype(np.float32)
    tk = exact_motion((g.random((15, 3)) * 2.0).astype(np.float32), 2)
    c = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()          # noqa: E731
    m = match(c(sd.astype(np.float32)), c(td.astype(np.float32)), c(sk), c(tk), use_mutual=False)
    s, t = m["src_keypts"][0].cpu().numpy(), m["tgt_keypts"][0].cpu().numpy()
    assert len(s) == 60 and len(np.unique(t, axis=0)) < 30
    return s, t, np.ones(len(s), np.float32)


@pytest.mark.parametrize("r", [0.10, 0.6])
def test_duplicate_rows(r):
    sets = list(duplicate_sets().values()) + [matched_without_mutual()]
    res = run_family(sets, r, max_iteration=2000)
    assert any((x["ratio"] <= DEGENERATE).any() for x in res)


# ---------------------------------------------------------------------------------------------------
# geometry: collinear, near-collinear, coincident
# ---------------------------------------------------------------------------------------------------
def test_geometry():
    sets = [collinear_set(o) for o in (0.0, 1e2, 1e4)] + [collinear_set(0.0, axis=0), collinear_set(1e2, axis=2)]
    sets += [near_collinear_triple(x) for x in NEAR_RATIOS]
    sets += list(point_sets().values())
    res = run_family(sets, 0.10, max_iteration=600)
    # the M = 3 triples draw every ordered triple, single-index ones (H = 0: R = I, t exact; checked by check_set) included
    for x in res[5:9]:
        d = x["draws"]
        assert ((d[:, 0] == d[:, 1]) & (d[:, 1] == d[:, 2])).any()
        assert (np.sort(d, 1) == [0, 1, 2]).all(1).any()
    # the near-collinear triples' full samples straddle the rank threshold sqrt(3.2e-30) = 1.8e-15 as built
    ratios = [float(x["ratio"][(np.sort(x["draws"], 1) == [0, 1, 2]).all(1)][0]) for x in res[5:9]]
    assert ratios[2] > 1.8e-14 and ratios[3] < 1.8e-15, ratios


# ---------------------------------------------------------------------------------------------------
# kernel edges: candidate tiles (kRansacTile = 256) and hypothesis chunks (kRansacChunk = 128)
# ---------------------------------------------------------------------------------------------------
def _mixed(Ms, seed=0):
    from pointdsc_b200.synth import make_pair
    sets = []
    for k, M in enumerate(Ms):
        pr = make_pair(seed + k, max(M, 1) + 3, "3dmatch", 0.5)
        s, t = pr["src_keypts"].numpy(), pr["tgt_keypts"].numpy()
        lab = np.zeros(len(s), np.float32)
        lab[:M] = 1.0
        sets.append((s, t, lab))
    return sets


def test_tile_edges():
    run_family(_mixed([255, 2, 256, 0, 257, 511, 1, 512, 513]), 0.10, max_iteration=300)


@pytest.mark.parametrize("max_iteration", [127, 128, 129, 255, 256, 257])
def test_chunk_edges(max_iteration):
    run_family(_mixed([40, 2, 300, 3]), 0.10, max_iteration=max_iteration)


# ---------------------------------------------------------------------------------------------------
# non-finite values
# ---------------------------------------------------------------------------------------------------
def test_non_finite_coordinates():
    from pointdsc_b200.synth import make_pair
    I, M = 30, 200
    seen = set(O.draws(O.DEFAULT_SEED, I, M).reshape(-1).tolist())
    drawn = sorted(seen)[:4]
    never = [k for k in range(M) if k not in seen][:4]
    sets = []
    for k, (rows, bad) in enumerate([(drawn, np.nan), (drawn, np.inf), (never, np.nan), (never, -np.inf)]):
        pr = make_pair(40 + k, M, "3dmatch", 0.6)
        s, t = pr["src_keypts"].numpy().copy(), pr["tgt_keypts"].numpy().copy()
        s[rows[0], 1] = bad
        t[rows[1], 2] = bad
        sets.append((s, t, np.ones(M, np.float32)))
    res = run_family(sets, 0.10, max_iteration=I)
    assert all(x["best"] >= 0 for x in res)


def test_label_values():
    """Rows labelled NaN, -0.0, +0.0, -inf are not candidates, rows labelled +inf and the smallest subnormal are.  The rows that are
    not candidates are exact copies of inlier correspondences, so counting one of them would change a key and the labels."""
    from pointdsc_b200.synth import make_pair
    pr = make_pair(7, 40, "3dmatch", 0.7)
    s, t = pr["src_keypts"].numpy(), pr["tgt_keypts"].numpy()
    special = np.float32([np.nan, -0.0, 0.0, -np.inf, np.inf, np.float32(1e-45)])
    assert special[5] > 0 and special[5] == np.float32(2.0 ** -149)
    copies = np.arange(len(special)) % 20
    s2, t2 = np.concatenate([s, s[copies]]), np.concatenate([t, t[copies]])
    lab = np.concatenate([np.ones(40, np.float32), special])
    lab[30:40] = np.where(np.arange(30, 40) % 2, -1.0, 0.5).astype(np.float32)
    sets = [(s2, t2, lab)]
    res = run_family(sets, 0.10, max_iteration=500)
    assert res[0]["M"] == 40 + 2 - 5


# ---------------------------------------------------------------------------------------------------
# pdsc_ransac_packed_hypotheses: the C entry point that adds hyp_trans to pdsc_ransac_packed
# ---------------------------------------------------------------------------------------------------
OUTS = [("trans", 4, lambda B, R, I: B * 16), ("labels", 4, lambda B, R, I: R), ("fitness", 8, lambda B, R, I: B),
        ("inlier_rmse", 8, lambda B, R, I: B), ("best_iteration", 4, lambda B, R, I: B), ("status", 4, lambda B, R, I: B),
        ("hyp_good", 4, lambda B, R, I: B * I), ("hyp_rmse", 8, lambda B, R, I: B * I), ("hyp_trans", 8, lambda B, R, I: B * I * 12)]


def _abi_group():
    return small_m_sets(4, "3dmatch", count=3) + [near_collinear_triple(1e-13)] + list(point_sets().values()) + _mixed([2, 300])


def _prepared(sets):
    """The group's device inputs, made once; returns call(fn, outs, scratch, nbytes, max_iteration, stream) -> status, which only
    launches (outs and scratch: device pointers as ints, tensors or None), so it can also be captured in a graph."""
    import ctypes as C
    from pointdsc_b200 import _capi
    lib, eng = _capi.load(), _capi.utility_engine(0)
    off = np.cumsum([0] + [len(s) for s, _, _ in sets]).tolist()
    cat = lambda i: torch.from_numpy(np.ascontiguousarray(np.concatenate([x[i] for x in sets]))).cuda()   # noqa: E731
    src, tgt, lab = cat(0), cat(1), cat(2)
    d_off = torch.tensor(off, dtype=torch.int32, device="cuda")
    h_off = (C.c_int32 * len(off))(*off)
    P = lambda x: None if x is None else C.c_void_p(x if isinstance(x, int) else x.data_ptr())           # noqa: E731

    def call(fn, outs, scratch, nbytes, max_iteration, stream=None):
        st = (stream or torch.cuda.current_stream()).cuda_stream
        return getattr(lib, fn)(eng, len(off) - 1, h_off, P(d_off), P(src), P(tgt), P(lab), 0.10, int(max_iteration),
                                C.c_uint64(O.DEFAULT_SEED), *[P(o) for o in outs], P(scratch), nbytes, C.c_void_p(st))
    torch.cuda.synchronize()
    return call


def _need(sets, I):
    import ctypes as C
    from pointdsc_b200 import _capi
    off = np.cumsum([0] + [len(s) for s, _, _ in sets]).tolist()
    return int(_capi.load().pdsc_ransac_packed_scratch_bytes(len(sets), (C.c_int32 * len(off))(*off), I))


def test_hypotheses_entry_point_memory_contract():
    """Every output of pdsc_ransac_packed_hypotheses, hyp_trans included, is written exactly within its bounds and equals the
    Python call's, whatever the buffers held; pdsc_ransac_packed writes the same bytes for the outputs it has."""
    from buffer_guards import PATTERNS, guarded_output, scratch_buffer
    sets, I = _abi_group(), 300
    B, R, need = len(sets), sum(len(s) for s, _, _ in sets), _need(sets, I)
    ref, _ = run(sets, 0.10, I)
    call = _prepared(sets)
    for pattern in PATTERNS:
        for fn, specs in (("pdsc_ransac_packed_hypotheses", OUTS), ("pdsc_ransac_packed", OUTS[:-1])):
            outs = [guarded_output(size * n(B, R, I), size, torch.device("cuda"), pattern) for _, size, n in specs]
            scratch = scratch_buffer(need, 16, pattern)
            assert call(fn, [g.ptr for g in outs], scratch.ptr, need, I) == 0, fn
            torch.cuda.synchronize()
            scratch.check((fn, "scratch", pattern))
            for (name, _, _), g in zip(specs, outs):
                g.check((fn, name, pattern))
                want = np.ascontiguousarray(ref[name]).view(np.uint8).reshape(-1)
                assert np.array_equal(g.inner.cpu().numpy(), want), (fn, name, pattern)


def test_hypotheses_entry_point_graph_and_errors():
    from pointdsc_b200 import _capi
    fn = "pdsc_ransac_packed_hypotheses"
    sets, I = _abi_group(), 129
    B, R, need = len(sets), sum(len(s) for s, _, _ in sets), _need(sets, I)
    scratch = _capi.scratch(need, torch.device("cuda"), 16)
    call = _prepared(sets)

    def outs():
        return [torch.empty(n(B, R, I) * size, dtype=torch.uint8, device="cuda") for _, size, n in OUTS]
    eager = outs()
    assert call(fn, eager, scratch, need, I) == 0
    graphed = outs()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            assert call(fn, graphed, scratch, need, I, stream=s) == 0
    torch.cuda.current_stream().wait_stream(s)
    for x in graphed:
        x.fill_(0xAB)
    g.replay()
    torch.cuda.synchronize()
    for (name, _, _), a, b in zip(OUTS, eager, graphed):
        assert torch.equal(a, b), name
    # errors: the checks of pdsc_ransac_packed, reported under this entry point's name
    lib = _capi.load()
    few = [eager[0], eager[1]] + [None] * 7
    assert call(fn, few, scratch, need, I) == 0
    assert call(fn, [None] + few[1:], scratch, need, I) == 1
    assert fn in lib.pdsc_last_error().decode()
    assert call(fn, few, scratch, need - 1, I) == 5
    assert call(fn, few, scratch, need, 0) == 1
    torch.cuda.synchronize()
