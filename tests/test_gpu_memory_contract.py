"""The memory contract of every entry point: no result depends on what the workspace, the scratch or the output buffers held
before the call, and no call writes outside them.

Every buffer a call gets is owned by the test (the C ABI, pointdsc_b200._capi) and lives inside a larger allocation:
64 KB of slack on either side, filled with a sentinel (inputs: NaN, so that a stray read past an input row changes a result
instead of passing unnoticed), the interior at exactly the alignment the header documents and no more (256 B for the
workspace, 8 B for match and FPFH scratch, 16 B for the eigenvector scratch, the element size for outputs and taps; inputs sit
at 16 B).  After the stream synchronises the slack must be byte-identical to its fill.

Poison.  Each configuration runs with a zeroed workspace and then with each poison; workspace, outputs and taps are prefilled
with it.  NaN alone hides in max-reductions (fmaxf drops it), so the float patterns are:
  zero         the baseline;
  0xFFFFFFFF   NaN in fp32, and 0xFFFF is NaN in fp16 and bf16 alike: it covers the tensor-core operand images in tc_scratch;
  0x7F7F7F7F   +3.4e38, finite: wins max-reductions and overflows sums;
  0xFF7F7F7F   -3.4e38.
Results must be bit-identical across patterns; every output and tap element must therefore have been written.  So must the
SC matrix in the workspace, whose pad columns the contract says are written as 0 (a pad column only feeds discarded query
rows, so no output shows it).

Workspace regions.  carve() (engine.cu) and plan_call() (sets.cuh) are restated in engine_rules.py (mirror_workspace),
including tc_scratch (encoder_tc.cu) and the key-split rules attn_set_split / attn_set_split_invariant / attn_call_splits
(sets.cuh), and every GPU test asserts that the restatement's total equals pdsc_workspace_bytes(_packed), so the map
cannot drift from the engine.  Float regions get the float patterns.  Control and index regions only get values that keep
every read in bounds, whatever a kernel does with them: seeds / knn / counts 0 or 1 (N >= 2), conv_mask 0 or all ones,
best_key 0 or 0xFFFFFFFF00000000, and zeros for the descriptor table and tile_set (a zero descriptor is N = 0, which every
kernel skips).

Scratch audit of the front end (which kernel initialises the scratch control data within the call, so poisoning it is safe):
  pdsc_match                row_idx [Ns] and col_idx [Nt] are written for every row by match_reduce_kernel (col_idx only with
                            the mutual check, and compact_center_kernel reads it only then); the (distance, index) partials by
                            match_rows_kernel for every (row, chunk) the reduction reads.
  pdsc_voxel_down_sample    vox_init_kernel resets the hash keys, sums, counts, the three min-bound keys and the counter;
                            ckeys / cslot are written by vox_compact_kernel for every slot below the counter vox_rank_kernel
                            reads.
  normals / FPFH            hybrid_search_kernel writes nb_idx [m, max_nn] and nb_cnt [m] for every point; spfh_kernel every
                            SPFH row fpfh_kernel reads.
  pdsc_leading_eigenvector  eig_init_kernel zeroes done [B] (and iters_run) and sets v to ones; u and the partial sums are
                            written by eig_gemv_kernel for every row and part eig_norm_kernel reads.
Output alignment audit: taps and outputs are written with scalar stores or cudaMemcpy*, except that the layer_debug tap's
PointCN plane was written with 16-byte stores (tc_unblock_f32_kernel), which a 4-byte aligned tap cannot take; it now stores
scalars.

The GPU tests need an H100 (`-m gpu`); the harness self-tests at the end run on the CPU.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from buffer_guards import (BEST_QWORD, FLOAT_WORD, INDEX_WORD, MASK_WORD, PATTERNS, SLACK, Call, Guarded, _capi, assert_same,
                           check_patterns, guarded_input, guarded_output, keypoints, make_inputs, poison_workspace,
                           run_guarded, scratch_buffer, surface, tiled)
from engine_rules import eig_plan, match_plan, mirror_workspace, num_seeds, search_plan
from gpu_models import get_model, sm_count


# ---------------------------------------------------------------------------------------------------
# forward entry points
# ---------------------------------------------------------------------------------------------------
ALL_TAPS = ["sc", "features", "normed", "confidence", "seeds", "knn_idx", "compat", "eig", "power_iters", "seed_trans",
            "inlier_counts", "best", "init_trans", "refine_solves", "layer_features", "layer_debug", "timeline"]
TAPS_NO_LAYER = [t for t in ALL_TAPS if t not in ("layer_features", "layer_debug")]

# (id, precision, N, B, invariant, expected split or None, layer tap)
UNIFORM = [
    ("fp16x3-split-1000", "fp16x3", 1000, 1, False, True, 11),
    ("fp16x3-split-5000", "fp16x3", 5000, 1, False, True, 0),
    ("fp16x3-unsplit-1003", "fp16x3", 1003, None, False, False, 11),
    ("fp16x3-16384", "fp16x3", 16384, 1, False, False, 0),
    ("fp16x3-2", "fp16x3", 2, 3, False, False, 0),
    ("fp16x3-3", "fp16x3", 3, 3, False, False, 11),
    ("fp16x3-63", "fp16x3", 63, 2, False, False, 0),
    ("fp16x3-64", "fp16x3", 64, 2, False, False, 11),
    ("fp16x3-65", "fp16x3", 65, 2, False, False, 0),
    ("fp16x3-127", "fp16x3", 127, 2, False, False, 11),
    ("fp16x3-129", "fp16x3", 129, 2, False, False, 0),
    ("fp16x3-65-many", "fp16x3", 65, 300, False, False, 11),      # S N % 4 != 0 in every set: the distance blocks' padding adds up
    ("fp32-2", "fp32", 2, 2, False, False, 11),
    ("fp32-65", "fp32", 65, 2, False, False, 0),
    ("fp32-129", "fp32", 129, 2, False, False, 11),
    ("fp32-1003", "fp32", 1003, 2, False, False, 0),
    ("bf16x3-split-1000", "bf16x3", 1000, 1, False, True, 0),
    ("bf16x3-129", "bf16x3", 129, 2, False, False, 11),
    ("bf16-split-1000", "bf16", 1000, 1, False, True, 11),
    ("bf16-65", "bf16", 65, 3, False, False, 0),
    ("invariant-513", "fp16x3", 513, 1, True, True, 11),
    ("invariant-5000", "fp16x3", 5000, 1, True, True, 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", UNIFORM, ids=[c[0] for c in UNIFORM])
def test_forward_poison_and_guards(case):
    """pdsc_forward with every tap, in every precision and attention regime, at ragged and whole tiles: bit-identical under
    every poison, nothing written outside its buffers."""
    name, precision, N, B, invariant, want_split, layer = case
    if B is None:                               # unsplit: the call's query tiles cover more than half of the SMs
        B = sm_count() // (2 * -(-N // 128)) + 1
    call = Call(precision, [N] * B, "forward", invariant, taps=ALL_TAPS, layer_tap=layer)
    split, per = call.regime()
    if precision != "fp32":
        assert split == want_split, (name, split, per)
    if invariant:
        sp, TS = per[0]
        assert sp % 4 and sp * TS > -(-N // 64), (sp, TS)      # the merge's clamped re-read and virtual key tiles
    check_patterns(call, (name,))


@pytest.mark.gpu
def test_forward_every_layer_tap_position():
    """layer_features / layer_debug at the first and last layer of one call shape in both SC layouts."""
    for precision in ("fp32", "fp16x3"):
        for layer in (0, 11):
            call = Call(precision, [129, 129], "forward", taps=["sc", "layer_features", "layer_debug"], layer_tap=layer)
            check_patterns(call, (precision, layer))


# one of each k family in one packed call (cfg.k = 100): k = 29 (<= 40), 59 (41-80, tensor-core Gram), 85 (81-88), 100 (> 88),
# beside sets without seeds (N = 9, 2) and ragged tiles
PACKED = [
    ("fp16x3-k100", "fp16x3", False, 100, [9, 30, 60, 86, 1000, 2, 65]),
    ("fp32-k100", "fp32", False, 100, [9, 30, 60, 86, 1000, 2, 65]),
    ("fp16x3-k40", "fp16x3", False, 40, [1000, 9, 3, 129, 513]),
    ("bf16-invariant", "bf16", True, 40, [513, 9, 1003, 64]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", PACKED, ids=[c[0] for c in PACKED])
def test_packed_poison_and_guards(case):
    name, precision, invariant, k, Ns = case
    call = Call(precision, Ns, "packed", invariant, k=k)
    ks = sorted({int(call.lib.pdsc_num_neighbours(call.e, n)) for n in Ns if num_seeds(n) > 0})
    if k == 100:
        assert any(k_ <= 40 for k_ in ks) and any(40 < k_ <= 80 for k_ in ks) and any(80 < k_ <= 88 for k_ in ks) \
            and any(k_ > 88 for k_ in ks), ks
    assert any(num_seeds(n) == 0 for n in Ns) and any(num_seeds(n) > 0 for n in Ns)
    call.regime()
    check_patterns(call, (name,))


EVAL = [("fp16x3-M", "fp16x3", 1000, 2, True), ("fp32-noM", "fp32", 129, 2, False), ("bf16x3-M-65", "bf16x3", 65, 3, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", EVAL, ids=[c[0] for c in EVAL])
def test_eval_poison_and_guards(case):
    """pdsc_forward_eval with and without d_M (zero diagonal written, not skipped), every tap."""
    name, precision, N, B, want_M = case
    call = Call(precision, [N] * B, "eval", taps=TAPS_NO_LAYER, want_M=want_M)
    call.regime()
    ref = check_patterns(call, (name,))
    if want_M:
        M = ref["M"].view(torch.float32).view(B, N, N)
        assert (torch.diagonal(M, dim1=1, dim2=2) == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("precision,N,B", [("fp16x3", 1000, 1), ("fp32", 65, 2)])
def test_graph_replay_with_poisoned_buffers(precision, N, B):
    """pdsc_forward_graph: captured on the first call, then replayed with the workspace and outputs re-poisoned in place;
    every replay equals an eager pdsc_forward of the same inputs."""
    eager = Call(precision, [N] * B, "forward", seed=5).run("zero")
    call = Call(precision, [N] * B, "graph", seed=5)
    for p in PATTERNS + ["ones", "zero"]:
        assert_same(eager, call.run(p), (precision, N, B, "graph", p))


@pytest.mark.gpu
@pytest.mark.parametrize("B,N", [(1, 1000), (2, 65), (4, 9000)])
def test_host_entry_points_write_whole_results(B, N):
    """pdsc_forward_host and _submit / _wait (engine-owned workspace) into NaN-prefilled host buffers with NaN slack:
    results equal pdsc_forward's, and nothing past them is written.  4 x 9000 rows takes the ungraphed host path."""
    lib = _capi().load()
    call = Call("fp16x3", [N] * B, "forward", seed=7)
    ref = call.run("ones")
    cp, s, t = make_inputs([N] * B, seed=7)
    e = call.e
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    slack = SLACK // 4

    def host_out(n):
        a = np.full(n + 2 * slack, np.nan, np.float32)
        return a, a[slack:slack + n]

    P = lambda a: C.c_void_p(a.ctypes.data)         # noqa: E731
    for mode in ("host", "submit"):
        for _ in range(2):
            (tr_all, tr), (lb_all, lb) = host_out(B * 16), host_out(B * N)
            if mode == "host":
                _capi().check(lib.pdsc_forward_host(e, B, N, P(cp), P(s), P(t), P(tr), P(lb), stream))
            else:
                slot = C.c_int32(-1)
                _capi().check(lib.pdsc_forward_host_submit(e, B, N, P(cp), P(s), P(t), P(tr), P(lb), stream, C.byref(slot)))
                _capi().check(lib.pdsc_forward_host_wait(e, slot.value))
            for a_all, a in ((tr_all, tr), (lb_all, lb)):
                assert np.isnan(a_all[:slack]).all() and np.isnan(a_all[slack + a.size:]).all(), (mode, "host slack written")
            assert tr.tobytes() == ref["final_trans"].cpu().numpy().tobytes(), (mode, B, N)
            assert lb.tobytes() == ref["final_labels"].cpu().numpy().tobytes(), (mode, B, N)


# ---------------------------------------------------------------------------------------------------
# call history: a module's cached workspace and graph buffers carry nothing from one call into the next
# ---------------------------------------------------------------------------------------------------
def history_calls():
    return [("run", 64, 5000), ("run", 1, 1000), ("run", 1, 2), ("many", [(2, 129), (1, 9), (1, 1000)]), ("eval", 2, 513),
            ("run", 64, 5000)]


def do_call(m, c, host=False, seed=11):
    def data(B, N, sd):
        cp, s, t = make_inputs([N] * B, sd)
        ts = [torch.from_numpy(x).view(B, N, -1) for x in (cp, s, t)]
        return ts if host else [x.cuda() for x in ts]
    if c[0] == "run":
        out = m.run(*data(c[1], c[2], seed))
        return [out["final_trans"].cpu(), out["final_labels"].cpu()]
    if c[0] == "eval":
        out = m.run_eval(*data(c[1], c[2], seed))
        return [out["final_trans"].cpu(), out["final_labels"].cpu(), out["M"].cpu()]
    batches = []
    for j, (B, N) in enumerate(c[1]):
        cp, s, t = data(B, N, seed + j)
        batches.append({"corr_pos": cp, "src_keypts": s, "tgt_keypts": t, "testing": True})
    return [x for o in m.forward_many(batches) for x in (o["final_trans"].cpu(), o["final_labels"].cpu())]


@pytest.mark.gpu
def test_call_history_on_one_module():
    """B = 64 x 5000, bs = 1 x 1000 (split, graph replay), N = 2, a packed call, an eval call, then the first shape again on
    one module: each equals the same call on a fresh module, bit for bit; then the uniform calls through the host path."""
    m = get_model(precision="fp16x3", fresh=True)
    fresh_results = []
    for c in history_calls():
        got = do_call(m, c)
        f = get_model(precision="fp16x3", fresh=True)
        want = do_call(f, c)
        f._release()
        del f
        fresh_results.append(want)
        for a, b in zip(got, want):
            assert a.numpy().tobytes() == b.numpy().tobytes(), c
    h = get_model(precision="fp16x3", fresh=True)
    for c, want in zip(history_calls(), fresh_results):
        if c[0] != "run":
            continue
        got = do_call(h, c, host=True)
        for a, b in zip(got, want):
            assert a.numpy().tobytes() == b.numpy().tobytes(), ("host", c)
    h._release()
    m._release()


# ---------------------------------------------------------------------------------------------------
# front-end entry points
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fp64", [False, True], ids=["fp32", "fp64"])
def test_match_poison_and_rows_past_m(fp64):
    """pdsc_match: scratch at exactly 8 B and pdsc_match_scratch_bytes, poisoned; outputs prefilled; rows >= M keep the
    prefill byte for byte (only the first M rows are written); mutual on and off; one chunk, several and the cap."""
    lib = _capi().load()
    dev = torch.device("cuda")
    e = _capi().utility_engine(0)
    sms = sm_count()
    D = 33 if fp64 else 32
    shapes = [(100, 1024 if fp64 else 2048), (5000, 700), (4 * sms * 128 + 5, 40)]   # the cap, several chunks, one
    kinds = set()
    for ns, nt in shapes:
        chunks = match_plan(ns, nt, D, fp64, sms)[0]
        kinds.add("1" if chunks == 1 else ("max" if chunks == 32 else "mid"))
        rng = np.random.default_rng(ns)
        dt = np.float64 if fp64 else np.float32
        t = rng.standard_normal((nt, D))
        t /= np.linalg.norm(t, axis=1, keepdims=True)
        s = t[rng.integers(0, nt, ns)] + 0.3 / np.sqrt(D) * rng.standard_normal((ns, D))
        s /= np.linalg.norm(s, axis=1, keepdims=True)
        ins = {"sd": guarded_input(s.astype(dt), dev), "td": guarded_input(t.astype(dt), dev),
               "sk": guarded_input(keypoints(rng, ns), dev), "tk": guarded_input(keypoints(rng, nt), dev)}
        need = int(lib.pdsc_match_scratch_bytes(ns, nt))
        for mutual in (0, 1):
            ref = None
            for p in PATTERNS:
                outs = {"corr": guarded_output(ns * 8, 4, dev, p), "count": guarded_output(4, 4, dev, p),
                        "corr_pos": guarded_output(ns * 24, 4, dev, p), "src": guarded_output(ns * 12, 4, dev, p),
                        "tgt": guarded_output(ns * 12, 4, dev, p)}
                sc = scratch_buffer(need, 8, p)
                P = lambda g: C.c_void_p(g.ptr)     # noqa: E731
                got = run_guarded((ns, nt, mutual, p), outs, sc, ins, lambda: lib.pdsc_match(
                    e, ns, nt, D, P(ins["sd"]), P(ins["td"]), int(fp64), P(ins["sk"]), P(ins["tk"]), mutual, P(outs["corr"]),
                    P(outs["count"]), P(outs["corr_pos"]), P(outs["src"]), P(outs["tgt"]), P(sc), need,
                    C.c_void_p(torch.cuda.current_stream().cuda_stream)))
                M = int(got["count"].view(torch.int32)[0])
                assert 0 < M <= ns and (mutual or M == ns)
                for name, row in (("corr", 8), ("corr_pos", 24), ("src", 12), ("tgt", 12)):
                    tail = got[name][M * row:]
                    assert torch.equal(tail, tiled(FLOAT_WORD[p], tail.numel(), dev)), (name, "row >= M written", ns, nt, p)
                    got[name] = got[name][:M * row]
                if ref is None:
                    ref = got
                else:
                    assert_same(ref, got, ("match", ns, nt, mutual, p))
    assert kinds == {"1", "mid", "max"}, kinds


@pytest.mark.gpu
def test_voxel_down_sample_poison():
    """pdsc_voxel_down_sample: poisoned scratch (the audit: every control word is reset by vox_init_kernel), count and
    status prefilled; both written on the stream."""
    lib = _capi().load()
    dev = torch.device("cuda")
    e = _capi().utility_engine(0)
    rng = np.random.default_rng(3)
    for n in (1, 700, 20000):
        pts = rng.uniform(0, 1, (n, 3)).astype(np.float32)
        ins = {"pts": guarded_input(pts, dev)}
        need = int(lib.pdsc_voxel_down_sample_scratch_bytes(n))
        ref = None
        for p in PATTERNS:
            outs = {"points": guarded_output(n * 12, 4, dev, p), "count": guarded_output(4, 4, dev, p),
                    "status": guarded_output(4, 4, dev, p)}
            sc = scratch_buffer(need, 8, p)
            P = lambda g: C.c_void_p(g.ptr)         # noqa: E731
            got = run_guarded(("voxel", n, p), outs, sc, ins, lambda: lib.pdsc_voxel_down_sample(
                e, n, P(ins["pts"]), 0.05, P(outs["points"]), P(outs["count"]), P(outs["status"]), P(sc), need,
                C.c_void_p(torch.cuda.current_stream().cuda_stream)))
            m = int(got["count"].view(torch.int32)[0])
            assert 1 <= m <= n and int(got["status"].view(torch.int32)[0]) == 0, (n, p, m)
            got["points"] = got["points"][:m * 12]
            if ref is None:
                ref = got
            else:
                assert_same(ref, got, ("voxel", n, p))


SIZE_CLASS_MAX_NN = [1, 3, 5, 9, 17, 33, 65, 129, 256]     # P = 2, 4, ..., 256: every bitonic size class of the search


@pytest.mark.gpu
def test_normals_and_fpfh_poison():
    assert sorted({search_plan(n)[0] for n in SIZE_CLASS_MAX_NN}) == [2 ** i for i in range(1, 9)]
    lib = _capi().load()
    dev = torch.device("cuda")
    e = _capi().utility_engine(0)
    m = 1203
    pts = surface(np.random.default_rng(9), m)
    for max_nn in SIZE_CLASS_MAX_NN:
        radius = float(np.sqrt(1.5 * max(max_nn, 4) / (np.pi * m)))
        ins = {"pts": guarded_input(pts, dev)}
        need = int(lib.pdsc_fpfh_scratch_bytes(m, max_nn))
        ref = None
        for p in PATTERNS:
            P = lambda g: C.c_void_p(g.ptr)         # noqa: E731
            st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            outs = {"normals": guarded_output(m * 24, 8, dev, p), "status": guarded_output(4, 4, dev, p)}
            sc = scratch_buffer(need, 8, p)
            got = run_guarded(("normals", max_nn, p), outs, sc, ins, lambda: lib.pdsc_estimate_normals(
                e, m, P(ins["pts"]), radius, max_nn, P(outs["normals"]), P(outs["status"]), P(sc), need, st))
            nrm = {"normals": Guarded(m * 24, 16, dev, slack="nan")}
            nrm["normals"].inner.copy_(got["normals"])
            outs2 = {"fpfh": guarded_output(m * 33 * 8, 8, dev, p), "status": guarded_output(4, 4, dev, p)}
            sc2 = scratch_buffer(need, 8, p)
            got2 = run_guarded(("fpfh", max_nn, p), outs2, sc2, {**ins, **nrm}, lambda: lib.pdsc_compute_fpfh(
                e, m, P(ins["pts"]), P(nrm["normals"]), radius, max_nn, 1, P(outs2["fpfh"]), P(outs2["status"]), P(sc2), need, st))
            res = {"normals": got["normals"], "status_n": got["status"], "fpfh": got2["fpfh"], "status_f": got2["status"]}
            assert int(res["status_n"].view(torch.int32)[0]) == 0 and int(res["status_f"].view(torch.int32)[0]) == 0, (max_nn, p)
            assert torch.isfinite(res["fpfh"].view(torch.float64)).all()
            if ref is None:
                ref = res
            else:
                assert_same(ref, res, ("normals/fpfh", max_nn, p))


@pytest.mark.gpu
def test_leading_eigenvector_poison():
    """Scratch at exactly 16 B and pdsc_leading_eigenvector_scratch_bytes, poisoned (done is reset by eig_init_kernel);
    iterations_run prefilled; early exit on and off; the bulk-copy path (N % 4 == 0) and the plain one."""
    lib = _capi().load()
    dev = torch.device("cuda")
    e = _capi().utility_engine(0)
    paths = set()
    for B, N in ((3, 1000), (2, 1001), (1, 4)):
        g = torch.Generator().manual_seed(N)
        M = torch.rand(B, N, N, generator=g)
        M = ((M + M.transpose(1, 2)) / 2).numpy().astype(np.float32)
        ins = {"M": guarded_input(M, dev)}
        paths.add(eig_plan(B, N, ins["M"].ptr, sm_count())["tma"])
        need = int(lib.pdsc_leading_eigenvector_scratch_bytes(B, N))
        for early in (0, 1):
            ref = None
            for p in PATTERNS:
                outs = {"v": guarded_output(B * N * 4, 4, dev, p), "iters": guarded_output(B * 4, 4, dev, p)}
                sc = scratch_buffer(need, 16, p)
                P = lambda g: C.c_void_p(g.ptr)     # noqa: E731
                got = run_guarded(("eig", B, N, early, p), outs, sc, ins, lambda: lib.pdsc_leading_eigenvector(
                    e, B, N, P(ins["M"]), 10, early, P(outs["v"]), P(outs["iters"]), P(sc), need,
                    C.c_void_p(torch.cuda.current_stream().cuda_stream)))
                it = got["iters"].view(torch.int32)
                assert ((it >= 1) & (it <= 10)).all() and (early or (it == 10).all()), (B, N, early, p, it)
                if ref is None:
                    ref = got
                else:
                    assert_same(ref, got, ("eig", B, N, early, p))
    assert paths == {True, False}


@pytest.mark.gpu
def test_eval_stats_poison():
    lib = _capi().load()
    dev = torch.device("cuda")
    e = _capi().utility_engine(0)
    rng = np.random.default_rng(4)
    for B, N in ((1, 1), (3, 257), (2, 5000)):
        eye = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
        pred = eye.copy()
        pred[:, :3, 3] = rng.normal(0, 0.1, (B, 3))
        ins = {"pred": guarded_input(pred, dev), "gt": guarded_input(eye, dev),
               "src": guarded_input(rng.uniform(-1, 1, (B, N, 3)).astype(np.float32), dev),
               "tgt": guarded_input(rng.uniform(-1, 1, (B, N, 3)).astype(np.float32), dev),
               "pl": guarded_input((rng.uniform(size=(B, N)) > 0.5).astype(np.float32), dev),
               "gl": guarded_input((rng.uniform(size=(B, N)) > 0.5).astype(np.float32), dev)}
        ref = None
        for p in PATTERNS:
            outs = {"stats": guarded_output(B * 40, 4, dev, p)}
            P = lambda g: C.c_void_p(g.ptr)         # noqa: E731
            dummy = Guarded(0, 4, dev)
            got = run_guarded(("stats", B, N, p), outs, dummy, ins, lambda: lib.pdsc_eval_stats(
                e, B, N, P(ins["pred"]), P(ins["gt"]), P(ins["src"]), P(ins["tgt"]), P(ins["pl"]), P(ins["gl"]), 15.0, 30.0,
                P(outs["stats"]), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
            if ref is None:
                ref = got
            else:
                assert_same(ref, got, ("stats", B, N, p))


# ---------------------------------------------------------------------------------------------------
# CPU: the harness itself
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("align", [4, 8, 16, 256])
def test_guard_catches_one_changed_byte_at_either_end(align):
    cpu = torch.device("cpu")
    for nbytes in (0, 1, 4, 1000, 4096):
        g = Guarded(nbytes, align, cpu)
        assert g.ptr % align == 0 and g.ptr % (2 * align) != 0          # exactly the alignment, not more
        assert g.off >= SLACK and g.raw.numel() - g.off - nbytes >= SLACK
        g.inner.fill_(0x11)
        assert g.violations() == []
        for rel in (-1, nbytes, -SLACK, nbytes + SLACK - 1):
            idx = g.off + rel
            old = int(g.raw[idx])
            g.raw[idx] = old ^ 0x01
            assert g.violations() == [rel], (nbytes, rel)
            g.raw[idx] = old
        assert g.violations() == []
    n = Guarded(64, 16, cpu, slack="nan")
    assert torch.isnan(n.raw[:n.off].view(torch.float32)).all()


MIRROR_SHAPES = [([1000], "fp16x3", False), ([5000], "fp16x3", False), ([1003] * 9, "fp16x3", False), ([2] * 3, "fp32", False),
                 ([9, 30, 60, 86, 1000, 2, 65], "fp16x3", False), ([9, 30, 60, 86, 1000, 2, 65], "fp32", False),
                 ([513], "fp16x3", True), ([5000], "bf16", True), ([16384], "fp16x3", False)]


@pytest.mark.parametrize("Ns,precision,invariant", MIRROR_SHAPES)
def test_region_map_covers_the_workspace_without_overlap(Ns, precision, invariant):
    regions, total = mirror_workspace(Ns, precision, invariant, 100 if 86 in Ns else 40, 132)
    assert total % 256 == 0
    end = 0
    names = [r[0] for r in regions]
    assert len(set(names)) == len(names)
    for name, off, n, kind in regions:
        assert off % 256 == 0 and off >= end and off - end < 256, (name, off, end)    # 256-byte steps, no overlap, no hole
        assert n > 0 or name == "sets", name
        end = off + n
    assert end <= total < end + 256
    assert {r[0] for r in regions if r[3] != "float"} == {"seeds", "knn", "counts", "conv_mask", "best_key", "sets", "tile_set"}


def test_each_pattern_reaches_every_word():
    Ns = [9, 30, 60, 86, 1000, 2, 65]
    regions, total = mirror_workspace(Ns, "fp16x3", False, 100, 132)
    for p in PATTERNS:
        ws = torch.empty(total, dtype=torch.uint8)
        ws.fill_(0xA5)                                      # a byte no pattern contains
        poison_workspace(ws, regions, p)
        assert not (ws == 0xA5).any(), p
        words = ws.view(torch.int32)
        for name, off, n, kind in regions:
            seg = ws[off:off + n]
            if kind == "float":
                want = FLOAT_WORD[p]
            elif kind == "index":
                want = INDEX_WORD[p]
            elif kind == "mask":
                want = MASK_WORD[p]
            elif kind == "zero":
                want = 0
            else:
                assert torch.equal(seg, tiled(BEST_QWORD[p], n, ws.device, 8)), p
                continue
            assert torch.equal(seg, tiled(want, n, ws.device)), (name, p)
        assert words.numel() * 4 == total
    # every float pattern is NaN / extreme where it should be, in the formats the images use
    ones = torch.tensor([0xFFFF], dtype=torch.int32).to(torch.int16)
    assert torch.isnan(ones.view(torch.float16)).all() and torch.isnan(ones.view(torch.bfloat16)).all()
    w = torch.tensor([FLOAT_WORD["fmax"], FLOAT_WORD["fmin"] - 2 ** 32, FLOAT_WORD["ones"] - 2 ** 32], dtype=torch.int64)
    f = w.to(torch.int32).view(torch.float32)
    assert float(f[0]) > 3e38 and float(f[1]) < -3e38 and torch.isnan(f[2])
