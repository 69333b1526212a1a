"""Mixed-size calls (pdsc_forward_packed / PointDSC.forward_many): sets of different N in one call.

Contract: a set's outputs depend only on its own inputs, its N and the call's attention regime (key split or not, DESIGN.md
§3).  Within one regime a set of a mixed call gives bit for bit what a uniform call holding that set gives."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import golden_cases, load_case, registration_ok
from gpu_models import as_batch, get_model, sm_count, synth_sets

pytestmark = pytest.mark.gpu

PRECISIONS = os.environ.get("PDSC_TEST_PRECISIONS", "fp32,fp16x3").split(",")


def single(m, pair):
    b = as_batch([pair])
    return m.run(b["corr_pos"], b["src_keypts"], b["tgt_keypts"])


def q_tiles(n):
    return (n + 127) // 128


@pytest.mark.parametrize("precision", PRECISIONS)
def test_large_regime_mixed_call_equals_uniform_calls(precision):
    """Interleaved sets of five sizes, enough copies of each that every size's uniform call is also in the large regime."""
    m = get_model("3dmatch", precision)
    sizes = [41, 257, 1000, 1003, 2000]
    copies = max(sm_count() // (2 * q_tiles(n)) + 1 for n in sizes)
    assert all(2 * copies * q_tiles(n) > sm_count() for n in sizes)
    groups = {n: synth_sets([n] * copies, seed0=1000 * n) for n in sizes}
    order = [(n, c) for c in range(copies) for n in sizes]          # interleaved: 41, 257, 1000, 1003, 2000, 41, ...
    out = m.forward_many([as_batch([groups[n][c]]) for n, c in order])
    for n in sizes:
        b = as_batch(groups[n])
        ref = m.run(b["corr_pos"], b["src_keypts"], b["tgt_keypts"])
        for i, (nn, c) in enumerate(order):
            if nn != n:
                continue
            assert out[i]["M"] is None and out[i]["final_labels"].shape == (1, n)
            assert torch.equal(out[i]["final_trans"][0], ref["final_trans"][c]), (n, c)
            assert torch.equal(out[i]["final_labels"][0], ref["final_labels"][c]), (n, c)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_split_regime_mixed_call_equals_single_calls(precision):
    """2 * sum(QT) = 40 <= SMs: the call is split per set exactly as each bs = 1 call is."""
    m = get_model("3dmatch", precision)
    sizes = [1000, 257, 41, 1003]
    assert 2 * sum(q_tiles(n) for n in sizes) <= sm_count()
    pairs = synth_sets(sizes, seed0=7)
    out = m.forward_many([as_batch([p]) for p in pairs])
    for p, o in zip(pairs, out):
        one = single(m, p)
        assert torch.equal(o["final_trans"], one["final_trans"])
        assert torch.equal(o["final_labels"], one["final_labels"])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_uniform_call_is_the_packed_call_with_equal_offsets(precision):
    """pdsc_forward(B, N) runs the packed call whose offsets are b * N: the same workspace and the same bytes, in both
    attention regimes (bs = 1 at N = 1000 is split, 64 sets are not)."""
    m = get_model("3dmatch", precision)
    lib = m._ensure_engine()
    for B, N in ((1, 2), (3, 9), (1, 1000), (64, 1000), (1, 16384), (2, 16384)):
        h = (C.c_int32 * (B + 1))(*range(0, (B + 1) * N, N))
        assert lib.pdsc_workspace_bytes(m._engine, B, N) == lib.pdsc_workspace_bytes_packed(m._engine, B, h) > 0, (B, N)
    for copies in (1, 64):
        b = as_batch(synth_sets([1000] * copies, seed0=90))
        ref = m.run(b["corr_pos"], b["src_keypts"], b["tgt_keypts"])
        out = m.forward_many([b])[0]
        assert torch.equal(out["final_trans"], ref["final_trans"]), copies
        assert torch.equal(out["final_labels"], ref["final_labels"]), copies


def test_batches_of_several_sets_keep_their_shapes():
    m = get_model("3dmatch", "fp16x3")
    a, b = synth_sets([300, 300], seed0=3), synth_sets([500], seed0=5)
    out = m.forward_many([as_batch(a), as_batch(b)])
    assert out[0]["final_trans"].shape == (2, 4, 4) and out[0]["final_labels"].shape == (2, 300)
    assert out[1]["final_trans"].shape == (1, 4, 4) and out[1]["final_labels"].shape == (1, 500)
    again = m.forward_many([as_batch(a), as_batch(b)])
    for x, y in zip(out, again):
        assert torch.equal(x["final_trans"], y["final_trans"]) and torch.equal(x["final_labels"], y["final_labels"])


def _check_against_fixture(c, T, labels, again_T):
    """test_end_to_end_vs_reference's checks for one set of a mixed call (labels: that set's [N] labels)."""
    R = T[:3, :3]
    assert np.abs(R @ R.T - np.eye(3)).max() < 1e-5 and abs(np.linalg.det(R) - 1) < 1e-5
    assert np.array_equal(T[3], np.array([0, 0, 0, 1], np.float32))
    if not registration_ok(c):
        # the reference failed on this pair (tied hypotheses): the call is reproducible, and the winning hypothesis (whose
        # inliers are the labels) holds at least as many inliers as the reference's best
        assert np.array_equal(again_T, T)
        n = len(c["final_labels"])
        assert int((labels > 0.5).sum()) + 2 >= int(round(float(c["fitness"].max()) * n))
        return
    assert np.abs(T - c["final_trans"]).max() < 1e-4
    assert (labels != c["final_labels"]).sum() <= 2


def _run_fixtures(cases, precision):
    m = get_model(cases[0]["meta"]["dataset"], precision, k=int(cases[0]["meta"].get("k", 40)))
    batches = [{"corr_pos": torch.from_numpy(np.ascontiguousarray(c["corr_pos"])).cuda()[None],
                "src_keypts": torch.from_numpy(np.ascontiguousarray(c["src_keypts"])).cuda()[None],
                "tgt_keypts": torch.from_numpy(np.ascontiguousarray(c["tgt_keypts"])).cuda()[None], "testing": True} for c in cases]
    out = m.forward_many(batches)
    again = m.forward_many(batches)
    for c, o, a in zip(cases, out, again):
        _check_against_fixture(c, o["final_trans"][0].cpu().numpy(), o["final_labels"][0].cpu().numpy(),
                               a["final_trans"][0].cpu().numpy())


@pytest.mark.parametrize("precision", PRECISIONS)
def test_3dmatch_fixtures_in_one_call_vs_reference(precision):
    cases = [load_case(p) for p in golden_cases("3dmatch", n_max=2000)]
    cases = [c for c in cases if int(c["meta"].get("k", 40)) == 40]
    assert len({int(c["meta"]["n"]) for c in cases}) >= 5
    _run_fixtures(cases, precision)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_kitti_fixtures_in_one_call_vs_reference(precision):
    cases = [load_case(p) for p in golden_cases("kitti")]
    cases = [c for c in cases if int(c["meta"]["n"]) == 5000] + [c for c in cases if int(c["meta"]["n"]) == 1000][:1]
    assert len(cases) == 3
    _run_fixtures(cases, precision)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_edge_sizes_in_one_call(precision):
    """N = 2, N < 10 (no seeds), N <= k and N = 16384 beside them: large regime in both calls (or too few key tiles to split)."""
    m = get_model("3dmatch", precision)
    sizes = [2, 7, 30, 16384, 9, 41]
    pairs = synth_sets(sizes, seed0=40)
    out = m.forward_many([as_batch([p]) for p in pairs])
    for n, p, o in zip(sizes, pairs, out):
        one = single(m, p)
        assert torch.equal(o["final_trans"], one["final_trans"]), n
        assert torch.equal(o["final_labels"], one["final_labels"]), n


@pytest.mark.parametrize("precision", PRECISIONS)
def test_sets_with_different_k_in_one_call(precision):
    """k = 80: N = 30 and N = 60 have k = N - 1 and run other power-iteration kernels than N = 1000 (k = 80)."""
    m = get_model("3dmatch", precision, k=80)
    sizes = [30, 1000, 60, 81]
    pairs = synth_sets(sizes, seed0=60)
    out = m.forward_many([as_batch([p]) for p in pairs])
    for n, p, o in zip(sizes, pairs, out):
        one = single(m, p)
        assert torch.equal(o["final_trans"], one["final_trans"]), n
        assert torch.equal(o["final_labels"], one["final_labels"]), n


def test_errors_are_loud():
    from pointdsc_b200 import _capi
    m = get_model("3dmatch", "fp16x3")
    lib = m._ensure_engine()
    pairs = synth_sets([50, 60], seed0=1)
    cp = torch.cat([p["corr_pos"] for p in pairs]).cuda()
    s = torch.cat([p["src_keypts"] for p in pairs]).cuda()
    t = torch.cat([p["tgt_keypts"] for p in pairs]).cuda()
    trans = torch.empty(2, 4, 4, device="cuda")
    labels = torch.empty(110, device="cuda")

    def call(offsets, ws_bytes=None):
        h = (C.c_int32 * len(offsets))(*offsets)
        d = torch.tensor(offsets, dtype=torch.int32, device="cuda")
        need = int(lib.pdsc_workspace_bytes_packed(m._engine, len(offsets) - 1, h))
        ws = torch.empty(max(need, 1 << 20), dtype=torch.uint8, device="cuda")
        rc = lib.pdsc_forward_packed(m._engine, len(offsets) - 1, h, C.c_void_p(d.data_ptr()), C.c_void_p(cp.data_ptr()),
                                     C.c_void_p(s.data_ptr()), C.c_void_p(t.data_ptr()), C.c_void_p(trans.data_ptr()),
                                     C.c_void_p(labels.data_ptr()), C.c_void_p(ws.data_ptr()),
                                     ws_bytes if ws_bytes is not None else ws.numel(), None)
        torch.cuda.synchronize()
        return rc, need

    rc, need = call([0, 50, 110])
    assert rc == 0 and need > 0
    for bad in ([1, 50, 110], [0, 60, 50], [0, 1, 110], [0, 50, 50]):
        rc, need = call(bad)
        assert rc == 3 and need == 0, bad
        with pytest.raises(_capi.PdscError):
            _capi.check(rc)
    rc, _ = call([0, 50, 110], ws_bytes=4096)
    assert rc == 5
    big = synth_sets([16385], seed0=2)[0]
    with pytest.raises(_capi.PdscError):
        m.forward_many([as_batch([big])])
    with pytest.raises(ValueError):
        m.forward_many([{k: v for k, v in as_batch([pairs[0]]).items() if k != "testing"}])
    with pytest.raises(ValueError):
        m.forward_many([{"corr_pos": pairs[0]["corr_pos"][None], "src_keypts": pairs[0]["src_keypts"][None],
                         "tgt_keypts": pairs[0]["tgt_keypts"][None], "testing": True}])


def test_evaluate_groups_equal_single_pairs():
    import evaluate
    s1, _ = evaluate.main(["--synthetic", "4", "--batch_size", "1"])
    s4, _ = evaluate.main(["--synthetic", "4", "--batch_size", "4"])
    assert s1.shape == s4.shape == (4, len(evaluate.COLUMNS))
    assert np.array_equal(s1[:, 0], s4[:, 0])
    ok = s1[:, 0] == 1
    # bs = 1 at these N (~6.7 k) is in the attention's key-split regime, the group of four is not: the two differ by fp32
    # rounding of the softmax sums, which the refinement carries into the transform (measured: 0.008 deg, 0.07 cm)
    assert np.abs(s1[ok, 1] - s4[ok, 1]).max(initial=0) < 1e-2 and np.abs(s1[ok, 2] - s4[ok, 2]).max(initial=0) < 0.1
    # the regimes' transforms keep or drop a few of the ~1.1 k inliers near the threshold
    assert np.abs(s1[:, 6] - s4[:, 6]).max() < 1e-2 and np.abs(s1[:, 7] - s4[:, 7]).max() < 1e-2
