"""Batch-invariant mode (PointDSC(batch_invariant=True), pdsc_set_batch_invariant).

Contract: in this mode a set's outputs depend only on its own inputs and its N: bit for bit the same at bs = 1, in a uniform
batch, in a mixed-size call, in any order, through every entry point and whatever the device's SM count.  The default mode is
left as it is (its own tests)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import golden_cases, load_case, registration_ok
from engine_rules import PARTIAL_BYTES, SPLIT_MAX_ITEMS
from gpu_models import as_batch, get_model, synth_sets

pytestmark = pytest.mark.gpu

PRECISIONS = list(dict.fromkeys(os.environ.get("PDSC_TEST_PRECISIONS", "fp32,fp16x3").split(",") + ["bf16x3"]))
TAPS = ["features", "seeds", "best"]


def args(b):
    return b["corr_pos"], b["src_keypts"], b["tgt_keypts"]


def invariant_tiles():
    """Key tiles per split of the invariant rule, read back from the workspace of one set of N = 16384 (KT = 256)."""
    m_def, m_inv = get_model(precision="fp16x3"), get_model(precision="fp16x3", invariant=True)
    lib = m_def._ensure_engine()
    m_inv._ensure_engine()
    diff = int(lib.pdsc_workspace_bytes(m_inv._engine, 1, 16384)) - int(lib.pdsc_workspace_bytes(m_def._engine, 1, 16384))
    items = diff // PARTIAL_BYTES + SPLIT_MAX_ITEMS
    assert diff % PARTIAL_BYTES == 0 and items % 128 == 0, diff
    return 256 // (items // 128)


def edge_sizes():
    """The issue's sizes and those where KT = TSI, TSI + 1 and 2 TSI + 1 (the first, second and third split of a set)."""
    tsi = invariant_tiles()
    return sorted({2, 7, 41, 257, 1000, 1003, 2000, 5000, 16384, 64 * tsi, 64 * tsi + 1, 128 * tsi + 1})


def assert_equal(a, b, what):
    for key in a:
        assert torch.equal(a[key].cpu(), b[key].cpu()), (what, key)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_single_uniform_and_mixed_calls_agree(precision):
    m = get_model(precision=precision, invariant=True)
    sizes = edge_sizes()
    pairs = synth_sets(sizes, seed0=500)
    uni = synth_sets([1000] * 64, seed0=900)
    picks = (0, 37, 63)
    # bs = 1 calls, eager with taps
    singles = [m.run(*args(as_batch([p])), taps=TAPS) for p in pairs]
    uni_singles = {i: m.run(*args(as_batch([uni[i]])), taps=TAPS) for i in picks}
    # one uniform batch of 64
    ub = m.run(*args(as_batch(uni)), taps=TAPS)
    for i in picks:
        row = {k: ub[k][i:i + 1] for k in ["final_trans", "final_labels"] + TAPS}
        assert_equal(uni_singles[i], row, ("uniform", i))
    # one mixed call: the edge sizes interleaved with the uniform sets
    order = []
    for j in range(max(len(pairs), len(uni))):
        if j < len(uni):
            order.append(("u", j))
        if j < len(pairs):
            order.append(("p", j))
    out = m.forward_many([as_batch([uni[j] if kind == "u" else pairs[j]]) for kind, j in order])
    for (kind, j), o in zip(order, out):
        if kind == "p":
            ref = {"final_trans": singles[j]["final_trans"], "final_labels": singles[j]["final_labels"]}
        else:
            ref = {"final_trans": ub["final_trans"][j:j + 1], "final_labels": ub["final_labels"][j:j + 1]}
        assert_equal(ref, {"final_trans": o["final_trans"], "final_labels": o["final_labels"]}, ("mixed", kind, j))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_permuted_batch(precision):
    m = get_model(precision=precision, invariant=True)
    pairs = synth_sets([1003] * 16, seed0=300)
    perm = np.random.default_rng(1).permutation(16)
    a = m.run(*args(as_batch(pairs)), taps=TAPS)
    b = m.run(*args(as_batch([pairs[i] for i in perm])), taps=TAPS)
    for pos, i in enumerate(perm):
        for key in ["final_trans", "final_labels"] + TAPS:
            assert torch.equal(a[key][i], b[key][pos]), (key, i)
    mixed = synth_sets([300, 5000, 41, 1000, 2000, 1025], seed0=330)
    perm = np.random.default_rng(2).permutation(len(mixed))
    x = m.forward_many([as_batch([p]) for p in mixed])
    y = m.forward_many([as_batch([mixed[i]]) for i in perm])
    for pos, i in enumerate(perm):
        assert_equal({k: x[i][k] for k in ("final_trans", "final_labels")},
                    {k: y[pos][k] for k in ("final_trans", "final_labels")}, ("mixed permuted", i))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_every_entry_point(precision):
    """Device (eager), graph replay, host (graph and eager), forward_stream, forward_many and forward() on the same sets."""
    m = get_model(precision=precision, invariant=True)
    pairs = synth_sets([1000] * 40, seed0=700)
    eager = [m.run(*args(as_batch([p])), taps=["best"]) for p in pairs[:3]]
    ref = [{"final_trans": e["final_trans"], "final_labels": e["final_labels"]} for e in eager]
    for _ in range(2):   # capture, then replay
        for r, p in zip(ref, pairs[:3]):
            assert_equal(r, m.run(*args(as_batch([p]))), "graph")
    for r, p in zip(ref, pairs[:3]):
        b = as_batch([p])
        assert_equal(r, m({k: v for k, v in b.items()}), "forward")
        assert_equal(r, m.run(*(x.cpu() for x in args(b))), "host, graph")
    big = as_batch(pairs)                                     # 40 000 rows: the host path's eager branch
    host = m.run(*(x.cpu() for x in args(big)))
    for i, r in enumerate(ref):
        assert_equal(r, {k: v[i:i + 1] for k, v in host.items()}, ("host, eager", i))
    stream_in = [{k: (v.cpu().pin_memory() if k != "testing" else v) for k, v in as_batch([p]).items()} for p in pairs[:3]]
    for r, o in zip(ref, m.forward_stream(iter(stream_in))):
        assert_equal(r, {"final_trans": o["final_trans"], "final_labels": o["final_labels"]}, "forward_stream")
    many = m.forward_many([as_batch([p]) for p in pairs[:3]])
    for r, o in zip(ref, many):
        assert_equal(r, {"final_trans": o["final_trans"], "final_labels": o["final_labels"]}, "forward_many")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_run_eval_logits_and_M_at_bs1_equal_batch_of_8(precision):
    """The validation forward: logits and M per set.  Its transform depends on the batch by design (the early exit of the
    power iteration spans the batch, reference PointDSC.py:176), so it is not compared."""
    m = get_model(precision=precision, invariant=True)
    pairs = synth_sets([1000] * 8, seed0=800)
    batch = m.run_eval(*args(as_batch(pairs)))
    for i in (0, 5, 7):
        one = m.run_eval(*args(as_batch([pairs[i]])))
        assert torch.equal(one["final_labels"][0], batch["final_labels"][i]), i
        assert torch.equal(one["M"][0], batch["M"][i]), i


SM_SIZES = [1000, 5000, 257, 2000, 41]


def _dump(path, precisions):
    """Subprocess side of test_sm_count_does_not_matter: invariant-mode outputs of bs = 1 calls and one mixed call."""
    out = {}
    pairs = synth_sets(SM_SIZES, seed0=1200)
    for prec in precisions:
        m = get_model(precision=prec, invariant=True)
        for n, p in zip(SM_SIZES, pairs):
            r = m.run(*args(as_batch([p])), taps=TAPS)
            for k, v in r.items():
                out[f"{prec}/single/{n}/{k}"] = v.cpu().numpy()
        for n, o in zip(SM_SIZES, m.forward_many([as_batch([p]) for p in pairs])):
            out[f"{prec}/many/{n}/trans"] = o["final_trans"].cpu().numpy()
            out[f"{prec}/many/{n}/labels"] = o["final_labels"].cpu().numpy()
    np.savez(path, **out)


def test_sm_count_does_not_matter(tmp_path):
    real = torch.cuda.get_device_properties(0).multi_processor_count
    runs = {}
    for sms in (None, 66, 114):
        env = dict(os.environ)
        env.pop("PDSC_SM_COUNT", None)
        if sms is not None:
            env["PDSC_SM_COUNT"] = str(sms)
        path = tmp_path / f"sm_{sms}.npz"
        subprocess.run([sys.executable, os.path.abspath(__file__), str(path), ",".join(PRECISIONS)], env=env, check=True,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        runs[sms] = np.load(path)
    base = runs[None]
    assert len(base.files) > 0
    for sms in (66, 114):
        assert sorted(runs[sms].files) == sorted(base.files)
        for key in base.files:
            assert np.array_equal(runs[sms][key], base[key]), (sms, real, key)


def test_golden_fixtures_in_invariant_fp16x3():
    """The reference fixtures at bs = 1 in the invariant mode still meet the 1e-4 R/t bar (or, where the reference itself
    failed on tied hypotheses, keep at least its inlier count)."""
    groups = {}
    for path in golden_cases():
        c = load_case(path)
        groups.setdefault((c["meta"]["dataset"], int(c["meta"].get("k", 40))), []).append(c)
    assert len(groups) >= 2
    for (dataset, k), cases in groups.items():
        m = get_model(dataset, "fp16x3", k=k, invariant=True)
        for c in cases:
            b = {key: torch.from_numpy(np.ascontiguousarray(c[key])).cuda()[None] for key in ("corr_pos", "src_keypts", "tgt_keypts")}
            o = m.run(*args(b))
            T, labels = o["final_trans"][0].cpu().numpy(), o["final_labels"][0].cpu().numpy()
            R = T[:3, :3]
            assert np.abs(R @ R.T - np.eye(3)).max() < 1e-5 and abs(np.linalg.det(R) - 1) < 1e-5
            if not registration_ok(c):
                n = len(c["final_labels"])
                assert int((labels > 0.5).sum()) + 2 >= int(round(float(c["fitness"].max()) * n)), c["meta"]
                continue
            assert np.abs(T - c["final_trans"]).max() < 1e-4, c["meta"]
            assert (labels != c["final_labels"]).sum() <= 2, c["meta"]


def test_fp32_flag_changes_nothing():
    on, off = get_model(precision="fp32", invariant=True), get_model(precision="fp32")
    lib = on._ensure_engine()
    off._ensure_engine()
    for B, N in ((1, 1000), (256, 1000), (1, 16384)):
        assert lib.pdsc_workspace_bytes(on._engine, B, N) == lib.pdsc_workspace_bytes(off._engine, B, N)
        assert lib.pdsc_launches_per_forward(on._engine, B, N) == lib.pdsc_launches_per_forward(off._engine, B, N)
    pairs = synth_sets([1000, 5000, 41], seed0=1300)
    for p in pairs:
        b = as_batch([p])
        assert_equal(off.run(*args(b), taps=TAPS), on.run(*args(b), taps=TAPS), "fp32 eager")
        assert_equal(off.run(*args(b)), on.run(*args(b)), "fp32 graph")
    for x, y in zip(off.forward_many([as_batch([p]) for p in pairs]), on.forward_many([as_batch([p]) for p in pairs])):
        assert torch.equal(x["final_trans"], y["final_trans"]) and torch.equal(x["final_labels"], y["final_labels"])


def test_launch_count_reports_the_merges():
    """12 layers: the invariant mode merges wherever a set has more than TSI key tiles, whatever the call."""
    tsi = invariant_tiles()
    inv, dft = get_model(precision="fp16x3", invariant=True), get_model(precision="fp16x3")
    lib = inv._ensure_engine()
    dft._ensure_engine()

    def launches(m, B, N):
        return int(lib.pdsc_launches_per_forward(m._engine, B, N))

    assert launches(inv, 256, 1000) - launches(dft, 256, 1000) == (12 if 1000 > 64 * tsi else 0)   # default: large regime
    assert launches(inv, 256, 64 * tsi) == launches(dft, 256, 64 * tsi)                           # neither splits
    assert launches(inv, 256, 64 * tsi + 1) == launches(dft, 256, 64 * tsi) + 12


@pytest.mark.parametrize("precision", ["fp16x3"])
def test_toggling_the_mode_on_one_module(precision):
    m = get_model(precision=precision, fresh=True)
    fresh = {mode: get_model(precision=precision, invariant=mode, fresh=True) for mode in (False, True)}
    p = synth_sets([5000], seed0=1400)[0]
    b = as_batch([p])
    host = [x.cpu() for x in args(b)]
    want = {mode: (fm.run(*args(b), taps=["features"]), fm.run(*args(b)), fm.run(*host)) for mode, fm in fresh.items()}
    # the two modes really associate the attention differently at this size (bs = 1 at N = 5000: split by both, unequally)
    assert not torch.equal(want[False][0]["features"], want[True][0]["features"])
    for mode in (False, True, False, True):
        m.set_batch_invariant(mode)
        assert m.batch_invariant is mode
        eager = m.run(*args(b), taps=["features"])
        assert_equal(want[mode][0], eager, ("eager", mode))
        assert_equal(want[mode][1], m.run(*args(b)), ("graph", mode))
        assert_equal(want[mode][1], m.run(*args(b)), ("graph replay", mode))
        assert_equal(want[mode][2], m.run(*host), ("host", mode))


def test_evaluate_groups_equal_single_pairs_in_invariant_mode():
    import evaluate
    s1, _ = evaluate.main(["--synthetic", "4", "--batch_size", "1", "--batch_invariant"])
    s4, _ = evaluate.main(["--synthetic", "4", "--batch_size", "4", "--batch_invariant"])
    assert s1.shape == s4.shape == (4, len(evaluate.COLUMNS))
    keep = [i for i, c in enumerate(evaluate.COLUMNS) if c not in ("model_time_s", "data_time_s")]
    assert np.array_equal(s1[:, keep], s4[:, keep])


if __name__ == "__main__":
    _dump(sys.argv[1], sys.argv[2].split(","))
