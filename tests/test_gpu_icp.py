"""Device ICP (pointdsc_b200.icp, csrc/icp.cu) against the float64 CPU restatement oracle/icp_oracle.py, on the packed interface
the evaluation loop uses, plus its memory, graph and error contracts and the evaluate.py --use_icp loop.

Parity is exact in the discrete decisions (iterations, fitness) and to rounding in the rest (rmse 1e-12 relative, T within 2 float32
ulps per entry).  That holds for a run whose every decision is further than rounding from its threshold: the oracle records the
margins (|d^2 - r^2_f|, the nearest / next distinct target gap, the |d rmse| criterion, sigma_2 / sigma_1 of every update) and each
case asserts they all exceed 1e-9.  The seeds below were chosen so that every case qualifies."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_snapshot
from gpu_models import ulps
from oracle import icp_oracle as O

pytestmark = pytest.mark.gpu

MARGIN = 1e-9
# (preset, N, seed) of pointdsc_b200.synth.make_pair: 3DMatch-like and KITTI-like correspondence sets
CASES = [("3dmatch", 2, 0), ("3dmatch", 41, 0), ("3dmatch", 1000, 0), ("3dmatch", 5000, 2), ("3dmatch", 12000, 2),
         ("kitti", 2, 2), ("kitti", 41, 0), ("kitti", 1000, 0), ("kitti", 5000, 0), ("kitti", 12000, 1)]


def _pair(preset, n, seed):
    from pointdsc_b200.synth import make_pair
    p = make_pair(seed, n, preset)
    return p["src_keypts"].numpy(), p["tgt_keypts"].numpy(), p["gt_trans"].numpy().astype(np.float32)


def _perturb(T, seed, deg=3.0, cm=3.0):
    """T composed with a rotation of `deg` degrees about a random axis and a translation of `cm` centimetres."""
    g = np.random.default_rng(seed)
    ax = g.normal(size=3)
    ax /= np.linalg.norm(ax)
    a = np.deg2rad(deg)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    P = np.eye(4)
    P[:3, :3] = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
    P[:3, 3] = g.normal(size=3) * cm / 100 / np.sqrt(3)
    return (P @ T.astype(np.float64)).astype(np.float32)


def _device(src, tgt, init, offsets=None, **kw):
    """icp_refine_packed with info on numpy inputs; returns numpy (trans [B,4,4], fitness, rmse, iterations, status)."""
    from pointdsc_b200.icp import icp_refine_packed
    init = np.asarray(init, np.float32).reshape(-1, 4, 4)
    if offsets is None:
        offsets = [0, len(src)]
    out, info = icp_refine_packed(torch.from_numpy(np.ascontiguousarray(src)).cuda(), torch.from_numpy(np.ascontiguousarray(tgt)).cuda(),
                                  torch.from_numpy(init).cuda(), offsets, info=True, **kw)
    torch.cuda.synchronize()
    return (out.cpu().numpy(), info["fitness"].cpu().numpy(), info["inlier_rmse"].cpu().numpy(), info["iterations"].cpu().numpy(),
            info["status"].cpu().numpy())


def _check(dev, b, ref):
    trans, fit, rmse, its, status = dev
    assert O.margin(ref) > MARGIN, ref["margins"]
    assert int(status[b]) == ref["status"]
    assert int(its[b]) == ref["iterations"], (int(its[b]), ref["iterations"])
    assert float(fit[b]) == ref["fitness"]
    assert abs(float(rmse[b]) - ref["inlier_rmse"]) <= 1e-12 * ref["inlier_rmse"]
    assert ulps(trans[b], ref["trans"]).max() <= 2, (trans[b], ref["trans"])


# ---------------------------------------------------------------------------------------------------
# 1. parity with the oracle
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("start", ["gt", "perturbed"])
@pytest.mark.parametrize("preset,n,seed", CASES, ids=[f"{p}-n{n}-s{s}" for p, n, s in CASES])
def test_parity_with_oracle(preset, n, seed, start):
    src, tgt, gt = _pair(preset, n, seed)
    init = gt if start == "gt" else _perturb(gt, seed)
    _check(_device(src, tgt, init), 0, O.icp(src, tgt, init))


def test_parity_demo_pair():
    z = np.load(os.path.join(GOLDEN, "demo_pair_3dmatch.npz"))
    ref = O.icp(z["src_keypts"], z["tgt_keypts"], z["final_trans"])
    assert ref["iterations"] == 9
    _check(_device(z["src_keypts"], z["tgt_keypts"], z["final_trans"]), 0, ref)


@pytest.fixture(scope="module")
def model_3dmatch():
    from pointdsc_b200 import PointDSC
    m = PointDSC(in_dim=6, num_layers=12, num_channels=128, num_iterations=10, ratio=0.1, inlier_threshold=0.10, sigma_d=0.10, k=40,
                 nms_radius=0.10)
    m.load_state_dict(load_snapshot("3dmatch"), strict=False)
    return m.cuda().eval()


@pytest.mark.parametrize("n,seed", [(1000, 0), (5000, 2)])
def test_parity_from_the_models_transform(model_3dmatch, n, seed):
    from pointdsc_b200.synth import make_pair
    p = make_pair(seed, n, "3dmatch")
    out = model_3dmatch({"corr_pos": p["corr_pos"][None].cuda(), "src_keypts": p["src_keypts"][None].cuda(),
                         "tgt_keypts": p["tgt_keypts"][None].cuda(), "testing": True})
    init = out["final_trans"][0].cpu().numpy()
    src, tgt = p["src_keypts"].numpy(), p["tgt_keypts"].numpy()
    _check(_device(src, tgt, init), 0, O.icp(src, tgt, init))


# ---------------------------------------------------------------------------------------------------
# 2. early iterations: the cap
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cap", [1, 2, 3])
@pytest.mark.parametrize("preset,n,seed", [("3dmatch", 1000, 0), ("3dmatch", 5000, 2)])
def test_iteration_cap(preset, n, seed, cap):
    src, tgt, gt = _pair(preset, n, seed)
    init = _perturb(gt, seed)
    ref = O.icp(src, tgt, init, max_iteration=cap)
    assert ref["iterations"] == cap
    _check(_device(src, tgt, init, max_iteration=cap), 0, ref)


# ---------------------------------------------------------------------------------------------------
# 3. a set's result is its own: packed == alone == reversed order, bit for bit
# ---------------------------------------------------------------------------------------------------
def _group():
    sets = []
    for preset, n, seed in [("3dmatch", 41, 0), ("3dmatch", 1000, 0), ("kitti", 1000, 0), ("3dmatch", 2, 0), ("3dmatch", 5000, 2),
                            ("3dmatch", 257, 3)]:
        s, t, gt = _pair(preset, n, seed)
        sets.append((s, t, _perturb(gt, seed)))
    s, t, gt = _pair("3dmatch", 1, 5)
    sets.insert(2, (s, t, gt))                                      # N = 1
    s, t, gt = _pair("3dmatch", 300, 6)
    sets.insert(4, (s, t + 100.0, gt))                              # no correspondence within 0.10
    s, t, gt = _pair("3dmatch", 120, 7)
    t = t.copy()
    t[17, 1] = np.nan
    sets.insert(6, (s, t, gt))                                      # status 1
    return sets


def _run_group(sets):
    off = np.cumsum([0] + [len(s) for s, _, _ in sets]).tolist()
    return _device(np.concatenate([s for s, _, _ in sets]), np.concatenate([t for _, t, _ in sets]), np.stack([i for _, _, i in sets]),
                   off)


def test_packed_equals_alone_and_reversed():
    sets = _group()
    assert len(sets) == 9
    packed = _run_group(sets)
    rev = _run_group(sets[::-1])
    for b, st in enumerate(sets):
        alone = _run_group([st])
        for k in range(5):
            assert np.array_equal(packed[k][b], alone[k][0], equal_nan=True), (b, k)
            assert np.array_equal(packed[k][b], rev[k][len(sets) - 1 - b], equal_nan=True), (b, k)
    trans, fit, rmse, its, status = packed
    assert list(status) == [0, 0, 0, 0, 0, 0, 1, 0, 0]
    assert np.array_equal(trans[6], sets[6][2]) and its[6] == 0
    assert fit[4] == 0.0 and rmse[4] == 0.0 and its[4] == 1 and np.array_equal(trans[4], sets[4][2])
    assert its[2] >= 1 and fit[2] in (0.0, 1.0)
    for b, (s, t, i) in enumerate(sets):
        if b != 6 and O.margin(O.icp(s, t, i)) > MARGIN:
            _check(packed, b, O.icp(s, t, i))


def test_icp_refine_equals_packed():
    from pointdsc_b200.icp import icp_refine, icp_refine_packed
    pairs = [_pair("3dmatch", 500, s) for s in (0, 1, 2)]
    src = torch.from_numpy(np.stack([p[0] for p in pairs])).cuda()
    tgt = torch.from_numpy(np.stack([p[1] for p in pairs])).cuda()
    init = torch.from_numpy(np.stack([_perturb(p[2], i) for i, p in enumerate(pairs)])).cuda()
    a = icp_refine(src, tgt, init)
    b = icp_refine_packed(src.reshape(-1, 3), tgt.reshape(-1, 3), init, [0, 500, 1000, 1500])
    assert a.shape == (3, 4, 4) and torch.equal(a, b)
    one = icp_refine(src[1:2], tgt[1:2], init[1:2])
    assert torch.equal(one[0], a[1])


# ---------------------------------------------------------------------------------------------------
# 4. memory contract (C ABI): scratch of exactly the reported size, poisoned; outputs guarded by NaN slack
# ---------------------------------------------------------------------------------------------------
def _raw_call(src, tgt, init, off, d_off, scratch, nbytes, outs, r=0.10, max_iteration=30):
    from pointdsc_b200 import _capi
    lib = _capi.load()
    eng = _capi.utility_engine(0)
    h = (C.c_int32 * len(off))(*off)
    trans, fit, rmse, its, status = outs
    return lib.pdsc_icp_packed(eng, len(off) - 1, h, C.c_void_p(d_off.data_ptr()), C.c_void_p(src.data_ptr()), C.c_void_p(tgt.data_ptr()),
                               C.c_void_p(init.data_ptr()), float(r), int(max_iteration), C.c_void_p(trans.data_ptr()),
                               C.c_void_p(fit.data_ptr()) if fit is not None else None,
                               C.c_void_p(rmse.data_ptr()) if rmse is not None else None,
                               C.c_void_p(its.data_ptr()) if its is not None else None,
                               C.c_void_p(status.data_ptr()) if status is not None else None,
                               C.c_void_p(scratch) if scratch is not None else None, nbytes,
                               C.c_void_p(torch.cuda.current_stream().cuda_stream))


def _group_tensors(sets):
    off = np.cumsum([0] + [len(s) for s, _, _ in sets]).tolist()
    src = torch.from_numpy(np.concatenate([s for s, _, _ in sets])).cuda()
    tgt = torch.from_numpy(np.concatenate([t for _, t, _ in sets])).cuda()
    init = torch.from_numpy(np.stack([i for _, _, i in sets])).cuda()
    return off, torch.tensor(off, dtype=torch.int32, device="cuda"), src, tgt, init


def test_memory_contract():
    from pointdsc_b200 import _capi
    sets = _group()
    off, d_off, src, tgt, init = _group_tensors(sets)
    B = len(sets)
    need = int(_capi.load().pdsc_icp_packed_scratch_bytes(B, (C.c_int32 * (B + 1))(*off)))
    assert need > 0
    ref = _run_group(sets)
    slack = 64
    for fill in ("zeros", "ones", "nan"):
        scratch = torch.empty(need + 2 * slack, dtype=torch.uint8, device="cuda")
        if fill == "zeros":
            scratch.zero_()
        elif fill == "ones":
            scratch.fill_(0xFF)
        else:
            scratch.view(torch.float32).fill_(float("nan"))
        guard = scratch.clone()
        bufs = [torch.full((B * 16 + 2 * slack,), float("nan"), device="cuda"),
                torch.full((B + 2 * slack,), float("nan"), dtype=torch.float64, device="cuda"),
                torch.full((B + 2 * slack,), float("nan"), dtype=torch.float64, device="cuda"),
                torch.full((B + 2 * slack,), -7, dtype=torch.int32, device="cuda"),
                torch.full((B + 2 * slack,), -7, dtype=torch.int32, device="cuda")]
        outs = [x[slack:slack + (B * 16 if k == 0 else B)] for k, x in enumerate(bufs)]
        assert _raw_call(src, tgt, init, off, d_off, scratch.data_ptr() + slack, need, outs) == 0
        torch.cuda.synchronize()
        got = [outs[0].view(B, 4, 4)] + outs[1:]
        for k in range(5):
            assert np.array_equal(got[k].cpu().numpy(), ref[k], equal_nan=True), (fill, k)
        for x in bufs:
            head, tail = x[:slack], x[-slack:]
            assert (torch.isnan(head).all() and torch.isnan(tail).all()) if x.is_floating_point() else \
                bool((head == -7).all() and (tail == -7).all())
        assert torch.equal(scratch[:slack], guard[:slack]) and torch.equal(scratch[slack + need:], guard[slack + need:])


# ---------------------------------------------------------------------------------------------------
# 5. CUDA graph capture and repeats
# ---------------------------------------------------------------------------------------------------
def test_graph_replay_and_repeats_are_bit_identical():
    from pointdsc_b200 import _capi
    sets = _group()
    off, d_off, src, tgt, init = _group_tensors(sets)
    B = len(sets)
    need = int(_capi.load().pdsc_icp_packed_scratch_bytes(B, (C.c_int32 * (B + 1))(*off)))
    scratch = torch.empty(need, dtype=torch.uint8, device="cuda")

    def outs():
        return [torch.empty(B, 4, 4, device="cuda"), torch.empty(B, dtype=torch.float64, device="cuda"),
                torch.empty(B, dtype=torch.float64, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda"),
                torch.empty(B, dtype=torch.int32, device="cuda")]
    eager = outs()
    assert _raw_call(src, tgt, init, off, d_off, scratch.data_ptr(), need, eager) == 0
    again = outs()
    assert _raw_call(src, tgt, init, off, d_off, scratch.data_ptr(), need, again) == 0
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(eager[:1] + eager[3:], again[:1] + again[3:]))
    assert all(np.array_equal(a.cpu().numpy(), b.cpu().numpy(), equal_nan=True) for a, b in zip(eager[1:3], again[1:3]))
    graphed = outs()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            assert _raw_call(src, tgt, init, off, d_off, scratch.data_ptr(), need, graphed) == 0
    torch.cuda.current_stream().wait_stream(s)
    for x in graphed:
        x.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, graphed):
        assert np.array_equal(a.cpu().numpy(), b.cpu().numpy(), equal_nan=True)


# ---------------------------------------------------------------------------------------------------
# 6. errors are loud, in C and in Python
# ---------------------------------------------------------------------------------------------------
def test_errors():
    from pointdsc_b200 import _capi
    from pointdsc_b200.icp import icp_refine, icp_refine_packed
    lib = _capi.load()
    sets = _group()[:3]
    off, d_off, src, tgt, init = _group_tensors(sets)
    B = len(sets)
    need = int(lib.pdsc_icp_packed_scratch_bytes(B, (C.c_int32 * (B + 1))(*off)))
    scratch = torch.empty(need + 16, dtype=torch.uint8, device="cuda")
    base = scratch.data_ptr()
    outs = [torch.empty(B, 4, 4, device="cuda"), None, None, None, None]
    assert _raw_call(src, tgt, init, off, d_off, base, need, outs) == 0
    # shapes
    assert _raw_call(src, tgt, init, [0, 5, 5, off[-1]], d_off, base, need, outs) == 3
    assert _raw_call(src, tgt, init, [1, 5, 9, off[-1]], d_off, base, need, outs) == 3
    assert lib.pdsc_icp_packed_scratch_bytes(3, (C.c_int32 * 4)(0, 5, 5, 9)) == 0
    assert lib.pdsc_icp_packed_scratch_bytes(0, (C.c_int32 * 1)(0)) == 0
    # arguments
    for r in (0.0, -0.1, float("nan"), float("inf")):
        assert _raw_call(src, tgt, init, off, d_off, base, need, outs, r=r) == 1, r
    assert _raw_call(src, tgt, init, off, d_off, base, need, outs, max_iteration=0) == 1
    # scratch
    assert _raw_call(src, tgt, init, off, d_off, base, need - 1, outs) == 5
    assert _raw_call(src, tgt, init, off, d_off, base + 4, need, outs) == 5
    assert _raw_call(src, tgt, init, off, d_off, None, need, outs) == 5
    assert "pdsc_icp_packed" in lib.pdsc_last_error().decode()
    # Python
    with pytest.raises(_capi.PdscError):
        icp_refine_packed(src, tgt, init, off, max_correspondence_distance=0.0)
    with pytest.raises(_capi.PdscError):
        icp_refine_packed(src, tgt, init, off, max_iteration=0)
    with pytest.raises(ValueError):
        icp_refine_packed(src, tgt, init, [0, 5, 5, off[-1]])
    with pytest.raises(ValueError):
        icp_refine_packed(src[1:], tgt[1:], init, off)
    with pytest.raises(ValueError):
        icp_refine(src[None], tgt[None, :-1], init[:1])
    with pytest.raises(_capi.PdscError):
        icp_refine_packed(src.cpu(), tgt.cpu(), init.cpu(), off)


# ---------------------------------------------------------------------------------------------------
# 7. evaluate.py --use_icp on synthetic pairs
# ---------------------------------------------------------------------------------------------------
def test_evaluate_use_icp():
    import evaluate
    from pointdsc_b200.frontend import match
    from pointdsc_b200.icp import icp_refine
    from pointdsc_b200.metrics import eval_stats
    flags = ["--synthetic", "4", "--batch_invariant"]
    s1, _ = evaluate.main(flags + ["--batch_size", "1", "--use_icp"])
    s4, _ = evaluate.main(flags + ["--batch_size", "4", "--use_icp"])
    plain, _ = evaluate.main(flags + ["--batch_size", "1"])
    cols = [c for c in range(len(evaluate.COLUMNS)) if c not in (9, 10)]
    assert np.array_equal(s1[:, cols], s4[:, cols])
    assert np.array_equal(s1[:, 3:9], plain[:, 3:9])                  # the labels stay the network's
    assert (np.abs(s1[:, 1:3] - plain[:, 1:3]) > 0).any()             # ICP moves RE / TE on at least one pair
    cfg = evaluate.load_config("PointDSC_3DMatch_release")
    model = evaluate.build_model("PointDSC_3DMatch_release", cfg, "cuda", batch_invariant=True)
    for p, (_, (sx, sd), (tx, td), gt) in enumerate(evaluate.synthetic_pairs(4, "cuda", 1.6 * cfg["downsample"])):
        data = match(sd, td, sx, tx)
        gt_t = torch.from_numpy(np.asarray(gt, dtype=np.float32)).cuda()
        labels = evaluate.gt_labels(data, gt_t, cfg["inlier_threshold"])
        data["testing"] = True
        res = model(data)
        row = eval_stats(icp_refine(data["src_keypts"], data["tgt_keypts"], res["final_trans"]), gt_t[None], data["src_keypts"],
                         data["tgt_keypts"], res["final_labels"], labels, re_thre=cfg["re_thre"], te_thre=cfg["te_thre"])
        row = row.double().cpu().numpy()[0]
        assert np.array_equal(s1[p, :9], row[:9]) and s1[p, 12] == row[9], p
