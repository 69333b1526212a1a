"""The forward outside the released configuration: every layer count, input width and seed ratio `pdsc_create` accepts.

The released snapshots are 12 layers deep and take in_dim 6 at ratio 0.1; the engine accepts num_layers and in_dim in [1, 64]
and any finite ratio.  The encoder's chain sequence depends on the layer count (layer 0 runs PCQ, later layers Q; every layer
but the last ends in MSGPC, which reads the next layer's W1; the last ends in MSG), layer0_kernel has a register path up to
in_dim 8 and a generic loop above, and the seed count S follows the reference's slice argsort(...)[:, 0:int(N * ratio)].

  (a) Layer counts L in {1, 2, 6, 13, 64}, all four precisions: layer i holds layer i mod 12 of the 3DMatch snapshot, so every
      operand has a trained scale.  PCQ / Q, KV, the attention (+ merge) and MSG / MSGPC are checked against float64 within
      the bounds of float64_bounds.py, in both attention regimes (bs = 1 at N = 1000 splits the keys, B = 64 at N = 300
      does not); then the end-to-end result against the oracle and the batch against its single-set calls.  Repeating the
      snapshot's layers grows the features from block to block: beyond the first repetition the logits grow until the
      attention's a-posteriori bound is vacuous (its relative logit factor above 1/2: at layer 31 of 64 on an H100, and
      within 0.03 of it at layer 13 in bf16x3), and at L = 64 the fp32 rounding the stack amplifies moves the transform by
      1.5e-4 to 2.8e-4 with the same labels.  So L = 64 is bound-checked up to layer 11, whose MSGPC reads the W1 of
      layer 12, past a 12-layer arena; its last layer is checked through the layer_features tap, and it is not compared
      with the oracle.
  (b) Input widths in_dim in {1, 3, 6, 8, 9, 12, 64} (8: the last register-path width, 9: the first of the generic loop), with
      corr_pos built by the reference loader's formulas and a seeded xavier-normal layer 0; the host-input path at odd
      R * in_dim, which leaves src_keypts 4-byte aligned in its slot.
  (c) The seed ratio: the slice rule on the CPU and in pdsc_num_seeds, forwards at ratios whose float32 rounding changed S, at
      ratios 0, 1, above 1 and below 0, the refinement switch's exact comparison with 0.10, and S = N = 16384.

Measured on an H100 80GB HBM3 (700 W power limit), worst error / bound over this module's bound checks:
                 fp32     fp16x3   bf16x3   bf16
    PCQ          0.076    0.245    0.228    0.544
    KV           0.062    0.245    0.232    0.526
    attention    0.242    0.693    0.189    0.929
    MSG          0.0070   0.029    0.033    0.063
The module's GPU tests took 187 s there.
"""
import math

import numpy as np
import pytest
import torch

from conftest import load_snapshot
from engine_rules import C_CH, num_seeds
from float64_bounds import (ALL_PRECISIONS, E_KNN, WORST, check_power, check_sets, check_transforms, run_case,
                            weighted_kabsch64)
from gpu_models import get_model, release_all, sm_count
from oracle import pointdsc_oracle as O

SNAP_LAYERS = 12
PDSC_ERR_INVALID_ARGUMENT = 1


# ---------------------------------------------------------------------------------------------------
# modules of any depth and input width
# ---------------------------------------------------------------------------------------------------
def stretched_state(L, in_dim=6, seed=0):
    """The 3DMatch snapshot as the state dict of an L-layer module: layer i is snapshot layer i mod 12, the head is the
    snapshot's.  in_dim != 6: layer 0 is xavier-normal (as PointDSC.__init__ initialises it, gain 1) from `seed`, its bias
    Conv1d's default uniform(+-1 / sqrt(fan_in))."""
    snap = load_snapshot("3dmatch")
    sd = {k: v for k, v in snap.items() if not k.startswith("encoder.blocks.")}
    for i in range(L):
        for kind in ("PointCN", "NonLocal"):
            pre = f"encoder.blocks.{kind}_layer_{i % SNAP_LAYERS}."
            for k, v in snap.items():
                if k.startswith(pre):
                    sd[f"encoder.blocks.{kind}_layer_{i}." + k[len(pre):]] = v
    if in_dim != 6:
        g = torch.Generator().manual_seed(1000 + seed)
        sd["encoder.layer0.weight"] = torch.randn(C_CH, in_dim, 1, generator=g) * math.sqrt(2.0 / (in_dim + C_CH))
        sd["encoder.layer0.bias"] = (torch.rand(C_CH, generator=g) * 2 - 1) / math.sqrt(in_dim)
    return sd


_states = {}


def config_model(precision="fp32", L=SNAP_LAYERS, in_dim=6, ratio=0.1, inlier_threshold=0.10, invariant=False):
    """(module, state dict, name of the state dict in float64_bounds' weight cache)."""
    name = f"config-L{L}-in{in_dim}"
    if name not in _states:
        _states[name] = stretched_state(L, in_dim)
    m = get_model(precision=precision, invariant=invariant, num_layers=L, in_dim=in_dim, ratio=ratio,
                  inlier_threshold=inlier_threshold, weights=(name, _states[name]))
    return m, _states[name], name


def oracle_cfg(L=SNAP_LAYERS, ratio=0.1, inlier_threshold=0.10):
    return dict(O.default_config("3dmatch"), num_layers=L, ratio=ratio, inlier_threshold=inlier_threshold)


def pair_inputs(seeds, N, in_dim=6, inlier_ratio=0.5):
    """Synthetic 3DMatch pairs with corr_pos of width in_dim, built as the reference's loader builds it
    (datasets/ThreeDMatch.py:144-157): 3 = src - tgt, 6 = [src, tgt] centred, 9 = [src, tgt, src - tgt], 12 = [src, tgt] and two
    unit normals.  Other widths: the first in_dim columns of [src, tgt] centred followed by seeded Gaussian columns of the
    coordinates' scale.  Returns host tensors corr_pos [B,N,in_dim], src, tgt [B,N,3] and gt [B,4,4]."""
    from pointdsc_b200.synth import make_pair
    cps, ss, ts, gts = [], [], [], []
    for sd in seeds:
        p = make_pair(sd, N, "3dmatch", inlier_ratio)
        s, t = p["src_keypts"], p["tgt_keypts"]
        g = torch.Generator().manual_seed(77 + sd)
        if in_dim == 3:
            cp = s - t
        elif in_dim == 6:
            cp = p["corr_pos"]
        elif in_dim == 9:
            cp = torch.cat([s, t, s - t], -1)
        elif in_dim == 12:
            nrm = torch.randn(2, N, 3, generator=g)
            nrm = nrm / nrm.norm(dim=-1, keepdim=True)
            cp = torch.cat([s, t, nrm[0], nrm[1]], -1)
        else:
            extra = torch.randn(N, max(in_dim - 6, 0), generator=g) * float(p["corr_pos"].std())
            cp = torch.cat([p["corr_pos"], extra], -1)[:, :in_dim]
        cps.append(cp.float().contiguous())
        ss.append(s)
        ts.append(t)
        gts.append(p["gt_trans"])
    return torch.stack(cps), torch.stack(ss), torch.stack(ts), torch.stack(gts)


def check_vs_oracle(out, sd, cfg, cp, s, t, gt, what):
    """The rule of test_gpu_parity.test_ragged_sizes_vs_oracle, per set: where the oracle registers the pair, the transform
    within 1e-4 and at most 2 labels flipped.  The oracle's selected hypothesis must register the pair too: a refinement that
    reaches the ground truth from a wrong hypothesis (one inlier) is chaotic.  Returns the number of sets compared."""
    compared = 0
    for b in range(cp.shape[0]):
        ref = O.forward_testing(sd, cfg, cp[b], s[b], t[b])
        if max(float((ref[x] - gt[b]).abs().max()) for x in ("init_trans", "final_trans")) < 0.05:
            compared += 1
            dT = float((out["final_trans"][b].cpu() - ref["final_trans"]).abs().max())
            flips = int((out["final_labels"][b].cpu() != ref["final_labels"]).sum())
            assert dT < 1e-4 and flips <= 2, (what, b, dT, flips)
    return compared


def per_layer_launches(precision, split):
    return 8 if precision == "fp32" else (5 if split else 4)


def summary(tag):
    for key in sorted(WORST):
        print(f"{tag}: {key[0]} ({key[1]}) worst error / bound so far {WORST[key]:.3g}")


# ---------------------------------------------------------------------------------------------------
# (a) layer counts
# ---------------------------------------------------------------------------------------------------
# L = 13: the snapshot's last layer ending in MSGPC (11) and its first layer's weights ending in MSG (12); L = 64: layers
# of a deep stack, 11 ending in the MSGPC that reads layer 12's W1
LAYERS_CHECKED = {1: [0], 2: [0, 1], 6: list(range(6)), 13: [0, 1, 11, 12], 64: [0, 1, 2, 10, 11]}
REGIMES = [(1, 1000), (64, 300)]      # bs = 1: the key-split attention; B = 64: unsplit


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ALL_PRECISIONS)
@pytest.mark.parametrize("L", sorted(LAYERS_CHECKED))
def test_layer_count_against_float64(L, precision):
    m, sd, name = config_model(precision, L)
    ref12, _, _ = config_model(precision, SNAP_LAYERS)
    sms = sm_count()
    for B, N in REGIMES:
        sets = [0] if B == 1 else check_sets(B, N)
        split, per = run_case(name, precision, B, N, LAYERS_CHECKED[L], sets, model=m, sd=sd, args=regime_inputs(B, N, L))
        if precision != "fp32" and sms >= 132:
            assert split == (B == 1), (B, N, split)                 # both attention regimes are reached
        # each layer adds its chain launches, the attention and (split) its merge, and nothing else
        diff = m.launches_per_forward(B, N) - ref12.launches_per_forward(B, N)
        assert diff == per_layer_launches(precision, split) * (L - SNAP_LAYERS), (L, B, N, diff)
        # the last layer's layer_features tap is the encoder output the head reads
        args = regime_inputs(B, N, L)
        out = m.run(*args, taps=["features", "layer_features"], layer_tap=L - 1)
        assert torch.equal(out["features"], out["layer_features"])
    summary(f"L={L}")


def regime_inputs(B, N, L):
    cp, s, t, _ = pair_inputs([50000 + 1000 * L + 7 * N + b for b in range(B)], N, 6, 0.5)
    return [x.cuda() for x in (cp, s, t)]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "fp16x3"])
@pytest.mark.parametrize("L", [1, 2, 6, 13])
def test_layer_count_end_to_end(L, precision):
    m, sd, _ = config_model(precision, L)
    cp, s, t, gt = pair_inputs([900 + L, 901 + L], 1000, 6, 0.5)
    out = m.run(cp.cuda(), s.cuda(), t.cuda())
    compared = check_vs_oracle(out, sd, oracle_cfg(L), cp, s, t, gt, f"L={L}")
    print(f"L={L} ({precision}): {compared} of 2 sets registered by the oracle and compared")
    if L in (1, 6):
        # a batch is the loop of its single-set calls, bit for bit (both calls split the attention by N alone)
        cp, s, t, _ = pair_inputs(range(21, 26), 500, 6, 0.3)
        cp, s, t = cp.cuda(), s.cuda(), t.cuda()
        full = m.run(cp, s, t, taps=["power_iters", "seeds"])
        for b in range(cp.shape[0]):
            one = m.run(cp[b:b + 1], s[b:b + 1], t[b:b + 1], taps=["power_iters", "seeds"])
            for key in ("final_trans", "final_labels", "seeds", "power_iters"):
                assert torch.equal(one[key][0], full[key][b]), (L, b, key)


# ---------------------------------------------------------------------------------------------------
# (b) input widths
# ---------------------------------------------------------------------------------------------------
IN_DIMS = [1, 3, 6, 8, 9, 12, 64]      # layer0_kernel: registers for in_dim <= 8, the generic loop from 9


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ALL_PRECISIONS)
@pytest.mark.parametrize("in_dim", IN_DIMS)
def test_input_width_against_float64(in_dim, precision):
    """Layer 0 (float64 within gamma(in_dim + 1) sum |terms|, carried into PCQ's bound) and layer 1 as in (a); end to end
    against the oracle in fp32 and fp16x3."""
    m, sd, name = config_model(precision, SNAP_LAYERS, in_dim)
    cp, s, t, gt = pair_inputs([700 + in_dim, 701 + in_dim], 1000, in_dim, 0.5)
    run_case(name, precision, 1, 1000, [0, 1], [0], model=m, sd=sd, args=[x[:1].cuda() for x in (cp, s, t)])
    if precision in ("fp32", "fp16x3"):
        out = m.run(cp.cuda(), s.cuda(), t.cuda())
        compared = check_vs_oracle(out, sd, oracle_cfg(), cp, s, t, gt, f"in_dim={in_dim}")
        print(f"in_dim={in_dim} ({precision}): {compared} of 2 sets registered by the oracle and compared")
    summary(f"in_dim={in_dim}")


@pytest.mark.gpu
@pytest.mark.parametrize("in_dim", [3, 9])
def test_host_path_at_odd_widths(in_dim):
    """pdsc_forward_host and the submit / wait pair equal the device path bit for bit where R * in_dim is odd, so that the
    slot's src_keypts starts 4-byte aligned only: a graphed size and an eager one (R above the 32,768 graph rows)."""
    m, _, _ = config_model("fp16x3", SNAP_LAYERS, in_dim)
    for B, N in ((1, 1001), (3, 16383)):
        assert (B * N * in_dim) % 2 == 1
        cp, s, t, _ = pair_inputs(range(60 + B, 60 + 2 * B), N, in_dim, 0.5)
        devo = m.run(cp.cuda(), s.cuda(), t.cuda())
        pinned = [x.pin_memory() for x in (cp, s, t)]
        host = m.run(*pinned)
        streamed = list(m.forward_stream([{"corr_pos": pinned[0], "src_keypts": pinned[1], "tgt_keypts": pinned[2],
                                           "testing": True}] * 2))
        for got in [host] + streamed:
            assert torch.equal(got["final_trans"], devo["final_trans"].cpu()), (in_dim, B, N)
            assert torch.equal(got["final_labels"], devo["final_labels"].cpu()), (in_dim, B, N)
    release_all()


# ---------------------------------------------------------------------------------------------------
# (c) the seed ratio
# ---------------------------------------------------------------------------------------------------
# 0.35, 0.45, 0.7 and 0.9 lie above their float32 roundings: a float32 ratio loses a seed wherever N * ratio is an integer
RATIOS = [0, 0.05, 0.1, 0.35, 0.45, 0.7, 0.9, 1, 1.5, -0.1]


@pytest.mark.parametrize("ratio", RATIOS + [0.2, 2.0, -1.0, -2.5, 1e-9])
def test_seed_rule_is_the_slice(ratio):
    from pointdsc_b200 import PointDSC
    m = PointDSC(num_layers=1, ratio=ratio)
    for N in list(range(0, 2049)) + [16383, 16384]:
        assert m.num_seeds(N) == num_seeds(N, ratio), (N, ratio)
    assert PointDSC(num_layers=1, ratio=0.7).num_seeds(10) == 7 == int(10 * 0.7)
    assert int(10 * float(np.float32(0.7))) == 6                  # what a float32 ratio gives


def engine_config(ratio):
    from pointdsc_b200 import _capi
    return _capi.Config(6, 1, C_CH, 10, ratio, 0.10, 0.10, 40, 0.10, _capi.PRECISIONS["fp32"], 0)


@pytest.mark.gpu
def test_num_seeds_sweep_and_non_finite_ratios():
    """pdsc_num_seeds (no launch) against the slice rule for every N in [2, 16384]; NaN and infinite ratios refused."""
    import ctypes
    from pointdsc_b200 import _capi
    lib = _capi.load()
    Ns = np.arange(2, 16385)
    for ratio in RATIOS:
        h = ctypes.c_void_p()
        _capi.check(lib.pdsc_create(ctypes.byref(engine_config(ratio)), ctypes.byref(h)))
        try:
            got = np.array([lib.pdsc_num_seeds(h, int(n)) for n in Ns])
        finally:
            lib.pdsc_destroy(h)
        want = np.array([num_seeds(int(n), ratio) for n in Ns])
        bad = Ns[got != want]
        assert bad.size == 0, (ratio, bad.size, bad[:5].tolist(), got[got != want][:5].tolist())
    for ratio in (math.nan, math.inf, -math.inf):
        h = ctypes.c_void_p()
        assert lib.pdsc_create(ctypes.byref(engine_config(ratio)), ctypes.byref(h)) == PDSC_ERR_INVALID_ARGUMENT, ratio
        assert b"ratio" in lib.pdsc_last_error()


def check_seeds(got, want, key):
    """Seeds against the oracle's: the same key at every rank, the same index wherever a key is unique, and every class of tied
    keys the prefix holds entirely (suppressed rows tie at +-0) as the same set."""
    assert len(set(got.tolist())) == len(got) and ((got >= 0) & (got < len(key))).all()
    kg, kw = key[got], key[want]
    assert np.array_equal(kg, kw)                                    # +0 == -0
    for v in np.unique(kw):
        pos = kw == v
        if np.count_nonzero(key == v) == np.count_nonzero(pos):
            assert set(got[pos].tolist()) == set(want[pos].tolist()), v


RATIO_CASES = [(0.7, 10), (0.7, 1000), (0.35, 20), (1.0, 1000), (1.5, 1000), (-0.1, 1000)]


@pytest.mark.gpu
@pytest.mark.parametrize("ratio,N", RATIO_CASES)
def test_seed_ratio_forward_vs_oracle(ratio, N):
    m, sd, _ = config_model("fp32", ratio=ratio)
    S = num_seeds(N, ratio)
    assert S != int(N * float(np.float32(ratio))) or ratio in (1.0, 1.5, -0.1)   # float32 would change S, or a new range
    cfg = oracle_cfg(ratio=ratio)
    cp, s, t, gt = pair_inputs([300 + N], N, 6, 0.5)
    ref = O.forward_testing(sd, cfg, cp[0], s[0], t[0])
    assert ref["seeds"].shape == (S,)
    args = [x.cuda() for x in (cp, s, t)]
    # the seeds given the oracle's features and confidence
    inj = {"features": ref["features"][None].cuda(), "confidence": ref["confidence"][None].cuda()}
    got = m.run(*args, taps=["seeds"], inject=inj)["seeds"][0].cpu().numpy()
    key = (ref["confidence"] * O.local_max_mask(ref["src_dist"], ref["confidence"], cfg["nms_radius"]).float()).numpy()
    check_seeds(got, ref["seeds"].numpy(), key)
    if S == N:
        assert np.array_equal(np.sort(got), np.arange(N))
    # end to end: the seed count, the transform and the labels
    out = m.run(*args, taps=["seeds", "power_iters"])
    assert out["seeds"].shape == (1, S) and 1 <= int(out["power_iters"][0]) <= 10
    compared = check_vs_oracle(out, sd, cfg, cp, s, t, gt, f"ratio={ratio} N={N}")
    print(f"ratio={ratio} N={N}: S={S}, {compared} set(s) registered by the oracle and compared")


@pytest.mark.gpu
def test_ratio_zero_takes_no_seeds():
    """S = 0: no power iteration, the identity is the initial transform, the labels are its inliers and the refinement starts
    from it (the reference itself cannot score zero hypotheses)."""
    m, _, _ = config_model("fp32", ratio=0.0)
    cp, s, t, _ = pair_inputs([808], 1000, 6, 0.5)
    t = t.clone()
    t[0, :500] = s[0, :500] + 0.02 * torch.randn(500, 3, generator=torch.Generator().manual_seed(8))   # inliers of the identity
    assert m.num_seeds(1000) == 0
    out = m.run(cp.cuda(), s.cuda(), t.cuda(), taps=["power_iters", "init_trans", "refine_solves"])
    assert int(out["power_iters"][0]) == 0
    assert torch.equal(out["init_trans"][0].cpu(), torch.eye(4))
    d = np.linalg.norm(s[0].double().numpy() - t[0].double().numpy(), axis=1)
    assert np.array_equal(out["final_labels"][0].cpu().numpy() > 0.5, d < 0.10)
    T, solves = O.post_refinement(torch.eye(4), s[0], t[0], 0.10)
    assert int(out["refine_solves"][0]) == solves >= 1
    assert float((out["final_trans"][0].cpu() - T).abs().max()) < 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [1.0, 1.5])
def test_validation_seeds_are_every_row(ratio):
    """The validation forward's seeds at ratio >= 1: all N rows, in confidence order (ties by index)."""
    m, _, _ = config_model("fp32", ratio=ratio)
    N = 300
    cp, s, t, _ = pair_inputs([41, 42], N, 6, 0.5)
    out = m.run_eval(cp.cuda(), s.cuda(), t.cuda(), want_M=False, taps=["seeds"])
    for b in range(2):
        seeds = out["seeds"][b].cpu().numpy()
        conf = out["final_labels"][b].cpu().numpy()
        assert np.array_equal(seeds, np.lexsort((np.arange(N), -conf)))


@pytest.mark.gpu
def test_refinement_switch_is_an_exact_comparison():
    """inlier_threshold = 0.1 + 1e-9 scores at float32 0.1, as the reference's float32 comparison does, and refines at 1.2,
    as `self.inlier_threshold == 0.10` decides; exactly 0.10 refines at 0.10."""
    near = 0.1 + 1e-9
    assert np.float32(near) == np.float32(0.1) and near != 0.10
    cp, s, t, gt = pair_inputs([606], 1000, 6, 0.5)
    args = [x.cuda() for x in (cp, s, t)]
    taps = ["inlier_counts", "init_trans", "refine_solves"]
    a = config_model("fp32", inlier_threshold=near)[0].run(*args, taps=taps)
    b = config_model("fp32", inlier_threshold=0.10)[0].run(*args, taps=taps)
    assert torch.equal(a["inlier_counts"], b["inlier_counts"]) and torch.equal(a["init_trans"], b["init_trans"])
    init = a["init_trans"][0].cpu()
    refs = {}
    for out, thr, tau in ((a, near, 1.2), (b, 0.10, 0.10)):
        assert O.refinement_threshold(thr) == tau
        T, solves = O.post_refinement(init, s[0], t[0], thr)
        refs[tau] = (T, solves)
        assert int(out["refine_solves"][0]) == solves, (thr, int(out["refine_solves"][0]), solves)
        assert float((out["final_trans"][0].cpu() - T).abs().max()) < 1e-4, thr
    # the two refinements differ, so the comparison decides the result
    (T12, n12), (T10, n10) = refs[1.2], refs[0.10]
    assert n12 != n10 or float((T12 - T10).abs().max()) > 1e-3
    # and the oracle's whole forward at 0.1 + 1e-9 agrees where it registers the pair
    sd = config_model("fp32", inlier_threshold=near)[1]
    assert check_vs_oracle(a, sd, oracle_cfg(inlier_threshold=near), cp, s, t, gt, "near 0.10") == 1


@pytest.mark.gpu
def test_every_row_a_seed_at_16384():
    """fp16x3, ratio 1, N = 16384: 16,384 seeds (a 1 GiB seed-row distance block).  kNN and the hypotheses of 64 sampled seeds
    and the power iteration of all of them against float64 (the rules of float64_bounds.py)."""
    release_all()
    N, k = 16384, 40
    m, _, _ = config_model("fp16x3", ratio=1.0)
    cp, s, t, _ = pair_inputs([4242], N, 6, 0.3)
    out = m.run(cp.cuda(), s.cuda(), t.cuda(),
                taps=["normed", "seeds", "knn_idx", "compat", "eig", "power_iters", "seed_trans"])
    seeds = out["seeds"][0].cpu().numpy().astype(np.int64)
    assert np.array_equal(np.sort(seeds), np.arange(N))
    pick = np.sort(np.random.default_rng(N).choice(N, 64, replace=False))
    pick[-1] = N - 1                                                    # the last seed slot
    nm = out["normed"][0].cpu().numpy().astype(np.float64)
    got = out["knn_idx"][0].cpu().numpy().astype(np.int64)[pick]
    assert all(len(set(r)) == k for r in got) and (got >= 0).all() and (got < N).all()
    dist = 2.0 - 2.0 * (nm[seeds[pick]] @ nm.T)
    order = np.argsort(dist, axis=1, kind="stable")
    ref = order[:, 1:k + 1]
    d_got, d_ref = np.take_along_axis(dist, got, 1), np.take_along_axis(dist, ref, 1)
    assert np.abs(d_got - d_ref).max() <= 2 * E_KNN
    full = np.take_along_axis(dist, order[:, :k + 2], 1)
    sep = (full[:, 1:k + 1] - full[:, 0:k] > 2 * E_KNN) & (full[:, 2:k + 2] - full[:, 1:k + 1] > 2 * E_KNN)
    assert sep.mean() > 0.2 and np.array_equal(got[sep], ref[sep])
    compat = out["compat"][0].cpu().numpy().reshape(N, k, k)
    eig = out["eig"][0].cpu().numpy().reshape(N, k)
    ratio, band, sure = check_power(compat, eig, int(out["power_iters"][0]), k, 10)
    src, tgt = s[0].double().numpy(), t[0].double().numpy()
    e = eig[pick].astype(np.float64)
    kab = weighted_kabsch64(src[got], tgt[got], e / (e.sum(1, keepdims=True) + 1e-6))
    check_transforms(out["seed_trans"][0].cpu().numpy()[pick], kab, "seed_trans N=16384 S=16384")
    print(f"N=S=16384: power iteration worst error / bound {ratio:.3g} (band {band:.3g}), exit compared: {sure}")
    release_all()
