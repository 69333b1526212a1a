"""The encoder's kernels against float64 on their own inputs, on every launch path they take: the 1x1-convolution chains
(tc_chain<PCQ / KV / MSG> in csrc/tc_chain.cuh, the SIMT `linear` in csrc/encoder_simt.cu), the attention (the persistent
tensor-core kernel and its key-split merge in csrc/tc_attention_p.cuh, the SIMT attention) and layer0.  The GPU tests need an
H100 (`-m gpu`); the CPU rehearsal at the end runs everywhere and checks the bound functions against emulated kernels.

Every layer l is driven through `PointDSC.run` taps: `layer_features` (layer l's output; layer l - 1's, from a second call, is
layer l's input, since forwards are bit-deterministic), `layer_debug` (feat1, q, k, v, msg: in the tensor-core modes q / k / v
are the decoded operand images hi + lo, q carries log2(e) / sqrt(C)) and `sc`.  Layer 0's input is the float64 layer0 of
corr_pos, its fp32 error bounded below.  Each kernel is compared with its own operation in float64 on the tapped fp32
inputs: the BatchNorm fold of oracle._lin + oracle._bn (checked against them on the CPU), and the SC-weighted softmax.  The
tests assert the attention regime, sp, TS and virtual-tile count they reach, from the split rules of sets.cuh as
engine_rules.py restates them and the SM count the engine sizes its launches for (PDSC_SM_COUNT).

Error model (float64_bounds.py implements it).  u = 2^-24; gamma(n) = n u / (1 - n u).  Every bound is a posteriori: float64
sums of the actual |terms| of a row.
  * Operand unit of a 16-bit format: uh = 2^-11 (fp16, 11-bit significand), 2^-8 (bf16).  x = hi + lo + r with
    |r| <= uh^2 |x| + fl in the x3 modes (fl = 2^-25 for fp16, whose lo part is subnormal below 2^-14; 0 for bf16) and
    |x - hi| <= uh |x| + fl in single bf16.  |lo| <= (uh |x| + fl)(1 + uh).
  * Weights: the engine folds BatchNorm in double, rounds to fp32 (engine.cu fold_conv), scales Q's in double by the fp32
    constant log2(e) / sqrt(C) and rounds again, then splits (encoder_tc.cu build_image).  The tests rebuild these images in
    numpy; |W64 - image| enters per weight.  The reference for q is the fold with that constant.
  * wgmma: products of 16-bit operands are exact.  The fp32 accumulation is not documented; the model, an ASSUMPTION, is
    that each k-step (16 products and the accumulator) returns their exact sum with an error of at most 2 ulps of the sum of
    their magnitudes (any rounding direction, plus one unit lost in alignment): 4 u (|acc| + sum |products|).  A contraction
    of `steps` k-steps over terms whose magnitudes sum to S is then within G(steps) S, G(s) = 4 u (s + 1) / (1 - 4 u (s + 1)).
    Hardware that aligns every term to the largest one's 24-bit window and truncates (as published measurements describe
    for earlier tensor cores) can lose up to one window ulp per term, about 17 ulps per k-step in the worst case, which this
    model does not cover.  The CPU rehearsal emulates that truncation too: on realistic operands it stays within the bounds
    (worst 0.38 of a chain bound, 0.57 of an attention bound), which is evidence, not proof.
  * SIMT fp32: fma chains, round to nearest: gamma(n) sum |terms|.  A single add / multiply / division: u.
  * The MSG chain's hidden activations are not tapped: their errors reach the output linearly through the composite
    W2 Theta1 W1 of the ReLU secant slopes (fc_message64), which keeps the cancellation inside the weights, so a GEMM of the
    chain that loses a cross product (x_lo w_hi) breaks the bound (CPU rehearsal: 3-6 times it).
  * The x3 contractions drop lo*lo: bounded by sum |a_lo| |w_lo| (|q_lo|, |k_lo|, |v_lo| exactly, by re-splitting the decoded
    images).
  * ex2.approx.ftz.f32 and expf: relative error 2^-22 (the PTX ISA's 2 ulp); FTZ only flushes results below 2^-126.
  * Attention.  Logits t = SC (q . k) (log2 units) with their bound Et; a kernel P_j = 2^(t_j - m) is the float64 one times
    (1 + delta_j), delta_j from Et_j, the rounding of t_j - m and ex2.  O and l share these factors, and the rescale factors
    of the online softmax multiply both alike, so the shared part enters as sum_j P_j delta_j |v_j - msg| / l.  O alone sees
    the P split (x3: (uh^2 P_j + fl) |v_j| + (uh P_j + fl) |v_lo_j| per key, bf16: uh P_j |v_j|; P is relative to the running
    maximum, so the final-frame P_j and the full floor are an upper bound) and the accumulation, 12 (4) k-steps per key tile
    whose accumulator is bounded by the tile prefix of sum P |v|, plus one rounding per rescale.  l: gamma(N + 6 tiles + 8);
    the final division 2 u.  The merge: each split's weight carries 2^-22 + ln2 u |m_s - m*|, its fma sums gamma(sp).

Measured on an H100 80GB HBM3 (700 W power limit), worst error / bound over every GPU test of this module (PCQ, KV and
attention were the same on a 400 W card):
                 fp32     fp16x3   bf16x3   bf16
    PCQ          0.061    0.253    0.265    0.491
    KV           0.054    0.256    0.236    0.529
    attention    0.231    0.918    0.271    0.892
    MSG          0.011    0.033    0.055    0.073
In fp16x3 the P floor makes up nearly all of the attention bound in the rows where that bound is tightest (share up to 0.98);
the module's GPU tests took 292 s there.
"""
import numpy as np
import pytest
import torch

from conftest import load_snapshot
from engine_rules import attn_set_split, call_split
from float64_bounds import (ALL_PRECISIONS, UNIT, attention_bound, check_sets, conv_bound, fc_message64, layer_convs,
                            run_case, split16)
from gpu_models import sm_count
from oracle import pointdsc_oracle as O


def tile_rows(N):
    """Query rows of the first, a middle and the last query tile."""
    QT = -(-N // 128)
    return np.concatenate([np.arange(t * 128, min(t * 128 + 128, N)) for t in sorted({0, QT // 2, QT - 1})])


# ---------------------------------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------------------------------
# The measured worst ratios are in the module docstring; each test prints the worst ratio per kernel so far.
@pytest.mark.gpu
@pytest.mark.parametrize("precision", ALL_PRECISIONS)
@pytest.mark.parametrize("dataset", ["3dmatch", "kitti"])
def test_all_layers_bs1(dataset, precision):
    """All 12 layers of one set of N = 1000 in every precision (bs = 1: one chain tile per CTA, the split regime)."""
    split, per = run_case(dataset, precision, 1, 1000, range(12), [0])
    if precision != "fp32":
        assert split == (attn_set_split(1000, sm_count())[0] > 1)


SPLIT_N = [257, 513, 1000, 3000, 5000]
SPLIT_AT_132 = {257: (3, 1), 513: (5, 1), 1000: (8, 0), 3000: (6, 1), 5000: (4, 1)}   # N: (sp, virtual tiles) at 132 SMs


@pytest.mark.gpu
@pytest.mark.parametrize("dataset", ["3dmatch", "kitti"])
def test_key_split_attention(dataset):
    """bs = 1 in the split regime: the merge with sp % 4 != 0 (its clamped re-read) and chunks ending in virtual tiles."""
    sms = sm_count()
    reached = []
    for N in SPLIT_N:
        if not call_split([N], sms, False)[0]:
            assert sms < 132, N                                # too few SMs for this N to split (PDSC_SM_COUNT)
            continue
        split, per = run_case(dataset, "fp16x3", 1, N, [0, 6, 11], [0], qrows=tile_rows(N) if N > 1000 else None)
        sp, TS = per[0]
        assert split and sp > 1, (N, per)
        if sms == 132:
            assert (sp, sp * TS - -(-N // 64)) == SPLIT_AT_132[N], (N, sp, TS)
        reached.append((sp, sp * TS - -(-N // 64)))
    assert len(reached) >= 3 and any(sp % 4 and virt for sp, virt in reached), reached


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "fp16x3", "bf16x3"])
@pytest.mark.parametrize("dataset", ["3dmatch", "kitti"])
def test_unsplit_small_sets(dataset, precision):
    """KT < 4: never split; ragged and whole key tiles."""
    for N in (2, 10, 63, 64, 65, 129, 192):
        split, per = run_case(dataset, precision, 1, N, [0, 6, 11], [0])
        assert not split and per[0][0] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp16x3", "bf16x3"])
def test_unsplit_batches(precision):
    """Several work items per persistent CTA (B QT >= 3 SMs), more than 3 chain tiles per CTA, a ragged last chain tile,
    tiles spanning sets with N % 128 in (64, 128) and (0, 64], and an odd key-tile count."""
    sms = sm_count()
    for N in (1000, 1003, 150):
        QT = -(-N // 128)
        B = max(-(-3 * sms // QT), (3 * sms * 128) // N + 1)
        assert B * QT >= 3 * sms and B * N > 3 * sms * 128
        if N == 1003:
            assert (B * N) % 128
        split, per = run_case("kitti" if N == 150 else "3dmatch", precision, B, N, [0, 6, 11], check_sets(B, N))
        assert not split
    assert 1000 % 128 > 64 and 0 < 150 % 128 <= 64 and (-(-150 // 64)) % 2 == 1


@pytest.mark.gpu
def test_large_set():
    """bs = 1, N = 16384: unsplit (its query tiles cover the SMs); the first, a middle and the last query tile against all keys."""
    split, per = run_case("3dmatch", "fp16x3", 1, 16384, [0, 11], [0], qrows=tile_rows(16384))
    assert not split


@pytest.mark.gpu
def test_batch_invariant_split():
    """The batch-invariant mode: N = 513 (sp = 2, a virtual tile), 1000, 5000 (sp = 10, a virtual tile) and a batch of 64."""
    for N, want in ((513, (2, 1)), (1000, (2, 0)), (5000, (10, 1))):
        split, per = run_case("3dmatch", "fp16x3", 1, N, [0, 11], [0], qrows=tile_rows(N) if N > 1000 else None,
                              invariant=True)
        sp, TS = per[0]
        assert split and (sp, sp * TS - -(-N // 64)) == want
    split, per = run_case("kitti", "fp16x3", 64, 1000, [0, 11], check_sets(64, 1000), invariant=True)
    assert split and per[0] == (2, 8)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp16x3", "bf16"])
def test_chain_tiles_with_many_set_starts(precision):
    """N = 2, 3, 4 in large batches: chain tiles in which more than 31 sets start walk past the set window (locate_row)."""
    for N in (2, 3, 4):
        B = 1000
        sets = list(range(0, 72)) + [B // 2, B - 1]
        if N < 4:
            assert 128 // N > 32                                   # rows of sets beyond the window's 32 lanes
        run_case("kitti", precision, B, N, [0, 11], sets)


# ---------------------------------------------------------------------------------------------------
# CPU rehearsal: emulated kernels satisfy the bounds, and an emulated defect breaks them
# ---------------------------------------------------------------------------------------------------
def rz32(x):
    """fp32 rounding toward zero: a rounding the wgmma model allows that round-to-nearest never produces."""
    r = x.astype(np.float32)
    fix = np.abs(r.astype(np.float64)) > np.abs(x)
    r[fix] = np.nextafter(r[fix], np.float32(0))
    return r


def mma(acc, pairs, align=False):
    """wgmma k-steps: acc [R,M] fp32; pairs of (A [R,K], W [M,K]) 16-bit operands.  Each k-step rounds its exact sum once
    toward zero; align: each of its 17 terms is first truncated to the 24-bit window of the largest of them (alignment
    without guard bits), then the sum is truncated."""
    acc = acc.astype(np.float32)
    for A, W in pairs:
        for k0 in range(0, A.shape[1], 16):
            a, w = A[:, k0:k0 + 16].astype(np.float64), W[:, k0:k0 + 16].astype(np.float64)
            if not align:
                acc = rz32(acc.astype(np.float64) + a @ w.T)
                continue
            terms = np.concatenate([acc.astype(np.float64)[:, :, None], a[:, None, :] * w[None, :, :]], axis=2)
            _, e = np.frexp(np.abs(terms).max(2, keepdims=True))
            q = np.ldexp(1.0, e - 24)
            acc = rz32(np.trunc(terms / q).sum(2) * q[:, :, 0])
    return acc


def emulate_conv(x, c, precision, relu, drop_lo_hi=False):
    """x fp32 [R,K] through one convolution, the way tc_chain / linear_simt_kernel compute it; drop_lo_hi leaves out the
    x_lo w_hi product of the x3 split."""
    R, K = x.shape
    if precision == "fp32":
        acc = np.zeros((R, c.img.shape[0]), np.float32)
        for k in range(K):                                 # fmaf chain in ascending k
            acc = (acc.astype(np.float64) + x[:, k:k + 1].astype(np.float64) * c.img[:, k][None]).astype(np.float32)
    else:
        split = UNIT[precision][2]
        xh, xl = split16(x, precision)
        wh = (c.img - c.wlo).astype(np.float32)
        wl = c.wlo.astype(np.float32)
        pairs = [(xh, wh), (xh, wl), (xl, wh)] if split else [(xh, wh)]
        acc = mma(np.zeros((R, c.img.shape[0])), pairs[:2] if drop_lo_hi else pairs)
    y = (acc + c.bimg.astype(np.float32)).astype(np.float32)
    return np.maximum(y, np.float32(0)) if relu else y


def emulate_attention(q, k, v, sc, precision, sp, TS, pv_single=False):
    """The persistent attention (+ merge) on fp32 operand images, rows vectorised; pv_single drops the P V lo products."""
    N = k.shape[0]
    KT = -(-N // 64)
    split = UNIT[precision][2]
    qh, ql = split16(q, precision)
    kh, kl = split16(k, precision)
    vh, vl = split16(v, precision)
    S = mma(np.zeros((q.shape[0], N)), [(qh, kh), (qh, kl), (ql, kh)] if split else [(qh, kh)])
    t = (S * sc).astype(np.float32)
    parts = []
    for s in range(sp):
        m = np.full((q.shape[0], 1), -np.inf, np.float32)
        lsum = np.zeros((q.shape[0], 1), np.float32)
        o = np.zeros((q.shape[0], 128), np.float32)
        for J in range(s * TS, (s + 1) * TS):
            cols = np.arange(J * 64, J * 64 + 64)
            real = np.minimum(cols, N - 1) if J < KT else np.arange((KT - 1) * 64, KT * 64).clip(max=N - 1)
            tt = np.where(cols[None] < N, t[:, real], -np.inf).astype(np.float32)
            mn = np.maximum(m, tt.max(1, keepdims=True))
            scale = np.where(mn > m, np.exp2((m - mn).astype(np.float32)), np.float32(1)).astype(np.float32)
            m = mn
            lsum = (lsum * scale).astype(np.float32)
            p = np.exp2((tt - m).astype(np.float32)).astype(np.float32)
            lsum = (lsum + p.sum(1, keepdims=True, dtype=np.float32)).astype(np.float32)
            o = (o * scale).astype(np.float32)
            ph, pl = split16(p, precision)
            vhj, vlj = vh[real].T, vl[real].T
            o = mma(o, [(ph, vhj)] if (pv_single or not split) else [(ph, vhj), (ph, vlj), (pl, vhj)])
        parts.append((o, m, lsum))
    if sp == 1:
        o, m, lsum = parts[0]
        return (o * (np.float32(1) / lsum)).astype(np.float32)
    mstar = np.max([p[1] for p in parts], axis=0)
    L = np.zeros_like(parts[0][2])
    acc = np.zeros_like(parts[0][0])
    for o, ms, ls in parts:
        w = np.exp2((ms - mstar).astype(np.float32)).astype(np.float32)
        L = (L.astype(np.float64) + ls.astype(np.float64) * w).astype(np.float32)
        acc = (acc.astype(np.float64) + o.astype(np.float64) * w).astype(np.float32)
    return (acc * (np.float32(1) / L)).astype(np.float32)


def rehearsal_inputs(rng, R, K, scale):
    """Activations like the encoder's: ReLU'd, a wide range of magnitudes, exact zeros and values below fp16's normal range."""
    x = np.maximum(rng.standard_normal((R, K)), 0) * rng.uniform(0.05, scale, (R, 1))
    x[:, ::7] *= 1e-6
    return x.astype(np.float32)


@pytest.mark.parametrize("align", [False, True])
@pytest.mark.parametrize("precision", ALL_PRECISIONS)
def test_rehearsal_conv_bounds(precision, align, monkeypatch):
    if align:
        if precision == "fp32":
            pytest.skip("no wgmma in fp32")
        plain = mma
        monkeypatch.setattr(__import__(__name__), "mma", lambda acc, pairs: plain(acc, pairs, align=True))
    rng = np.random.default_rng(5)
    cv = layer_convs("3dmatch", precision, 5)
    x = rehearsal_inputs(rng, 96, 128, 40.0)
    # the float64 folds are oracle._lin followed by oracle._bn (PointCN, fc_message.0-1)
    sd = {k: v.double() for k, v in load_snapshot("3dmatch").items()}
    x64 = torch.from_numpy(x.astype(np.float64))
    for name, conv, bn in (("w1", "encoder.blocks.PointCN_layer_5.0", "encoder.blocks.PointCN_layer_5.1"),
                           ("wm0", "encoder.blocks.NonLocal_layer_5.fc_message.0", "encoder.blocks.NonLocal_layer_5.fc_message.1")):
        ref = O._bn(O._lin(x64, sd[conv + ".weight"], sd[conv + ".bias"]), sd, bn).numpy()
        y = x.astype(np.float64) @ cv[name].Wref.T + cv[name].bref
        assert np.abs(y - ref).max() <= 1e-12 * (1 + np.abs(ref).max())
    worst = 0.0
    for name, relu in (("w1", True), ("wq", False), ("wk", False), ("wv", False), ("wm0", True)):
        got = emulate_conv(x, cv[name], precision, relu)
        y, e = conv_bound(x.astype(np.float64), 0.0, cv[name], precision)
        want = np.maximum(y, 0.0) if relu else y
        err = np.abs(got - want)
        assert (err <= e).all(), (name, float((err / e).max()))
        worst = max(worst, float((err / e).max()))
    # the MSG chain with its propagated input error
    msg = (rng.standard_normal((96, 128)) * 5).astype(np.float32)
    f1 = rehearsal_inputs(rng, 96, 128, 20.0)
    h = emulate_conv(msg, cv["wm0"], precision, True)
    h = emulate_conv(h, cv["wm1"], precision, True)
    o = emulate_conv(h, cv["wm2"], precision, False)
    got = (f1 + o).astype(np.float32)
    want, e = fc_message64(msg.astype(np.float64), f1.astype(np.float64), cv, precision)
    err = np.abs(got - want)
    assert (err <= e).all(), float((err / e).max())
    worst = max(worst, float((err / e).max()))
    assert worst > 0
    print(f"rehearsal convs ({precision}, align={align}): worst error / bound {worst:.3g}")
    if UNIT[precision] and UNIT[precision][2]:
        # an MSG chain whose GEMMs lose a cross product (x_lo w_hi) breaks the bound, whichever GEMM loses it
        for drop in ("wm0", "wm1", "wm2"):
            h = emulate_conv(msg, cv["wm0"], precision, True, drop == "wm0")
            h = emulate_conv(h, cv["wm1"], precision, True, drop == "wm1")
            o = emulate_conv(h, cv["wm2"], precision, False, drop == "wm2")
            assert (np.abs(f1 + o - want) > e).any(), drop


@pytest.mark.parametrize("precision", ["fp16x3", "bf16x3", "bf16"])
@pytest.mark.parametrize("N,sp,TS,spread,align", [(200, 1, 4, 0.3, False), (200, 2, 2, 0.3, False), (300, 3, 2, 0.3, False),
                                                   (300, 3, 2, 2.0, False), (200, 2, 2, 2.0, True)])


def test_rehearsal_attention_bound(precision, N, sp, TS, spread, align, monkeypatch):
    """spread 2.0: logits over a range of ~100 (log2 units), so that most P lie below 2^-14 and many below 2^-24, where the
    fp16 floor makes up the bound."""
    if align:
        plain = mma
        monkeypatch.setattr(__import__(__name__), "mma", lambda acc, pairs: plain(acc, pairs, align=True))
    rng = np.random.default_rng(N + sp)
    R = 64
    def image(a):
        hi, lo = split16(a.astype(np.float32), precision)
        return (hi + lo).astype(np.float32)
    q = image(rng.standard_normal((R, 128)) * spread)
    k = image(rng.standard_normal((N, 128)) * spread)
    v = image(rng.standard_normal((N, 128)) * 4.0)
    sc = np.where(rng.uniform(size=(R, N)) < 0.5, 0.0, rng.uniform(size=(R, N))).astype(np.float32)
    got = emulate_attention(q, k, v, sc, precision, sp, TS)
    msg, bound, floor = attention_bound(q, k, v, sc, precision, sp, TS)
    err = np.abs(got - msg)
    assert (err <= bound).all(), float((err / bound).max())
    if spread > 1:
        t = sc.astype(np.float64) * (q.astype(np.float64) @ k.astype(np.float64).T)
        p = np.exp2(t - t.max(1, keepdims=True))
        assert (p < 2.0 ** -14).mean() > 0.5 and (p < 2.0 ** -24).mean() > 0.1
        if precision == "fp16x3":
            assert (floor / bound).max() > 0.5                 # the floor dominates some rows' bounds
    print(f"rehearsal attention ({precision}, N={N}, sp={sp}, spread={spread}, align={align}): worst error / bound {float((err / bound).max()):.3g}, "
          f"floor share {float((floor / bound).max()):.3g}")
    if precision == "fp16x3":
        # a P V that drops its lo products (the x3 split off) breaks the bound
        bad = emulate_attention(q, k, v, sc, precision, sp, TS, pv_single=True)
        assert (np.abs(bad - msg) > bound).any()
