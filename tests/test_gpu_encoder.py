"""The encoder's kernels against float64 on their own inputs, on every launch path they take: the 1x1-convolution chains
(tc_chain<PCQ / KV / MSG> in csrc/tc_chain.cuh, the SIMT `linear` in csrc/encoder_simt.cu), the attention (the persistent
tensor-core kernel and its key-split merge in csrc/tc_attention_p.cuh, the SIMT attention) and layer0.  The GPU tests need an
H100 (`-m gpu`); the CPU rehearsal at the end runs everywhere and checks the bound functions against emulated kernels.

Every layer l is driven through `PointDSC.run` taps: `layer_features` (layer l's output; layer l - 1's, from a second call, is
layer l's input, since forwards are bit-deterministic), `layer_debug` (feat1, q, k, v, msg: in the tensor-core modes q / k / v
are the decoded operand images hi + lo, q carries log2(e) / sqrt(C)) and `sc`.  Layer 0's input is the float64 layer0 of
corr_pos, its fp32 error bounded below.  Each kernel is compared with its own operation in float64 on the tapped fp32
inputs: the BatchNorm fold of oracle._lin + oracle._bn (checked against them on the CPU), and the SC-weighted softmax.  The tests restate attn_set_split / attn_set_split_invariant (sets.cuh) and assert the
regime, sp, TS and virtual-tile count they reach, from the SM count the engine sizes its launches for (PDSC_SM_COUNT).

Error model.  u = 2^-24; gamma(n) = n u / (1 - n u).  Every bound is a posteriori: float64 sums of the actual |terms| of a row.
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
import math
import os

import numpy as np
import pytest
import torch

from conftest import load_snapshot
from oracle import pointdsc_oracle as O

U = 2.0 ** -24
EX2 = 2.0 ** -22
KQ = float(np.float32(1.4426950408889634) / np.float32(11.313708498984761))   # tc_common.cuh kQScale
C32 = float(np.float32(1.0) / np.sqrt(np.float32(128.0)))                      # encoder_simt.cu inv_sqrt_c
UNIT = {"fp32": None, "fp16x3": (2.0 ** -11, 2.0 ** -25, True), "bf16x3": (2.0 ** -8, 0.0, True),
        "bf16": (2.0 ** -8, 0.0, False)}
ALL_PRECISIONS = ["fp32", "fp16x3", "bf16x3", "bf16"]
HEADROOM = 65504.0        # tc_ptx.cuh: fp16 operands need |x| < 65504
TSI = 8                   # sets.cuh kAttnInvariantTiles
SPLIT_MAX_ITEMS = 320     # encoder_tc.cu kAttnSplitMaxItems
# worst error / bound per (kernel, precision) over the module's tests, printed at the end of each test
WORST = {}


def gamma(n):
    return n * U / (1.0 - n * U)


def G(steps):
    return 4 * U * (steps + 1) / (1.0 - 4 * U * (steps + 1))


# ---------------------------------------------------------------------------------------------------
# 16-bit operands and folded weights, as the engine forms them
# ---------------------------------------------------------------------------------------------------
def round16(x, precision):
    """fp32 -> the nearest fp16 / bf16 value (ties to even), as fp32."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    if precision == "fp16x3":
        return x.astype(np.float16).astype(np.float32)
    b = x.view(np.uint32).astype(np.uint64)
    b = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    return b.astype(np.uint32).view(np.float32)


def split16(x, precision):
    """tc_ptx.cuh split_pair: hi = round16(x), lo = round16(x - hi) (x3 modes; single bf16 has no lo)."""
    x = np.asarray(x, dtype=np.float32)
    hi = round16(x, precision)
    lo = round16(x - hi, precision) if UNIT[precision][2] else np.zeros_like(hi)
    return hi, lo


class Conv:
    """One folded 1x1 convolution: the float64 fold (Wref, bref: the reference operation), the operand the kernel multiplies
    (img: fp32 W in SIMT, hi + lo or hi in the tensor-core modes), its lo part and the fp32 bias the epilogue adds."""

    def __init__(self, sd, conv, bn, scale, precision):
        W = sd[conv + ".weight"].double().numpy()[:, :, 0]
        b = sd[conv + ".bias"].double().numpy()
        s, sh = np.ones(len(b)), np.zeros(len(b))
        if bn:
            s = sd[bn + ".weight"].double().numpy() / np.sqrt(sd[bn + ".running_var"].double().numpy() + O.BN_EPS)
            sh = sd[bn + ".bias"].double().numpy() - sd[bn + ".running_mean"].double().numpy() * s
        W64, b64 = W * s[:, None], b * s + sh
        W32, b32 = W64.astype(np.float32), b64.astype(np.float32)
        if precision == "fp32":
            scale = 1.0
            self.img, self.wlo, self.bimg = W32.astype(np.float64), np.zeros_like(W64), b32.astype(np.float64)
        else:
            src = (W32.astype(np.float64) * scale).astype(np.float32)
            hi, lo = split16(src, precision)
            self.img, self.wlo = hi.astype(np.float64) + lo, lo.astype(np.float64)
            self.bimg = (b32.astype(np.float64) * scale).astype(np.float32).astype(np.float64)
        self.Wref, self.bref, self.scale = W64 * scale, b64 * scale, scale


_convs = {}


def layer_convs(dataset, precision, l, sd=None):
    """Layer l's folded convolutions of the state dict sd (default: the dataset's snapshot; `dataset` names sd in the
    cache)."""
    key = (dataset, precision, l)
    if key not in _convs:
        sd = load_snapshot(dataset) if sd is None else sd
        pc, nl = f"encoder.blocks.PointCN_layer_{l}", f"encoder.blocks.NonLocal_layer_{l}"
        _convs[key] = {
            "w1": Conv(sd, pc + ".0", pc + ".1", 1.0, precision),
            "wq": Conv(sd, nl + ".projection_q", None, KQ, precision),
            "wk": Conv(sd, nl + ".projection_k", None, 1.0, precision),
            "wv": Conv(sd, nl + ".projection_v", None, 1.0, precision),
            "wm0": Conv(sd, nl + ".fc_message.0", nl + ".fc_message.1", 1.0, precision),
            "wm1": Conv(sd, nl + ".fc_message.3", nl + ".fc_message.4", 1.0, precision),
            "wm2": Conv(sd, nl + ".fc_message.6", None, 1.0, precision),
        }
    return _convs[key]


# ---------------------------------------------------------------------------------------------------
# bounds
# ---------------------------------------------------------------------------------------------------
def rho(a, precision):
    """|x - (what the kernel's operand represents)| for |x| <= a."""
    uh, fl, split = UNIT[precision]
    return (uh * uh if split else uh) * a + fl


def conv_bound(x, ex, c, precision, own=False):
    """A convolution whose kernel input lies within ex of the float64 x [R,K]: the float64 y = x Wref^T + bref and the bound
    of |y32 - y|, y32 the fp32 accumulator plus bias the epilogue forms (before its ReLU / split).  own: the bound of
    |y32 - (x_k Wref^T + bref)| instead, x_k the kernel's input (the input error is then propagated by the caller)."""
    K = x.shape[1]
    ex = np.broadcast_to(np.asarray(ex, np.float64), x.shape)
    ax = np.abs(x)
    xa = ax + ex
    ia = np.abs(c.img)
    y = x @ c.Wref.T + c.bref
    if own:
        prop = ex @ np.abs(c.Wref).T
        e = xa @ np.abs(c.Wref - c.img).T + np.abs(c.bref - c.bimg)
    else:
        prop = 0.0
        e = ax @ np.abs(c.Wref - c.img).T + np.abs(c.bref - c.bimg) + ex @ ia.T
    if precision == "fp32":
        e += gamma(K) * (xa @ ia.T)
    else:
        uh, fl, split = UNIT[precision]
        e += rho(xa, precision) @ ia.T
        if split:                                           # the dropped lo*lo
            e += ((uh * xa + fl) * (1 + uh)) @ np.abs(c.wlo).T
        e += G((3 if split else 1) * K // 16) * (1 + 3 * uh) * (xa @ ia.T)
    return y, e + U * (np.abs(y) + e + prop)


def decoded(y, e, precision):
    """Bound of a decoded hi + lo (hi) operand image of the fp32 y32 within e of y."""
    return e if precision == "fp32" else e + rho(np.abs(y) + e, precision)


def layer0_64(cp, sd):
    """float64 layer0 of corr_pos [R,6] and the bound of layer0_kernel's fp32 (6 fmas, then the bias)."""
    W = sd["encoder.layer0.weight"].double()
    b = sd["encoder.layer0.bias"].double()
    x = torch.from_numpy(cp.astype(np.float64))
    y = O._lin(x, W, b).numpy()
    e = gamma(cp.shape[1] + 1) * (np.abs(cp.astype(np.float64)) @ np.abs(W[:, :, 0].numpy()).T + np.abs(b.numpy()))
    return y, e


def attention_bound(q, k, v, sc, precision, sp, TS):
    """Query rows q [R,C] of a set with keys k, v [N,C] and SC rows sc [R,N] (fp32 taps): the float64 msg of the kernel's
    operation, the bound of the kernel's error, and the share of that bound the fp16 P floor accounts for."""
    R, N = q.shape[0], k.shape[0]
    KT = -(-N // 64)
    tiles = sp * TS
    q64, k64, v64, sc = (np.asarray(a, np.float64) for a in (q, k, v, sc))
    qk = q64 @ k64.T
    Sabs = np.abs(q64) @ np.abs(k64).T
    if precision == "fp32":
        c = 1.0 / math.sqrt(128.0)
        t = sc * qk * c
        Et = sc * c * gamma(128) * Sabs + sc * np.abs(qk) * abs(C32 - c) + 3 * U * np.abs(t)
        lnb = 1.0
    else:
        uh, fl, split = UNIT[precision]
        ES = G(24 if split else 8) * (1 + 3 * uh) * Sabs
        if split:
            ES += np.abs(q64 - round16(q, precision)) @ np.abs(k64 - round16(k, precision)).T
        t = sc * qk
        Et = sc * ES + U * (np.abs(t) + sc * ES)
        lnb = math.log(2.0)
    m = t.max(1, keepdims=True)
    P = np.exp(lnb * (t - m))
    l = P.sum(1, keepdims=True)
    msg = (P @ v64) / l
    Tmax = (np.abs(t) + Et).max(1, keepdims=True)
    delta = np.expm1(lnb * (Et + U * (np.abs(t) + Tmax))) * (1 + EX2) + EX2
    dmax = delta.max(1, keepdims=True)
    assert (dmax < 0.5).all(), "the logit bound is vacuous"
    lk = l * (1 - dmax)
    Pk = P * (1 + delta)
    va = np.abs(v64)
    A = np.empty_like(msg)
    for r0 in range(0, R, 16):
        A[r0:r0 + 16] = np.einsum("rj,rjc->rc", (P * delta)[r0:r0 + 16], np.abs(v64[None] - msg[r0:r0 + 16, None]))
    bound = A / lk + (gamma(N + 6 * tiles + 8) + 2 * U) * np.abs(msg)
    pv = Pk @ va
    floor = np.zeros_like(msg)
    if precision == "fp32":
        bound += gamma(N + KT) * pv / lk
    else:
        if split:
            vlo = np.abs(v64 - round16(v, precision))
            floor = fl * (va.sum(0) + vlo.sum(0))[None] / lk
            bound += ((uh * uh * Pk) @ va + (uh * Pk) @ vlo) / lk + floor
        else:
            bound += uh * pv / lk
        ST = 12 if split else 4
        pad = KT * 64 - N
        Pt = np.pad(Pk, ((0, 0), (0, pad))).reshape(R, KT, 64)
        Tt = np.einsum("rtj,tjc->rtc", Pt, np.pad(va, ((0, pad), (0, 0))).reshape(KT, 64, -1)) * (1 + uh) ** 2
        Ac = np.cumsum(Tt, axis=1)
        bound += ((4 * U * ST + U) * (Ac.sum(1) + (tiles - KT) * Ac[:, -1]) + 4 * U * ST * Tt.sum(1)) / lk
        if sp > 1:                                          # the merge
            for s in range(sp):
                cols = slice(s * TS * 64, min((s + 1) * TS * 64, N))
                ms = t[:, cols].max(1, keepdims=True)
                eps = EX2 + math.log(2.0) * U * (m - ms + 2 * Tmax)
                bound += eps * (Pk[:, cols] @ va[cols] + Pk[:, cols].sum(1, keepdims=True) * np.abs(msg)) / lk
            bound += gamma(sp) * (pv / lk + np.abs(msg)) + 2 * U * np.abs(msg)
    return msg, bound, floor


def relu_masks(y, e):
    """The units a ReLU certainly passes (y > e) and those whose state the error e leaves open (|y| <= e)."""
    return (y > e).astype(np.float64), (np.abs(y) <= e).astype(np.float64)


def fc_message64(msg, f1, cv, precision):
    """feat = feat1 + fc_message(msg) in float64 (Conv.Wref / bref: the fold of oracle._lin + oracle._bn, see
    test_rehearsal_conv_bounds) and the bound of the MSG chain's fp32 result on the tapped msg and feat1.

    The hidden activations are not tapped, so their errors are carried to the output linearly, keeping the cancellation
    inside the weights: with eps_i the error of convolution i at the kernel's own input and Theta = diag(theta) the ReLU's
    secant slopes (relu(y + d) - relu(y) = theta d, theta in [0, 1]; 1 / 0 where the ReLU's state is certain),
        feat_k - feat = W2 Theta1 W1 Theta0 eps0 + W2 Theta1 eps1 + eps2 (+ the roundings of the bias and residual adds),
    bounded by |W2 A1 W1| |Theta0 eps0| + |W2| K1 |W1| |Theta0 eps0| + |W2| (A1 + K1) |eps1| + |eps2|, A1 / K1 the certain /
    open units of the second ReLU."""
    c0, c1, c2 = cv["wm0"], cv["wm1"], cv["wm2"]
    y0, e0 = conv_bound(msg, 0.0, c0, precision)
    a0, k0 = relu_masks(y0, e0)
    h0, d0 = np.maximum(y0, 0.0), e0 * (a0 + k0)
    W1a, W2a = np.abs(c1.Wref), np.abs(c2.Wref)
    y1, e1 = conv_bound(h0, d0, c1, precision, own=True)
    p1 = d0 @ W1a.T + e1
    a1, k1 = relu_masks(y1, p1)
    h1 = np.maximum(y1, 0.0)
    o, e2 = conv_bound(h1, p1 * (a1 + k1), c2, precision, own=True)
    E = e2 + ((a1 + k1) * e1 + k1 * (d0 @ W1a.T)) @ W2a.T
    for r0 in range(0, len(o), 256):
        M = (c2.Wref[None] * a1[r0:r0 + 256, None, :]) @ c1.Wref
        E[r0:r0 + 256] += np.einsum("rok,rk->ro", np.abs(M), d0[r0:r0 + 256])
    feat = f1 + o
    return feat, E + U * (np.abs(feat) + E)


# ---------------------------------------------------------------------------------------------------
# the regime a call reaches (sets.cuh, encoder_tc.cu tc_packed_split)
# ---------------------------------------------------------------------------------------------------
def attn_set_split(N, sms):
    QT, KT = -(-N // 128), -(-N // 64)
    if KT < 4:
        return 1, KT
    want = -(-sms // QT)
    ts = max(-(-KT // want), 2)
    s = -(-KT // ts)
    return (s, ts) if s >= 2 else (1, KT)


def attn_set_split_invariant(N):
    KT = -(-N // 64)
    sp = -(-KT // TSI)
    return sp, -(-KT // sp)


def call_split(Ns, sms, invariant):
    """(split?, [(sp, TS)] per set) of a tensor-core call."""
    per = [attn_set_split_invariant(n) if invariant else attn_set_split(n, sms) for n in Ns]
    qtiles = sum(-(-n // 128) for n in Ns)
    items = sum(-(-n // 128) * sp for n, (sp, _) in zip(Ns, per))
    split = items > qtiles if invariant else (2 * qtiles <= sms and qtiles < items <= SPLIT_MAX_ITEMS)
    return split, (per if split else [(1, -(-n // 64)) for n in Ns])


def sm_count():
    n = torch.cuda.get_device_properties(0).multi_processor_count
    env = os.environ.get("PDSC_SM_COUNT", "")
    return min(n, int(env)) if env.isdigit() and int(env) > 0 else n


# ---------------------------------------------------------------------------------------------------
# one call, layer by layer
# ---------------------------------------------------------------------------------------------------
_models = {}


def get_model(dataset, precision, invariant=False):
    from pointdsc_b200 import PointDSC
    key = (dataset, precision, invariant)
    if key not in _models:
        cfg = O.default_config(dataset)
        m = PointDSC(in_dim=6, num_layers=12, num_channels=128, num_iterations=10, ratio=0.1,
                     inlier_threshold=cfg["inlier_threshold"], sigma_d=cfg["sigma_d"], k=40,
                     nms_radius=cfg["nms_radius"], precision=precision, batch_invariant=invariant)
        res = m.load_state_dict(load_snapshot(dataset), strict=False)
        assert res.missing_keys == [] and res.unexpected_keys == ["gamma"]
        _models[key] = m.cuda().eval()
    return _models[key]


def note(kernel, precision, err, bound):
    r = float((err / bound).max()) if err.size else 0.0
    WORST[(kernel, precision)] = max(WORST.get((kernel, precision), 0.0), r)
    return r


def check(kernel, precision, got, want, bound, where):
    got = got.astype(np.float64)
    assert np.isfinite(got).all() and (np.abs(got) < HEADROOM).all(), (kernel, where, "operand headroom")
    err = np.abs(got - want)
    bad = err > bound
    assert not bad.any(), (kernel, precision, where, np.argwhere(bad)[:4], float(err.max()), float((err / bound).max()))
    note(kernel, precision, err, bound)


def run_case(dataset, precision, B, N, layers, sets, qrows=None, invariant=False, seed=0, model=None, sd=None, args=None):
    """Runs B sets of N correspondences and checks, at every layer in `layers`, PCQ, KV, the attention and MSG on the rows of
    `sets` (qrows: the query rows within a set the attention is checked at, default all).  Returns (split, [(sp, TS)]).
    model / sd: the module and the state dict it holds (default: the dataset's 12-layer snapshot model; `dataset` then names
    sd in the weight cache); args: the call's device inputs (default: synthetic pairs of the dataset's geometry)."""
    from pointdsc_b200.synth import make_pair
    m = get_model(dataset, precision, invariant) if model is None else model
    sms = sm_count()
    if args is None:
        pairs = [make_pair(10000 * seed + 17 * N + b, N, dataset, 0.3 + 0.4 * (b % 3) / 2) for b in range(B)]
        args = [torch.stack([p[x] for p in pairs]).cuda() for x in ("corr_pos", "src_keypts", "tgt_keypts")]
    if precision == "fp32":
        split, per = False, [(1, -(-N // 64))] * B
    else:
        split, per = call_split([N] * B, sms, invariant)
        enc = m.launches_per_forward(B, N) - 12
        assert enc == 2 + (5 if split else 4) * m.num_layers, (enc, split)   # the engine ran the regime restated here
    qrows = np.arange(N) if qrows is None else np.asarray(qrows)
    sd = load_snapshot(dataset) if sd is None else sd
    sc_all = m.run(*args, taps=["sc"])["sc"]
    scs = {b: sc_all[b][torch.from_numpy(qrows).cuda()].cpu().numpy() for b in sets}
    del sc_all
    cp = args[0].cpu().numpy()
    floor_share = 0.0
    prev = {}
    for l in layers:
        out = m.run(*args, taps=["layer_features", "layer_debug"], layer_tap=l)
        if l > 0 and l - 1 not in prev:
            p = m.run(*args, taps=["layer_features"], layer_tap=l - 1)["layer_features"]
            prev[l - 1] = {b: p[b].cpu().numpy() for b in sets}
        cv = layer_convs(dataset, precision, l, sd)
        feats = {}
        for b in sets:
            dbg = out["layer_debug"][:, b].cpu().numpy()          # feat1, q, k, v, msg [N,C]
            feats[b] = out["layer_features"][b].cpu().numpy()
            where = (dataset, N, B, b, l)
            if l == 0:
                x, ex = layer0_64(cp[b], sd)
            else:
                x, ex = prev[l - 1][b].astype(np.float64), 0.0
                assert (np.abs(x) < HEADROOM).all()
            # PCQ: feat1 = relu(BN(W1 x + b1)), q from feat1
            y, e = conv_bound(x, ex, cv["w1"], precision)
            check("pcq", precision, dbg[0], np.maximum(y, 0.0), e, where)
            f1 = dbg[0].astype(np.float64)
            y, e = conv_bound(f1, 0.0, cv["wq"], precision)
            check("pcq", precision, dbg[1], y, decoded(y, e, precision), where)
            # KV
            for i, name in ((2, "wk"), (3, "wv")):
                y, e = conv_bound(f1, 0.0, cv[name], precision)
                check("kv", precision, dbg[i], y, decoded(y, e, precision), where)
            # attention (+ merge)
            sp, TS = per[b]
            msg, bound, floor = attention_bound(dbg[1][qrows], dbg[2], dbg[3], scs[b], precision, sp, TS)
            check("attention", precision, dbg[4][qrows], msg, bound, where)
            floor_share = max(floor_share, float((floor / bound).max()))
            # MSG
            feat, e = fc_message64(dbg[4].astype(np.float64), f1, cv, precision)
            check("msg", precision, feats[b], feat, e, where)
        prev = {l: feats}
    for key in sorted(k for k in WORST if k[1] == precision):
        print(f"{key[0]} ({precision}): worst error / bound so far {WORST[key]:.3g}")
    if precision == "fp16x3":
        print(f"fp16 P floor: largest share of an attention bound {floor_share:.3g}")
    return split, per


def check_sets(B, N):
    """The first and last sets and sets whose rows straddle 128-row chain tiles."""
    out = {0, B - 1}
    for b in (1, B // 2, B // 2 + 1):
        if b < B and (b * N) % 128 and (b * N) // 128 != (b * N + N - 1) // 128:
            out.add(b)
    return sorted(out)


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
