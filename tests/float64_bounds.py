"""The float64 error model of the GPU tests and the bound checkers more than one test module uses.

u = 2^-24 and u64 = 2^-53 are the fp32 and float64 unit roundoffs, eps = 2^-23 and eps64 = 2^-52 the machine epsilons;
gamma(n) = n u / (1 - n u) bounds the relative error of an n-term sum in any order, fma or not (gamma64 with u64).  Every
reference is float64 on the engine's own fp32 inputs or taps, and every bound is derived beside its constant.
  * The encoder (tc_chain.cuh, encoder_simt.cu, tc_attention_p.cuh): conv_bound, attention_bound, fc_message64 and run_case,
    which checks every kernel of a forward's encoder layers; test_gpu_encoder.py sets out their error model.
  * Kabsch (svd3.cuh): weighted_kabsch64 and check_transforms; test_gpu_kabsch.py sets out the solver's bound.
  * The seed-row kNN (E_KNN) and the power iteration (check_power) of test_gpu_stages.py.
  * The spectral-matching baseline's compatibility entries (entry_width); test_gpu_spectral_matching.py sets out their bound.
"""
import math

import numpy as np
import torch

from conftest import load_snapshot
from engine_rules import call_split
from gpu_models import get_model, sm_count
from oracle import pointdsc_oracle as O

U = 2.0 ** -24
U64 = 2.0 ** -53
EPS = 2.0 ** -23
EPS64 = 2.0 ** -52      # float64 machine epsilon: the bound of the double solver (ICP's updates) uses it in place of eps


def gamma(n):
    return n * U / (1.0 - n * U)


def gamma64(n):
    return n * U64 / (1.0 - n * U64)


# ---------------------------------------------------------------------------------------------------
# the encoder
# ---------------------------------------------------------------------------------------------------
EX2 = 2.0 ** -22
KQ = float(np.float32(1.4426950408889634) / np.float32(11.313708498984761))   # tc_common.cuh kQScale
C32 = float(np.float32(1.0) / np.sqrt(np.float32(128.0)))                      # encoder_simt.cu inv_sqrt_c
UNIT = {"fp32": None, "fp16x3": (2.0 ** -11, 2.0 ** -25, True), "bf16x3": (2.0 ** -8, 0.0, True),
        "bf16": (2.0 ** -8, 0.0, False)}
ALL_PRECISIONS = ["fp32", "fp16x3", "bf16x3", "bf16"]
HEADROOM = 65504.0        # tc_ptx.cuh: fp16 operands need |x| < 65504
# worst error / bound per (kernel, precision) over the session's encoder checks, printed at the end of each test
WORST = {}


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
    m = get_model(dataset, precision, invariant=invariant) if model is None else model
    sms = sm_count()
    if args is None:
        pairs = [make_pair(10000 * seed + 17 * N + b, N, dataset, 0.3 + 0.4 * (b % 3) / 2) for b in range(B)]
        args = [torch.stack([p[x] for p in pairs]).cuda() for x in ("corr_pos", "src_keypts", "tgt_keypts")]
    if precision == "fp32":
        split, per = False, [(1, -(-N // 64))] * B
    else:
        split, _, per = call_split([N] * B, sms, invariant)
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


# ---------------------------------------------------------------------------------------------------
# Kabsch
# ---------------------------------------------------------------------------------------------------
# Solver constant: |R - R64|max <= C_SVD * eps * s1 / (s2 + d s3).  Worst measured on an H100 over the ~1.1e5 matrices of
# part 1: 5.2 (repeated singular values; random 4.7, ill-conditioned 3.8, reflected 1.8, rank 2 1.8), so 16 leaves 3x.
C_SVD = 16.0
# Pre-solver fp32 term (`_h_error`): per-entry bound on |H32 - H64| in units of eps * (its magnitude terms).  Derivation: a
# weighted centroid is a 4-term fma chain per lane, a 5-level warp tree and a division by a sum with the same error, so it
# is off by <= 20 eps * max|a|; a centred coordinate then by <= 21 eps * max|a|; each H entry sums k products of such terms
# (4 fma per lane + the tree: 10 eps relative).  32 covers all three with margin.  Measured on an H100 (part 2's degenerate
# neighbourhoods): the worst error is 0.002 of the rotation tolerance, 0.018 of the translation one and 0.008 of the centroid
# one; the bounds are worst cases, the typical rounding errors cancel.
C_PRE = 32.0


def kabsch64(H):
    """R = V diag(1, 1, det(V U^T)) U^T of H [..., 3, 3] (float64, H = U S V^T, H = sum w a b^T so that b ~= R a).
    Returns R, singular values s [..., 3] (descending), d = det(V U^T), U, V."""
    U, s, Vt = np.linalg.svd(H)
    V = np.swapaxes(Vt, -1, -2)
    d = np.sign(np.linalg.det(V @ np.swapaxes(U, -1, -2)))
    D = np.broadcast_to(np.eye(3), H.shape).copy()
    D[..., 2, 2] = d
    return V @ D @ np.swapaxes(U, -1, -2), s, d, U, V


def kabsch_ld(H, sweeps=12):
    """kabsch64's R, s, d, U, V for float64 H, computed in long double (64-bit significand, 2^-11 of float64's roundoff).
    LAPACK's float64 SVD is itself off by up to ~50 eps64 s1 / (s2 + d s3) on part 1's families, as much as the solver under
    test, so the double solver is checked against this: one-sided Jacobi on the columns of H, R = V diag(1, 1, d) U^T in
    the form v1 u1^T + v2 u2^T + (v1 x v2)(u1 x u2)^T, which needs no u3 (rank-2 H included).  Rows of rank < 2 get the
    same form with an arbitrary u2 and are not compared (their gap s2 + d s3 is 0)."""
    H = np.asarray(H, np.float64)
    m = np.abs(H).max(axis=(1, 2))
    e = np.where(m > 0, np.floor(np.log2(np.where(m > 0, m, 1.0))), 0.0)
    G = H.astype(np.longdouble) * np.exp2(-e).astype(np.longdouble)[:, None, None]     # exact power-of-two scaling
    V = np.broadcast_to(np.eye(3, dtype=np.longdouble), G.shape).copy()
    one = np.longdouble(1)
    for _ in range(sweeps):
        for p, q in ((0, 1), (0, 2), (1, 2)):
            gp, gq = G[:, :, p].copy(), G[:, :, q].copy()
            a, b, g = (gp * gp).sum(1), (gq * gq).sum(1), (gp * gq).sum(1)
            rot = g != 0
            z = np.where(rot, (b - a) / np.where(rot, 2 * g, one), one)
            t = np.where(rot, np.sign(z) / (np.abs(z) + np.sqrt(one + z * z)), 0)
            c = one / np.sqrt(one + t * t)
            s = c * t
            G[:, :, p], G[:, :, q] = c[:, None] * gp - s[:, None] * gq, s[:, None] * gp + c[:, None] * gq
            vp, vq = V[:, :, p].copy(), V[:, :, q].copy()
            V[:, :, p], V[:, :, q] = c[:, None] * vp - s[:, None] * vq, s[:, None] * vp + c[:, None] * vq
    n = np.sqrt((G * G).sum(1))                                                         # [P, 3] singular values
    order = np.argsort(-n, axis=1, kind="stable")
    n = np.take_along_axis(n, order, 1)
    G = np.take_along_axis(G, order[:, None, :], 2)
    V = np.take_along_axis(V, order[:, None, :], 2)
    safe = lambda x: np.where(x > 0, x, one)  # noqa: E731
    u1 = G[:, :, 0] / safe(n[:, 0])[:, None]
    u2 = G[:, :, 1] - u1 * (G[:, :, 1] * u1).sum(1)[:, None]
    u2 = u2 / safe(np.sqrt((u2 * u2).sum(1)))[:, None]
    v1, v2 = V[:, :, 0], V[:, :, 1]
    R = (v1[:, :, None] * u1[:, None, :] + v2[:, :, None] * u2[:, None, :]
         + np.cross(v1, v2)[:, :, None] * np.cross(u1, u2)[:, None, :])
    U = np.stack([u1, u2, np.cross(u1, u2)], 2)
    d = np.where(np.linalg.det(H) < 0, -1.0, 1.0)          # sign(det H) = det(U) det(V) wherever s3 > 0
    s = (n * np.exp2(e).astype(np.longdouble)[:, None]).astype(np.float64)
    return R.astype(np.float64), s, d, U.astype(np.float64), V.astype(np.float64)


def _gap(s, d):
    return s[..., 1] + d * s[..., 2]


def _h_error(w, a, b, m, n):
    """Per-entry bound on |H32 - H64| from fp32 centroids, centring and sums.  w [P,k], a/b the points [P,k,3], m/n the
    centred points [P,k,3] (all float64).  Ma, Mb: the coordinates' magnitude, which the centroid errors scale with."""
    Ma, Mb = np.abs(a).max(axis=(1, 2)), np.abs(b).max(axis=(1, 2))
    mi, ni = np.abs(m).max(axis=2), np.abs(n).max(axis=2)
    return C_PRE * EPS * (Ma * (w * ni).sum(1) + Mb * (w * mi).sum(1) + (w * mi * ni).sum(1)), Ma, Mb


def weighted_kabsch64(a, b, w):
    """oracle.pointdsc_oracle.weighted_kabsch in float64 (the oracle builds its identity in float32): negative weights -> 0,
    centroids over sum(w) + 1e-6, H = Am^T diag(w) Bm, t = cb - R ca.  a, b [P,k,3], w [P,k].
    Returns R [P,3,3], t [P,3], ca, cb, H, and the H error bound with its magnitudes."""
    w = np.where(w < 0, 0.0, w)
    den = w.sum(1) + 1e-6
    ca = (a * w[..., None]).sum(1) / den[:, None]
    cb = (b * w[..., None]).sum(1) / den[:, None]
    m, n = a - ca[:, None], b - cb[:, None]
    H = np.einsum("pki,pkj,pk->pij", m, n, w)
    R, s, d, U, V = kabsch64(H)
    t = cb - np.einsum("pij,pj->pi", R, ca)
    EH, Ma, Mb = _h_error(w, a, b, m, n)
    return dict(R=R, t=t, ca=ca, cb=cb, H=H, s=s, d=d, U=U, V=V, EH=EH, Ma=Ma, Mb=Mb)


def assert_rotations(R, what, tol=1e-6):
    """Finite, orthonormal and det = +1 to `tol`.  1e-6 is ~8 fp32 roundings of a product of unit vectors; the worst measured
    on an H100 over every part-1 input is 8.6e-7 (|R R^T - I|) and 8.9e-7 (|det R - 1|)."""
    R = np.asarray(R, np.float64)
    assert np.isfinite(R).all(), what
    orth = np.abs(R @ np.swapaxes(R, -1, -2) - np.eye(3)).max(axis=(-1, -2))
    det = np.abs(np.linalg.det(R) - 1.0)
    assert orth.max() <= tol and det.max() <= tol, (what, float(orth.max()), float(det.max()))


def check_transforms(T, ref, what):
    """Engine transforms T [P,4,4] against a weighted_kabsch64 result.  Returns the worst ratios (error / tolerance)."""
    T = np.asarray(T, np.float64)
    R, t = T[:, :3, :3], T[:, :3, 3]
    assert_rotations(R, what)
    s, d, EH, Ma, Mb = ref["s"], ref["d"], ref["EH"], ref["Ma"], ref["Mb"]
    gap = _gap(s, d)
    with np.errstate(divide="ignore", invalid="ignore"):
        # rotation: solver term + pre-solver term over the signed gap; >= 2 is vacuous (entries of two rotations)
        tol_R = np.where(gap > 0, (C_SVD * EPS * s[:, 0] + 6.0 * EH) / gap, np.inf)
        # the first singular pair is defined whenever s1 > s2, the gap of singular vectors: R u1 = v1 (rank 1 included)
        tol_u1 = np.where(s[:, 0] > s[:, 1], (C_SVD * EPS * s[:, 0] + 6.0 * EH) / (s[:, 0] - s[:, 1]), np.inf)
    err_R = np.abs(R - ref["R"]).max(axis=(1, 2))
    assert (err_R <= tol_R).all(), (what, np.flatnonzero(err_R > tol_R)[:8], err_R[err_R > tol_R][:8], tol_R[err_R > tol_R][:8])
    err_u1 = np.abs(np.einsum("pij,pj->pi", R, ref["U"][:, :, 0]) - ref["V"][:, :, 0]).max(1)
    assert (err_u1 <= tol_u1).all(), (what, err_u1[err_u1 > tol_u1][:8], tol_u1[err_u1 > tol_u1][:8])
    # t = cb - R ca: its error is the rotation's error at the centroid plus the centroids' own (<= 20 eps Ma, see C_PRE)
    tol_t = 3.0 * np.minimum(tol_R, 2.0) * Ma + C_PRE * EPS * (Ma + Mb)
    err_t = np.abs(t - ref["t"]).max(1)
    assert (err_t <= tol_t).all(), (what, err_t[err_t > tol_t][:8], tol_t[err_t > tol_t][:8])
    # whatever R is, it maps the weighted centroid onto the target centroid (no division by a gap): the centroids' errors
    # (<= 20 eps each), R times the source one (3 terms) and the rounding of t = cb - R ca: 96 eps (Ma + Mb)
    err_c = np.abs(np.einsum("pij,pj->pi", R, ref["ca"]) + t - ref["cb"]).max(1)
    tol_c = 96.0 * EPS * (Ma + Mb)
    assert (err_c <= tol_c).all(), (what, err_c[err_c > tol_c][:8], tol_c[err_c > tol_c][:8])
    ratio = lambda e, tl: float(np.max(np.where(np.isfinite(tl) & (tl < 2), e / tl, 0.0), initial=0.0))  # noqa: E731
    return dict(R=ratio(err_R, tol_R), u1=ratio(err_u1, tol_u1), t=ratio(err_t, tol_t), c=ratio(err_c, tol_c), tol_R=tol_R)


# ---------------------------------------------------------------------------------------------------
# the seed-row kNN and the power iteration
# ---------------------------------------------------------------------------------------------------
# A distance 2 - 2 f_s . f_j of unit rows: the fp32 dot of 128 terms is within gamma(128) sum |f_s| |f_j| <= gamma(128)
# (Cauchy-Schwarz), doubled, plus u 4 for 2 - 2x: E_KNN = 2 gamma(128) + 4 u = 1.55e-5.  The tensor-core mode's fp16
# hi/lo split drops lo*lo and the lo parts' own rounding: <= 3 2^-22 + 2^-25 (|f_s|_1 + |f_j|_1) = 1.4e-6, and its fp32
# accumulation over the 24 k-steps adds <= 48 u: below E_KNN.  Two ranks can swap only if their float64 distances are
# within 2 E_KNN.  Measured on an H100 (80GB HBM3): worst |d64(got) - d64(ref)| / (2 E_KNN) = 0.025 (fp32, N = 16384,
# k = 128); 91-95 % of the ranks are separated.  Identical rows came out with bitwise identical distances in both modes.
E_KNN = 2 * gamma(128) + 4 * U

# M and the iterates are non-negative, so one fp32 step is the exact step followed by a per-entry relative perturbation:
# (M v)_i within gamma(k + 2) (k fmas and the two butterfly adds) and the division by the norm u; the norm's own rounding
# scales every entry alike.  Non-negative matrices do not expand Hilbert's projective metric, and the normalisation does not
# change it, so after t steps d_H(v32, v64) <= D_t = 2.01 t gamma(k + 3), linear in t.  Both vectors have the norm
# nrm / (nrm + 1e-6), the fp32 one within ((k + 1) / 2 + 4) u and one more D_t: per entry
#   |v32 - v64| <= (2 (e^D_t - 1) + ((k + 1) / 2 + 4) u) v64 + 1e-30.
# Measured on an H100 (80GB HBM3) over the sweep and the caps: worst error / bound = 0.032 (cap 1, k = 40).
#
# The exit iteration.  That worst case is wider than allclose's own rtol of 1e-5, so it cannot decide whether fp32 and
# float64 take the same exit.  The per-step roundings are independent: their sum grows like the square root of their number,
# so the band is B_t = C_BAND sqrt(t (k + 3)) u v64, C_BAND = 4, and the test asserts that the engine's eig stays inside
# that band at its exit iteration (measured on an H100: worst error / band 0.12).  An entry's allclose margin |v_t - v_t-1| - (1e-8 + 1e-5 v_t-1)
# is then known to within B_t + B_t-1 + 3 u (|v_t - v_t-1| + 1e-8 + 1e-5 v_t-1) (the fp32 comparison's own roundings).
# An iteration's all-seeds decision is sure when every margin is below minus that or one margin is above it; where every
# decision up to the float64 exit is sure, power_iters must equal the float64 exit (220 of the sweep's 320 sets on an H100).
C_BAND = 4.0


def power64(M, iters):
    """The reference iteration in float64 on M [S,k,k]: every iterate [iters,S,k], the exit (first iteration at which
    allclose holds for all seeds, else the cap) and the margins [iters,S,k] (<= 0: the entry passes)."""
    v = np.ones(M.shape[:2])
    its, margins, exit_t = [], [], iters
    for t in range(1, iters + 1):
        w = np.einsum("sij,sj->si", M, v)
        w = w / (np.linalg.norm(w, axis=1, keepdims=True) + 1e-6)
        margin = np.abs(w - v) - (1e-8 + 1e-5 * np.abs(v))
        its.append(w)
        margins.append(margin)
        if exit_t == iters and (margin <= 0).all():
            exit_t = t
        v = w
    return np.stack(its), exit_t, np.stack(margins)


def check_power(compat, eig, power_iters, k, iters):
    """One set: eig against the float64 iterate at the engine's exit, power_iters against the float64 exit where sure.
    Returns (eig error / bound, eig error / band, exit compared)."""
    M = compat.astype(np.float64)
    its, exit64, margins = power64(M, iters)
    t = int(power_iters)
    assert 1 <= t <= iters
    v64 = its[t - 1]
    D = 2.01 * t * gamma(k + 3)
    tol = (2 * math.expm1(D) + ((k + 1) / 2 + 4) * U) * v64 + 1e-30
    err = np.abs(eig.astype(np.float64) - v64)
    assert (err <= tol).all(), (t, float(err.max()), np.argwhere(err > tol)[:4])
    band = lambda tt: C_BAND * math.sqrt(tt * (k + 3)) * U * its[tt - 1]             # noqa: E731
    assert (err <= band(t) + 1e-30).all(), ("the statistical band", t, float((err / (band(t) + 1e-30)).max()))
    sure = True
    for tt in range(1, exit64 + 1):
        prev = its[tt - 2] if tt > 1 else np.ones_like(v64)
        w = band(tt) + (band(tt - 1) if tt > 1 else 0.0) + 3 * U * (np.abs(its[tt - 1] - prev) + 1e-8 + 1e-5 * prev)
        mg = margins[tt - 1]
        sure &= bool((mg < -w).all() or (mg > w).any())
    if sure:
        assert t == exit64, (t, exit64)
    return float((err / tol).max()), float((err / (band(t) + 1e-30)).max()), sure


# ---------------------------------------------------------------------------------------------------
# the spectral-matching baseline
# ---------------------------------------------------------------------------------------------------
def entry_width(corr, thr):
    """W [N,N] float64 (on corr's device) of test_gpu_spectral_matching.py's header: the bound of |M' - M| per entry."""
    c = corr.to(torch.float64)
    ds = torch.cdist(c[:, :3], c[:, :3], compute_mode="donot_use_mm_for_euclid_dist")
    dt = torch.cdist(c[:, 3:], c[:, 3:], compute_mode="donot_use_mm_for_euclid_dist")
    m = (ds - dt).abs()
    em = gamma(5) * (ds + dt) * (1 + 1e-12)
    del ds, dt
    cf = 4.5 / thr ** 2
    e = (2 * m * em + em * em) * cf * (1 + gamma(3)) + gamma(3) * cf * m * m + 4.5 * U
    mu = 4.5 - m * m * cf
    W = (mu + e).clamp_min(0.0) - (mu - e).clamp_min(0.0)
    W.fill_diagonal_(0.0)
    return W
