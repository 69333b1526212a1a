"""Guarded buffers for the memory contract's tests, and the inputs those tests share with the float64 ones.

Every buffer a call gets is owned by the test and lives inside a larger allocation: SLACK bytes of sentinel on either side
(inputs: NaN, so that a stray read past an input row changes a result instead of passing unnoticed), the interior at exactly
the alignment asked for and no more.  After the stream synchronises the slack must be byte-identical to its fill.  Outputs,
scratch and the workspace are prefilled with one of PATTERNS (test_gpu_memory_contract.py sets out why these four); `Call`
runs one forward configuration through the C ABI that way.  The front-end cases at the end are the inputs of the float64
tests of test_gpu_front_end.py, which test_gpu_packed_eval.py runs through the packed entry points.
"""
import ctypes as C
import math

import numpy as np
import torch

from engine_rules import C_CH, call_split, mirror_workspace, num_seeds
from float64_bounds import U64, gamma64
from gpu_models import get_model, sm_count

SLACK = 64 * 1024
SENTINEL = 0x3CC35AA5
NAN32 = 0x7FC00000
PATTERNS = ["zero", "ones", "fmax", "fmin"]
FLOAT_WORD = {"zero": 0x00000000, "ones": 0xFFFFFFFF, "fmax": 0x7F7F7F7F, "fmin": 0xFF7F7F7F}
INDEX_WORD = {"zero": 0, "ones": 1, "fmax": 1, "fmin": 0}
MASK_WORD = {"zero": 0, "ones": 0xFFFFFFFF, "fmax": 0, "fmin": 0xFFFFFFFF}
BEST_QWORD = {"zero": 0, "ones": 0xFFFFFFFF00000000, "fmax": 0, "fmin": 0xFFFFFFFF00000000}


# ---------------------------------------------------------------------------------------------------
# guarded buffers
# ---------------------------------------------------------------------------------------------------
def tiled(word, n, device, width=4):
    """n bytes of the little-endian `width`-byte word repeated."""
    pat = torch.tensor(list(int(word).to_bytes(width, "little")), dtype=torch.uint8)
    return pat.repeat(n // width + 1)[:n].to(device)


def fill_words(buf, word, width=4):
    """Fill a uint8 tensor (length a multiple of `width`) with a repeated word, without a temporary of its size."""
    n = buf.numel()
    assert n % width == 0, (n, width)
    if n:
        pat = torch.tensor(list(int(word).to_bytes(width, "little")), dtype=torch.uint8, device=buf.device)
        buf.view(-1, width).copy_(pat.expand(n // width, width))


class Guarded:
    """`nbytes` at exactly `align` (an address that is a multiple of align but not of 2 align), with at least SLACK bytes of
    sentinel (or NaN) on either side, all inside one allocation."""

    def __init__(self, nbytes, align, device, slack="sentinel"):
        self.nbytes, self.align = int(nbytes), int(align)
        self.raw = torch.empty(2 * SLACK + 2 * self.align + self.nbytes, dtype=torch.uint8, device=device)
        base = self.raw.data_ptr()
        addr = -(-(base + SLACK) // self.align) * self.align
        if addr % (2 * self.align) == 0:
            addr += self.align
        self.off = addr - base
        self.inner = self.raw[self.off:self.off + self.nbytes]
        word = SENTINEL if slack == "sentinel" else NAN32
        self.pre_want = tiled(word, self.off, device)
        self.post_want = tiled(word, self.raw.numel() - self.off - self.nbytes, device)
        self.raw[:self.off].copy_(self.pre_want)
        self.raw[self.off + self.nbytes:].copy_(self.post_want)

    @property
    def ptr(self):
        return self.raw.data_ptr() + self.off       # (an empty slice reports address 0)

    def typed(self, dtype, shape):
        return self.inner.view(dtype).view(shape)

    def violations(self):
        """Offsets, relative to the buffer's first byte, of slack bytes that changed."""
        pre = torch.nonzero(self.raw[:self.off] != self.pre_want).flatten() - self.off
        post = torch.nonzero(self.raw[self.off + self.nbytes:] != self.post_want).flatten() + self.nbytes
        return pre.tolist() + post.tolist()

    def check(self, what):
        v = self.violations()
        assert not v, f"{what}: {len(v)} guard bytes changed, first at offsets {v[:8]} from the buffer's first byte"


def guarded_input(arr, device):
    """A float32 / float64 / int32 host array as a device input at 16 B with NaN slack."""
    arr = np.ascontiguousarray(arr)
    g = Guarded(arr.nbytes, 16, device, slack="nan")
    g.inner.copy_(torch.from_numpy(arr.view(np.uint8).reshape(-1)))
    return g


def guarded_output(nbytes, align, device, pattern):
    g = Guarded(nbytes, align, device)
    fill_words(g.inner, FLOAT_WORD[pattern]) if nbytes % 4 == 0 else g.inner.copy_(tiled(FLOAT_WORD[pattern], nbytes, device))
    return g


def scratch_buffer(nbytes, align, pattern):
    g = Guarded(nbytes, align, torch.device("cuda"))
    g.inner.copy_(tiled(FLOAT_WORD[pattern], nbytes, g.inner.device))
    return g


def run_guarded(where, outs, scratch, inputs, call):
    """call(), synchronise, check every guard; returns {name: bytes} of the outputs."""
    _capi().check(call())
    torch.cuda.synchronize()
    for name, g in list(outs.items()) + list(inputs.items()) + [("scratch", scratch)]:
        g.check((name,) + where)
    return {n: g.inner.clone() for n, g in outs.items()}


def assert_same(ref, got, where):
    assert ref.keys() == got.keys()
    for name in ref:
        if not torch.equal(ref[name], got[name]):
            diff = torch.nonzero(ref[name] != got[name]).flatten()
            raise AssertionError(f"{where}: {name} differs in {diff.numel()} bytes, first at byte {int(diff[0])}")


def check_patterns(call, where):
    ref = call.run("zero")
    for p in PATTERNS[1:]:
        assert_same(ref, call.run(p), where + (p,))
    return ref


# ---------------------------------------------------------------------------------------------------
# one forward configuration through the C ABI
# ---------------------------------------------------------------------------------------------------
def poison_workspace(ws, regions, pattern):
    fill_words(ws, FLOAT_WORD[pattern])
    for name, off, n, kind in regions:
        seg = ws[off:off + n]
        if kind == "index":
            fill_words(seg, INDEX_WORD[pattern])
        elif kind == "mask":
            fill_words(seg, MASK_WORD[pattern])
        elif kind == "best":
            fill_words(seg, BEST_QWORD[pattern], 8)
        elif kind == "zero":
            seg.zero_()


def make_inputs(Ns, seed=0):
    """Packed corr_pos [R,6], src [R,3], tgt [R,3] float32 (numpy) of sets with N = Ns[b]."""
    from pointdsc_b200.synth import make_pair
    pairs = [make_pair(1000 * seed + 37 * n + b, n, "3dmatch", 0.3 + 0.2 * (b % 3)) for b, n in enumerate(Ns)]
    return [np.concatenate([p[x].numpy() for p in pairs]).astype(np.float32) for x in ("corr_pos", "src_keypts", "tgt_keypts")]


def tap_spec(name, B, N, S, k):
    from pointdsc_b200.model import _TAP_SPECS
    dtype, shape = _TAP_SPECS[name]
    return dtype, shape(B, N, S, k, C_CH)


def nbytes_of(dtype, shape):
    return int(np.prod(shape, dtype=np.int64)) * torch.empty((), dtype=dtype).element_size()


class Call:
    """One configuration: its engine, entry point, sets and taps.  run(pattern) runs it on freshly poisoned buffers and
    returns {output name: device bytes}, having checked every guard."""

    def __init__(self, precision, Ns, entry="forward", invariant=False, k=40, taps=(), layer_tap=0, want_M=False, seed=0):
        assert entry in ("forward", "packed", "eval", "graph")
        assert entry == "packed" or len(set(Ns)) == 1
        self.precision, self.Ns, self.entry, self.taps, self.layer_tap, self.want_M = precision, list(Ns), entry, list(taps), \
            layer_tap, want_M
        self.m = get_model("3dmatch", precision, invariant=invariant, k=k)
        self.lib, self.e = self.m._ensure_engine(), self.m._engine
        self.dev = torch.device("cuda")
        self.B, self.R, self.N = len(Ns), sum(Ns), Ns[0]
        self.S, self.k = int(self.lib.pdsc_num_seeds(self.e, self.N)), int(self.lib.pdsc_num_neighbours(self.e, self.N))
        self.offsets = np.concatenate([[0], np.cumsum(Ns)]).astype(np.int32)
        self.h_off = (C.c_int32 * (self.B + 1))(*self.offsets.tolist())
        if entry == "packed":
            self.need = int(self.lib.pdsc_workspace_bytes_packed(self.e, self.B, self.h_off))
        else:
            self.need = int(self.lib.pdsc_workspace_bytes(self.e, self.B, self.N))
        self.regions, total = mirror_workspace(Ns, precision, invariant, k, sm_count())
        assert total == self.need, ("workspace map drifted from the engine", total, self.need)
        for n in set(Ns):
            assert int(self.lib.pdsc_num_seeds(self.e, n)) == num_seeds(n)
        cp, s, t = make_inputs(Ns, seed)
        self.inputs = {"corr_pos": guarded_input(cp, self.dev), "src": guarded_input(s, self.dev), "tgt": guarded_input(t, self.dev),
                       "d_offsets": guarded_input(self.offsets, self.dev)}
        self.ws = Guarded(self.need, 256, self.dev)
        self.outs = None
        # the SC matrix (workspace offset 0) is written whole, pad columns as 0: row-major [N, round_up(N, 64)] in fp32,
        # 64 x 128 tiles of every (key tile, query tile) in the tensor-core modes
        self.sc_bytes = 4 * (sum(n * (-(-n // 64) * 64) for n in Ns) if precision == "fp32"
                             else sum(-(-n // 64) * -(-n // 128) * 8192 for n in Ns))

    def _outputs(self, pattern):
        B, R, N = self.B, self.R, self.N
        specs = {"final_trans": (torch.float32, (B, 4, 4)), "final_labels": (torch.float32, (R,))}
        if self.want_M:
            specs["M"] = (torch.float32, (B, N, N))
        for name in self.taps:
            specs[name] = tap_spec(name, B, N, self.S, self.k)
        outs = {}
        for name, (dtype, shape) in specs.items():
            size = torch.empty((), dtype=dtype).element_size()
            outs[name] = guarded_output(nbytes_of(dtype, shape), size, self.dev, pattern)
        return outs

    def _poison(self, pattern):
        poison_workspace(self.ws.inner, self.regions, pattern)
        if self.outs is None or self.entry != "graph":
            self.outs = self._outputs(pattern)
        else:                                     # a replayed graph keeps its output addresses: refill them in place
            for g in self.outs.values():
                fill_words(g.inner, FLOAT_WORD[pattern])

    def run(self, pattern):
        self._poison(pattern)
        lib, e, o, i = self.lib, self.e, self.outs, self.inputs
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        io_ptr = None
        if self.taps:
            io = self._io = _capi().StageIO()
            for name in self.taps:
                setattr(io, "out_" + name, o[name].ptr)
            io.layer_tap = int(self.layer_tap)
            io_ptr = C.byref(io)
        P = C.c_void_p
        args_in = (P(i["corr_pos"].ptr), P(i["src"].ptr), P(i["tgt"].ptr))
        outs2 = (P(o["final_trans"].ptr), P(o["final_labels"].ptr))
        if self.entry == "forward":
            rc = lib.pdsc_forward(e, self.B, self.N, *args_in, *outs2, io_ptr, P(self.ws.ptr), self.need, stream)
        elif self.entry == "eval":
            rc = lib.pdsc_forward_eval(e, self.B, self.N, *args_in, *outs2, P(o["M"].ptr) if self.want_M else None, io_ptr,
                                       P(self.ws.ptr), self.need, stream)
        elif self.entry == "packed":
            rc = lib.pdsc_forward_packed(e, self.B, self.h_off, P(i["d_offsets"].ptr), *args_in, *outs2, P(self.ws.ptr), self.need,
                                         stream)
        else:
            rc = lib.pdsc_forward_graph(e, self.B, self.N, *args_in, *outs2, P(self.ws.ptr), self.need, stream)
        _capi().check(rc)
        torch.cuda.synchronize()
        where = (self.precision, self.entry, self.Ns[:8], pattern)
        self.ws.check(("workspace",) + where)
        for name, g in list(o.items()) + list(i.items()):
            g.check((name,) + where)
        res = {}
        for name, g in o.items():
            if name == "timeline":                # documented as never written: it keeps the prefill
                assert torch.equal(g.inner, tiled(FLOAT_WORD[pattern], g.nbytes, self.dev)), ("timeline written",) + where
                continue
            dtype = tap_spec(name, 1, 1, 1, 1)[0] if name in self.taps else torch.float32
            if dtype == torch.float32 and g.nbytes:
                assert torch.isfinite(g.inner.view(torch.float32)).all(), (name, "non-finite") + where
            res[name] = g.inner.clone()
        res["workspace sc"] = self.ws.inner[:self.sc_bytes].clone()
        return res

    def regime(self):
        """(split?, [(sp, TS)]) the engine ran, asserted against pdsc_launches_per_forward for uniform tensor-core calls."""
        if self.precision == "fp32":
            return False, [(1, -(-n // 64)) for n in self.Ns]
        split, _, per = call_split(self.Ns, sm_count(), self.m.batch_invariant)
        if self.entry != "packed":
            enc = int(self.lib.pdsc_launches_per_forward(self.e, self.B, self.N)) - 12
            assert enc == 2 + (5 if split else 4) * 12, (enc, split)
        return split, per


def _capi():
    from pointdsc_b200 import _capi as capi
    return capi


# ---------------------------------------------------------------------------------------------------
# front-end cases
# ---------------------------------------------------------------------------------------------------
RE_THRE, TE_THRE = 15.0, 25.0


def keypoints(rng, n):
    return rng.uniform(-3, 3, (n, 3)).astype(np.float32)


def surface(rng, m):
    """m points on a smooth, gently curved patch of the unit square (continuous: no ties, no bin-edge features)."""
    xy = rng.uniform(0, 1, (m, 2))
    z = 0.1 * np.sin(3 * xy[:, 0]) * np.cos(2 * xy[:, 1]) + 0.002 * rng.standard_normal(m)
    return np.concatenate([xy, z[:, None]], 1).astype(np.float32)


def match_descriptors(rng, ns, nt, D, dtype):
    """Sources near random targets; among the targets and the sources a few exact copies and (D > 1) copies one ulp away in
    one channel, which no float64 argmin can separate from their original."""
    unit = lambda f: f / np.linalg.norm(f, axis=1, keepdims=True)      # noqa: E731
    if D == 1:
        t, s = rng.uniform(-1, 1, (nt, 1)), rng.uniform(-1, 1, (ns, 1))
    else:
        t = unit(rng.standard_normal((nt, D)))
        s = unit(t[rng.integers(0, nt, ns)] + 0.3 / math.sqrt(D) * rng.standard_normal((ns, D)))
    t, s = t.astype(dtype), s.astype(dtype)
    for f in (t, s):
        n = len(f)
        if n >= 4:
            k = max(1, n // 30)
            f[rng.choice(n, k, replace=False)] = f[rng.integers(0, n, k)]
            if D > 1:
                dst, src = rng.choice(n, k, replace=False), rng.integers(0, n, k)
                f[dst] = f[src]
                c = rng.integers(0, D, k)
                f[dst, c] = np.nextafter(f[dst, c], dtype(2))
    return s, t


def run_match(sd, td, sk, tk, mutual):
    from pointdsc_b200.frontend import match
    d = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()      # noqa: E731
    out = match(d(sd), d(td), d(sk), d(tk), use_mutual=mutual)
    return {"corr": out["corr"].cpu().numpy(), "corr_pos": out["corr_pos"][0].cpu().numpy(),
            "src": out["src_keypts"][0].cpu().numpy(), "tgt": out["tgt_keypts"][0].cpu().numpy()}


def mean_candidates(col, exact):
    """The fp32 means the kernel may form for one column of corr_pos: an fp64 sum in any order (within gamma64(M) sum |v|),
    divided by M (one rounding) and rounded to fp32; `exact`: the fp64 sum is exact (dyadic inputs), one candidate."""
    x = col.astype(np.float64)
    mean = math.fsum(x) / len(x)
    if exact:
        return [np.float32(mean)]
    d = gamma64(len(x)) * np.abs(x).sum() / len(x) + 4 * U64 * abs(mean)
    out, hi = [np.float32(mean - d)], np.float32(mean + d)
    while out[-1] < hi:
        out.append(np.nextafter(out[-1], np.float32(np.inf)))
    return out


def check_network_input(out, sk, tk, exact):
    """Exact gathers, and corr_pos = fl32(v - m32) bit for bit for one admissible fp32 mean m32 per column."""
    corr = out["corr"]
    assert np.array_equal(out["src"], sk[corr[:, 0]]) and np.array_equal(out["tgt"], tk[corr[:, 1]])
    if len(corr) == 0:
        return
    v = np.concatenate([sk[corr[:, 0]], tk[corr[:, 1]]], 1)
    for c in range(6):
        cands = mean_candidates(v[:, c], exact)
        assert any(np.array_equal(out["corr_pos"][:, c], v[:, c] - m) for m in cands), (c, cands)


def rotations(rng, n):
    q, r = np.linalg.qr(rng.standard_normal((n, 3, 3)))
    q *= np.sign(np.diagonal(r, axis1=1, axis2=2))[:, None, :]
    q[np.linalg.det(q) < 0, :, 0] *= -1
    return q


def axis_rotation(axis, ang):
    a = axis / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(ang) * K + (1 - math.cos(ang)) * K @ K


def stats_case(rng, B, N):
    """B sets of N correspondences; from B >= 8 the first sets are the constructed edges: pred == gt (a signed permutation),
    a 180 degree relative rotation with the clamp active, TE == te_thre exactly, and the label edges (pred all <= 0 with
    exact +0 and -0, pred all > 0, gt all zero, gt all zero with pred all <= 0, gt all one)."""
    Rg = rotations(rng, B)
    gt = np.tile(np.eye(4), (B, 1, 1))
    gt[:, :3, :3], gt[:, :3, 3] = Rg, rng.uniform(-1, 1, (B, 3))
    ang = rng.uniform(0, 30, B) * math.pi / 180
    pred = gt.copy()
    for b in range(B):
        pred[b, :3, :3] = Rg[b] @ axis_rotation(rng.standard_normal(3), ang[b])
    pred[:, :3, 3] += rng.standard_normal((B, 3)) * rng.uniform(0, 0.2, (B, 1))
    gt, pred = gt.astype(np.float32), pred.astype(np.float32)
    src = rng.uniform(-2, 2, (B, N, 3)).astype(np.float32)
    inl = rng.uniform(size=(B, N)) < rng.uniform(0.05, 0.9, (B, 1))
    tgt = np.einsum("bck,bnk->bnc", gt[:, :3, :3].astype(np.float64), src) + gt[:, None, :3, 3]
    tgt = np.where(inl[..., None], tgt + 0.01 * rng.standard_normal(tgt.shape), rng.uniform(-2, 2, tgt.shape)).astype(np.float32)
    gl = inl.astype(np.float32)
    pl = rng.standard_normal((B, N)).astype(np.float32)
    pl[:, ::7], pl[:, 3::11] = 0.0, -0.0
    if B >= 8:
        perm = np.array([[0, -1, 0], [0, 0, 1], [-1, 0, 0]], np.float32)
        gt[0, :3, :3] = pred[0, :3, :3] = perm
        pred[0, :3, 3] = gt[0, :3, 3]
        # 180 degrees, scaled by 1 + 2^-12 as a nearly orthonormal estimate may be: the trace lies below -1 in any rounding
        pred[1, :3, :3] = Rg[1] @ axis_rotation(rng.standard_normal(3), math.pi) * (1 + 2.0 ** -12)
        gt[2, :3, :3] = pred[2, :3, :3] = np.eye(3, dtype=np.float32)
        gt[2, :3, 3] = 0.0
        pred[2, :3, 3] = (TE_THRE / 100, 0.0, 0.0)                        # 0.25 m: TE = 25 cm exactly
        pl[3] = -np.abs(pl[3])
        pl[4] = np.abs(pl[4]) + 1.0
        gl[5] = 0.0
        gl[6], pl[6] = 0.0, -np.abs(pl[6])
        pl[[3, 6], ::5] = 0.0                                               # +0 and -0 beside negatives: none kept
        gl[7] = 1.0
    return pred, gt, src, tgt, pl, gl
