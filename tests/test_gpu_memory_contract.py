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

Workspace regions.  carve() and call_shape() (engine.cu) are restated below (mirror_workspace), including
tc_scratch_bytes_tiles and the key-split rules attn_set_split / attn_set_split_invariant / tc_packed_split (sets.cuh,
encoder_tc.cu), and every GPU test asserts that the restatement's total equals pdsc_workspace_bytes(_packed), so the map
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
import os

import numpy as np
import pytest
import torch

from conftest import load_snapshot

SLACK = 64 * 1024
SENTINEL = 0x3CC35AA5
NAN32 = 0x7FC00000
PATTERNS = ["zero", "ones", "fmax", "fmin"]
FLOAT_WORD = {"zero": 0x00000000, "ones": 0xFFFFFFFF, "fmax": 0x7F7F7F7F, "fmin": 0xFF7F7F7F}
INDEX_WORD = {"zero": 0, "ones": 1, "fmax": 1, "fmin": 0}
MASK_WORD = {"zero": 0, "ones": 0xFFFFFFFF, "fmax": 0, "fmin": 0xFFFFFFFF}
BEST_QWORD = {"zero": 0, "ones": 0xFFFFFFFF00000000, "fmax": 0, "fmin": 0xFFFFFFFF00000000}
C_CH = 128                      # num_channels
SETDESC_BYTES = 72              # sets.cuh SetDesc: 12 int32 + 3 int64
TSI = 8                         # sets.cuh kAttnInvariantTiles
SPLIT_MAX_ITEMS = 320           # encoder_tc.cu kAttnSplitMaxItems
PARTIAL_BYTES = 65536 + 1024    # encoder_tc.cu kAttnPartialBytes
RATIO = 0.1                     # cfg.ratio


# ---------------------------------------------------------------------------------------------------
# harness
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


# ---------------------------------------------------------------------------------------------------
# the workspace, restated (engine.cu call_shape / carve, encoder_tc.cu tc_packed_split / tc_scratch_bytes_tiles, sets.cuh)
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


def tc_packed_split(Ns, invariant, sms):
    """(split, items, [(sp, TS)] per set) of a tensor-core call."""
    per = [attn_set_split_invariant(n) if invariant else attn_set_split(n, sms) for n in Ns]
    qtiles = sum(-(-n // 128) for n in Ns)
    items = sum(-(-n // 128) * sp for n, (sp, _) in zip(Ns, per))
    split = items > qtiles if invariant else (2 * qtiles <= sms and qtiles < items <= SPLIT_MAX_ITEMS)
    return split, (items if split else qtiles), per


def num_seeds(N):
    m = int(N * RATIO)                  # sets.cuh num_seeds: the length of range(N)[:m]
    return min(m, N) if m >= 0 else max(N + m, 0)


def mirror_workspace(Ns, precision, invariant, k_cfg, sms, iters=10):
    """[(name, offset, bytes, kind)] and the total of carve(call_shape(Ns)); kind: float / index / mask / best / zero."""
    R = sum(Ns)
    B = len(Ns)
    seeds = sum(num_seeds(n) for n in Ns)
    dist = sum((num_seeds(n) * n + 3) & ~3 for n in Ns)
    knn = sum(num_seeds(n) * max(min(k_cfg, n - 1), 0) for n in Ns)
    sc_row = sum(n * (-(-n // 64) * 64) for n in Ns)
    sc_tiled = sum(-(-n // 64) * -(-n // 128) * 8192 for n in Ns)
    qtiles, ktiles = sum(-(-n // 128) for n in Ns), sum(-(-n // 64) for n in Ns)
    regions, off = [], 0

    def take(name, count, size, kind):
        nonlocal off
        off = -(-off // 256) * 256
        regions.append((name, off, count * size, kind))
        off += count * size

    take("sc", max(sc_row, sc_tiled), 4, "float")
    take("feat_a", R * C_CH, 4, "float")
    take("feat_b", -(-R // 128) * 128 * C_CH, 4, "float")
    take("msg", R * C_CH, 4, "float")
    if precision == "fp32":
        for name in ("q", "k", "v"):
            take(name, R * C_CH, 4, "float")
        take("h1", R * 64, 4, "float")
        take("h2", R * 64, 4, "float")
    else:
        split, items, _ = tc_packed_split(Ns, invariant, sms)
        partial = (items if split else 0) if invariant else SPLIT_MAX_ITEMS
        take("tc_scratch", (qtiles + ktiles) * 65536 + 1024 + partial * PARTIAL_BYTES, 1, "float")
    take("normed", R * C_CH, 4, "float")
    take("conf", R, 4, "float")
    take("key", R, 4, "float")
    take("seeds", seeds + 1, 4, "index")
    take("seedfeat", seeds * C_CH + 1, 4, "float")
    take("dist", dist + 1, 4, "float")
    take("knn", knn + 1, 4, "index")
    take("iterates", knn * iters + 1, 4, "float")
    take("seed_trans", seeds * 16 + 16, 4, "float")
    take("counts", seeds + 1, 4, "index")
    take("conv_mask", B, 4, "mask")
    take("best_key", B, 8, "best")
    take("sets", B * SETDESC_BYTES, 1, "zero")
    take("tile_set", -(-R // 128), 4, "zero")
    return regions, -(-off // 256) * 256


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


# ---------------------------------------------------------------------------------------------------
# driving the engine
# ---------------------------------------------------------------------------------------------------
ALL_TAPS = ["sc", "features", "normed", "confidence", "seeds", "knn_idx", "compat", "eig", "power_iters", "seed_trans",
            "inlier_counts", "best", "init_trans", "refine_solves", "layer_features", "layer_debug", "timeline"]


def sm_count():
    n = torch.cuda.get_device_properties(0).multi_processor_count
    env = os.environ.get("PDSC_SM_COUNT", "")
    return min(n, int(env)) if env.isdigit() and int(env) > 0 else n


_models = {}


def get_model(precision, invariant=False, k=40, fresh=False):
    from oracle import pointdsc_oracle as O
    from pointdsc_b200 import PointDSC
    key = (precision, invariant, k)
    if fresh or key not in _models:
        cfg = O.default_config("3dmatch")
        m = PointDSC(in_dim=6, num_layers=12, num_channels=128, num_iterations=10, ratio=0.1,
                     inlier_threshold=cfg["inlier_threshold"], sigma_d=cfg["sigma_d"], k=k,
                     nms_radius=cfg["nms_radius"], precision=precision, batch_invariant=invariant)
        res = m.load_state_dict(load_snapshot("3dmatch"), strict=False)
        assert res.missing_keys == [] and res.unexpected_keys == ["gamma"]
        m = m.cuda().eval()
        m._ensure_engine()
        if fresh:
            return m
        _models[key] = m
    return _models[key]


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
        self.m = get_model(precision, invariant, k)
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
        split, _, per = tc_packed_split(self.Ns, self.m.batch_invariant, sm_count())
        if self.entry != "packed":
            enc = int(self.lib.pdsc_launches_per_forward(self.e, self.B, self.N)) - 12
            assert enc == 2 + (5 if split else 4) * 12, (enc, split)
        return split, per


def _capi():
    from pointdsc_b200 import _capi as capi
    return capi


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
# forward entry points
# ---------------------------------------------------------------------------------------------------
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
    m = get_model("fp16x3", fresh=True)
    fresh_results = []
    for c in history_calls():
        got = do_call(m, c)
        f = get_model("fp16x3", fresh=True)
        want = do_call(f, c)
        f._release()
        del f
        fresh_results.append(want)
        for a, b in zip(got, want):
            assert a.numpy().tobytes() == b.numpy().tobytes(), c
    h = get_model("fp16x3", fresh=True)
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


@pytest.mark.gpu
@pytest.mark.parametrize("fp64", [False, True], ids=["fp32", "fp64"])
def test_match_poison_and_rows_past_m(fp64):
    """pdsc_match: scratch at exactly 8 B and pdsc_match_scratch_bytes, poisoned; outputs prefilled; rows >= M keep the
    prefill byte for byte (only the first M rows are written); mutual on and off; one chunk, several and the cap."""
    from test_gpu_front_end import match_plan, keypoints
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
    from test_gpu_front_end import search_plan, surface
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
    from test_gpu_front_end import eig_plan
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


def test_split_rules_match_the_encoder_tests():
    """The restated split rules agree with test_gpu_encoder's on the shapes both use."""
    import test_gpu_encoder as T
    for n in (2, 65, 257, 513, 1000, 3000, 5000, 16384):
        for sms in (132, 114, 66):
            assert attn_set_split(n, sms) == T.attn_set_split(n, sms)
        assert attn_set_split_invariant(n) == T.attn_set_split_invariant(n)
    for Ns in ([1000], [5000], [1003] * 17, [513, 9, 1003, 64]):
        for inv in (False, True):
            split, _, per = tc_packed_split(Ns, inv, 132)
            t_split, t_per = T.call_split(Ns, 132, inv)
            assert split == t_split and (not split or per == t_per)
