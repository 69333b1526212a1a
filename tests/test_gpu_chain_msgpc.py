"""The encoder's MSGPC chain mode (tc_chain.cuh): layer l's fc_message and residual, then layer l + 1's PointCN, written in
place over feat1, so that feat goes to HBM only for the head (after the last layer, in plain MSG) and for the layer_features
tap.  Layers 1 and up start with the Q mode, which reads that feat1.

The split only moves arithmetic between kernels, so what the taps do must not change a single bit:
- final outputs and every layer tap are byte-identical with and without layer_features / layer_debug taps, in every
  tensor-core precision, at row counts with a ragged last chain tile, tiles spanning sets and tiles in which more than 31 sets
  start (the set-window walk of the Q mode);
- a mixed-size call in the batch-invariant mode gives each set what a call holding it alone gives;
- results do not depend on what the workspace held (the in-place feat1 update under every poison of the memory contract);
- feat1(l + 1), from layer_debug at layer l + 1, is PointCN(l + 1) of layer_features at layer l within the float64 bound of
  float64_bounds.conv_bound.
"""
import numpy as np
import pytest
import torch

from buffer_guards import Call, check_patterns
from float64_bounds import check, conv_bound, layer_convs
from gpu_models import get_model, same

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp16x3", "bf16x3", "bf16"]
TAP_LAYERS = [0, 5, 10, 11]


def batch(Ns, seed, dataset="3dmatch"):
    """Device tensors [B, N, ...] of B = len(Ns) sets of equal N."""
    from pointdsc_b200.synth import make_pair
    pairs = [make_pair(1000 * seed + 31 * n + b, n, dataset, 0.3 + 0.2 * (b % 3)) for b, n in enumerate(Ns)]
    return [torch.stack([p[x] for p in pairs]).cuda() for x in ("corr_pos", "src_keypts", "tgt_keypts")]


def check_taps(precision, N, B, layers, dataset="3dmatch"):
    """Runs B sets of N with no tap, then with layer_features and layer_debug at each layer of `layers`, together and apart.
    Final outputs must not move, each tap must be the same with or without the other, and feat1 of layer l + 1 must be
    PointCN(l + 1) of layer l's output."""
    m = get_model(dataset, precision)
    args = batch([N] * B, seed=N, dataset=dataset)
    ref = m.run(*args)
    debug = {}
    for l in layers:
        both = m.run(*args, taps=["layer_features", "layer_debug"], layer_tap=l)
        feat = m.run(*args, taps=["layer_features"], layer_tap=l)
        dbg = m.run(*args, taps=["layer_debug"], layer_tap=l)
        for name, out in (("both", both), ("layer_features", feat), ("layer_debug", dbg)):
            for key in ("final_trans", "final_labels"):
                assert same(out[key], ref[key]), (precision, N, B, l, name, key)
        assert same(both["layer_features"], feat["layer_features"]), (precision, N, B, l)
        assert same(both["layer_debug"], dbg["layer_debug"]), (precision, N, B, l)
        assert torch.isfinite(both["layer_features"]).all() and torch.isfinite(both["layer_debug"]).all()
        debug[l] = both
    for l in layers:
        if l + 1 >= 12:
            continue
        nxt = debug[l + 1]["layer_debug"] if l + 1 in debug else m.run(*args, taps=["layer_debug"], layer_tap=l + 1)["layer_debug"]
        w1 = layer_convs(dataset, precision, l + 1)["w1"]
        for b in sorted({0, B // 2, B - 1}):
            x = debug[l]["layer_features"][b].cpu().numpy().astype(np.float64)
            y, e = conv_bound(x, 0.0, w1, precision)
            check("pcq", precision, nxt[0, b].cpu().numpy(), np.maximum(y, 0.0), e, (dataset, N, B, b, l + 1))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_taps_ragged_tiles(precision):
    """N = 129, B = 3: the last chain tile is ragged and the tiles span sets."""
    assert (3 * 129) % 128 and 129 % 128
    check_taps(precision, 129, 3, TAP_LAYERS)


@pytest.mark.parametrize("precision", ["fp16x3", "bf16"])
def test_taps_many_set_starts(precision):
    """N = 2 and 4, B = 300: chain tiles in which 64 and 32 sets start, past the Q mode's 32-lane set window."""
    for N in (2, 4):
        assert 128 // N >= 32
        check_taps(precision, N, 300, [0, 10, 11], dataset="kitti")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_mixed_call_equals_single_calls(precision):
    """Sets of N = 2, 5, 127, 129, 1000, 4097 in one batch-invariant call, 36 sets of N = 2 first so that the first chain tile
    holds 41 set starts: each set's outputs are those of a call holding it alone."""
    from pointdsc_b200.synth import make_pair
    m = get_model("3dmatch", precision, invariant=True)
    sizes = [2] * 36 + [5] * 4 + [127, 129, 1000, 4097]
    assert sum(1 for r in np.cumsum([0] + sizes[:-1]) if r < 128) > 31
    pairs = [make_pair(5000 + i, n, "3dmatch", 0.3 + 0.2 * (i % 3)) for i, n in enumerate(sizes)]
    dev = [{k: p[k][None].cuda() for k in ("corr_pos", "src_keypts", "tgt_keypts")} for p in pairs]
    out = m.forward_many([{**d, "testing": True} for d in dev])
    for i in [0, 17, 35, 36, 39] + list(range(40, len(sizes))):
        one = m.run(dev[i]["corr_pos"], dev[i]["src_keypts"], dev[i]["tgt_keypts"])
        assert same(out[i]["final_trans"], one["final_trans"]), (precision, i, sizes[i])
        assert same(out[i]["final_labels"], one["final_labels"]), (precision, i, sizes[i])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_in_place_feat1_under_poison(precision):
    """The in-place feat1 update reads nothing it did not write: a uniform call with both layer taps (at a middle layer, whose
    MSGPC also writes feat) and a mixed-size call, bit-identical under every workspace and output poison."""
    check_patterns(Call(precision, [129] * 3, "forward", taps=["layer_features", "layer_debug"], layer_tap=5), (precision, 5))
    check_patterns(Call(precision, [2, 5, 127, 129, 1000, 3], "packed"), (precision, "packed"))
