#!/usr/bin/env python
"""Developer tool: localise the run-to-run differences of the tensor-core encoder (DESIGN.md, "Run-to-run reproducibility").

Every repetition runs the same B x N batch with the per-layer debug taps of ONE layer L (cycled over the layers):
    layer_debug[0..4] = feat1 (PointCN output: chain<PCQ> at layer 0, the previous layer's chain<MSGPC> after it), Q, K, V
                        (decoded operand images), msg (attention output)
    layer_features    = the layer's output (chain<MSGPC>, chain<MSG> at the last layer)
and compares them with the first run that tapped the same layer.  For a repetition that differs, the FIRST differing
tensor in data-flow order names the kernel (feat1 differs: the layer's input already differed or PointCN; only Q differs:
chain<Q>, or the Q GEMM of chain<PCQ>; K / V: chain<KV>; msg: attention; layer_features: chain<MSGPC / MSG>), and the row range tells which
128-row tile (flat row tiles for the chain kernels, per-set query tiles for attention) and which CTA / iteration made it."""
import os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointdsc_b200 import PointDSC
from pointdsc_b200.synth import make_pair
root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
z = np.load(os.path.join(root, "tests/golden/snapshot_3dmatch.npz")); sd = {k: torch.from_numpy(z[k]) for k in z.files}
m = PointDSC(num_layers=12, precision=os.environ.get("PDSC_PRECISION", "fp16x3")); m.load_state_dict(sd, strict=False); m = m.cuda().eval()
B, N = int(os.environ.get("PDSC_B", "256")), int(os.environ.get("PDSC_N", "1000"))
reps = int(os.environ.get("PDSC_REPS", "240"))
layers = [int(x) for x in os.environ.get("PDSC_LAYERS", ",".join(str(i) for i in range(12))).split(",")]
ratios = [0.05, 0.1, 0.2, 0.4]
pairs = [make_pair(g, N, "3dmatch", ratios[g % 4]) for g in range(B)]
cp, s, t = (torch.stack([p[k] for p in pairs]).cuda() for k in ("corr_pos", "src_keypts", "tgt_keypts"))
names = ["feat1", "Q", "K", "V", "msg", "layer_features"]
SMS = torch.cuda.get_device_properties(0).multi_processor_count

def run(layer):
    o = m.run(cp, s, t, taps=["layer_debug", "layer_features"], layer_tap=layer)
    d = o["layer_debug"]
    return [d[0], d[1], d[2], d[3], d[4], o["layer_features"]]

ref = {}
events = {}
for rep in range(reps):
    L = layers[rep % len(layers)]
    cur = run(L)
    torch.cuda.synchronize()
    if L not in ref:
        ref[L] = [x.clone() for x in cur]
        continue
    for name, a, b in zip(names, cur, ref[L]):
        diff = (a != b).reshape(B * N, -1).any(dim=1)
        if bool(diff.any()):
            rows = diff.nonzero().flatten()
            r0, r1, n = int(rows[0]), int(rows[-1]), int(rows.numel())
            b0, b1 = r0 // N, r1 // N
            flat_tile0, flat_tile1 = r0 // 128, r1 // 128
            qt0 = (r0 % N) // 128
            item = b0 * ((N + 127) // 128) + qt0
            md = float((a - b).abs().max())
            print(f"rep {rep} layer {L}: first differing tensor {name}: {n} rows in [{r0}, {r1}] (sets {b0}..{b1}), max |delta| {md:.3e}; "
                  f"flat tiles {flat_tile0}..{flat_tile1} (CTA {flat_tile0 % SMS}, iteration {flat_tile0 // SMS}); "
                  f"attention item {item} (CTA {item % SMS}, iteration {item // SMS})")
            events[name] = events.get(name, 0) + 1
            break
print("events by first differing tensor:", events if events else "none (deterministic)")
