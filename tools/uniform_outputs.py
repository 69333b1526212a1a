#!/usr/bin/env python
"""Every output of bs = 1 uniform forwards, for comparing two builds of the engine byte for byte.

    python tools/uniform_outputs.py --out DIR/uniform_outputs.npz
    python tools/uniform_outputs.py --compare A.npz B.npz

Seeded synthetic pairs (pointdsc_b200.synth, released 3DMatch weights) at N = 41, 257, 1003 and 5000 in every precision with
k = 40, and at N = 41, 257 and 1003 in fp32 and fp16x3 with k = 80 and k = 128 (keys "<precision>/k<k>/..."), so that every
NSM kernel runs: N = 41 falls back to k = 40 under the larger configurations.  N = 5000 at bs = 1 runs the attention's key
split, the others are too small to split or split into few chunks.  Per (precision, k, N) the file holds the testing-mode
forward with every stage tap (SC, features, the layer-0 internals, seeds, kNN, compatibility, eigenvectors, hypotheses,
refinement) and the eval-mode forward (confidence, M) with its taps.  Per precision it also holds the testing-mode forwards at
the same N in the batch-invariant mode (keys "<precision>/inv/..."), and one mixed-size forward_many call of the sets in MIXED,
with the mode off and on (keys "<precision>/mixed/..." and "<precision>/inv/mixed/..."): in the invariant mode the N = 5000
set of that call runs the key split and its merge at B > 1.  --compare exits non-zero unless both files hold the same arrays
with the same bytes."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = (41, 257, 1003, 5000)
PRECISIONS = ("fp32", "fp16x3", "bf16x3", "bf16")
# (k, precisions, sizes) beside k = 40: k = 80 and 128 reach the four-warp NSM kernels of both Gram forms
LARGE_K = ((80, ("fp32", "fp16x3"), (41, 257, 1003)), (128, ("fp32", "fp16x3"), (41, 257, 1003)))
MIXED = ((1, 41), (1, 257), (2, 1003), (1, 5000))   # (bs, N) batches of the mixed-size call
TAPS = ("sc", "features", "normed", "confidence", "seeds", "knn_idx", "compat", "eig", "power_iters", "seed_trans",
        "inlier_counts", "best", "init_trans", "refine_solves", "layer_features", "layer_debug")
EVAL_TAPS = ("features", "confidence", "seeds", "knn_idx", "compat", "eig", "power_iters", "seed_trans", "inlier_counts",
             "best", "init_trans")


def collect():
    import bench
    from pointdsc_b200 import PointDSC
    from pointdsc_b200.synth import make_pair
    out = {}
    configs = [(40, precision, SIZES, "") for precision in PRECISIONS]
    configs += [(k, precision, sizes, f"k{k}/") for k, precisions, sizes in LARGE_K for precision in precisions]
    for k, precision, sizes, prefix in configs:
        m = PointDSC(num_layers=12, k=k, precision=precision, **bench.CTOR["3dmatch"])
        m.load_state_dict(bench.load_snapshot("3dmatch"), strict=False)
        m = m.cuda().eval()
        for n in sizes:
            p = make_pair(n, n, "3dmatch", 0.3)
            cp, s, t = (p[key][None].cuda() for key in ("corr_pos", "src_keypts", "tgt_keypts"))
            for mode, res in (("test", m.run(cp, s, t, taps=TAPS)), ("eval", m.run_eval(cp, s, t, taps=EVAL_TAPS))):
                for name, v in res.items():
                    if v is not None:
                        out[f"{precision}/{prefix}{n}/{mode}/{name}"] = v.cpu().numpy()
        torch.cuda.synchronize()
    for precision in PRECISIONS:
        m = PointDSC(num_layers=12, k=40, precision=precision, **bench.CTOR["3dmatch"])
        m.load_state_dict(bench.load_snapshot("3dmatch"), strict=False)
        m = m.cuda().eval()
        batches = []
        for i, (bs, n) in enumerate(MIXED):
            pairs = [make_pair(n + 1000 * i + b, n, "3dmatch", 0.3) for b in range(bs)]
            batches.append({key: torch.stack([p[key] for p in pairs]).cuda() for key in ("corr_pos", "src_keypts", "tgt_keypts")})
            batches[-1]["testing"] = True
        for invariant in (False, True):
            m.set_batch_invariant(invariant)
            prefix = "inv/" if invariant else ""
            if invariant:
                for n in SIZES:
                    p = make_pair(n, n, "3dmatch", 0.3)
                    cp, s, t = (p[key][None].cuda() for key in ("corr_pos", "src_keypts", "tgt_keypts"))
                    for name, v in m.run(cp, s, t, taps=TAPS).items():
                        if v is not None:
                            out[f"{precision}/inv/{n}/test/{name}"] = v.cpu().numpy()
            for i, res in enumerate(m.forward_many(batches)):
                for name, v in res.items():
                    if isinstance(v, torch.Tensor):
                        out[f"{precision}/{prefix}mixed/{i}/{name}"] = v.cpu().numpy()
        torch.cuda.synchronize()
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args(argv)
    if args.compare:
        a, b = (np.load(f) for f in args.compare)
        bad = sorted(set(a.files) ^ set(b.files)) + [k for k in sorted(set(a.files) & set(b.files))
                                                      if a[k].dtype != b[k].dtype or a[k].tobytes() != b[k].tobytes()]
        print(f"{len(a.files)} arrays, {len(bad)} differ" + (": " + ", ".join(bad) if bad else ""))
        return 1 if bad else 0
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this tool runs the engine")
    np.savez(args.out, **collect())
    return 0


if __name__ == "__main__":
    sys.exit(main())
