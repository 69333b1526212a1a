#!/usr/bin/env python
"""Time of the spectral-matching baseline (pdsc_spectral_matching_packed) against a torch eager restatement of the reference's
`SM` (baseline_scripts/baseline_3DMatch.py:19-53: the [N,N,6] difference tensor, ten bmm power steps, argsort, the weighted
Kabsch with torch.svd) on the same GPU, one set at a time as the baseline script runs it, and `evaluate.py --synthetic 64
--batch_size 8 --method SM` in pairs/s.

    python tools/sm_bench.py [--repeats 5] [--out profiles/sm_bench.jsonl]

Cases: one set of N = 1,000 / 5,000 / 12,000 rows (the sizes of tools/ransac_bench.py), and groups of 8 and 64 sets drawn from
tools/mixed_batch_bench.py's 3DMatch-like mix.  Medians of alternated repeats; one JSON line per case, with the card's name and
power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from mixed_batch_bench import card, draw_sizes, timed  # noqa: E402


def eager_sm(corr, src, tgt, thr):
    """The reference's SM restated in torch eager, one set [1,N,*] per call (the [N,N,6] temporary included)."""
    diff = corr - corr.permute(1, 0, 2)
    M = torch.sum(diff[:, :, 0:3] ** 2, dim=-1) ** 0.5 - torch.sum(diff[:, :, 3:6] ** 2, dim=-1) ** 0.5
    M = M[None]
    sigma = thr / 3
    M = torch.max(torch.zeros_like(M), 4.5 - M ** 2 / 2 / sigma ** 2)
    M[:, torch.arange(M.shape[1]), torch.arange(M.shape[1])] = 0
    v = torch.ones_like(M[:, :, 0:1])
    for _ in range(10):
        v = torch.bmm(M, v)
        v = v / (torch.norm(v, dim=1, keepdim=True) + 1e-6)
    v = v.squeeze(-1)
    top = torch.argsort(v, dim=1, descending=True)[:, 0:int(v.shape[1] * 0.1)]
    labels = torch.zeros_like(v)
    labels[0, top[0]] = 1
    w = v * labels
    ca = (src * w[:, :, None]).sum(1, keepdim=True) / (w.sum(1, keepdim=True)[:, :, None] + 1e-6)
    cb = (tgt * w[:, :, None]).sum(1, keepdim=True) / (w.sum(1, keepdim=True)[:, :, None] + 1e-6)
    H = (src - ca).permute(0, 2, 1) @ torch.diag_embed(w) @ (tgt - cb)
    U, S, V = torch.svd(H.cpu())
    U, V = U.to(w.device), V.to(w.device)
    eye = torch.eye(3, device=w.device)[None].repeat(1, 1, 1)
    eye[:, -1, -1] = torch.det(V @ U.permute(0, 2, 1))
    R = V @ eye @ U.permute(0, 2, 1)
    t = cb.permute(0, 2, 1) - R @ ca.permute(0, 2, 1)
    return R, t, labels


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "sm_bench.jsonl"))
    ap.add_argument("--skip-evaluate", action="store_true")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("sm_bench.py measures on the GPU: no CUDA device")
    from pointdsc_b200.spectral import spectral_matching_packed
    from pointdsc_b200.synth import make_pair
    name, power = card()
    cases = [("bs1", [1000]), ("bs1", [5000]), ("bs1", [12000]), ("mix8", draw_sizes("3dmatch", 8, 100)),
             ("mix64", draw_sizes("3dmatch", 64, 101))]
    records = []
    for kind, sizes in cases:
        pairs = [make_pair(500 + i, n, "3dmatch", 0.3) for i, n in enumerate(sizes)]
        off = np.cumsum([0] + sizes).tolist()
        dev = {k: torch.cat([p[k] for p in pairs]).cuda() for k in ("corr_pos", "src_keypts", "tgt_keypts")}
        d_off = torch.tensor(off, dtype=torch.int32, device="cuda")
        one = [{k: p[k][None].cuda() for k in ("corr_pos", "src_keypts", "tgt_keypts")} for p in pairs]

        def device():
            spectral_matching_packed(dev["corr_pos"], dev["src_keypts"], dev["tgt_keypts"], off, d_offsets=d_off, inlier_threshold=0.10)

        def eager():
            for d in one:
                eager_sm(d["corr_pos"], d["src_keypts"], d["tgt_keypts"], 0.10)
        arms = {"device": device, "torch_eager": eager}
        for fn in arms.values():       # warm-up: module loads, cuBLAS / cuSOLVER plans, the caching allocator
            fn()
        times = {k: [] for k in arms}
        for _ in range(args.repeats):
            for k, fn in arms.items():
                times[k].append(timed(fn))
        med = {k: float(np.median(v)) for k, v in times.items()}
        rec = {"tool": "sm_bench", "case": kind, "sets": len(sizes), "rows": int(off[-1]), "n_max": max(sizes),
               "device_ms": med["device"] * 1e3, "torch_eager_ms": med["torch_eager"] * 1e3,
               "eager_over_device": med["torch_eager"] / med["device"],
               "device_ms_all": [x * 1e3 for x in times["device"]], "torch_eager_ms_all": [x * 1e3 for x in times["torch_eager"]],
               "gpu": name, "power_limit": power}
        print(json.dumps(rec))
        records.append(rec)
        del dev, one
        torch.cuda.empty_cache()
    if not args.skip_evaluate:
        import evaluate
        evaluate.main(["--synthetic", "8", "--method", "SM", "--batch_size", "8"])      # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        stats, _ = evaluate.main(["--synthetic", "64", "--method", "SM", "--batch_size", "8"])
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        rec = {"tool": "sm_bench", "case": "evaluate --synthetic 64 --batch_size 8 --method SM", "pairs": int(len(stats)),
               "pairs_per_s": len(stats) / dt, "model_ms_per_pair": float(stats[:, 9].mean() * 1e3), "gpu": name,
               "power_limit": power}
        print(json.dumps(rec))
        records.append(rec)
    if args.out:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as f:
            for r in records:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
