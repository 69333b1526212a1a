#!/usr/bin/env python
"""Cost of the device ICP (pointdsc_b200.icp, row f5) and what it adds to the evaluation loop.

    python tools/icp_bench.py [--repeats 5] [--pairs 64] [--out profiles/icp_bench.jsonl]

Records, one JSON line each, with the card's name and power limit read in the same run; medians over alternated repeats:
  icp_bs1        device time (CUDA events) of one icp_refine call on one synthetic 3DMatch-like set (synth.make_pair), N = 1000,
                 5000, 12000, started 3 degrees / 3 cm off the ground truth
  icp_group      device time of one icp_refine_packed call on groups of 8 and 64 sets drawn from tools/mixed_batch_bench.py's
                 3DMatch-like mix, started as above, and of one forward_packed on the same group, for scale
  evaluate       evaluate.py --synthetic P --batch_size 8 pairs/s with and without --use_icp (pairs generated once, FPFH on the device,
                 and reused by both arms: the arms differ by the ICP only)
  oracle_cpu     the float64 CPU restatement's time per pair (oracle/icp_oracle.py, scipy k-d tree) on the 64-set mix: a stand-in for
                 the open3d call the reference makes, which is not installed here and is NOT what was timed"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def perturbed(gt, seed, deg=3.0, cm=3.0):
    g = np.random.default_rng(seed)
    ax = g.normal(size=3)
    ax /= np.linalg.norm(ax)
    a = np.deg2rad(deg)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    P = np.eye(4)
    P[:3, :3] = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
    P[:3, 3] = g.normal(size=3) * cm / 100 / np.sqrt(3)
    return (P @ np.asarray(gt, np.float64)).astype(np.float32)


def group(sizes, seed):
    from pointdsc_b200.synth import make_pair
    pairs = [make_pair(seed + i, n, "3dmatch") for i, n in enumerate(sizes)]
    off = np.cumsum([0] + list(sizes)).tolist()
    cat = lambda k: torch.cat([p[k] for p in pairs]).cuda()          # noqa: E731
    init = torch.from_numpy(np.stack([perturbed(p["gt_trans"].numpy(), seed + i) for i, p in enumerate(pairs)])).cuda()
    return {"corr_pos": cat("corr_pos"), "src": cat("src_keypts"), "tgt": cat("tgt_keypts"), "init": init, "offsets": off,
            "d_offsets": torch.tensor(off, dtype=torch.int32, device="cuda"), "pairs": pairs}


def device_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def alternate(arms, repeats, reps):
    for fn in arms.values():                     # warm-up
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(repeats):
        for k, fn in arms.items():
            times[k].append(device_ms(fn, reps))
    return {k: statistics.median(v) for k, v in times.items()}, times


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "icp_bench.jsonl"))
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the GPU")
    import evaluate
    from mixed_batch_bench import card, draw_sizes
    from oracle import icp_oracle as O
    from pointdsc_b200.icp import icp_refine_packed
    name, power = card()
    lines = []

    def emit(rec):
        rec.update({"tool": "icp_bench", "gpu": name, "power_limit": power, "repeats": args.repeats})
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    def icp_call(g):
        return lambda: icp_refine_packed(g["src"], g["tgt"], g["init"], g["offsets"], d_offsets=g["d_offsets"])

    # bs = 1
    singles = {n: group([n], 11) for n in (1000, 5000, 12000)}
    med, allt = alternate({str(n): icp_call(g) for n, g in singles.items()}, args.repeats, 20)
    its = {}
    for n, g in singles.items():
        _, info = icp_refine_packed(g["src"], g["tgt"], g["init"], g["offsets"], d_offsets=g["d_offsets"], info=True)
        its[str(n)] = int(info["iterations"][0])
    emit({"what": "icp_bs1", "ms_median": med, "ms_all": allt, "iterations": its})

    # groups of the 3DMatch-like mix, against the forward of the same group
    cfg = evaluate.load_config("PointDSC_3DMatch_release")
    model = evaluate.build_model("PointDSC_3DMatch_release", cfg, "cuda")
    for P in (8, 64):
        g = group(draw_sizes("3dmatch", P, 5), 100)
        fwd = lambda: model.forward_packed(g["corr_pos"], g["src"], g["tgt"], g["offsets"], d_offsets=g["d_offsets"])  # noqa: E731
        med, allt = alternate({"icp": icp_call(g), "forward_packed": fwd}, args.repeats, 5)
        _, info = icp_refine_packed(g["src"], g["tgt"], g["init"], g["offsets"], d_offsets=g["d_offsets"], info=True)
        sizes = np.diff(g["offsets"])
        emit({"what": "icp_group", "group": P, "n_min": int(sizes.min()), "n_max": int(sizes.max()), "n_mean": float(sizes.mean()),
              "ms_median": med, "ms_all": allt, "icp_over_forward": med["icp"] / med["forward_packed"],
              "iterations_max": int(info["iterations"].max()), "iterations_mean": float(info["iterations"].double().mean())})
        if P == 64:
            t0 = time.perf_counter()
            for i, p in enumerate(g["pairs"]):
                O.icp(p["src_keypts"].numpy(), p["tgt_keypts"].numpy(), g["init"][i].cpu().numpy())
            emit({"what": "oracle_cpu", "group": P, "n_mean": float(sizes.mean()),
                  "ms_per_pair": (time.perf_counter() - t0) * 1e3 / P,
                  "note": "float64 numpy / scipy restatement on the host CPU, a stand-in for open3d (absent): not open3d's time"})

    # evaluate.py --synthetic P --batch_size 8, with and without --use_icp, on the same generated pairs
    pairs = list(evaluate.synthetic_pairs(args.pairs, "cuda", 1.6 * cfg["downsample"]))
    arms = {"plain": lambda: evaluate.evaluate(model, iter(pairs), cfg, batch_size=8),
            "use_icp": lambda: evaluate.evaluate(model, iter(pairs), cfg, batch_size=8, use_icp=True)}
    for fn in arms.values():
        fn()
    times = {k: [] for k in arms}
    for _ in range(args.repeats):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    med = {k: statistics.median(v) for k, v in times.items()}
    emit({"what": "evaluate", "pairs": len(pairs), "batch_size": 8, "pairs_per_s": {k: len(pairs) / v for k, v in med.items()},
          "seconds_all": times, "note": "descriptors computed once before timing; the loop matches, runs, refines and scores"})

    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
