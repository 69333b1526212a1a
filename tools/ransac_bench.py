#!/usr/bin/env python
"""Cost of the device RANSAC (pointdsc_b200.ransac, row f6) and what it adds to the evaluation loop.

    python tools/ransac_bench.py [--repeats 5] [--pairs 64] [--out profiles/ransac_bench.jsonl]

Records, one JSON line each, with the card's name and power limit read in the same run; medians over alternated repeats:
  ransac_bs1     device time (CUDA events) of one ransac_packed call (5,000 iterations) on one synthetic 3DMatch-like set
                 (synth.make_pair), N = 1000, 5000, 12000, over the forward's labels; M = the candidates the forward kept.  Also
                 the scoring kernel's achieved fp64 rate, from a torch.profiler run of its own: the distance tests' fp64
                 operations (FP64_PER_TEST each, an FMA counted as 2) over the kernel's time, and that rate as a share of the data
                 sheet's H100 SXM FP64 (non-tensor) rate, 34 TFLOP/s at 700 W
  ransac_group   device time of one ransac_packed call on groups of 8 and 64 sets drawn from tools/mixed_batch_bench.py's
                 3DMatch-like mix, over the forward's labels, and of one forward_packed on the same group
  evaluate       evaluate.py --synthetic P --batch_size 8 pairs/s with and without --solver RANSAC (pairs generated once, FPFH on
                 the device, and reused by both arms: the arms differ by the RANSAC only)
  oracle_cpu     the float64 CPU restatement's time per pair (oracle/ransac_oracle.py, numpy) on the 8-set group: a stand-in for the
                 open3d call the reference makes, which is not installed here and is NOT what was timed"""
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

FP64_PER_TEST = 27          # R p + t: 9 FMA; minus q: 3; d^2: 1 MUL + 2 FMA; the sum of an inlier: 1 (an FMA counted as 2)
FP64_PEAK = 34e12           # H100 SXM data sheet, FP64 without tensor cores


def group(model, sizes, seed):
    from pointdsc_b200.synth import make_pair
    pairs = [make_pair(seed + i, n, "3dmatch") for i, n in enumerate(sizes)]
    off = np.cumsum([0] + list(sizes)).tolist()
    cat = lambda k: torch.cat([p[k] for p in pairs]).cuda()          # noqa: E731
    g = {"corr_pos": cat("corr_pos"), "src": cat("src_keypts"), "tgt": cat("tgt_keypts"), "offsets": off,
         "d_offsets": torch.tensor(off, dtype=torch.int32, device="cuda"), "pairs": pairs}
    g["labels"] = model.forward_packed(g["corr_pos"], g["src"], g["tgt"], off, d_offsets=g["d_offsets"])["final_labels"].float()
    return g


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


def score_kernel_ms(fn, reps):
    """Mean device time of ransac_score_kernel over `reps` calls, from torch.profiler's CUDA activity."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = [e.device_time_total for e in prof.key_averages() if "ransac_score_kernel" in e.key]
    return sum(us) / 1e3 / reps


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "ransac_bench.jsonl"))
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the GPU")
    import evaluate
    from mixed_batch_bench import card, draw_sizes
    from oracle import ransac_oracle as O
    from pointdsc_b200.ransac import ransac_packed
    name, power = card()
    lines = []

    def emit(rec):
        rec.update({"tool": "ransac_bench", "gpu": name, "power_limit": power, "repeats": args.repeats})
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    def call(g):
        return lambda: ransac_packed(g["src"], g["tgt"], g["labels"], g["offsets"], d_offsets=g["d_offsets"])

    cfg = evaluate.load_config("PointDSC_3DMatch_release")
    model = evaluate.build_model("PointDSC_3DMatch_release", cfg, "cuda")

    # bs = 1
    singles = {n: group(model, [n], 11) for n in (1000, 5000, 12000)}
    med, allt = alternate({str(n): call(g) for n, g in singles.items()}, args.repeats, 20)
    Ms, rate = {}, {}
    for n, g in singles.items():
        M = int((g["labels"] > 0).sum())
        Ms[str(n)] = M
        ms = score_kernel_ms(call(g), 20)
        flops = 5000.0 * M * FP64_PER_TEST
        rate[str(n)] = {"score_kernel_ms": ms, "fp64_tflops": flops / (ms * 1e-3) / 1e12 if ms > 0 else None,
                        "share_of_datasheet_fp64": flops / (ms * 1e-3) / FP64_PEAK if ms > 0 else None}
    emit({"what": "ransac_bs1", "ms_median": med, "ms_all": allt, "M": Ms, "score_kernel": rate})

    # groups of the 3DMatch-like mix, against the forward of the same group
    for P in (8, 64):
        g = group(model, draw_sizes("3dmatch", P, 5), 100)
        fwd = lambda: model.forward_packed(g["corr_pos"], g["src"], g["tgt"], g["offsets"], d_offsets=g["d_offsets"])  # noqa: E731
        med, allt = alternate({"ransac": call(g), "forward_packed": fwd}, args.repeats, 5)
        sizes = np.diff(g["offsets"])
        M = [int((g["labels"][a:b] > 0).sum()) for a, b in zip(g["offsets"][:-1], g["offsets"][1:])]
        emit({"what": "ransac_group", "group": P, "n_min": int(sizes.min()), "n_max": int(sizes.max()), "n_mean": float(sizes.mean()),
              "m_mean": float(np.mean(M)), "ms_median": med, "ms_all": allt, "ransac_over_forward": med["ransac"] / med["forward_packed"]})
        if P == 8:
            lab = g["labels"].cpu().numpy()
            t0 = time.perf_counter()
            for i, p in enumerate(g["pairs"]):
                a, b = g["offsets"][i], g["offsets"][i + 1]
                O.ransac(p["src_keypts"].numpy(), p["tgt_keypts"].numpy(), lab[a:b], 0.10)
            emit({"what": "oracle_cpu", "group": P, "n_mean": float(sizes.mean()), "m_mean": float(np.mean(M)),
                  "ms_per_pair": (time.perf_counter() - t0) * 1e3 / P,
                  "note": "float64 numpy restatement on the host CPU, a stand-in for open3d (absent): not open3d's time"})

    # evaluate.py --synthetic P --batch_size 8, with and without --solver RANSAC, on the same generated pairs
    pairs = list(evaluate.synthetic_pairs(args.pairs, "cuda", 1.6 * cfg["downsample"]))
    arms = {"svd": lambda: evaluate.evaluate(model, iter(pairs), cfg, batch_size=8),
            "ransac": lambda: evaluate.evaluate(model, iter(pairs), cfg, batch_size=8, solver="RANSAC")}
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
          "seconds_all": times, "note": "descriptors computed once before timing; the loop matches, runs, post-processes and scores"})

    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
