#!/usr/bin/env python
"""Throughput of mixed-size calls (PointDSC.forward_many -> pdsc_forward_packed) against the loop the evaluation drivers run
today, at the same total work.

    python tools/mixed_batch_bench.py [--sets 64] [--repeats 5] [--precision fp16x3] [--out profiles/mixed_batch_bench.jsonl]

Seeded synthetic sets (pointdsc_b200.synth, released 3DMatch weights), N drawn from two stated mixes:
  uniform   N uniform on [500, 5000]
  3dmatch   a 3DMatch-like spread of correspondence counts: 10 % on [200, 1000), 60 % on [1000, 3000), 30 % on [3000, 6000]
Arms, alternated within every repeat, medians reported:
  mixed        one forward_many call over all sets
  loop_graph   the drivers' bs = 1 loop: model.run per set (graph capture / replay per shape, as model.run does it)
  loop_eager   the same loop with graph replay off
  uniform_mean one uniform call of the same number of sets at the mix's mean N (a ceiling for the mixed call)
One JSON line per mix, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def draw_sizes(mix, count, seed):
    rng = np.random.default_rng(seed)
    if mix == "uniform":
        return [int(x) for x in rng.integers(500, 5001, size=count)]
    u = rng.random(count)
    lo = np.where(u < 0.1, 200, np.where(u < 0.7, 1000, 3000))
    hi = np.where(u < 0.1, 1000, np.where(u < 0.7, 3000, 6001))
    return [int(rng.integers(a, b)) for a, b in zip(lo, hi)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["unknown, unknown"])[0].split(", ")
    return name, power


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--sets", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--precision", default="fp16x3")
    ap.add_argument("--mixes", default="uniform,3dmatch")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "mixed_batch_bench.jsonl"))
    args = ap.parse_args(argv)
    import bench
    from pointdsc_b200 import PointDSC
    from pointdsc_b200.synth import make_batch, make_pair
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the GPU")
    m = PointDSC(num_layers=12, k=40, precision=args.precision, **bench.CTOR["3dmatch"])
    m.load_state_dict(bench.load_snapshot("3dmatch"), strict=False)
    m = m.cuda().eval()
    name, power = card()
    lines = []
    for mi, mix in enumerate(args.mixes.split(",")):
        sizes = draw_sizes(mix, args.sets, 100 + mi)
        sets = []
        for i, n in enumerate(sizes):
            p = make_pair(10_000 * mi + i, n, "3dmatch", 0.3)
            sets.append({k: p[k].cuda()[None] for k in ("corr_pos", "src_keypts", "tgt_keypts")})
            sets[-1]["testing"] = True
        n_mean = int(round(sum(sizes) / len(sizes)))
        ub = make_batch(list(range(len(sizes))), n_mean, "3dmatch", 0.3)
        ucp, us, ut = (ub[k].cuda() for k in ("corr_pos", "src_keypts", "tgt_keypts"))

        def mixed():
            m.forward_many(sets)

        def loop():
            for d in sets:
                m.run(d["corr_pos"], d["src_keypts"], d["tgt_keypts"])

        def loop_eager():
            rows, m.graph_rows = m.graph_rows, 0
            try:
                loop()
            finally:
                m.graph_rows = rows

        def uniform():
            m.run(ucp, us, ut)

        arms = {"mixed": mixed, "loop_graph": loop, "loop_eager": loop_eager, "uniform_mean": uniform}
        for fn in arms.values():      # warm-up: modules, graphs of the loop's shapes, workspaces
            fn()
        times = {k: [] for k in arms}
        for _ in range(args.repeats):
            for k, fn in arms.items():
                times[k].append(timed(fn))
        med = {k: statistics.median(v) for k, v in times.items()}
        rec = {"tool": "mixed_batch_bench", "mix": mix, "sets": len(sizes), "rows": sum(sizes), "n_min": min(sizes),
               "n_max": max(sizes), "n_mean": n_mean, "precision": args.precision, "repeats": args.repeats,
               "sets_per_s": {k: len(sizes) / v for k, v in med.items()}, "seconds_median": med,
               "seconds_all": times, "gpu": name, "power_limit": power}
        rec["mixed_over_loop_graph"] = med["loop_graph"] / med["mixed"]
        rec["mixed_over_uniform_mean"] = med["uniform_mean"] / med["mixed"]
        print(json.dumps(rec))
        lines.append(rec)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
