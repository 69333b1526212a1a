#!/usr/bin/env python
"""FPFH descriptors of a group of clouds: the per-cloud loop against one call per stage for the whole group.

    python tools/fpfh_group_bench.py [--points 60000] [--voxel 0.08] [--groups 16 64] [--repeats 5]
                                     [--out profiles/fpfh_group_bench.jsonl]

Seeded synth_scene clouds of 60,000 points each at voxel 0.08 (the sizes `evaluate.py --synthetic` uses), already on the device.
Arms, alternated within every repeat, medians of clouds/s reported:
  per_cloud  `descriptors.fpfh_descriptors` cloud by cloud: three launches of the front end and three host reads per cloud
  packed     `descriptors.fpfh_descriptors_many` on the whole group: one call per stage and two host reads per group
Both arms return normalised FPFH; the tool checks that every cloud's key points and descriptors agree bit for bit.  One JSON
line per group size, with the card's name and power limit read in the same run."""
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


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--points", type=int, default=60000)
    ap.add_argument("--voxel", type=float, default=0.08)
    ap.add_argument("--groups", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "fpfh_group_bench.jsonl"))
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the GPU")
    from mixed_batch_bench import card
    from pointdsc_b200.descriptors import fpfh_descriptors, fpfh_descriptors_many
    from pointdsc_b200.synth_scene import scene
    name, power = card()
    clouds = [torch.from_numpy(scene(args.points, seed=100 + i)).cuda() for i in range(max(args.groups))]
    lines = []
    for P in args.groups:
        group = clouds[:P]
        arms = {"per_cloud": lambda: [fpfh_descriptors(c, args.voxel) for c in group],
                "packed": lambda: fpfh_descriptors_many(group, args.voxel)}
        per, (kp, feat, off, _) = arms["per_cloud"](), arms["packed"]()       # warm-up, and the outputs compared
        same = all(torch.equal(per[p][0], kp[off[p]:off[p + 1]]) and torch.equal(per[p][1], feat[off[p]:off[p + 1]])
                   for p in range(P))
        times = {k: [] for k in arms}
        for _ in range(args.repeats):
            for k, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()                     # both arms end in a host read of their status words
                torch.cuda.synchronize()
                times[k].append(time.perf_counter() - t0)
        med = {k: statistics.median(v) for k, v in times.items()}
        keypts = [off[p + 1] - off[p] for p in range(P)]
        rec = {"tool": "fpfh_group_bench", "clouds": P, "points_per_cloud": args.points, "voxel": args.voxel,
               "keypoints_min": min(keypts), "keypoints_max": max(keypts), "keypoints_mean": float(np.mean(keypts)),
               "repeats": args.repeats, "clouds_per_s": {k: P / v for k, v in med.items()}, "seconds_median": med,
               "seconds_all": times, "packed_over_per_cloud": med["per_cloud"] / med["packed"], "bit_identical": same,
               "gpu": name, "power_limit": power}
        print(json.dumps(rec))
        lines.append(rec)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
